"""Exact reference for numeric sum / avg on the GPU path, with no GPU and nothing of the product in it.

A value is an (unscaled int, scale) pair of Python integers.  sum is the exact sum at the argument's display scale (+ and -
take the larger scale of their operands, * the sum of their scales).  avg restates numeric_avg -> numeric_div: the result
scale from select_div_scale (16 significant digits judged from the base-10000 weights and first digits of the operands, at
least the operands' display scales) and the quotient rounded half away from zero at that scale.  test_device_emu.py holds
this restatement to the reference's own answers (golden/numeric_kat.json) before the GPU tests lean on it.

The device keeps a numeric as a 64-bit integer at its scale and refuses (GG_ERR_UNSUPPORTED, the plan stays on the CPU)
what does not fit.  `refusal` says when it must refuse, when it must not, and when either is right."""
from fractions import Fraction

from greengage_b200 import capi

R63, R62 = 1 << 63, 1 << 62
REQUIRED, FORBIDDEN, EITHER = "refusal required", "refusal forbidden", "either"


def typmod(precision, scale):
    return ((precision << 16) | scale) + 4


def rescale(v, frm, to):
    assert to >= frm
    return v * 10 ** (to - frm)


def weight_first(mag, scale):
    """base-10000 weight and first (most significant, non-zero) digit of mag / 10^scale; zero: (0, 0)"""
    if mag == 0:
        return 0, 0
    x = Fraction(mag, 10 ** scale)
    w = 0
    while x >= Fraction(10000) ** (w + 1):
        w += 1
    while x < Fraction(10000) ** w:
        w -= 1
    return w, int(x / Fraction(10000) ** w)


def div_scale(sum_unscaled, sscale, n):
    """select_div_scale(sum, n::numeric): n has display scale 0"""
    w1, f1 = weight_first(abs(sum_unscaled), sscale)
    w2, f2 = weight_first(n, 0)
    qweight = w1 - w2
    if f1 <= f2:
        qweight -= 1
    return min(max(16 - 4 * qweight, sscale, 0), 1000)


def avg(sum_unscaled, sscale, n):
    """numeric_avg over n inputs that sum to sum_unscaled at scale sscale: (unscaled, result scale)"""
    rs = div_scale(sum_unscaled, sscale, n)
    q = Fraction(abs(sum_unscaled) * 10 ** rs, 10 ** sscale * n)
    r = int(q + Fraction(1, 2))                      # round half away from zero (div_var with round = true)
    return (-r if sum_unscaled < 0 else r), rs


def text(v, scale):
    return capi.numeric_text(v, scale)


def sum_text(values, scale):
    """values: unscaled ints at `scale`, None for NULL -> sum as numeric_out prints it, or None (no input)"""
    vs = [v for v in values if v is not None]
    return text(sum(vs), scale) if vs else None


def avg_text(values, scale):
    vs = [v for v in values if v is not None]
    return text(*avg(sum(vs), scale, len(vs))) if vs else None


def refusal(required, produced):
    """required: every input at its column scale and every + - * result at its display scale, of the rows that reach an
    aggregate; produced: every value at the scale the compiler produces it (an operand rescaled for + - or a comparison).
    Refusal is required when one of `required` has magnitude >= 2^63, forbidden when all of `produced` (and `required`) are
    below 2^62; in between (rescaling overflow, the decoder's conservative refusal of -2^63) either outcome is right."""
    if any(v >= R63 or v < -R63 for v in required):
        return REQUIRED
    if all(abs(v) < R62 for v in list(required) + list(produced)):
        return FORBIDDEN
    return EITHER


def is_numeric_refusal(exc):
    return isinstance(exc, capi.GGError) and exc.code == -6 and "numeric" in str(exc)


def long_header_payload(unscaled, dscale):
    """the same value with the 4-byte NumericLong header (sign and display scale word, then the int16 weight), which
    older on-disk data still carries even where the short header would do"""
    import struct
    short = capi.numeric_payload(unscaled, dscale)
    hdr = struct.unpack("<H", short[:2])[0]
    if not hdr & 0x8000:
        return short
    neg = bool(hdr & 0x2000)
    weight = (hdr & 0x3F) - (0x40 if hdr & 0x40 else 0)
    return struct.pack("<Hh", (0x4000 if neg else 0) | (dscale & 0x3FFF), weight) + short[2:]
