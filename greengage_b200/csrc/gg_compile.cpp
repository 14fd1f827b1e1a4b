/*
 * gg_compile.cpp — host-side plan compiler: gg_plan.h PODs -> ggp_program.
 *
 * Stands where ExecInitExpr / ExecInitAgg prepare ExprState trees and per-agg
 * state (execQual.c:5378, nodeAgg.c:1875-2300): the plan is checked for
 * eligibility (anything outside the accelerated subset returns
 * GG_ERR_UNSUPPORTED so the caller keeps the CPU node), referenced columns get
 * slots, attcacheoff is precomputed the way slot_deform_tuple memoises it
 * (heaptuple.c:1160-1190), and the scan qual, the grouping keys and every
 * aggregate argument are flattened into one accumulator-machine program
 * (gg_program.h).
 */
#include <cstdio>
#include <cstring>
#include <cstdarg>
#include <cstdlib>
#include "gg_program.h"
#include "../../include/ggb200.h"

namespace {

struct Ctx {
	const gg_exprpool *pool;
	ggp_program *prog;
	ggp_side *outer;
	ggp_side *inner;          /* may be null */
	const gg_tupdesc *odesc;
	const gg_tupdesc *idesc;
	char *err;
	int errlen;
	int temps_busy;           /* bit t: temporary t holds a live value */
	int npersist;
	int persist_root[4], persist_temp[4];   /* common subexpressions kept in temporaries for later aggregate arguments */
	int persist_scale[4];     /* numeric subexpressions: the scale the temporary holds the value at */
	bool inner_as_outer;      /* build program of a join: the inner tuple is the scanned one */
	bool failed;
};

void fail(Ctx &c, const char *fmt, ...)
{
	if (c.failed) return;
	c.failed = true;
	va_list ap;
	va_start(ap, fmt);
	vsnprintf(c.err, (size_t) c.errlen, fmt, ap);
	va_end(ap);
}

int loadtype_of(int32_t typid)
{
	switch (typid)
	{
		case GG_INT4OID: case GG_DATEOID: return GGP_LT_I4;
		case GG_INT8OID: case GG_FLOAT8OID: case GG_TIMESTAMPOID: return GGP_LT_I8;
		case GG_BPCHAROID: return GGP_LT_BPCHAR;
		case GG_VARCHAROID: case GG_TEXTOID: return GGP_LT_VARCHAR;
		case GG_BOOLOID: return GGP_LT_BOOL;
		case GG_NUMERICOID: return GGP_LT_NUM;
	}
	return 0;
}

long align_nominal(long off, char a)
{
	switch (a) { case 'i': return (off + 3) & ~3L; case 'c': return off; case 'd': return (off + 7) & ~7L; default: return (off + 1) & ~1L; }
}

/* attcacheoff as slot_deform_tuple memoises it (heaptuple.c:1160-1200): valid for the fixed-width
 * prefix, and for the first varlena iff its offset is already aligned */
void init_side(ggp_side *s, const gg_tupdesc *d)
{
	memset(s, 0, sizeof *s);
	s->natts = d->natts;
	if (d->format == GG_FMT_DATUMROWS)
	{
		/* every column is one 64-bit word at a constant offset behind the NULL-mask word */
		s->rowwords = 1 + d->natts;
		s->first_walk = d->natts;
		for (int i = 0; i < d->natts && i < GG_MAX_ATTS; i++)
		{
			s->att[i].attlen = 8;
			s->att[i].attalign = 'd';
			s->att[i].slot = -1;
			s->att[i].cacheoff = (int16_t) (8 * i);
			s->att[i].notnull = d->attrs[i].attnotnull;
		}
		return;
	}
	for (int i = 0; i < d->natts && i < GG_MAX_ATTS; i++)
	{
		s->att[i].attlen = d->attrs[i].attlen;
		s->att[i].attalign = d->attrs[i].attalign;
		s->att[i].slot = -1;
		s->att[i].cacheoff = -1;
		s->att[i].notnull = d->attrs[i].attnotnull;
	}
	long off = 0;
	s->first_walk = s->natts;
	for (int i = 0; i < s->natts; i++)
	{
		if (s->att[i].attlen == -1)
		{
			if (off == align_nominal(off, s->att[i].attalign))
			{
				s->att[i].cacheoff = (int16_t) off;
				s->first_walk = i + 1;      /* the varlena's own offset is constant; what follows is not */
			}
			else
				s->first_walk = i;
			break;
		}
		off = align_nominal(off, s->att[i].attalign);
		s->att[i].cacheoff = (int16_t) off;
		off += s->att[i].attlen;
	}
}

/* slot of (varno, attno), allocating on first use */
int col_slot(Ctx &c, int varno, int attno)
{
	const bool inner = varno == 1 && !c.inner_as_outer;
	if (c.inner_as_outer && varno != 1) { fail(c, "outer Var in an inner-only expression"); return 0; }
	ggp_side *s = inner ? c.inner : c.outer;
	const gg_tupdesc *d = inner ? c.idesc : c.odesc;

	if (!s || !d) { fail(c, "Var references a side that does not exist (varno %d)", varno); return 0; }
	if (attno < 1 || attno > d->natts) { fail(c, "Var attno %d out of range", attno); return 0; }
	int a = attno - 1;
	if (s->att[a].slot >= 0) return s->att[a].slot;
	int lt = loadtype_of(d->attrs[a].atttypid);
	if (!lt) { fail(c, "column %d: type %d not supported on the GPU path", attno, d->attrs[a].atttypid); return 0; }
	if (d->format == GG_FMT_DATUMROWS && lt == GGP_LT_NUM) { fail(c, "numeric columns do not travel as datum rows yet"); return 0; }
	if (d->format == GG_FMT_DATUMROWS) lt = GGP_LT_I8;       /* already in loaded form */
	if (s->ncols >= GGP_MAX_COLS) { fail(c, "too many referenced columns"); return 0; }
	int slot = s->ncols++;
	s->att[a].slot = (int8_t) slot;
	s->coltype[slot] = (uint8_t) lt;
	s->colatt[slot] = (uint8_t) a;
	if (a + 1 > s->natts_walk) s->natts_walk = a + 1;
	if (!d->attrs[a].attnotnull) c.prog->nullable = 1;
	if (inner && slot >= GGP_MAX_PAYLOAD) { fail(c, "too many inner columns referenced above the join"); return 0; }
	return slot;
}

int add_const(Ctx &c, int64_t v, bool isnull)
{
	ggp_program *p = c.prog;
	for (int i = 0; i < p->nconst; i++)
		if (p->consts[i] == v && (((p->constnull >> i) & 1) != 0) == isnull) return i;
	if (p->nconst >= GGP_MAX_CONSTS) { fail(c, "too many constants"); return 0; }
	p->consts[p->nconst] = v;
	if (isnull) { p->constnull |= 1 << p->nconst; p->nullable = 1; }
	return p->nconst++;
}

bool is_col_op(int op)
{
	switch (op)
	{
		case GGP_LD_C4: case GGP_LD_C8: case GGP_LD_BP: case GGP_LD_VS: case GGP_LD_BOOL:
		case GGP_ADD_C: case GGP_SUB_C: case GGP_RSUB_C: case GGP_MUL_C: case GGP_DIV_C: case GGP_RDIV_C:
		case GGP_CMPF_C: case GGP_CMPI_C4: case GGP_CMPI_C8: case GGP_LD_NUM:
			return true;
	}
	return false;
}

void emit(Ctx &c, int op, int idx = 0, int aux = 0)
{
	ggp_program *p = c.prog;
	if (p->ncode >= GGP_MAX_CODE - 1) { fail(c, "expression program too long"); return; }
	ggp_op o;
	memset(&o, 0, sizeof o);
	o.op = (uint8_t) op; o.idx = (uint8_t) idx; o.aux = (uint8_t) aux;
	o.off = 0xFFFF;
	if (is_col_op(op) && !(idx & 0x80))
	{
		const ggp_side *s = c.outer;
		int a = s->colatt[idx & 0x7F];
		if (s->att[a].cacheoff >= 0) o.off = (uint16_t) s->att[a].cacheoff;
	}
	p->code[p->ncode++] = o;
}

/* attach a post-action to the op that produced the current accumulator value */
ggp_op *last_op(Ctx &c, int start)
{
	ggp_program *p = c.prog;
	if (p->ncode <= start) emit(c, GGP_NOP);
	return &p->code[p->ncode - 1];
}

bool expr_equal(const gg_exprpool *pool, int a, int b)
{
	if (a == b) return true;
	if (a < 0 || b < 0) return false;
	const gg_expr &x = pool->nodes[a], &y = pool->nodes[b];
	if (x.kind != y.kind) return false;
	switch (x.kind)
	{
		case GG_E_VAR: return x.varno == y.varno && x.varattno == y.varattno;
		case GG_E_CONST: return x.constvalue == y.constvalue && x.constisnull == y.constisnull && x.constlen == y.constlen;
		case GG_E_FUNC:
			if (x.funcid != y.funcid || x.nargs != y.nargs) return false;
			for (int i = 0; i < x.nargs; i++) if (!expr_equal(pool, x.args[i], y.args[i])) return false;
			return true;
		case GG_E_NOT: case GG_E_ISNULL: case GG_E_ISNOTNULL: return expr_equal(pool, x.args[0], y.args[0]);
		default: return expr_equal(pool, x.args[0], y.args[0]) && expr_equal(pool, x.args[1], y.args[1]);
	}
}

/* does tree `root` contain a subtree equal to `sub`? */
bool contains(const gg_exprpool *pool, int root, int sub)
{
	if (root < 0) return false;
	if (expr_equal(pool, root, sub)) return true;
	const gg_expr &e = pool->nodes[root];
	if (e.kind == GG_E_VAR || e.kind == GG_E_CONST) return false;
	for (int i = 0; i < e.nargs && i < 2; i++)
		if (contains(pool, e.args[i], sub)) return true;
	return false;
}

/* operand kinds a binary op can take directly */
enum { OPD_NONE = 0, OPD_C8, OPD_C4, OPD_STR, OPD_K, OPD_T };
struct Operand { int kind; int idx; };

/* a node that can be used as a direct operand: Var, Const, or a subtree already kept in a temporary */
Operand operand_of(Ctx &c, int root)
{
	Operand o = { OPD_NONE, 0 };
	const gg_expr &e = c.pool->nodes[root];
	for (int i = 0; i < c.npersist; i++)
		if (expr_equal(c.pool, c.persist_root[i], root)) { o.kind = OPD_T; o.idx = c.persist_temp[i]; return o; }
	if (e.kind == GG_E_VAR)
	{
		int slot = col_slot(c, e.varno, e.varattno);
		const bool inner = e.varno == 1 && !c.inner_as_outer;
		const ggp_side *s = inner ? c.inner : c.outer;
		if (c.failed) return o;
		int lt = s->coltype[slot];
		o.idx = slot | (inner ? 0x80 : 0);
		o.kind = lt == GGP_LT_I4 ? OPD_C4 : lt == GGP_LT_I8 ? OPD_C8 : OPD_STR;
		if (lt == GGP_LT_BOOL || lt == GGP_LT_NUM) o.kind = OPD_NONE;
	}
	else if (e.kind == GG_E_CONST && e.rettype != GG_NUMERICOID)
	{
		o.kind = OPD_K;
		o.idx = add_const(c, e.constvalue, e.constisnull != 0);
	}
	return o;
}

int swap_cc(int cc)
{
	switch (cc) { case GGP_LT: return GGP_GT; case GGP_LE: return GGP_GE; case GGP_GT: return GGP_LT; case GGP_GE: return GGP_LE; }
	return cc;
}

enum { K_F8ADD = 1, K_F8SUB, K_F8MUL, K_F8DIV, K_CMPF, K_CMPI, K_CMPS, K_AND, K_OR, K_NADD, K_NSUB, K_NMUL, K_NCMP };
struct BinInfo { int k, cc; bool isbin; };

bool func_info(int funcid, BinInfo *b, int *unary_op)
{
	*unary_op = 0;
	b->isbin = true; b->cc = 0;
	switch (funcid)
	{
		case GG_F_FLOAT8PL:  b->k = K_F8ADD; return true;
		case GG_F_FLOAT8MUL: b->k = K_F8MUL; return true;
		case GG_F_FLOAT8MI:  b->k = K_F8SUB; return true;
		case GG_F_FLOAT8DIV: b->k = K_F8DIV; return true;
		case GG_F_NUMERIC_ADD: b->k = K_NADD; return true;
		case GG_F_NUMERIC_SUB: b->k = K_NSUB; return true;
		case GG_F_NUMERIC_MUL: b->k = K_NMUL; return true;
#define CMPCASE(F, K, CC) case F: b->k = K; b->cc = CC; return true;
		CMPCASE(GG_F_FLOAT8LT, K_CMPF, GGP_LT) CMPCASE(GG_F_FLOAT8LE, K_CMPF, GGP_LE)
		CMPCASE(GG_F_FLOAT8EQ, K_CMPF, GGP_EQ) CMPCASE(GG_F_FLOAT8NE, K_CMPF, GGP_NE)
		CMPCASE(GG_F_FLOAT8GT, K_CMPF, GGP_GT) CMPCASE(GG_F_FLOAT8GE, K_CMPF, GGP_GE)
		CMPCASE(GG_F_INT4LT, K_CMPI, GGP_LT) CMPCASE(GG_F_INT4LE, K_CMPI, GGP_LE)
		CMPCASE(GG_F_INT4EQ, K_CMPI, GGP_EQ) CMPCASE(GG_F_INT4NE, K_CMPI, GGP_NE)
		CMPCASE(GG_F_INT4GT, K_CMPI, GGP_GT) CMPCASE(GG_F_INT4GE, K_CMPI, GGP_GE)
		CMPCASE(GG_F_INT8LT, K_CMPI, GGP_LT) CMPCASE(GG_F_INT8LE, K_CMPI, GGP_LE)
		CMPCASE(GG_F_INT8EQ, K_CMPI, GGP_EQ) CMPCASE(GG_F_INT8NE, K_CMPI, GGP_NE)
		CMPCASE(GG_F_INT8GT, K_CMPI, GGP_GT) CMPCASE(GG_F_INT8GE, K_CMPI, GGP_GE)
		CMPCASE(GG_F_DATE_LT, K_CMPI, GGP_LT) CMPCASE(GG_F_DATE_LE, K_CMPI, GGP_LE)
		CMPCASE(GG_F_DATE_EQ, K_CMPI, GGP_EQ) CMPCASE(GG_F_DATE_NE, K_CMPI, GGP_NE)
		CMPCASE(GG_F_DATE_GT, K_CMPI, GGP_GT) CMPCASE(GG_F_DATE_GE, K_CMPI, GGP_GE)
		CMPCASE(GG_F_BPCHAREQ, K_CMPS, GGP_EQ) CMPCASE(GG_F_BPCHARNE, K_CMPS, GGP_NE)
		CMPCASE(GG_F_NUMERIC_LT, K_NCMP, GGP_LT) CMPCASE(GG_F_NUMERIC_LE, K_NCMP, GGP_LE)
		CMPCASE(GG_F_NUMERIC_EQ, K_NCMP, GGP_EQ) CMPCASE(GG_F_NUMERIC_NE, K_NCMP, GGP_NE)
		CMPCASE(GG_F_NUMERIC_GT, K_NCMP, GGP_GT) CMPCASE(GG_F_NUMERIC_GE, K_NCMP, GGP_GE)
#undef CMPCASE
		case GG_F_INT48: b->isbin = false; *unary_op = -1; return true;     /* loads already sign-extend */
		case GG_F_I4TOD: case GG_F_I8TOD: b->isbin = false; *unary_op = GGP_I2F8; return true;
	}
	return false;
}

int date_ts_cc(int funcid)
{
	switch (funcid)
	{
		case GG_F_DATE_LT_TIMESTAMP: return GGP_LT; case GG_F_DATE_LE_TIMESTAMP: return GGP_LE;
		case GG_F_DATE_EQ_TIMESTAMP: return GGP_EQ; case GG_F_DATE_GT_TIMESTAMP: return GGP_GT;
		case GG_F_DATE_GE_TIMESTAMP: return GGP_GE; case GG_F_DATE_NE_TIMESTAMP: return GGP_NE;
	}
	return -1;
}

void gen(Ctx &c, int root);

void emit_load(Ctx &c, const Operand &o, int root)
{
	const gg_expr &e = c.pool->nodes[root];
	switch (o.kind)
	{
		case OPD_C8: emit(c, GGP_LD_C8, o.idx); return;
		case OPD_C4: emit(c, GGP_LD_C4, o.idx); return;
		case OPD_K: emit(c, GGP_LD_K, o.idx); return;
		case OPD_T: emit(c, GGP_LD_T, o.idx); return;
		case OPD_STR: emit(c, e.rettype == GG_BPCHAROID ? GGP_LD_BP : GGP_LD_VS, o.idx); return;
	}
	if (e.kind == GG_E_VAR && !c.failed)      /* bool column */
	{
		emit(c, GGP_LD_BOOL, col_slot(c, e.varno, e.varattno) | ((e.varno == 1 && !c.inner_as_outer) ? 0x80 : 0));
		return;
	}
	fail(c, "operand cannot be loaded");
}

/* acc = acc OP operand (reversed=false) or operand OP acc (reversed=true) */
void emit_binop(Ctx &c, int k, int cc, const Operand &o, bool reversed)
{
	int base = 0;
	switch (k)
	{
		case K_F8ADD: base = GGP_ADD_C; break;
		case K_F8MUL: base = GGP_MUL_C; break;
		case K_F8SUB: base = reversed ? GGP_RSUB_C : GGP_SUB_C; break;
		case K_F8DIV: base = reversed ? GGP_RDIV_C : GGP_DIV_C; break;
		case K_CMPF:
			if (reversed) cc = swap_cc(cc);
			if (o.kind == OPD_C8) emit(c, GGP_CMPF_C, o.idx, cc);
			else if (o.kind == OPD_K) emit(c, GGP_CMPF_K, o.idx, cc);
			else if (o.kind == OPD_T) emit(c, GGP_CMPF_T, o.idx, cc);
			else fail(c, "float8 comparison with a non-float8 operand");
			return;
		case K_CMPI:
			if (reversed) cc = swap_cc(cc);
			if (o.kind == OPD_C8) emit(c, GGP_CMPI_C8, o.idx, cc);
			else if (o.kind == OPD_C4) emit(c, GGP_CMPI_C4, o.idx, cc);
			else if (o.kind == OPD_K) emit(c, GGP_CMPI_K, o.idx, cc);
			else if (o.kind == OPD_T) emit(c, GGP_CMPI_T, o.idx, cc);
			else fail(c, "integer comparison with a non-integer operand");
			return;
		case K_CMPS:
			if (o.kind == OPD_K) emit(c, GGP_CMPS_K, o.idx, cc);
			else if (o.kind == OPD_T) emit(c, GGP_CMPS_T, o.idx, cc);
			else fail(c, "string comparison operand must be a constant or a temporary");
			return;
		case K_AND: case K_OR:
			if (o.kind != OPD_T) { fail(c, "boolean operand must be a temporary"); return; }
			emit(c, k == K_AND ? GGP_AND_T : GGP_OR_T, o.idx);
			return;
	}
	if (o.kind == OPD_C8) emit(c, base, o.idx);
	else if (o.kind == OPD_K) emit(c, base + 1, o.idx);
	else if (o.kind == OPD_T) emit(c, base + 2, o.idx);
	else fail(c, "float8 arithmetic on a non-float8 operand (missing cast)");
}

int alloc_temp(Ctx &c)
{
	for (int t = 0; t < 4; t++)
		if (!(c.temps_busy & (1 << t))) { c.temps_busy |= 1 << t; return t; }
	fail(c, "expression too deep");
	return 0;
}

/* temp[t] = acc, as a post-action of the op that produced acc */
void store_temp(Ctx &c, int t)
{
	if (c.failed) return;
	if (c.prog->ncode == 0 || (c.prog->code[c.prog->ncode - 1].flags & GGP_F_ST)) emit(c, GGP_NOP);
	if (c.prog->ncode == 0) return;
	ggp_op *o = &c.prog->code[c.prog->ncode - 1];
	o->flags |= GGP_F_ST;
	o->aux = (uint8_t) ((o->aux & ~0x30) | (t << 4));
}

void gen_binary(Ctx &c, int lroot, int rroot, int k, int cc)
{
	bool commut = (k == K_F8ADD || k == K_F8MUL || k == K_AND || k == K_OR);
	bool logical = (k == K_AND || k == K_OR);
	Operand ro = operand_of(c, rroot), lo = operand_of(c, lroot);
	if (logical)
	{
		/* AND/OR take their second operand from a temporary only */
		if (ro.kind != OPD_T) ro.kind = OPD_NONE;
		if (lo.kind != OPD_T) lo.kind = OPD_NONE;
	}
	if (k == K_CMPS)
	{
		if (ro.kind == OPD_STR) ro.kind = OPD_NONE;     /* two string columns: one goes through a temp */
		if (lo.kind == OPD_STR) lo.kind = OPD_NONE;
	}
	if (ro.kind != OPD_NONE)
	{
		gen(c, lroot);
		emit_binop(c, k, cc, ro, false);
	}
	else if (lo.kind != OPD_NONE)
	{
		gen(c, rroot);
		emit_binop(c, k, cc, lo, !commut);
	}
	else
	{
		gen(c, lroot);
		int t = alloc_temp(c);
		store_temp(c, t);
		/* ExecEvalAnd / ExecEvalOr (execQual.c:3321-3450) do not evaluate the second arm once the first has decided the
		 * result: lanes where it has are not live while the arm runs, so what it would have raised is not raised */
		if (logical) emit(c, k == K_AND ? GGP_GUARD_AND : GGP_GUARD_OR, t);
		gen(c, rroot);
		if (logical) emit(c, GGP_UNGUARD);
		Operand to = { OPD_T, t };
		emit_binop(c, k, cc, to, !commut);
		c.temps_busy &= ~(1 << t);
	}
}

/* ---- numeric as scaled 64-bit integers (gg_plan.h "numeric") ---- */
static const int64_t kPow10[19] = { 1LL, 10LL, 100LL, 1000LL, 10000LL, 100000LL, 1000000LL, 10000000LL, 100000000LL, 1000000000LL, 10000000000LL,
                                    100000000000LL, 1000000000000LL, 10000000000000LL, 100000000000000LL, 1000000000000000LL,
                                    10000000000000000LL, 100000000000000000LL, 1000000000000000000LL };
#define GG_NUM_MAX_SCALE 15            /* a load op carries its scale in four bits */

/* display scale of a numeric expression, as numeric.c computes it: a column's declared scale; add / sub: the larger of the
 * operands' (numeric.c:1659,1698 -> add_var / sub_var: res_dscale = Max); mul: their sum (numeric.c:1735 -> mul_var rscale) */
int num_scale(Ctx &c, int root)
{
	if (c.failed) return 0;
	if (root < 0 || root >= c.pool->nnodes) { fail(c, "bad expression index %d", root); return 0; }
	const gg_expr &e = c.pool->nodes[root];
	if (e.rettype != GG_NUMERICOID) { fail(c, "numeric operator applied to a value of type %d (missing cast)", e.rettype); return 0; }
	if (e.kind == GG_E_VAR)
	{
		const bool inner = e.varno == 1 && !c.inner_as_outer;
		const gg_tupdesc *d = inner ? c.idesc : c.odesc;
		if (!d || e.varattno < 1 || e.varattno > d->natts) { fail(c, "Var attno %d out of range", e.varattno); return 0; }
		const int32_t typmod = d->attrs[e.varattno - 1].atttypmod;
		if (typmod < 4) { fail(c, "numeric column %d has no declared scale: only numeric(p,s) runs on the GPU path", e.varattno); return 0; }
		const int sc = (typmod - 4) & 0xFFFF;
		if (sc > GG_NUM_MAX_SCALE) { fail(c, "numeric column %d: scale %d not supported on the GPU path", e.varattno, sc); return 0; }
		return sc;
	}
	if (e.kind == GG_E_CONST)
	{
		if (e.constlen < 0 || e.constlen > GG_NUM_MAX_SCALE) { fail(c, "numeric constant with display scale %d", e.constlen); return 0; }
		return e.constlen;
	}
	if (e.kind == GG_E_FUNC)
	{
		BinInfo b; int un;
		if (func_info(e.funcid, &b, &un) && b.isbin && (b.k == K_NADD || b.k == K_NSUB || b.k == K_NMUL))
		{
			const int l = num_scale(c, e.args[0]), r = num_scale(c, e.args[1]);
			const int sc = b.k == K_NMUL ? l + r : (l > r ? l : r);
			if (sc > GG_NUM_MAX_SCALE) { fail(c, "numeric expression with display scale %d not supported on the GPU path", sc); return 0; }
			return sc;
		}
	}
	fail(c, "numeric expression (kind %d, function %d) not supported on the GPU path", e.kind, e.funcid);
	return 0;
}

int num_const(Ctx &c, const gg_expr &e, int want)
{
	/* the constant at the wanted scale, computed here: a constant that does not fit is a plan this path does not take */
	__int128 v = (__int128) e.constvalue * (__int128) kPow10[want - e.constlen];
	if (v > INT64_MAX || v < INT64_MIN) { fail(c, "numeric constant out of the 64-bit range at scale %d", want); return 0; }
	return add_const(c, (int64_t) v, e.constisnull != 0);
}

/* acc = value(root) * 10^want, want >= the expression's own scale */
void gen_num(Ctx &c, int root, int want)
{
	if (c.failed) return;
	const gg_expr &e = c.pool->nodes[root];
	const int own = num_scale(c, root);
	if (c.failed) return;
	if (want < own || want > GG_NUM_MAX_SCALE) { fail(c, "numeric expression needs scale %d", want); return; }
	for (int i = 0; i < c.npersist; i++)
		if (expr_equal(c.pool, c.persist_root[i], root))
		{
			emit(c, GGP_LD_T, c.persist_temp[i]);
			if (want > c.persist_scale[i]) emit(c, GGP_IMUL_K, add_const(c, kPow10[want - c.persist_scale[i]], false));
			return;
		}
	if (e.kind == GG_E_VAR)
	{
		const int slot = col_slot(c, e.varno, e.varattno);
		if (c.failed) return;
		if (e.varno == 1 && !c.inner_as_outer)
		{
			/* an inner column above a join: the build program stored it at its own scale (ggp_compile_join) */
			emit(c, GGP_LD_NUM, slot | 0x80, own);
			if (want > own) emit(c, GGP_IMUL_K, add_const(c, kPow10[want - own], false));
			return;
		}
		emit(c, GGP_LD_NUM, slot, want);
		return;
	}
	if (e.kind == GG_E_CONST) { emit(c, GGP_LD_K, num_const(c, e, want)); return; }
	BinInfo b; int un;
	func_info(e.funcid, &b, &un);
	const gg_expr &l = c.pool->nodes[e.args[0]], &r = c.pool->nodes[e.args[1]];
	if (b.k == K_NADD || b.k == K_NSUB)
	{
		/* (a +- b) * 10^k = a * 10^k +- b * 10^k: both operands are produced at the wanted scale */
		if (r.kind == GG_E_CONST) { gen_num(c, e.args[0], want); emit(c, b.k == K_NADD ? GGP_IADD_K : GGP_ISUB_K, num_const(c, r, want)); return; }
		if (l.kind == GG_E_CONST) { gen_num(c, e.args[1], want); emit(c, b.k == K_NADD ? GGP_IADD_K : GGP_IRSUB_K, num_const(c, l, want)); return; }
		gen_num(c, e.args[0], want);
		const int t = alloc_temp(c);
		store_temp(c, t);
		gen_num(c, e.args[1], want);
		emit(c, b.k == K_NADD ? GGP_IADD_T : GGP_IRSUB_T, t);
		c.temps_busy &= ~(1 << t);
		return;
	}
	/* mul: scales add; whatever the caller wants beyond that goes into the left operand */
	const int ls = num_scale(c, e.args[0]), rs = num_scale(c, e.args[1]);
	const int extra = want - (ls + rs);
	if (r.kind == GG_E_CONST) { gen_num(c, e.args[0], ls + extra); emit(c, GGP_IMUL_K, num_const(c, r, rs)); return; }
	if (l.kind == GG_E_CONST) { gen_num(c, e.args[1], rs + extra); emit(c, GGP_IMUL_K, num_const(c, l, ls)); return; }
	gen_num(c, e.args[0], ls + extra);
	const int t = alloc_temp(c);
	store_temp(c, t);
	gen_num(c, e.args[1], rs);
	emit(c, GGP_IMUL_T, t);
	c.temps_busy &= ~(1 << t);
}

/* numeric comparison: both sides at the larger scale, then a signed integer compare (numeric_cmp, numeric.c:1512, orders
 * values, not representations: 1.0 = 1.00) */
void gen_num_cmp(Ctx &c, int lroot, int rroot, int cc)
{
	const int ls = num_scale(c, lroot), rs = num_scale(c, rroot);
	if (c.failed) return;
	const int sc = ls > rs ? ls : rs;
	const gg_expr &r = c.pool->nodes[rroot], &l = c.pool->nodes[lroot];
	if (r.kind == GG_E_CONST) { gen_num(c, lroot, sc); emit(c, GGP_CMPI_K, num_const(c, r, sc), cc); return; }
	if (l.kind == GG_E_CONST) { gen_num(c, rroot, sc); emit(c, GGP_CMPI_K, num_const(c, l, sc), swap_cc(cc)); return; }
	gen_num(c, lroot, sc);
	const int t = alloc_temp(c);
	store_temp(c, t);
	gen_num(c, rroot, sc);
	emit(c, GGP_CMPI_T, t, swap_cc(cc));          /* acc = right, temp = left: left cc right == right swap(cc) left */
	c.temps_busy &= ~(1 << t);
}

void gen(Ctx &c, int root)
{
	if (c.failed) return;
	if (root < 0 || root >= c.pool->nnodes) { fail(c, "bad expression index %d", root); return; }
	const gg_expr &e = c.pool->nodes[root];
	if (e.rettype == GG_NUMERICOID && (e.kind == GG_E_VAR || e.kind == GG_E_CONST || e.kind == GG_E_FUNC)) { gen_num(c, root, num_scale(c, root)); return; }
	Operand o = operand_of(c, root);
	if (o.kind != OPD_NONE || e.kind == GG_E_VAR) { emit_load(c, o, root); return; }

	switch (e.kind)
	{
		case GG_E_FUNC:
		{
			int cc = date_ts_cc(e.funcid);
			if (cc >= 0)
			{
				/* date_xx_timestamp(date, ts): promote the date, then integer compare (date.c:560-640) */
				Operand ro = operand_of(c, e.args[1]);
				if (ro.kind == OPD_K || ro.kind == OPD_C8 || ro.kind == OPD_T)
				{
					gen(c, e.args[0]);
					emit(c, GGP_DATE2TS);
					emit_binop(c, K_CMPI, cc, ro, false);
				}
				else
				{
					gen(c, e.args[1]);
					int t = alloc_temp(c);
					store_temp(c, t);
					gen(c, e.args[0]);
					emit(c, GGP_DATE2TS);
					Operand to = { OPD_T, t };
					emit_binop(c, K_CMPI, cc, to, false);
					c.temps_busy &= ~(1 << t);
				}
				return;
			}
			BinInfo b; int un;
			if (!func_info(e.funcid, &b, &un)) { fail(c, "function %d not supported on the GPU path", e.funcid); return; }
			if (b.k == K_NCMP) { gen_num_cmp(c, e.args[0], e.args[1], b.cc); return; }
			/* the argument types must be the function's own (a planner never emits anything else; a
			 * hand-built plan that does is refused rather than reinterpreting Datum bits) */
			{
				auto is_int = [](int32_t t) { return t == GG_INT4OID || t == GG_INT8OID || t == GG_DATEOID || t == GG_TIMESTAMPOID; };
				auto is_str = [](int32_t t) { return t == GG_BPCHAROID || t == GG_VARCHAROID || t == GG_TEXTOID; };
				int32_t t0 = c.pool->nodes[e.args[0]].rettype;
				int32_t t1 = b.isbin ? c.pool->nodes[e.args[1]].rettype : t0;
				bool ok = true;
				if (b.isbin && (b.k == K_F8ADD || b.k == K_F8SUB || b.k == K_F8MUL || b.k == K_F8DIV || b.k == K_CMPF)) ok = t0 == GG_FLOAT8OID && t1 == GG_FLOAT8OID;
				else if (b.isbin && b.k == K_CMPI) ok = is_int(t0) && is_int(t1);
				else if (b.isbin && b.k == K_CMPS) ok = is_str(t0) && is_str(t1);
				else if (!b.isbin) ok = is_int(t0);
				if (!ok) { fail(c, "function %d applied to arguments of type %d, %d", e.funcid, t0, t1); return; }
			}
			if (!b.isbin)
			{
				gen(c, e.args[0]);
				if (un > 0) emit(c, un);
				return;
			}
			gen_binary(c, e.args[0], e.args[1], b.k, b.cc);
			return;
		}
		case GG_E_AND:
		case GG_E_OR:
			gen_binary(c, e.args[0], e.args[1], e.kind == GG_E_AND ? K_AND : K_OR, 0);
			return;
		case GG_E_NOT: gen(c, e.args[0]); emit(c, GGP_NOT); return;
		case GG_E_ISNULL: gen(c, e.args[0]); emit(c, GGP_ISNULL); c.prog->nullable = 1; return;
		case GG_E_ISNOTNULL: gen(c, e.args[0]); emit(c, GGP_ISNOTNULL); c.prog->nullable = 1; return;
	}
	fail(c, "expression kind %d not supported", e.kind);
}

/* generate an expression whose value must end in a fresh op (so that post-actions can attach) */
ggp_op *gen_value(Ctx &c, int root)
{
	int start = c.prog->ncode;
	c.temps_busy = 0;
	for (int i = 0; i < c.npersist; i++) c.temps_busy |= 1 << c.persist_temp[i];
	gen(c, root);
	return last_op(c, start);
}

/* A plan qual is an implicit-AND list of clauses that ExecQual walks until one is not true (execQual.c:6260-6310; the
 * planner flattens every top-level AND, make_ands_implicit): one FILTER per clause.  A row that failed a clause is not
 * live for the clauses behind it, so they raise nothing for it — what the reference does by never reaching them — and a
 * specialised kernel lets such lanes skip nothing they need. */
void gen_qual(Ctx &c, int qual)
{
	if (qual < 0) return;
	const gg_exprpool *pool = c.pool;
	ggp_program *prog = c.prog;
	int stack[GG_MAX_EXPR_NODES], sp = 0, clauses[GG_MAX_EXPR_NODES], nc = 0, steps = 0;
	stack[sp++] = qual;
	while (sp > 0 && !c.failed)
	{
		const int r = stack[--sp];
		const gg_expr &e = pool->nodes[r];
		/* a pool is a DAG: AND nodes sharing children could be walked exponentially often — bounded, then refused */
		if (++steps > 4 * GG_MAX_EXPR_NODES || nc >= GG_MAX_EXPR_NODES) { fail(c, "qual with too many clauses"); break; }
		if (e.kind == GG_E_AND && sp + 2 <= GG_MAX_EXPR_NODES) { stack[sp++] = e.args[1]; stack[sp++] = e.args[0]; }   /* left clause first */
		else clauses[nc++] = r;
	}
	for (int k = 0; k < nc && !c.failed; k++)
	{
		ggp_op *o = gen_value(c, clauses[k]);
		if (c.failed) break;
		if (o->flags & GGP_F_FILTER) { emit(c, GGP_NOP); o = &prog->code[prog->ncode - 1]; }
		o->flags |= GGP_F_FILTER;
	}
}

}  // namespace

/* grouping keys, GROUP and the aggregate arguments: the part of the row program that is the same for a
 * plain scan and for the per-match segment of a join */
static void compile_agg_part(Ctx &c, const gg_agg *agg, ggp_aggmap *aggmap)
{
	ggp_program *prog = c.prog;
	const gg_exprpool *pool = c.pool;
	/* ---- grouping keys ---- */
	if (agg->numCols < 0 || agg->numCols > GG_MAX_KEYS) fail(c, "too many grouping columns");
	prog->nkeys = agg->numCols;
	for (int i = 0; i < agg->numCols && !c.failed; i++)
	{
		int32_t t = pool->nodes[agg->grpCol[i]].rettype;
		switch (t)
		{
			case GG_INT4OID: case GG_INT8OID: case GG_DATEOID: case GG_TIMESTAMPOID: case GG_BOOLOID: prog->keytype[i] = 1; break;
			case GG_FLOAT8OID: prog->keytype[i] = 2; break;
			case GG_BPCHAROID: case GG_VARCHAROID: case GG_TEXTOID: prog->keytype[i] = 3; break;
			default: fail(c, "grouping column type %d not supported", t);
		}
		ggp_op *o = gen_value(c, agg->grpCol[i]);
		if (c.failed) break;
		if (o->flags & GGP_F_KEY) { emit(c, GGP_NOP); o = &prog->code[prog->ncode - 1]; }
		o->flags |= GGP_F_KEY;
		o->aux = (uint8_t) ((o->aux & 0x3F) | (i << 6));
		if (i == agg->numCols - 1) o->flags |= GGP_F_GROUP;
	}
	if (agg->numCols == 0 && !c.failed)
	{
		emit(c, GGP_NOP);
		prog->code[prog->ncode - 1].flags |= GGP_F_GROUP;
	}
	if (agg->numAggs < 0 || agg->numAggs > GG_MAX_AGGS) fail(c, "too many aggregates");
	if (agg->aggstage == GG_AGGSTAGE_FINAL) fail(c, "FINAL stage runs through gg_agg_final");

	/* ---- aggregate arguments -> deduplicated accumulator columns ---- */
	int accroot[GGP_MAX_ACCS];
	int accnum[GGP_MAX_ACCS];          /* numeric sums live in two int64 columns: 1 = low 32 bits of every input, 2 = the rest */
	bool needsq[GGP_MAX_ACCS], checksq[GGP_MAX_ACCS];
	for (int j = 0; j < GGP_MAX_ACCS; j++) accnum[j] = 0;
	for (int i = 0; i < agg->numAggs && !c.failed; i++)
	{
		const gg_aggref &ar = agg->aggs[i];
		const int kind = ggp_acckind_of(ar.aggfnoid);
		aggmap[i].scale = 0;
		if (kind < 0) { fail(c, "aggregate %d not supported on the GPU path", ar.aggfnoid); continue; }
		if (kind == 0) { aggmap[i].col = -1; continue; }              /* count(*) */
		/* float8_accum also maintains sumX2, which float8_avg ignores (float.c:1982): only a PARTIAL stage,
		 * whose transition state {N, sumX, sumX2} is shipped to another process, has to produce it */
		const int sq = ar.aggfnoid == GG_AGG_AVG_FLOAT8 && agg->aggstage == GG_AGGSTAGE_PARTIAL && !(agg->flags & GG_AGGF_DEVICE_FINAL);
		/* numeric_avg_accum (numeric.c:3057): N and an exact running sum — here a 128-bit integer at the argument's
		 * scale, kept as two int64 sums of the inputs' halves */
		const bool isnum = ar.aggfnoid == GG_AGG_SUM_NUMERIC || ar.aggfnoid == GG_AGG_AVG_NUMERIC;
		if (isnum && agg->aggstage != GG_AGGSTAGE_NORMAL) fail(c, "numeric aggregates run as one-stage aggregates on the GPU path");
		if (ar.arg < 0) { fail(c, "aggregate %d needs an argument", ar.aggfnoid); continue; }
		int found = -1;
		for (int j = 0; j < prog->nacc; j++)
		{
			/* every column kind also counts its non-NULL inputs, so count(x) rides on any column over x —
			 * and a column created for count(x) is upgraded when sum/min/max(x) comes later */
			bool compat = prog->acckind[j] == kind || kind == GGP_ACC_COUNT || prog->acckind[j] == GGP_ACC_COUNT;
			/* a numeric sum is a PAIR of columns: another numeric aggregate over the same argument shares it, count(x) rides on
			 * its low half, nothing else does — and it never takes over a column made for count(x) */
			if (isnum) compat = accnum[j] == 1;
			else if (accnum[j] != 0) compat = kind == GGP_ACC_COUNT && accnum[j] == 1;
			if (compat && expr_equal(pool, accroot[j], ar.arg))
			{
				found = j;
				if (prog->acckind[j] == GGP_ACC_COUNT) prog->acckind[j] = (uint8_t) kind;
				break;
			}
		}
		if (found < 0)
		{
			if (prog->nacc >= GGP_MAX_ACCS) { fail(c, "too many distinct aggregate arguments"); continue; }
			found = prog->nacc++;
			accroot[found] = ar.arg;
			needsq[found] = false;
			checksq[found] = false;
			prog->acckind[found] = (uint8_t) kind;
			if (isnum)
			{
				if (prog->nacc >= GGP_MAX_ACCS) { fail(c, "too many distinct aggregate arguments"); continue; }
				accnum[found] = 1;
				const int hi = prog->nacc++;
				accroot[hi] = ar.arg; accnum[hi] = 2; needsq[hi] = checksq[hi] = false;
				prog->acckind[hi] = GGP_ACC_I8SUM;
			}
		}
		if (isnum) aggmap[i].scale = num_scale(c, ar.arg);
		if (sq) needsq[found] = true;
		/* float8_accum squares every input and CHECKFLOATVALs the running sumX2 (float.c:1895): an avg over a finite value
		 * whose square is not finite is "value out of range: overflow" in the reference even where sumX2 itself is not kept */
		if (ar.aggfnoid == GG_AGG_AVG_FLOAT8 && !sq) checksq[found] = true;
		aggmap[i].col = found;
	}
	/* value slots: column j -> slot j; sums of squares get the slots after them */
	prog->nslots = prog->nacc;
	for (int j = 0; j < prog->nacc; j++)
	{
		prog->accsq[j] = -1;
		if (needsq[j]) prog->accsq[j] = (int8_t) prog->nslots++;
	}
	if (prog->nslots > GGP_MAX_SLOTS) fail(c, "too many aggregate value slots");
	/* A complex argument that reappears inside a later argument stays in a temporary
	 * (e.g. Q1's l_extendedprice*(1-l_discount) inside sum_charge). */
	c.npersist = 0;
	for (int j = 0; j < prog->nacc && !c.failed; j++)
	{
		if (accnum[j] == 2) continue;          /* written together with its low half */
		if (accnum[j] == 1)
		{
			/* acc = the argument at its own scale; kept in a temporary so that both halves can be taken from it (and, when a
			 * later argument contains it — Q1's l_extendedprice * (1 - l_discount) inside sum_charge — for that one too) */
			const int sc = num_scale(c, accroot[j]);
			c.temps_busy = 0;
			for (int i = 0; i < c.npersist; i++) c.temps_busy |= 1 << c.persist_temp[i];
			int t = -1;
			bool persisted = false;
			for (int i = 0; i < c.npersist; i++)
				if (expr_equal(pool, c.persist_root[i], accroot[j]) && c.persist_scale[i] == sc) { t = c.persist_temp[i]; persisted = true; }
			if (t < 0)
			{
				gen_num(c, accroot[j], sc);
				if (c.failed) break;
				t = alloc_temp(c);
				store_temp(c, t);
				const gg_expr &e = pool->nodes[accroot[j]];
				bool reused = false;
				for (int k = j + 2; k < prog->nacc && e.kind == GG_E_FUNC; k++)
					if (accnum[k] == 1 && contains(pool, accroot[k], accroot[j]) && !expr_equal(pool, accroot[k], accroot[j])) reused = true;
				if (reused && c.npersist < 2)
				{
					c.persist_root[c.npersist] = accroot[j]; c.persist_temp[c.npersist] = t; c.persist_scale[c.npersist] = sc;
					c.npersist++;
					persisted = true;
				}
			}
			emit(c, GGP_LD_T, t);
			emit(c, GGP_LO32);
			prog->code[prog->ncode - 1].flags |= GGP_F_OUT; prog->code[prog->ncode - 1].out = (uint8_t) j;
			emit(c, GGP_LD_T, t);
			emit(c, GGP_SAR32);
			prog->code[prog->ncode - 1].flags |= GGP_F_OUT; prog->code[prog->ncode - 1].out = (uint8_t) (j + 1);
			if (!persisted) c.temps_busy &= ~(1 << t);
			continue;
		}
		ggp_op *o = gen_value(c, accroot[j]);
		if (c.failed) break;
		const gg_expr &e = pool->nodes[accroot[j]];
		bool complex_expr = !(e.kind == GG_E_VAR || e.kind == GG_E_CONST);
		bool reused = false;
		for (int k = j + 1; k < prog->nacc && complex_expr; k++)
			if (contains(pool, accroot[k], accroot[j]) && !expr_equal(pool, accroot[k], accroot[j])) reused = true;
		if (reused && c.npersist < 2 && operand_of(c, accroot[j]).kind != OPD_T)
		{
			int t = alloc_temp(c);
			store_temp(c, t);
			o = &prog->code[prog->ncode - 1];
			c.persist_root[c.npersist] = accroot[j];
			c.persist_temp[c.npersist] = t;
			c.persist_scale[c.npersist] = 0;
			c.npersist++;
		}
		if (o->flags & (GGP_F_OUT | GGP_F_OUTSQ)) { emit(c, GGP_NOP); o = &prog->code[prog->ncode - 1]; }
		o->flags |= GGP_F_OUT;
		o->out = (uint8_t) j;
		if (prog->accsq[j] >= 0) { o->flags |= GGP_F_OUTSQ; o->out2 = (uint8_t) prog->accsq[j]; }
		else if (checksq[j]) { o->flags |= GGP_F_OUTSQ; o->out2 = GGP_OUTSQ_CHECK_ONLY; }
	}
	emit(c, GGP_END);
	c.npersist = 0;

	/* private-accumulator kernel: NOT NULL float8 sums and int64 sums (int4_sum over a NOT NULL argument, the halves of a
	 * numeric sum): both are plain adds into a per-thread accumulator */
	prog->priv_ok = !prog->nullable;
	for (int j = 0; j < prog->nacc; j++)
		if (prog->acckind[j] != GGP_ACC_F8SUM && prog->acckind[j] != GGP_ACC_I8SUM) prog->priv_ok = 0;
}


/* ---- structural validation of what crosses the C-ABI ----
 * Nothing below indexes the pool, a descriptor or the aggregate list with a value that was not checked here: a malformed
 * plan is GG_ERR_ARG with a message, never a crash of the backend that loaded the library.  A pool lists children before
 * their parents (gg_plan.h), which is also what rules out cycles; only the nodes reachable from the plan's roots are looked
 * at (a pool may hold the expressions of other pipelines of the same plan tree). */
struct Roots {
	int n = 0;
	int r[4 + 2 * GG_MAX_KEYS + GG_MAX_AGGS + GGP_MAX_ACCS];
	bool ok = true;
	void add(Ctx &c, const gg_exprpool *pool, int root, bool optional, const char *what)
	{
		if (optional && root == -1) return;
		if (root < 0 || root >= pool->nnodes) { fail(c, "%s: node %d is not in the pool (%d nodes)", what, root, pool->nnodes); ok = false; return; }
		if (n < (int) (sizeof r / sizeof r[0])) r[n++] = root;
	}
};

static bool valid_nodes(Ctx &c, const gg_exprpool *pool, const gg_tupdesc *odesc, const gg_tupdesc *idesc, const Roots &roots)
{
	bool used[GG_MAX_EXPR_NODES];
	memset(used, 0, sizeof used);
	for (int i = 0; i < roots.n; i++) used[roots.r[i]] = true;
	for (int i = pool->nnodes - 1; i >= 0; i--)        /* children have smaller indices: one descending sweep reaches everything */
	{
		if (!used[i]) continue;
		const gg_expr &e = pool->nodes[i];
		int need = 0;
		switch (e.kind)
		{
			case GG_E_VAR:
			{
				const gg_tupdesc *d = e.varno == 0 ? odesc : (e.varno == 1 ? idesc : nullptr);
				if (!d) { fail(c, "node %d: Var of relation %d, which this plan does not have", i, e.varno); return false; }
				if (e.varattno < 1 || e.varattno > d->natts) { fail(c, "node %d: Var attribute %d out of range (1..%d)", i, e.varattno, d->natts); return false; }
				break;
			}
			case GG_E_CONST: break;
			case GG_E_FUNC:
			{
				BinInfo b; int un;
				need = (func_info(e.funcid, &b, &un) && b.isbin) ? 2 : 1;     /* an unknown function is refused where it is compiled */
				break;
			}
			case GG_E_AND: case GG_E_OR: need = 2; break;
			case GG_E_NOT: case GG_E_ISNULL: case GG_E_ISNOTNULL: need = 1; break;
			default: fail(c, "node %d: expression kind %d not supported", i, e.kind); return false;
		}
		if (need && (e.nargs < need || e.nargs > 2)) { fail(c, "node %d: %d arguments where %d are needed", i, e.nargs, need); return false; }
		for (int k = 0; k < need; k++)
		{
			if (e.args[k] < 0 || e.args[k] >= i) { fail(c, "node %d: argument %d is node %d (children come before their parents)", i, k, e.args[k]); return false; }
			used[e.args[k]] = true;
		}
	}
	return true;
}

static bool valid_header(Ctx &c, const gg_exprpool *pool, const gg_tupdesc *odesc, const gg_tupdesc *idesc)
{
	if (pool->nnodes < 0 || pool->nnodes > GG_MAX_EXPR_NODES) { fail(c, "expression pool with %d nodes (0..%d)", pool->nnodes, GG_MAX_EXPR_NODES); return false; }
	if (odesc->natts < 0 || odesc->natts > GG_MAX_ATTS || (idesc && (idesc->natts < 0 || idesc->natts > GG_MAX_ATTS))) { fail(c, "descriptor with too many attributes"); return false; }
	return true;
}

static bool add_agg_roots(Ctx &c, const gg_agg *agg, const gg_exprpool *pool, Roots &roots)
{
	if (agg->numCols < 0 || agg->numCols > GG_MAX_KEYS) { fail(c, "%d grouping columns (0..%d)", agg->numCols, GG_MAX_KEYS); return false; }
	if (agg->numAggs < 0 || agg->numAggs > GG_MAX_AGGS) { fail(c, "%d aggregates (0..%d)", agg->numAggs, GG_MAX_AGGS); return false; }
	if (agg->aggstage == GG_AGGSTAGE_FINAL) return true;            /* grpCol carries type OIDs there; refused by compile_agg_part */
	for (int i = 0; i < agg->numCols; i++) roots.add(c, pool, agg->grpCol[i], false, "grouping column");
	for (int i = 0; i < agg->numAggs; i++) roots.add(c, pool, agg->aggs[i].arg, true, "aggregate argument");
	return roots.ok;
}

int ggp_compile_scanagg(const gg_scan *scan, const gg_agg *agg, const gg_exprpool *pool,
                        ggp_program *prog, ggp_aggmap *aggmap, char *err, int errlen)
{
	Ctx c;
	memset(prog, 0, sizeof *prog);
	memset(&c, 0, sizeof c);
	c.pool = pool; c.prog = prog; c.outer = &prog->outer; c.inner = nullptr;
	c.odesc = &scan->desc; c.idesc = nullptr; c.err = err; c.errlen = errlen;
	if (err && errlen) err[0] = 0;
	{
		Roots roots;
		if (!valid_header(c, pool, &scan->desc, nullptr)) return GG_ERR_ARG;
		roots.add(c, pool, scan->qual, true, "scan qual");
		if (!add_agg_roots(c, agg, pool, roots) || !roots.ok || !valid_nodes(c, pool, &scan->desc, nullptr, roots)) return GG_ERR_ARG;
	}

	if (scan->desc.natts < 0 || scan->desc.natts > GG_MAX_ATTS) { fail(c, "too many attributes"); return GG_ERR_UNSUPPORTED; }
	for (int i = 0; i < scan->desc.natts; i++)
	{
		const gg_attr &a = scan->desc.attrs[i];
		if (!(a.attlen == -1 || a.attlen == 1 || a.attlen == 2 || a.attlen == 4 || a.attlen == 8))
		{ fail(c, "attribute %d: attlen %d not supported", i + 1, a.attlen); return GG_ERR_UNSUPPORTED; }
	}
	init_side(&prog->outer, &scan->desc);

	/* ---- scan qual ---- */
	gen_qual(c, scan->qual);
	compile_agg_part(c, agg, aggmap);
	if (c.failed) return GG_ERR_UNSUPPORTED;
	return GG_OK;
}

static bool check_desc(Ctx &c, const gg_tupdesc *d)
{
	if (d->natts < 0 || d->natts > GG_MAX_ATTS) { fail(c, "too many attributes"); return false; }
	if (d->format == GG_FMT_DATUMROWS) return true;
	for (int i = 0; i < d->natts; i++)
	{
		const gg_attr &a = d->attrs[i];
		if (!(a.attlen == -1 || a.attlen == 1 || a.attlen == 2 || a.attlen == 4 || a.attlen == 8))
		{ fail(c, "attribute %d: attlen %d not supported", i + 1, a.attlen); return false; }
	}
	return true;
}

/* The key type (ggp_program::keytype) of a join key pair, or 0 when the reference cannot hash-join the pair: both sides must
 * be in one hash opfamily (pg_amop.h:557-565 and the hash opclasses of pg_opclass.h).  Only integer_ops is cross-type here
 * (int4 = int8; both load sign-extended to 64 bits and hashint8 agrees with hashint4 on int4 values).  Date, timestamp, bool,
 * float8 and bpchar each hash only against their own type — date = timestamp compares days with microseconds, bpchar strips
 * blanks where text does not — and varchar uses text's operators (text_ops). */
static int join_keytype(int32_t outer, int32_t inner)
{
	const bool oint = outer == GG_INT4OID || outer == GG_INT8OID, iint = inner == GG_INT4OID || inner == GG_INT8OID;
	const bool otext = outer == GG_VARCHAROID || outer == GG_TEXTOID, itext = inner == GG_VARCHAROID || inner == GG_TEXTOID;
	if (oint && iint) return 1;
	if (otext && itext) return 3;
	if (outer != inner) return 0;
	switch (outer)
	{
		case GG_DATEOID: case GG_TIMESTAMPOID: case GG_BOOLOID: return 1;
		case GG_FLOAT8OID: return 2;
		case GG_BPCHAROID: return 3;
	}
	return 0;
}

/* does the expression at `root` (a validated pool) read a column of side `varno` */
static bool refs_side(const gg_exprpool *pool, int root, int varno)
{
	const gg_expr &e = pool->nodes[root];
	if (e.kind == GG_E_VAR) return e.varno == varno;
	const int n = e.kind == GG_E_CONST ? 0 : (e.nargs < 2 ? e.nargs : 2);
	for (int k = 0; k < n; k++)
		if (e.args[k] >= 0 && e.args[k] < root && refs_side(pool, e.args[k], varno)) return true;     /* children come first */
	return false;
}

/* the per-match piece of a join with a target list: claim a row, then one output column per target (what ggp_compile_motion
 * gives its payload, without the hash keys) */
static void compile_rows_part(Ctx &c, const int32_t *targets, int ntargets)
{
	ggp_program *prog = c.prog;
	emit(c, GGP_NOP);
	prog->code[prog->ncode - 1].flags |= GGP_F_GROUP;
	for (int p = 0; p < ntargets && !c.failed; p++)
	{
		const int32_t t = c.pool->nodes[targets[p]].rettype;
		if (t == GG_NUMERICOID) { fail(c, "join target %d: numeric columns do not travel as datum rows yet", p); break; }
		if (!loadtype_of(t)) { fail(c, "join target %d: type %d not supported", p, t); break; }
		ggp_op *o = gen_value(c, targets[p]);
		if (c.failed) break;
		if (o->flags & (GGP_F_OUT | GGP_F_GROUP)) { emit(c, GGP_NOP); o = &prog->code[prog->ncode - 1]; }
		o->flags |= GGP_F_OUT;
		o->out = (uint8_t) p;
	}
	emit(c, GGP_END);
	prog->nkeys = 0;
	prog->nslots = ntargets;
	prog->priv_ok = 0;
}

/* HashJoin + Agg (agg != nullptr), or HashJoin with a target list (agg == nullptr): see ggp_joinprog in gg_program.h.  Stands
 * where ExecInitHashJoin / ExecInitHash prepare hj_OuterHashKeys / hashkeys and the hash functions (nodeHashjoin.c:540-750,
 * nodeHash.c:270-450). */
static int compile_join(const gg_scan *outer, const gg_scan *inner, const gg_hashjoin *hj, const gg_agg *agg, const int32_t *targets,
                        int ntargets, const gg_exprpool *pool, ggp_joinprog *jp, ggp_aggmap *aggmap, char *err, int errlen)
{
	Ctx c;
	memset(jp, 0, sizeof *jp);
	memset(&c, 0, sizeof c);
	c.pool = pool; c.err = err; c.errlen = errlen;
	if (err && errlen) err[0] = 0;
	if (hj->nkeys < 1 || hj->nkeys > 2) { fail(c, "hash join with %d keys not supported (1 or 2)", hj->nkeys); return GG_ERR_UNSUPPORTED; }
	if (!agg && (ntargets < 1 || ntargets > 16)) { fail(c, "join projecting %d columns (1..16 travel as datum rows)", ntargets); return GG_ERR_UNSUPPORTED; }
	{
		Roots roots;
		if (!valid_header(c, pool, &outer->desc, &inner->desc)) return GG_ERR_ARG;
		roots.add(c, pool, outer->qual, true, "outer scan qual");
		roots.add(c, pool, inner->qual, true, "inner scan qual");
		roots.add(c, pool, hj->joinqual, true, "join qual");
		for (int k = 0; k < hj->nkeys; k++)
		{
			roots.add(c, pool, hj->outerkey[k], false, "outer join key");
			roots.add(c, pool, hj->innerkey[k], false, "inner join key");
		}
		if (agg) { if (!add_agg_roots(c, agg, pool, roots)) return GG_ERR_ARG; }
		else
			for (int p = 0; p < ntargets; p++) roots.add(c, pool, targets[p], false, "join target");
		if (!roots.ok || !valid_nodes(c, pool, &outer->desc, &inner->desc, roots)) return GG_ERR_ARG;
	}
	switch (hj->jointype)
	{
		case GG_JOIN_INNER: case GG_JOIN_LEFT: case GG_JOIN_FULL: case GG_JOIN_RIGHT:
		case GG_JOIN_SEMI: case GG_JOIN_ANTI: case GG_JOIN_LASJ_NOTIN:
			break;
		default:
			fail(c, "join type %d not supported", hj->jointype);
			return GG_ERR_UNSUPPORTED;
	}
	/* a semi / anti join returns outer rows only (the matched inner row is not part of its result) */
	if (!agg && (hj->jointype == GG_JOIN_SEMI || hj->jointype == GG_JOIN_ANTI || hj->jointype == GG_JOIN_LASJ_NOTIN))
		for (int p = 0; p < ntargets; p++)
			if (refs_side(pool, targets[p], 1))
			{ fail(c, "join target %d reads an inner column: a semi or anti join returns outer rows only", p); return GG_ERR_UNSUPPORTED; }
	/* a side that can come back null-extended makes every expression above the join nullable */
	const bool nullext = hj->jointype != GG_JOIN_INNER && hj->jointype != GG_JOIN_SEMI;
	jp->nkeys = hj->nkeys;
	jp->jointype = hj->jointype;

	/* ---- probe program: outer tuple scanned, inner columns = payload slots ---- */
	c.prog = &jp->probe;
	c.outer = &jp->probe.outer;
	ggp_side innerside;
	c.inner = &innerside;
	c.odesc = &outer->desc;
	c.idesc = &inner->desc;
	if (!check_desc(c, &outer->desc) || !check_desc(c, &inner->desc)) return GG_ERR_UNSUPPORTED;
	init_side(&jp->probe.outer, &outer->desc);
	init_side(&innerside, &inner->desc);
	gen_qual(c, outer->qual);
	for (int k = 0; k < hj->nkeys && !c.failed; k++)
	{
		const int kt = join_keytype(pool->nodes[hj->outerkey[k]].rettype, pool->nodes[hj->innerkey[k]].rettype);
		if (!kt) { fail(c, "join key %d: types %d / %d share no hash opfamily", k, pool->nodes[hj->outerkey[k]].rettype, pool->nodes[hj->innerkey[k]].rettype); break; }
		jp->keytype[k] = (uint8_t) kt;
		ggp_op *o = gen_value(c, hj->outerkey[k]);
		if (c.failed) break;
		if (o->flags & GGP_F_KEY) { emit(c, GGP_NOP); o = &jp->probe.code[jp->probe.ncode - 1]; }
		o->flags |= GGP_F_KEY;
		o->aux = (uint8_t) ((o->aux & 0x3F) | (k << 6));
		if (k == hj->nkeys - 1) o->flags |= GGP_F_PROBE;
	}
	jp->probe_pc = jp->probe.ncode;
	if (hj->joinqual >= 0 && !c.failed)
	{
		/* one FILTER for the whole join qual: an ANTI join evaluates it on a match without emitting (the sink takes the
		 * lane out after the FILTER), so clauses cannot be separate FILTERs here; AND arms are guarded all the same */
		ggp_op *o = gen_value(c, hj->joinqual);
		if (!c.failed) o->flags |= GGP_F_FILTER;
	}
	if (nullext) jp->probe.nullable = 1;
	if (!c.failed) { if (agg) compile_agg_part(c, agg, aggmap); else compile_rows_part(c, targets, ntargets); }
	jp->npayload = innerside.ncols;
	if (nullext) { jp->probe.nullable = 1; jp->probe.priv_ok = 0; }

	/* ---- build program: inner tuple scanned; keys, then the payload columns in slot order ---- */
	Ctx b;
	memset(&b, 0, sizeof b);
	b.pool = pool; b.err = err; b.errlen = errlen;
	b.failed = c.failed;
	b.prog = &jp->build;
	b.outer = &jp->build.outer;
	b.inner = nullptr;
	b.odesc = &inner->desc;
	b.idesc = nullptr;
	b.inner_as_outer = true;
	init_side(&jp->build.outer, &inner->desc);
	if (!b.failed) gen_qual(b, inner->qual);
	for (int k = 0; k < hj->nkeys && !b.failed; k++)
	{
		ggp_op *o = gen_value(b, hj->innerkey[k]);
		if (b.failed) break;
		if (o->flags & GGP_F_KEY) { emit(b, GGP_NOP); o = &jp->build.code[jp->build.ncode - 1]; }
		o->flags |= GGP_F_KEY;
		o->aux = (uint8_t) ((o->aux & 0x3F) | (k << 6));
		if (k == hj->nkeys - 1) o->flags |= GGP_F_GROUP;       /* keys complete: claim the hash-table slot */
	}
	for (int p = 0; p < innerside.ncols && !b.failed; p++)
	{
		/* payload slot p = inner attribute colatt[p], loaded the way the probe side expects to read it */
		int att = innerside.colatt[p];
		int slot = col_slot(b, 1, att + 1);
		if (b.failed) break;
		int lt = innerside.coltype[p];
		if (lt == GGP_LT_NUM)
		{
			/* a numeric travels as its scaled integer at the column's declared scale; the probe rescales it (gen_num) */
			const int32_t typmod = inner->desc.attrs[att].atttypmod;
			const int sc = (typmod - 4) & 0xFFFF;
			if (typmod < 4 || sc > GG_NUM_MAX_SCALE) { fail(b, "numeric inner column %d: only numeric(p,s) with s <= %d travels above a join", att + 1, GG_NUM_MAX_SCALE); break; }
			emit(b, GGP_LD_NUM, slot, sc);
		}
		else
			emit(b, lt == GGP_LT_I4 ? GGP_LD_C4 : lt == GGP_LT_I8 ? GGP_LD_C8 : lt == GGP_LT_BPCHAR ? GGP_LD_BP : lt == GGP_LT_VARCHAR ? GGP_LD_VS : GGP_LD_BOOL, slot);
		ggp_op *o = &jp->build.code[jp->build.ncode - 1];
		o->flags |= GGP_F_OUT;
		o->out = (uint8_t) p;
	}
	if (!b.failed) emit(b, GGP_END);
	jp->build.nkeys = hj->nkeys;
	for (int k = 0; k < hj->nkeys; k++) jp->build.keytype[k] = jp->keytype[k];
	if (c.failed || b.failed) return GG_ERR_UNSUPPORTED;
	return GG_OK;
}

int ggp_compile_join(const gg_scan *outer, const gg_scan *inner, const gg_hashjoin *hj, const gg_agg *agg,
                     const gg_exprpool *pool, ggp_joinprog *jp, ggp_aggmap *aggmap, char *err, int errlen)
{
	return compile_join(outer, inner, hj, agg, nullptr, 0, pool, jp, aggmap, err, errlen);
}

int ggp_compile_joinrows(const gg_scan *outer, const gg_scan *inner, const gg_hashjoin *hj, const int32_t *targets, int ntargets,
                         const gg_exprpool *pool, ggp_joinprog *jp, char *err, int errlen)
{
	return compile_join(outer, inner, hj, nullptr, targets, ntargets, pool, jp, nullptr, err, errlen);
}

/* Redistribute Motion (nodeMotion.c:1481-1687): which tuples go where, and what travels */
int ggp_compile_motion(const gg_scan *scan, const gg_exprpool *pool, const int32_t *hashkeys, int nkeys,
                       const int32_t *payload, int npayload, ggp_program *prog, uint8_t *hashtype,
                       char *err, int errlen)
{
	Ctx c;
	memset(prog, 0, sizeof *prog);
	memset(&c, 0, sizeof c);
	c.pool = pool; c.prog = prog; c.outer = &prog->outer; c.odesc = &scan->desc; c.err = err; c.errlen = errlen;
	if (err && errlen) err[0] = 0;
	if (nkeys < 1 || nkeys > GG_MAX_KEYS) { fail(c, "motion with %d hash keys not supported", nkeys); return GG_ERR_UNSUPPORTED; }
	if (npayload < 1 || npayload > GGP_MAX_ACCS) { fail(c, "motion with %d output columns not supported (1..%d)", npayload, GGP_MAX_ACCS); return GG_ERR_UNSUPPORTED; }
	{
		Roots roots;
		if (!valid_header(c, pool, &scan->desc, nullptr)) return GG_ERR_ARG;
		roots.add(c, pool, scan->qual, true, "scan qual");
		for (int k = 0; k < nkeys; k++) roots.add(c, pool, hashkeys[k], false, "hash key");
		for (int k = 0; k < npayload; k++) roots.add(c, pool, payload[k], false, "output column");
		if (!roots.ok || !valid_nodes(c, pool, &scan->desc, nullptr, roots)) return GG_ERR_ARG;
	}
	if (!check_desc(c, &scan->desc)) return GG_ERR_UNSUPPORTED;
	init_side(&prog->outer, &scan->desc);
	gen_qual(c, scan->qual);
	for (int k = 0; k < nkeys && !c.failed; k++)
	{
		hashtype[k] = (uint8_t) ggp_hashtype_of(pool->nodes[hashkeys[k]].rettype);
		if (!hashtype[k]) { fail(c, "hash key %d: type %d has no GPU hash function", k, pool->nodes[hashkeys[k]].rettype); break; }
		ggp_op *o = gen_value(c, hashkeys[k]);
		if (c.failed) break;
		if (o->flags & GGP_F_KEY) { emit(c, GGP_NOP); o = &prog->code[prog->ncode - 1]; }
		o->flags |= GGP_F_KEY;
		o->aux = (uint8_t) ((o->aux & 0x3F) | (k << 6));
		if (k == nkeys - 1) o->flags |= GGP_F_GROUP;
	}
	for (int p = 0; p < npayload && !c.failed; p++)
	{
		if (!loadtype_of(pool->nodes[payload[p]].rettype)) { fail(c, "output column %d: type %d not supported", p, pool->nodes[payload[p]].rettype); break; }
		ggp_op *o = gen_value(c, payload[p]);
		if (c.failed) break;
		if (o->flags & (GGP_F_OUT | GGP_F_GROUP)) { emit(c, GGP_NOP); o = &prog->code[prog->ncode - 1]; }
		o->flags |= GGP_F_OUT;
		o->out = (uint8_t) p;
	}
	if (!c.failed) emit(c, GGP_END);
	prog->nkeys = nkeys;
	prog->nslots = npayload;
	if (c.failed) return GG_ERR_UNSUPPORTED;
	return GG_OK;
}

/* human-readable listing of a compiled program (debugging, DESIGN.md examples) */
int ggp_disasm(const ggp_program *p, char *buf, int cap)
{
	static const char *const N[] = { "END", "LD_C4", "LD_C8", "LD_BP", "LD_VS", "LD_BOOL", "LD_K", "LD_T",
		"ADD_C", "ADD_K", "ADD_T", "SUB_C", "SUB_K", "SUB_T", "RSUB_C", "RSUB_K", "RSUB_T", "MUL_C", "MUL_K", "MUL_T",
		"DIV_C", "DIV_K", "DIV_T", "RDIV_C", "RDIV_K", "RDIV_T", "CMPF_C", "CMPF_K", "CMPF_T",
		"CMPI_C4", "CMPI_C8", "CMPI_K", "CMPI_T", "CMPS_K", "CMPS_T", "DATE2TS", "I2F8", "AND_T", "OR_T",
		"NOT", "ISNULL", "ISNOTNULL", "NOP", "GUARD_AND", "GUARD_OR", "UNGUARD",
		"LD_NUM", "IADD_K", "IADD_T", "ISUB_K", "ISUB_T", "IRSUB_K", "IRSUB_T", "IMUL_K", "IMUL_T", "LO32", "SAR32" };
	int n = 0;
	for (int i = 0; i < p->ncode && n < cap - 96; i++)
	{
		const ggp_op &o = p->code[i];
		n += snprintf(buf + n, (size_t) (cap - n), "%3d %-8s idx=%-3d cc=%d off=%-5d", i,
		              o.op < GGP_NOPS ? N[o.op] : "?", o.idx, o.aux & 7, o.off == 0xFFFF ? -1 : (int) o.off);
		if (o.flags & GGP_F_ST) n += snprintf(buf + n, (size_t) (cap - n), " ST t%d", (o.aux >> 4) & 3);
		if (o.flags & GGP_F_FILTER) n += snprintf(buf + n, (size_t) (cap - n), " FILTER");
		if (o.flags & GGP_F_KEY) n += snprintf(buf + n, (size_t) (cap - n), " KEY%d", (o.aux >> 6) & 3);
		if (o.flags & GGP_F_GROUP) n += snprintf(buf + n, (size_t) (cap - n), " GROUP");
		if (o.flags & GGP_F_PROBE) n += snprintf(buf + n, (size_t) (cap - n), " PROBE");
		if (o.flags & GGP_F_OUT) n += snprintf(buf + n, (size_t) (cap - n), " OUT%d", o.out);
		if (o.flags & GGP_F_OUTSQ) n += o.out2 == GGP_OUTSQ_CHECK_ONLY ? snprintf(buf + n, (size_t) (cap - n), " SQCHECK") : snprintf(buf + n, (size_t) (cap - n), " OUTSQ%d", o.out2);
		n += snprintf(buf + n, (size_t) (cap - n), "\n");
	}
	return n;
}
