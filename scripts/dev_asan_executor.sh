#!/bin/bash
# Run the executor-node host code (greengage_b200/host/gg_executor.c + gg_motion_host.c) under AddressSanitizer +
# UndefinedBehaviorSanitizer on a CPU-only box: the oracle-backed stand-in for the device library (tests/mock/ggb200_mock.c)
# answers the C-ABI, the single-segment control-flow checks and the two-segment dispatched Q1 / co-located join of
# tests/test_executor_multiseg.py drive it; the single-segment case of tests/test_executor_window.py drives the datum-row paths
# (hand-up, read-back, upload) over the window stand-in (tests/mock/ggb200_mock_window.c).  Prints the sanitizer reports, if any.
# Usage: scripts/dev_asan_executor.sh
set -e
cd "$(dirname "$0")/.."
OUT=$(mktemp -d)
SAN="-O1 -g -fPIC -fsanitize=address,undefined -fno-omit-frame-pointer"
for f in greengage_b200/host/gg_executor.c greengage_b200/host/gg_motion_host.c greengage_b200/host/gg_tupser.c tests/mock/ggb200_mock.c; do gcc $SAN -std=gnu11 -c $f -o "$OUT/$(basename $f).o"; done
for f in tests/mock/compile_glue.cpp greengage_b200/csrc/gg_compile.cpp; do g++ $SAN -std=c++17 -c $f -o "$OUT/$(basename $f).o"; done
g++ -shared -fsanitize=address,undefined -o "$OUT/libggexec_mock_asan.so" "$OUT"/*.o -L oracle -lggoracle -Wl,-rpath,"$PWD/oracle" -lm
# the window stand-in: ggb200_mock.c with its refusing relation functions renamed out of the way, as the test builds it
mkdir "$OUT/window"
RENAMES=$(for f in gg_relation_create gg_relation_attach_rows gg_relation_read gg_relation_device_ptr gg_relation_free gg_sort_datumrows; do echo "-D$f=mockbase_${f#gg_}"; done)
gcc $SAN -std=gnu11 $RENAMES -c tests/mock/ggb200_mock.c -o "$OUT/window/ggb200_mock.c.o"
for f in tests/mock/ggb200_mock_window.c tests/window_ref.c; do gcc $SAN -std=gnu11 -c $f -o "$OUT/window/$(basename $f).o"; done
g++ -shared -fsanitize=address,undefined -o "$OUT/libggexec_mock_window_asan.so" $(ls "$OUT"/*.o | grep -v '/ggb200_mock\.c\.o$') "$OUT"/window/*.o \
    -L oracle -lggoracle -Wl,-rpath,"$PWD/oracle" -lm
cat > "$OUT/worker.py" <<PY
import ctypes as C, sys
sys.path.insert(0, "$PWD"); sys.path.insert(0, "$PWD/tests")
import test_executor_multiseg as t
class Q:
    def put(self, x):
        print("RESULT", x[0], x[1], x[2] if x[0] == "err" else (x[2], x[3] if x[2] == "single" else len(x[3])))
t._worker(int(sys.argv[1]), int(sys.argv[2]), 29871, "$OUT/libggexec_mock_asan.so", sys.argv[3], Q())
PY
export LD_PRELOAD="$(gcc -print-file-name=libasan.so) $(gcc -print-file-name=libubsan.so)" ASAN_OPTIONS=detect_leaks=0
python "$OUT/worker.py" 0 1 single 2>&1 | grep -E "RESULT|AddressSanitizer|runtime error" || true
cat > "$OUT/window_worker.py" <<PY
import sys
sys.path.insert(0, "$PWD"); sys.path.insert(0, "$PWD/tests")
import test_executor_window as t
class Q:
    def put(self, x):
        print("RESULT window", x[0], x[2])
t._worker(0, 1, 29871, "$OUT/libggexec_mock_window_asan.so", "single", Q())
PY
python "$OUT/window_worker.py" 2>&1 | grep -E "RESULT|AddressSanitizer|runtime error" || true
for c in q1 join; do
    for r in 0 1; do python "$OUT/worker.py" $r 2 $c > "$OUT/$c.$r.log" 2>&1 & done
    wait
    grep -hE "RESULT|AddressSanitizer|runtime error" "$OUT"/$c.*.log || true
done
rm -rf "$OUT"
