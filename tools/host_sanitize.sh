#!/bin/bash
# AddressSanitizer + UndefinedBehaviorSanitizer over the HOST side of the library (handle management, the explicit
# host path of every family, the C ABI): builds a sanitized copy of libbsuite_b200.so under /tmp and runs the whole
# CPU test-suite and the ABI fuzzer (tools/fuzz_abi.py) against it (BSB_LIBRARY points the ctypes binding at that
# build).  No GPU needed.
#   bash tools/host_sanitize.sh [logfile]
set -e
OUT=/tmp/bsb_asan
LOG=${1:-/tmp/bsb_asan/run.log}
mkdir -p $OUT && rm -f $OUT/*.o
cd "$(dirname "$0")/../bsuite_b200/csrc"
# the translation units of the library as bsuite_b200/build.py lists them: "name source [defines]" per line
python -c "import sys; sys.path.insert(0, '../..'); from bsuite_b200 import build
for name, source, defines in build.UNITS: print(name, source, *defines)" \
  | xargs -P 16 -L 1 sh -c "nvcc -gencode arch=compute_90a,code=sm_90a -O1 -std=c++17 --fmad=false \
  -Xcompiler -fPIC,-ffp-contract=off,-O1,-g,-fsanitize=address,-fsanitize=undefined,-fno-omit-frame-pointer \$2 -c \$1 -o $OUT/\$0.o"
nvcc -shared -o $OUT/libbsuite_b200.so $OUT/*.o -cudart static -ldl -Xcompiler -fsanitize=address,-fsanitize=undefined 2>/dev/null
cd ../..
set +e
LD_PRELOAD="$(gcc -print-file-name=libasan.so) $(gcc -print-file-name=libubsan.so)" ASAN_OPTIONS=detect_leaks=0 \
  UBSAN_OPTIONS=print_stacktrace=1 BSB_LIBRARY=$OUT/libbsuite_b200.so \
  python -m pytest tests -q -m "not gpu" -p no:cacheprovider > "$LOG" 2>&1
echo "pytest rc=$?" >> "$LOG"
LD_PRELOAD="$(gcc -print-file-name=libasan.so) $(gcc -print-file-name=libubsan.so)" ASAN_OPTIONS=detect_leaks=0 \
  UBSAN_OPTIONS=print_stacktrace=1 BSB_LIBRARY=$OUT/libbsuite_b200.so python tools/fuzz_abi.py 3000 0 >> "$LOG" 2>&1
echo "fuzz rc=$?" >> "$LOG"
echo "sanitizer reports: $(grep -c 'runtime error\|AddressSanitizer' "$LOG")" >> "$LOG"
tail -5 "$LOG"
