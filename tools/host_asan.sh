#!/bin/bash
# Host-side sanitizer pass (no GPU needed): rebuild rb200_host.cu / rb200_shard.cu with
# -fsanitize=address,undefined, link them with the product's device objects into a scratch library
# and run the CPU-executable paths (portable (de)serializer, blob algebra, mutation fuzz, host ABI
# tests) against it.      bash tools/host_asan.sh > host_asan.txt 2>&1
set -e
ROOT=$(cd "$(dirname "$0")/.." && pwd)
OUT=${TMPDIR:-/tmp}/rb200_asan
mkdir -p "$OUT"
python -m croaring_b200.build > /dev/null            # the product's objects (device code)
cd "$ROOT/croaring_b200/csrc"
for f in rb200_host rb200_shard; do
  nvcc -O1 -g -std=c++17 -gencode arch=compute_90a,code=sm_90a --expt-relaxed-constexpr -cudart static -DRB200_BUILDING_LIBRARY \
       -Xcompiler -fPIC,-fvisibility=hidden,-fsanitize=address,-fsanitize=undefined,-fno-omit-frame-pointer \
       -c $f.cu -o "$OUT/$f.o" 2>&1 | grep -v deprecated || true
done
nvcc -shared -cudart static -o "$OUT/libroaring_b200_asan.so" "$OUT/rb200_host.o" "$OUT/rb200_shard.o" \
     rb200_kernels.o rb200_many.o rb200_many2.o rb200_convert.o rb200_fused.o \
     -Xlinker -Bsymbolic -ldl -lpthread -Xcompiler -fsanitize=address,-fsanitize=undefined 2>&1 | grep -v deprecated || true
cd "$ROOT"
export RB200_LIB="$OUT/libroaring_b200_asan.so" ASAN_OPTIONS=detect_leaks=0 UBSAN_OPTIONS=print_stacktrace=1
export LD_PRELOAD="$(gcc -print-file-name=libasan.so) $(gcc -print-file-name=libubsan.so)"
python -m pytest tests/test_host_abi.py tests/test_sharding_gloo.py -q -k "not world2 and not exports and not type_rules" 2>&1 | tail -n 4
