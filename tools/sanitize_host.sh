#!/bin/bash
# AddressSanitizer + UBSan over the HOST side of the library (layout, quant schedule, sparse format, VLC walker / parser):
# builds an instrumented copy, swaps it in for the CPU tests, restores the real library.  No GPU needed.
set -e
cd "$(dirname "$0")/.."
LIB=cineform-sdk_b200/libcfhd_b200.so
TMP=$(mktemp -d)
(cd cineform-sdk_b200/csrc && ${NVCC:-/usr/local/cuda/bin/nvcc} -gencode arch=compute_90a,code=sm_90a -O1 -g -std=c++17 \
    -Xcompiler -fPIC,-fvisibility=hidden,-fsanitize=address,-fsanitize=undefined,-fno-omit-frame-pointer -cudart static -shared \
    -o "$TMP/libsan.so" *.cu -lpthread)
cp "$LIB" "$TMP/real.so"
trap 'cp "$TMP/real.so" "$LIB"; rm -rf "$TMP"' EXIT
cp "$TMP/libsan.so" "$LIB"
export ASAN_OPTIONS=detect_leaks=0 UBSAN_OPTIONS=print_stacktrace=1
export LD_PRELOAD="$(gcc -print-file-name=libasan.so) $(gcc -print-file-name=libubsan.so)"
if [ "$1" = "--fuzz" ]; then
    python tools/fuzz_host.py "${2:-300}"        # random code sets / band streams / damaged sparse buffers
else
    python -m pytest tests -q -m "not gpu" -x -s -p no:cacheprovider --deselect tests/test_c_example.py --ignore tests/test_launch_geometry.py
fi
