#!/usr/bin/env bash
# Build libfastlivo_b200.so in-tree for sm_90a (H100; cross-compiles without a GPU).
#   -fmad=false : every a*b+c rounds twice, like the reference's x86-64 build (no FMA
#                 contraction) -- this is what makes the float32 plane fit / photometric
#                 taps bit-exact against the oracle.
set -euo pipefail
HERE="$(cd "$(dirname "${BASH_SOURCE[0]}")" && pwd)"
NVCC="${NVCC:-/usr/local/cuda/bin/nvcc}"
OUT="$HERE/libfastlivo_b200.so"
"$NVCC" -std=c++17 -O3 -gencode arch=compute_90a,code=sm_90a -lineinfo -fmad=false \
    -ccbin /usr/bin/g++ -Xcompiler -fPIC,-O3,-Wall,-Wno-unknown-pragmas,-ffp-contract=off -shared \
    ${FLB_PTXAS_V:+-Xptxas -v} \
    -o "$OUT" "$HERE/csrc/flb_capi.cu" -ldl
echo "built $OUT"
