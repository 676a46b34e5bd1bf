#!/usr/bin/env bash
# TEST INFRASTRUCTURE.  Builds the UNMODIFIED reference CUDA kernels for sm_90 into
# oracle/_ref/ (git-ignored; travels to the GPU box with gpurun).  Sources are compiled
# where they lie under /root/reference; nothing is copied into the repo.  Only the BVH
# builder needs a one-line patched copy (SURVEY.md §8c-addendum), generated into
# oracle/_ref/ at build time and printed here.
set -euo pipefail
HERE="$(cd "$(dirname "${BASH_SOURCE[0]}")" && pwd)"
REF="${R3DG_REFERENCE:-/root/reference}"
OUT="$HERE/_ref"
[ -d "$REF" ] || { echo "[build_ref] $REF absent — skipping (prebuilt oracle/_ref is used if present)"; exit 0; }
mkdir -p "$OUT"
NVCC="${NVCC:-/usr/local/cuda/bin/nvcc}"
ARCH="-gencode arch=compute_90,code=sm_90"
# Flags = the reference's own (r3dg-rasterization/setup.py:30-33: -O3 + glm include) plus
# what torch's BuildExtension always adds, plus the two header papering pre-includes.
TORCHISH="-D__CUDA_NO_HALF_OPERATORS__ -D__CUDA_NO_HALF_CONVERSIONS__ -D__CUDA_NO_BFLOAT16_CONVERSIONS__ -D__CUDA_NO_HALF2_OPERATORS__ --expt-relaxed-constexpr -std=c++17"
RAS="$REF/r3dg-rasterization"
if [ ! -f "$OUT/libref_raster.so" ] || [ "$HERE/ref_shim_raster.cu" -nt "$OUT/libref_raster.so" ]; then
  echo "[build_ref] rasterizer (forward.cu backward.cu rasterizer_impl.cu + shim)"
  for f in forward backward rasterizer_impl; do
    $NVCC $ARCH -O3 $TORCHISH --pre-include cstdint -I"$RAS/third_party/glm" -I"$RAS" \
      -Xcompiler -fPIC -c "$RAS/cuda_rasterizer/$f.cu" -o "$OUT/ref_$f.o" &
  done
  $NVCC $ARCH -O3 $TORCHISH --pre-include cstdint -I"$RAS/third_party/glm" -I"$RAS" \
      -Xcompiler -fPIC -c "$HERE/ref_shim_raster.cu" -o "$OUT/ref_shim_raster.o" &
  wait
  $NVCC -shared -o "$OUT/libref_raster.so" "$OUT"/ref_forward.o "$OUT"/ref_backward.o \
      "$OUT"/ref_rasterizer_impl.o "$OUT"/ref_shim_raster.o -lcudart
  rm -f "$OUT"/ref_forward.o "$OUT"/ref_backward.o "$OUT"/ref_rasterizer_impl.o "$OUT"/ref_shim_raster.o
fi
if [ -f "$HERE/ref_shim_bvh.cu" ]; then
 if [ ! -f "$OUT/libref_bvh.so" ] || [ "$HERE/ref_shim_bvh.cu" -nt "$OUT/libref_bvh.so" ]; then
  echo "[build_ref] bvh (construct.cu[patched copy] trace.cu + shim)"
  BVH="$REF/bvh"
  sed '166s/rhs)[[:space:]]*{/rhs) -> aabb_type {/' "$BVH/src/construct.cu" > "$OUT/construct_patched.cu"
  echo "[build_ref] one-line patch applied to the COPY of bvh/src/construct.cu:166:"
  diff "$BVH/src/construct.cu" "$OUT/construct_patched.cu" || true
  $NVCC $ARCH -O3 $TORCHISH --expt-extended-lambda -I"$BVH/include" -Xcompiler -fPIC \
      -c "$OUT/construct_patched.cu" -o "$OUT/ref_construct.o" &
  $NVCC $ARCH -O3 $TORCHISH --expt-extended-lambda -I"$BVH/include" -Xcompiler -fPIC \
      -c "$BVH/src/trace.cu" -o "$OUT/ref_trace.o" &
  $NVCC $ARCH -O3 $TORCHISH --expt-extended-lambda -I"$BVH/include" -Xcompiler -fPIC \
      -c "$HERE/ref_shim_bvh.cu" -o "$OUT/ref_shim_bvh.o" &
  wait
  $NVCC -shared -o "$OUT/libref_bvh.so" "$OUT"/ref_construct.o "$OUT"/ref_trace.o "$OUT"/ref_shim_bvh.o -lcudart
  rm -f "$OUT"/ref_construct.o "$OUT"/ref_trace.o "$OUT"/ref_shim_bvh.o
 fi
fi
echo "[build_ref] done: $(ls "$OUT")"
