#!/bin/bash
# Build oracle/_ref/libref_ops.so: the reference's own CUDA kernels (compiled where they lie under
# $REF/ops, never copied) against the stand-in TensorFlow headers of oracle/tf_stub, plus the C wrapper.
# Needs the reference tree, i.e. runs in the build container; the .so travels to the GPU box.
set -e
HERE="$(cd "$(dirname "$0")" && pwd)"
ORACLE="$(dirname "$HERE")"
REF="${UNFLOW_REFERENCE:-/root/reference}"
OUT="$ORACLE/_ref"
NVCC="${NVCC:-/usr/local/cuda/bin/nvcc}"
[ -d "$REF/ops" ] || { echo "reference tree not found at $REF (nothing built)"; exit 0; }
mkdir -p "$OUT"
LIB="$OUT/libref_ops.so"
if [ -f "$LIB" ] && [ -z "$UNFLOW_FORCE_BUILD" ]; then
  stale=0
  for f in "$REF"/ops/*.cu.cc "$REF"/ops/*.h "$HERE/wrapper.cu" "$HERE/build.sh" $(find "$ORACLE/tf_stub" -type f); do
    [ "$f" -nt "$LIB" ] && stale=1
  done
  [ $stale -eq 0 ] && { echo "up to date: $LIB"; exit 0; }
fi
unset CC CXX
FLAGS="-gencode arch=compute_90a,code=sm_90a -O2 -lineinfo -std=c++17 -DGOOGLE_CUDA=1 -Xcompiler -fPIC -I $ORACLE/tf_stub -I $REF/ops"
OBJS=""
for f in correlation_op backward_warp_op forward_warp_op downsample_op; do
  "$NVCC" $FLAGS -x cu -c "$REF/ops/$f.cu.cc" -o "$OUT/$f.o"
  OBJS="$OBJS $OUT/$f.o"
done
"$NVCC" $FLAGS -c "$HERE/wrapper.cu" -o "$OUT/wrapper.o"
"$NVCC" -shared -o "$OUT/libref_ops.so" $OBJS "$OUT/wrapper.o" -gencode arch=compute_90a,code=sm_90a -Xcompiler -fPIC
rm -f $OBJS "$OUT/wrapper.o"
echo "built $OUT/libref_ops.so"
