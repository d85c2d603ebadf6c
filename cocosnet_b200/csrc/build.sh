#!/bin/bash
# Build libcocos_b200.so in-tree for sm_90a (nvcc cross-compiles without a GPU).  One object per source, compiled in
# parallel and only when the source (or a header) is newer than its object.
set -e
cd "$(dirname "$0")"
NVCC=${NVCC:-/usr/local/cuda/bin/nvcc}
OUT=../libcocos_b200.so
OBJ=build
mkdir -p $OBJ
FLAGS="-std=c++17 -O3 -lineinfo -gencode arch=compute_90a,code=sm_90a -Xcompiler -fPIC ${COCOS_NVCC_EXTRA}"
newest_hdr=$(ls -t *.h *.cuh ../../include/*.h | head -1)
pids=()
for src in *.cu; do
  obj=$OBJ/${src%.cu}.o
  if [ ! -f $obj ] || [ $src -nt $obj ] || [ $newest_hdr -nt $obj ] || [ build.sh -nt $obj ]; then
    $NVCC $FLAGS -c -o $obj $src &
    pids+=($!)
  fi
done
for p in "${pids[@]}"; do wait $p; done
# objects of sources that no longer exist must not be linked
for obj in $OBJ/*.o; do
  [ -f "$(basename ${obj%.o}).cu" ] || rm -f $obj
done
$NVCC -shared -gencode arch=compute_90a,code=sm_90a -o $OUT $OBJ/*.o -lcudart
echo "built $(readlink -f $OUT)"
