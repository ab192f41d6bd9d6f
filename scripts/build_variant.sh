#!/bin/bash
# build an experimental variant of libcommpy_b200.so:  scripts/build_variant.sh <tag> [-DFLAG=VALUE ...]
# VARIANT_FILES="bcjr ..." names the sources the flags apply to (default: viterbi)
# -> build/variants/libcommpy_b200_<tag>.so   (use with COMMPY_B200_LIB=...)
set -e
cd "$(dirname "$0")/.."
tag=$1; shift
mkdir -p build/variants/$tag
for f in common viterbi bcjr ldpc demap count pipeline hostapi txlink turbolink; do
  [ -f commpy_b200/csrc/$f.cu ] || continue
  if [[ " ${VARIANT_FILES:-viterbi} " == *" $f "* ]] || [ ! -f build/$f.o ] || [ -n "$VARIANT_ALL" ]; then
    /usr/local/cuda/bin/nvcc -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 -Xcompiler -fPIC --fmad=true -DCPB_BUILDING=1 "$@" -c commpy_b200/csrc/$f.cu -o build/variants/$tag/$f.o &
  else
    cp build/$f.o build/variants/$tag/$f.o
  fi
done
wait
/usr/local/cuda/bin/nvcc -shared -o build/variants/libcommpy_b200_$tag.so build/variants/$tag/*.o -gencode arch=compute_90a,code=sm_90a -Xcompiler -fPIC -lcudart
echo build/variants/libcommpy_b200_$tag.so
