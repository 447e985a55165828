#!/bin/bash
# A/B builds of the filter's mean stage: tools/build_variants.sh  ->  safe_learning_b200/variants/libslb200_<name>.so
# (loaded through SLB200_LIB by tools/mean_variants.py)
set -e
cd "$(dirname "$0")/../safe_learning_b200/csrc"
mkdir -p ../variants
FLAGS="-gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -std=c++17 -Xcompiler -fPIC"
build() {  # name, extra flags...
  name=$1; shift
  nvcc $FLAGS "$@" -c filter.cu -o ../variants/filter_$name.o
  objs=$(ls build/*.o | grep -v "build/filter.o")
  nvcc -shared -gencode arch=compute_90a,code=sm_90a -o ../variants/libslb200_$name.so $objs ../variants/filter_$name.o
  echo built $name
}
build u4 &
build u8 -DSLB_MEAN_UNROLL=8 &
build ft128 -DSLB_FT=128 -DSLB_MEAN_MINB=4 &
build u8b5 -DSLB_MEAN_UNROLL=8 -DSLB_MEAN_MINB=5 &
wait
