#!/bin/bash
# experimental builds of libsonarfe with different cfar.cu knobs -> scratch/lib_<tag>.so (run after the main build)
set -e
cd "$(dirname "$0")/.."
mkdir -p scratch
B=sonar_slam_b200/build
FL="-gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 -Xcompiler -fPIC -Xcompiler -fvisibility=hidden --expt-relaxed-constexpr"
build() { tag=$1; shift
  nvcc $FL "$@" -c sonar_slam_b200/csrc/cfar.cu -o scratch/cfar_$tag.o
  objs=$(ls $B/*.o | grep -v "/cfar.o")
  nvcc -shared -o scratch/lib_$tag.so scratch/cfar_$tag.o $objs -gencode arch=compute_90a,code=sm_90a -lcudart
}
build ns2b4 -DSFE_CG_NS=2 -DSFE_CG_MINB=4 &
build ns2b3 -DSFE_CG_NS=2 -DSFE_CG_MINB=3 &
wait
ls -la scratch/*.so
