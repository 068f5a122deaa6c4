#!/bin/bash
# experimental build of libsonarfe with cloud.cu knobs (run after the main build):
#   scratch/lib_dsphases.so  per-phase cycle counts of the down-sample kernels (-DSFE_DS_PHASE_CLOCKS, tools/ds_phases.py)
# (the build in which every cloud takes the grid-wide path: tools/build_map_class_variant.sh)
set -e
cd "$(dirname "$0")/.."
mkdir -p scratch
B=sonar_slam_b200/build
FL="-gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 -Xcompiler -fPIC -Xcompiler -fvisibility=hidden --expt-relaxed-constexpr"
objs=$(ls $B/*.o | grep -v "/cloud.o")
build() { tag=$1; shift
  nvcc $FL "$@" -c sonar_slam_b200/csrc/cloud.cu -o scratch/cloud_$tag.o
  nvcc -shared -o scratch/lib_$tag.so scratch/cloud_$tag.o $objs -gencode arch=compute_90a,code=sm_90a -lcudart
}
build dsphases -DSFE_DS_PHASE_CLOCKS
ls -la scratch/lib_dsphases.so
