#!/bin/bash
# experimental builds of libsonarfe with different icp.cu knobs -> scratch/lib_<tag>.so (run after the main build)
set -e
cd "$(dirname "$0")/.."
mkdir -p scratch
B=sonar_slam_b200/build
FL="-gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 -Xcompiler -fPIC -Xcompiler -fvisibility=hidden --expt-relaxed-constexpr"
build() { tag=$1; shift
  nvcc $FL "$@" -c sonar_slam_b200/csrc/icp.cu -o scratch/icp_$tag.o
  objs=$(ls $B/*.o | grep -v "/icp.o")
  nvcc -shared -o scratch/lib_$tag.so scratch/icp_$tag.o $objs -gencode arch=compute_90a,code=sm_90a -lcudart
}
rm -f scratch/lib_*.so
build pipe128 -DSFE_SEQ_PIPE_MIN=128
build phases -DSFE_ICP_PHASE_CLOCKS  # per-phase cycle counts of icp_kernel (tools/icp_phases.py)
ls -la scratch/*.so
