#!/bin/bash
# experimental build of libsonarfe where every down-sampled cloud takes the grid-wide path -> scratch/lib_dsgrid.so
# (run after the main build; tools/bench_map_downsample.py compares it with the one-CTA kernel)
set -e
cd "$(dirname "$0")/.."
mkdir -p scratch
B=sonar_slam_b200/build
FL="-gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 -Xcompiler -fPIC -Xcompiler -fvisibility=hidden --expt-relaxed-constexpr"
nvcc $FL -DSFE_DS_GRID_ALL -c sonar_slam_b200/csrc/cloud.cu -o scratch/cloud_dsgrid.o
objs=$(ls $B/*.o | grep -v "/cloud.o")
nvcc -shared -o scratch/lib_dsgrid.so scratch/cloud_dsgrid.o $objs -gencode arch=compute_90a,code=sm_90a -lcudart
ls -la scratch/lib_dsgrid.so
