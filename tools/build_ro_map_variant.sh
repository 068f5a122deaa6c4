#!/bin/bash
# experimental build of libsonarfe in which every outlier-filtered cloud takes the map class (run after the main build):
#   scratch/lib_romap.so   cloud.cu with -DSFE_RO_MAP_ALL (tools/bench_map_outlier.py compares it with the one-CTA
#                          kernel on clouds both paths hold)
set -e
cd "$(dirname "$0")/.."
mkdir -p scratch
B=sonar_slam_b200/build
FL="-gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 -Xcompiler -fPIC -Xcompiler -fvisibility=hidden --expt-relaxed-constexpr"
objs=$(ls $B/*.o | grep -v "/cloud.o")
nvcc $FL -DSFE_RO_MAP_ALL -c sonar_slam_b200/csrc/cloud.cu -o scratch/cloud_romap.o
nvcc -shared -o scratch/lib_romap.so scratch/cloud_romap.o $objs -gencode arch=compute_90a,code=sm_90a -lcudart
ls -la scratch/lib_romap.so
