#!/bin/bash
# experimental build of libsonarfe in which every scan-match target takes the map class (run after the main build):
#   scratch/lib_icpmap.so   icp.cu with -DSFE_ICP_MAP_ALL (tools/bench_map_icp.py compares it with the in-CTA kernel
#                           on a target both layouts hold)
set -e
cd "$(dirname "$0")/.."
mkdir -p scratch
B=sonar_slam_b200/build
FL="-gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 -Xcompiler -fPIC -Xcompiler -fvisibility=hidden --expt-relaxed-constexpr"
objs=$(ls $B/*.o | grep -v "/icp.o")
nvcc $FL -DSFE_ICP_MAP_ALL -c sonar_slam_b200/csrc/icp.cu -o scratch/icp_icpmap.o
nvcc -shared -o scratch/lib_icpmap.so scratch/icp_icpmap.o $objs -gencode arch=compute_90a,code=sm_90a -lcudart
ls -la scratch/lib_icpmap.so
