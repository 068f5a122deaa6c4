#!/bin/bash
# experimental build of libsonarfe in which every cloud takes the large-cloud path (run after the main build):
#   scratch/lib_mapclass.so   cloud.cu and icp.cu with -DSFE_MAP_CLASS_ALL: pcl.downsample on the grid-wide path,
#                             pcl.remove_outlier, ICP targets and pcl.match references in the map class
#                             (tools/bench_map_downsample.py, bench_map_outlier.py and bench_map_icp.py compare it with
#                             the one-CTA kernels on clouds both hold)
set -e
cd "$(dirname "$0")/.."
mkdir -p scratch
B=sonar_slam_b200/build
FL="-gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 -Xcompiler -fPIC -Xcompiler -fvisibility=hidden --expt-relaxed-constexpr"
objs=$(ls $B/*.o | grep -v -e "/cloud.o" -e "/icp.o")
for f in cloud icp; do
  nvcc $FL -DSFE_MAP_CLASS_ALL -c sonar_slam_b200/csrc/$f.cu -o scratch/${f}_mapclass.o
done
nvcc -shared -o scratch/lib_mapclass.so scratch/cloud_mapclass.o scratch/icp_mapclass.o $objs \
  -gencode arch=compute_90a,code=sm_90a -lcudart
ls -la scratch/lib_mapclass.so
