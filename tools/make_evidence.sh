#!/bin/bash
# Condense one gpurun round (tag $1, files gpurun_out/$1_*) into the committed evidence under profiles/ (round $2).
# Run here (ncu / cuobjdump are installed; no GPU needed):   bash tools/make_evidence.sh r02z r02
set -e
tag=$1; rnd=${2:-r02}
cd "$(dirname "$0")/.."
G=gpurun_out; P=profiles
[ -f $G/${tag}_bench.json ] && grep '^{' $G/${tag}_bench.json | tail -1 > $P/${rnd}_bench_n1.json
[ -f $G/${tag}_bench_plane.json ] && grep '^{' $G/${tag}_bench_plane.json | tail -1 > $P/${rnd}_bench_n1_plane.json
[ -f $G/${tag}_bench_ref.json ] && grep '^{' $G/${tag}_bench_ref.json | tail -1 > $P/${rnd}_bench_reference_arm.json
for n in 2 4 8; do f=$G/${tag}_bench_n$n.json; [ -f "$f" ] || f=$(ls -t $G/*_bench_n$n.json 2>/dev/null | head -1); [ -n "$f" ] && [ -f "$f" ] && grep '^{' $f | tail -1 > $P/${rnd}_bench_n$n.json; done
[ -f $G/icp_parity_sweep.json ] && cp $G/icp_parity_sweep.json $P/${rnd}_icp_parity_sweep.json
[ -f $G/${tag}_launches.csv ] && cp $G/${tag}_launches.csv $P/${rnd}_launch_list_ncu.csv && \
  python tools/launch_summary.py $P/${rnd}_launch_list_ncu.csv $P/${rnd}_launch_list_summary.csv 2 28 > /dev/null
args=""
[ -f $G/${tag}_prof_cfar_u8gate4.ncu-rep ] && args="$args prof_cfar_u8gate4=$G/${tag}_prof_cfar_u8gate4.ncu-rep"
[ -f $G/${tag}_prof_cfar_u8lut.ncu-rep ] && args="$args prof_cfar_u8lut=$G/${tag}_prof_cfar_u8lut.ncu-rep"
[ -f $G/${tag}_prof_icp_config3.ncu-rep ] && args="$args prof_icp_config3=$G/${tag}_prof_icp_config3.ncu-rep"
if [ -f $G/${tag}_prof_pipeline.ncu-rep ]; then
  args="$args pipeline_cart_scatter=$G/${tag}_prof_pipeline.ncu-rep@cart_scatter"
  args="$args pipeline_downsample_frames=$G/${tag}_prof_pipeline.ncu-rep@downsample#2"
  args="$args pipeline_downsample_submaps=$G/${tag}_prof_pipeline.ncu-rep@downsample#0"
  args="$args pipeline_remove_outlier=$G/${tag}_prof_pipeline.ncu-rep@remove_outlier"
  args="$args pipeline_icp_128=$G/${tag}_prof_pipeline.ncu-rep@icp_kernel<128"
fi
[ -f $G/${tag}_prof_plane.ncu-rep ] && args="$args pipeline_icp_128_plane=$G/${tag}_prof_plane.ncu-rep@icp_kernel<128"
[ -n "$args" ] && python tools/ncu_summary.py $P/${rnd}_ncu_full_summaries.json $args
{
  echo "# hot source lines (ncu --set full --import-source on; tools/ncu_hot_lines.py) -- round $rnd, gpurun tag $tag"
  [ -f $G/${tag}_prof_cfar_u8gate4.ncu-rep ] && python tools/ncu_hot_lines.py $G/${tag}_prof_cfar_u8gate4.ncu-rep cfar_u8_gate4 sonar_slam_b200/libsonarfe.so 16
  [ -f $G/${tag}_prof_icp_config3.ncu-rep ] && python tools/ncu_hot_lines.py $G/${tag}_prof_icp_config3.ncu-rep icp_kernel sonar_slam_b200/libsonarfe.so 20
  if [ -f $G/${tag}_prof_pipeline.ncu-rep ]; then
    python tools/ncu_hot_lines.py $G/${tag}_prof_pipeline.ncu-rep cart_scatter sonar_slam_b200/libsonarfe.so 14
    python tools/ncu_hot_lines.py $G/${tag}_prof_pipeline.ncu-rep "downsample#2" sonar_slam_b200/libsonarfe.so 14
    python tools/ncu_hot_lines.py $G/${tag}_prof_pipeline.ncu-rep "icp_kernel<(int)128" sonar_slam_b200/libsonarfe.so 20
  fi
  [ -f $G/${tag}_prof_plane.ncu-rep ] && python tools/ncu_hot_lines.py $G/${tag}_prof_plane.ncu-rep "icp_kernel<(int)128" sonar_slam_b200/libsonarfe.so 14
} > $P/${rnd}_hot_lines.txt 2>&1 || true
# per call site (everything inlined below a call site of the kernel's own file folded into it)
{
  echo "# per call site: ncu source page joined with nvdisasm -gi (tools/ncu_call_sites.py) -- round $rnd, gpurun tag $tag"
  td=$(mktemp -d); (cd $td && cuobjdump -xelf all $OLDPWD/sonar_slam_b200/libsonarfe.so > /dev/null 2>&1)
  [ -f $G/${tag}_prof_icp_config3.ncu-rep ] && { echo "== icp_kernel<512,1,false,false,false,false>, 296 problems of 2 000 x 20 000 points"; python tools/ncu_call_sites.py $G/${tag}_prof_icp_config3.ncu-rep icp_kernel $td/icp.sm_90a.cubin icp_kernelILi512ELi1ELb0ELb0ELb0ELb0E icp.cu 12; }
  if [ -f $G/${tag}_prof_pipeline.ncu-rep ]; then
    echo "== icp_kernel<128,8,false,false,false,false>, the front end's class, 1024 frames"; python tools/ncu_call_sites.py $G/${tag}_prof_pipeline.ncu-rep "icp_kernel<(int)128" $td/icp.sm_90a.cubin icp_kernelILi128ELi8ELb0ELb0ELb0ELb0E icp.cu 12
    echo "== cart_scatter_kernel, 1024 frames"; python tools/ncu_call_sites.py $G/${tag}_prof_pipeline.ncu-rep cart_scatter $td/featx.sm_90a.cubin cart_scatter featx.cu 10
    echo "== downsample_cta_kernel (frames), 1024 frames"; python tools/ncu_call_sites.py $G/${tag}_prof_pipeline.ncu-rep "downsample#2" $td/cloud.sm_90a.cubin downsample_cta_kernel cloud.cu 12
  fi
  [ -f $G/${tag}_prof_plane.ncu-rep ] && { echo "== icp_kernel<128,8,true,false,false,false> (point-to-plane), 1024 frames"; python tools/ncu_call_sites.py $G/${tag}_prof_plane.ncu-rep "icp_kernel<(int)128" $td/icp.sm_90a.cubin icp_kernelILi128ELi8ELb1ELb0ELb0ELb0E icp.cu 10; }
  rm -rf $td
} > $P/${rnd}_call_sites.txt 2>&1 || true
# SASS excerpt: the interior 16-row block of the pipeline's CFAR kernel + the TMA / mbarrier instructions of the library
{
  echo "# cuobjdump -sass sonar_slam_b200/libsonarfe.so -- cfar_u8_gate4_kernel<SOCA, bits>: one interior 16-row block"
  echo "# (rows are branch-free: LDS.32 of 4 beams, PRMT to 16-bit lanes, IADD3 window sums, VIMNMX.U16x2, gate test, predicated parking)"
  cuobjdump -sass -fun '_ZN3sfe20cfar_u8_gate4_kernelILi1ELb0ELb1EEEv14CUtensorMap_stNS_10CfarParamsEPKtij' sonar_slam_b200/libsonarfe.so 2>/dev/null \
    | grep -E '^\s+/\*[0-9a-f]{4}\*/' | sed -E 's/\s+\/\* 0x[0-9a-f]+ \*\///' > /tmp/_g4.txt
  first=$(grep -n "SYNCS.PHASECHK" /tmp/_g4.txt | sed -n 3p | cut -d: -f1)
  sed -n "${first},$((first+150))p" /tmp/_g4.txt
  echo; echo "# opcode histogram of the whole kernel"; awk '{print $2}' /tmp/_g4.txt | sed 's/\..*//' | sort | uniq -c | sort -rn | head -24
  echo; echo "# TMA / mbarrier instructions in libsonarfe.so (all kernels)"
  cuobjdump -sass sonar_slam_b200/libsonarfe.so | grep -oE "UTMALDG[.A-Z0-9]*|UTMASTG[.A-Z0-9]*|SYNCS[.A-Z0-9]*|UTMACMDFLUSH|VIMNMX.U16x2|ATOMS[.A-Z0-9]*" | sort | uniq -c
} > $P/${rnd}_sass_cfar_gate4.txt 2>&1 || true
ls -la $P | tail -20
