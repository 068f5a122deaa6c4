#!/bin/bash
# One gpurun call: GPU tests, stage micro-benchmarks, the bench line, ncu launch list and full captures.
#   gpurun --timeout 2400 -- 'bash tools/gpu_round.sh [tag] [steps...]'
# Every step writes its own log under gpurun_out/<tag>_*; a failing step does not stop the rest.
tag=${1:-r02a}; shift
steps=${*:-"tests cfar icp bench ncu_list ncu_cfar ncu_icp"}
export PYTHONPATH=$PWD
mkdir -p gpurun_out
for s in $steps; do
  echo "=== $s $(date +%T)"
  case $s in
    tests)    timeout 1200 python -m pytest tests -m gpu -q -x --timeout 900 > gpurun_out/${tag}_pytest.log 2>&1; tail -5 gpurun_out/${tag}_pytest.log ;;
    tests_all) timeout 1500 python -m pytest tests -m gpu -q --timeout 900 > gpurun_out/${tag}_pytest.log 2>&1; tail -15 gpurun_out/${tag}_pytest.log ;;
    cfar)
              timeout 300 python tools/bench_cfar.py 4096 noise > gpurun_out/${tag}_cfar_noise.log 2>&1; timeout 300 python tools/bench_cfar.py 4096 replay > gpurun_out/${tag}_cfar.log 2>&1; cp gpurun_out/bench_cfar.json gpurun_out/${tag}_bench_cfar.json
              ;;
    icp)      timeout 600 python tools/icp_scaling.py > gpurun_out/${tag}_icp_scaling.log 2>&1; cat gpurun_out/${tag}_icp_scaling.log ;;
    stages)   timeout 600 python tools/bench_stages.py 4096 1184 > gpurun_out/${tag}_stages.log 2>&1; cat gpurun_out/${tag}_stages.log ;;
    bench)    timeout 900 python bench.py > gpurun_out/${tag}_bench.json 2> gpurun_out/${tag}_bench.err; tail -c 3000 gpurun_out/${tag}_bench.json; tail -3 gpurun_out/${tag}_bench.err ;;
    bench_plane) timeout 900 python bench.py --minimizer plane --pairs 0 --cpu-sample 64 > gpurun_out/${tag}_bench_plane.json 2> gpurun_out/${tag}_bench_plane.err; tail -c 2500 gpurun_out/${tag}_bench_plane.json; tail -3 gpurun_out/${tag}_bench_plane.err ;;
    icp_variants) for so in sonar_slam_b200/libsonarfe.so scratch/lib_*.so; do echo "== $so"; SFE_LIB_PATH=$PWD/$so timeout 300 python bench.py --pairs 0 --cpu-sample 8 --steps 5 2>/dev/null | python -c "import sys,json; d=json.loads(sys.stdin.read()); print({k: round(v,3) for k,v in d['stage_ms_per_step'].items()}, round(d['ms_per_step'],3), round(d['config3_icp']['fixed20']['ms_per_wave'],3))"; done ;;
    cfar_variants) for so in scratch/lib_*.so; do echo "== $so"; SFE_LIB_PATH=$PWD/$so timeout 300 python tools/bench_cfar.py 4096 replay 2>&1 | grep -E "u8_SOCA_bits|u8_SOCA_mask " | cut -c1-120; done ;;
    bench_ref) timeout 900 python bench.py --impl reference --steps 3 --warmup 1 > gpurun_out/${tag}_bench_ref.json 2> gpurun_out/${tag}_bench_ref.err; cat gpurun_out/${tag}_bench_ref.json ;;
    ncu_list) timeout 900 ncu --metrics gpu__time_duration.sum --clock-control none -k regex:"cfar|cart_|downsample|outlier|assemble|icp_|fill_off|match_|flip_|feat" -c 400 --csv \
                --log-file gpurun_out/${tag}_launches.csv python bench.py --steps 2 --warmup 1 --pairs 0 --cpu-sample 8 > gpurun_out/${tag}_bench_under_ncu.log 2>&1; tail -2 gpurun_out/${tag}_launches.csv ;;
    ncu_cfar) timeout 600 ncu --set full --clock-control none --import-source on -k regex:cfar_u8 -s 2 -c 1 -f -o gpurun_out/${tag}_prof_cfar_u8gate4 \
                python tools/prof_cfar.py 4096 u8 bits > gpurun_out/${tag}_ncu_cfar.log 2>&1; tail -2 gpurun_out/${tag}_ncu_cfar.log
              ;;
    ncu_icp)  timeout 900 ncu --set full --clock-control none --import-source on -k regex:icp_kernel -s 2 -c 1 -f -o gpurun_out/${tag}_prof_icp_config3 \
                python tools/prof_icp.py 296 > gpurun_out/${tag}_ncu_icp.log 2>&1; tail -2 gpurun_out/${tag}_ncu_icp.log ;;
    ncu_pipe) timeout 900 ncu --set full --clock-control none --import-source on -k regex:"icp_kernel|feat|cart_|downsample|outlier|assemble" -s 14 -c 7 -f -o gpurun_out/${tag}_prof_pipeline \
                python tools/prof_pipeline.py 1024 > gpurun_out/${tag}_ncu_pipe.log 2>&1; tail -2 gpurun_out/${tag}_ncu_pipe.log ;;
    ncu_plane) timeout 900 ncu --set full --clock-control none --import-source on -k regex:"icp_kernel" -s 4 -c 2 -f -o gpurun_out/${tag}_prof_plane \
                python tools/prof_pipeline.py 1024 1 > gpurun_out/${tag}_ncu_plane.log 2>&1; tail -2 gpurun_out/${tag}_ncu_plane.log ;;
    n2)       timeout 900 python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29511 bench.py --gpus 2 \
                > gpurun_out/${tag}_bench_n2.json 2> gpurun_out/${tag}_bench_n2.err; tail -c 2500 gpurun_out/${tag}_bench_n2.json; tail -5 gpurun_out/${tag}_bench_n2.err ;;
    n8)       NCCL_DEBUG=INFO timeout 900 python -m torch.distributed.run --nnodes=1 --nproc-per-node 8 --master-addr 127.0.0.1 --master-port 29512 bench.py --gpus 8 \
                > gpurun_out/${tag}_bench_n8.json 2> gpurun_out/${tag}_bench_n8.err; tail -c 2500 gpurun_out/${tag}_bench_n8.json; grep -c "NCCL INFO" gpurun_out/${tag}_bench_n8.err ;;
  esac
done
echo "=== done $(date +%T)"
