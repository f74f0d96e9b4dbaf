#!/bin/bash
# GPU validation commands (run from the repo root on an H100 box):
#   bash scripts/gpu_checks.sh tests            # 1 GPU: kernel + model tests, smoke
#   bash scripts/gpu_checks.sh tests-mgpu       # >= 2 GPUs: pipeline / expert-parallel parity
#   bash scripts/gpu_checks.sh bench N          # headline bench on N GPUs (N > 1: both shardings)
#   bash scripts/gpu_checks.sh micro N          # boundary (2 GPUs) and expert-parallel block micro-benchmarks
#   bash scripts/gpu_checks.sh profile          # 1 GPU: ncu captures + launch list + memcheck (outputs in gpurun_out/)
set -u
mkdir -p gpurun_out
TR() { python -m torch.distributed.run --nnodes=1 --nproc-per-node "$1" --master-addr 127.0.0.1 --master-port 29610 "${@:2}"; }
case "${1:-tests}" in
  tests)
    python -m pytest tests/test_kernels_gpu.py tests/test_models_gpu.py -m gpu -q --timeout 600
    python -c "import __graft_entry__ as g; g.smoke()" ;;
  tests-mgpu)
    python -m pytest tests/test_multigpu.py -m gpu -q --timeout 900 ;;
  bench)
    N=${2:-1}
    if [ "$N" = 1 ]; then python bench.py; else TR "$N" bench.py --gpus "$N" --steps 24 --warmup 4; fi ;;
  micro)
    N=${2:-2}
    [ "$N" = 2 ] && TR 2 bench/boundary_bench.py
    TR "$N" bench/ep_bench.py --tokens 64 --breakdown ;;
  profile)
    NCU="ncu --set full --clock-control none --import-source on --kernel-name-base demangled"
    B="python bench.py --layers 3 --steps 1 --warmup 1 --no-graphs --no-e2e"
    $NCU -k 'regex:gemm_persistent_kernel<\(int\)64, \(bool\)1' -s 2 -c 1 -o gpurun_out/ncu_experts_gateup_decode $B
    $NCU -k 'regex:gemm_swapab_kernel<\(int\)64, \(bool\)0' -s 6 -c 1 -o gpurun_out/ncu_splitk_decode $B
    $NCU -k 'regex:paged_attn_kernel' -s 4 -c 1 -o gpurun_out/ncu_attn_decode $B
    ncu --metrics gpu__time_duration.sum --clock-control none --csv --log-file gpurun_out/launches_decode.csv \
        python bench.py --steps 1 --warmup 3 --no-graphs --no-e2e
    compute-sanitizer --tool memcheck --error-exitcode 7 --log-file gpurun_out/memcheck.log python -m pytest tests/test_kernels_gpu.py \
        -m gpu -q -x -k "linear or gated_up or moe_experts or moe_route or rmsnorm or mla_rope or paged_attention" ;;
  *) echo "unknown mode $1"; exit 2 ;;
esac
