#!/bin/bash
# Full GPU validation pass (run on the GPU box): kernel parity, model parity, smoke, benches.
mkdir -p gpurun_out
run() { echo "=== $1"; shift; timeout ${TMO:-240} "$@" 2>&1 | grep -vE "Warning|warn\(|^$" | tail -${TAILN:-12}; }
run "ops" python -m pytest tests/test_ops_gpu.py -q -m gpu --tb=line -p no:cacheprovider
run "gemm conformance" python -m pytest tests/test_gemm_conformance_gpu.py -q -m gpu --tb=short -p no:cacheprovider
run "attention conformance" python -m pytest tests/test_attn_conformance_gpu.py -q -m gpu --tb=short -p no:cacheprovider
run "norm conformance" python -m pytest tests/test_norm_conformance_gpu.py -q -m gpu --tb=short -p no:cacheprovider
run "dwconv conformance" python -m pytest tests/test_dwconv_conformance_gpu.py -q -m gpu --tb=short -p no:cacheprovider
run "optimizer conformance" python -m pytest tests/test_optim_conformance_gpu.py -q -m gpu --tb=short -p no:cacheprovider
run "token conformance" python -m pytest tests/test_token_conformance_gpu.py -q -m gpu --tb=short -p no:cacheprovider
run "operand conformance" python -m pytest tests/test_operand_conformance_gpu.py -q -m gpu --tb=short -p no:cacheprovider
run "vit ops" python -m pytest tests/test_vit_ops_gpu.py -q -m gpu --tb=short -p no:cacheprovider
TAILN=40 run "resnet model" python -m pytest tests/test_resnet_gpu.py -q -m gpu -s --tb=line -p no:cacheprovider
TAILN=40 run "darknet model" python -m pytest tests/test_darknet_gpu.py -q -m gpu -s --tb=line -p no:cacheprovider
TAILN=30 run "vit model" python -m pytest tests/test_vit_gpu.py -q -m gpu -s --tb=short -p no:cacheprovider
run "smoke" python __graft_entry__.py smoke
timeout 300 python bench.py --steps 5 --warmup 3 --no-cpu-baseline --dump-ops gpurun_out/ops_r50.csv > gpurun_out/bench_r50.log 2>&1; tail -1 gpurun_out/bench_r50.log
timeout 300 python bench.py --model vit_base_patch16 --steps 5 --warmup 3 --no-cpu-baseline --dump-ops gpurun_out/ops_vit.csv > gpurun_out/bench_vit.log 2>&1; tail -2 gpurun_out/bench_vit.log
