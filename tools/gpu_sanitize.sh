#!/bin/bash
# compute-sanitizer evidence (VERDICT item 9): memcheck + racecheck over the tensor-core operator tests, the weight-gradient tests and
# one FlowNet2-C forward + backward with graph replay off.  Summaries go to the output directory.
cd "$(dirname "$0")/.."
mkdir -p gpurun_out
export FN2_NO_GRAPH=1
run() {  # name tool args...
    local name=$1 tool=$2; shift 2
    timeout 900 compute-sanitizer --tool $tool --print-limit 20 "$@" > gpurun_out/san_${name}_${tool}.log 2>&1
    echo "== $name / $tool: exit $?" >> gpurun_out/r02_sanitizer_summary.txt
    grep -E "ERROR SUMMARY|RACECHECK SUMMARY|passed|failed" gpurun_out/san_${name}_${tool}.log | tail -4 >> gpurun_out/r02_sanitizer_summary.txt
}
: > gpurun_out/r02_sanitizer_summary.txt
run tc_ops memcheck python -m pytest tests/test_ops_gpu.py -q -x -k "tensor_core or taps_on_n"
run tc_ops racecheck python -m pytest tests/test_ops_gpu.py -q -x -k "tensor_core or taps_on_n"
run wgrad memcheck python -m pytest tests/test_train_gpu.py -q -x -k "conv_backward"
run wgrad racecheck python -m pytest tests/test_train_gpu.py -q -x -k "c3x3_s1_wide or c5x5_s2_w57 or d4x4_s2_wide"
run net_c memcheck python -m pytest tests/test_train_gpu.py -q -x -k "without_fusion"
run corr_bwd memcheck python -m pytest tests/test_ops_gpu.py -q -x -k "correlation_backward"
run corr_bwd racecheck python -m pytest tests/test_ops_gpu.py -q -x -k "correlation_backward_fast"
run warp_block memcheck python -m pytest tests/test_net_gpu.py -q -x -k "fused_warp_block"
run train_layers memcheck python -m pytest tests/test_train_gpu.py -q -x -k "training_layers or random_shapes"
cat gpurun_out/r02_sanitizer_summary.txt
