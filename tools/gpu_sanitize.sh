#!/usr/bin/env bash
# compute-sanitizer pass over the single-rank GPU kernel tests (run on an H100):
#   tools/gpu_sanitize.sh memcheck|racecheck|synccheck|initcheck [all]
# Only world=1 cases are selected: the multi-rank kernels spin on each other's flags and the sanitizer serialises
# kernel launches, so virtual-cluster tests would dead-lock under it (the spin watchdog would trap).
# Default: one case per kernel family; `all` selects every world-1 case (several minutes).
set -euo pipefail
TOOL=${1:-memcheck}
ROOT=$(cd "$(dirname "$0")/.." && pwd)
cd "$ROOT"
OUT=${SANITIZER_OUT:-/tmp/byteps_b200_sanitizer}   # logs go outside the tree
mkdir -p "$OUT"
if [ "${2:-}" = "all" ]; then
  SEL=(tests/test_gpu_kernels.py tests/test_gpu_ring.py tests/test_gpu_compress.py -k "1] and not multigpu")
else
  SEL=("tests/test_gpu_kernels.py::test_inplace_pushpull_virtual[bf16-1]"
       "tests/test_gpu_kernels.py::test_inplace_pushpull_tma_virtual[bf16-1]"
       "tests/test_gpu_kernels.py::test_packed_pushpull_virtual[f32-bf16-True-1]"
       "tests/test_gpu_kernels.py::test_fused_optimizer_virtual[lsu-bf16-adam-1]"
       "tests/test_gpu_kernels.py::test_fused_optimizer_virtual[tma-bf16-sgd-1]"
       "tests/test_gpu_ring.py::test_ring_allreduce_virtual[True-bf16-1]"
       "tests/test_gpu_compress.py::test_gpu_compressor_matches_cpu_reference[kw0-1]"
       "tests/test_gpu_compress.py::test_gpu_compressor_matches_cpu_reference[kw1-1]"
       "tests/test_gpu_bn_act_junction.py::test_two_gradients_match_torch_sum[3x8x5x7-bfloat16-full]"
       "tests/test_gpu_bn_act_junction.py::test_two_gradients_match_torch_sum[3x8x5x7-float32-part]"
       "tests/test_gpu_bn_act_junction.py::test_two_gradients_match_torch_sum[2x40x9x7-float16-none]"
       "tests/test_gpu_bn_act_junction.py::test_two_gradients_match_torch_sum[1x24x37x3-bfloat16-part]"
       "tests/test_gpu_bn_act_junction.py::test_two_gradients_match_torch_sum[64x1024x14x14-bfloat16-part]"
       "tests/test_gpu_bn_act_junction.py::test_second_gradient_fallbacks[3x8x5x7-bfloat16-misaligned]"
       "tests/test_gpu_bn_act_junction.py::test_second_gradient_fallbacks[2x40x9x7-float32-nchw]"
       "tests/test_gpu_bn_act_pool.py::test_pooled_matches_stock_chain[3x8x5x7-bfloat16-full]"
       "tests/test_gpu_bn_act_pool.py::test_pooled_matches_stock_chain[2x40x9x7-float32-part]"
       "tests/test_gpu_bn_act_pool.py::test_pooled_matches_stock_chain[1x8x1x6-float16-none]"
       "tests/test_gpu_bn_act_pool.py::test_pooled_matches_stock_chain[2x16x7x1-bfloat16-none]"
       "tests/test_gpu_attn.py::test_matches_float64[bfloat16-3x17x2-bool-p0]"
       "tests/test_gpu_attn.py::test_matches_float64[bfloat16-3x100x2-none-p01]"
       "tests/test_gpu_attn.py::test_matches_float64[bfloat16-2x512x3-none-p0]")
fi
timeout 1200 compute-sanitizer --tool "$TOOL" --error-exitcode 3 \
  --log-file "$OUT"/sanitizer_"$TOOL".log \
  python -m pytest -q -p no:cacheprovider --timeout 600 "${SEL[@]}" || true
tail -30 "$OUT"/sanitizer_"$TOOL".log
