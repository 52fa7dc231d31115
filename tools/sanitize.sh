#!/bin/bash
# compute-sanitizer targets (run on an H100 box: `bash tools/sanitize.sh [OUT_DIR]`; add a second GPU for the handoff
# target).  memcheck: out-of-bounds / misaligned accesses incl. TMA and DSMEM; racecheck: shared-memory (and distributed
# shared memory) hazards of the split-K reduce-scatter, the cluster sampler and the attention kernels; synccheck: barrier
# misuse.  Not yet run on H100.
set -u
OUT=${1:-gpurun_out/sanitizer}
mkdir -p "$OUT"
export B2B_ALLOW_RANDOM_WEIGHTS=1
CS="compute-sanitizer --error-exitcode 9 --launch-timeout 0"
SEL_GEMM='test_gemm_splitk_cluster or test_gemm_fused_epilogues_chain or test_gemm_mxfp8'
SEL_SAMP='sampler'
SEL_ATTN='test_attention_decode or test_attention_prefill_tcgen05_long'
run() {   # name, tool, pytest selection
  local name=$1 tool=$2 sel=$3
  timeout 900 $CS --tool "$tool" python -m pytest tests/test_kernels_gpu.py -x -q -m gpu -k "$sel" > "$OUT/$name.$tool.log" 2>&1
  echo "$name $tool rc=$? $(grep -E 'ERROR SUMMARY|RACECHECK SUMMARY' "$OUT/$name.$tool.log" | tail -1) $(tail -1 "$OUT/$name.$tool.log")"
}
if [ "${SANITIZE_ONLY:-all}" != "handoff" ]; then
run gemm memcheck "$SEL_GEMM"
run gemm racecheck "$SEL_GEMM"
run sampler memcheck "$SEL_SAMP"
run sampler racecheck "$SEL_SAMP"
run attention memcheck "$SEL_ATTN"
run gemm synccheck "$SEL_GEMM"
# engine end to end (graph prefill, decode graphs, fetch_window into mapped host memory)
timeout 900 $CS --tool memcheck python -c "import __graft_entry__ as g; g.smoke()" > "$OUT/smoke.memcheck.log" 2>&1
echo "smoke memcheck rc=$? $(grep 'ERROR SUMMARY' "$OUT/smoke.memcheck.log" | tail -1)"
fi
if [ "$(nvidia-smi -L | wc -l)" -ge 2 ]; then
  # 2-rank NVLink handoff: peer stores + .sys flags + double-buffered prefill channel, every rank under memcheck
  B2B_PROMPTS=bigsmall B2B_PF_TOKENS=64 B2B_STEPS=4 B2B_GROUPS=2 B2B_BATCH=4 timeout 1200 $CS --tool memcheck --target-processes all \
    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29733 tools/mp_check.py \
    > "$OUT/handoff.memcheck.log" 2>&1
  echo "handoff(2 ranks) memcheck rc=$? $(grep -c 'ERROR SUMMARY: 0 errors' "$OUT/handoff.memcheck.log") clean process summaries; $(grep RESULT "$OUT/handoff.memcheck.log" | cut -c1-80)"
fi
