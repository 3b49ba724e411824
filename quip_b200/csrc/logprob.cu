// Continuation scoring: per-row log-probability of a target token and whether it is the row's argmax, from fp16
// logits (R, V) with row stride ld, without a full-vocab fp32 tensor.  The rule is stated in include/quip_b200.h
// (quip_token_logprobs); oracle/loglik.py restates it in float64.
//
// One CTA per row, one pass over the row (logprob_row.cuh: the partition and combine order fix the bits, and
// csrc/topk_logprobs.cu runs the same pass).  Thread 0 reads the target logit (never dereferenced outside [0, V)).
#include "logprob_row.cuh"

namespace quip {

namespace {

__global__ void __launch_bounds__(LP_THREADS) token_logprobs_kernel(const __half* __restrict__ logits, int64_t ld,
                                                                    const int64_t* __restrict__ targets,
                                                                    float* __restrict__ logprob,
                                                                    uint8_t* __restrict__ is_greedy, int V) {
  __shared__ RowStat part[LP_WARPS];
  const int r = blockIdx.x;
  const __half* x = logits + (size_t)r * (size_t)ld;
  const RowStat t = row_stat(x, V, part);
  if (threadIdx.x != 0) return;
  const int64_t tg = targets[r];
  if (t.nan || tg < 0 || tg >= V) {
    logprob[r] = __int_as_float(0x7FC00000);
    is_greedy[r] = 0;
    return;
  }
  const float xt = __half2float(x[tg]);
  logprob[r] = (xt - t.m) - logf(t.s);
  is_greedy[r] = (int64_t)t.bi == tg ? 1 : 0;
}

}  // namespace

}  // namespace quip

using namespace quip;

extern "C" int quip_token_logprobs(const void* logits, int64_t ld, const int64_t* targets, float* logprob,
                                   uint8_t* is_greedy, int32_t R, int32_t V, void* stream) {
  QUIP_CHECK_ARG(R >= 0 && V >= 1 && ld >= V,
                 "quip_token_logprobs: bad sizes (R %d, V %d, ld %lld): need R >= 0, V >= 1 and ld >= V", R, V,
                 (long long)ld);
  QUIP_CHECK_ARG(logits && targets && logprob && is_greedy, "quip_token_logprobs: null pointer");
  QUIP_CHECK_ARG(((uintptr_t)logits & 1) == 0 && ((uintptr_t)targets & 7) == 0 && ((uintptr_t)logprob & 3) == 0,
                 "quip_token_logprobs: logits must be 2-byte, targets 8-byte and logprob 4-byte aligned");
  if (R == 0) return QUIP_OK;
  token_logprobs_kernel<<<(unsigned)R, LP_THREADS, 0, (cudaStream_t)stream>>>((const __half*)logits, ld, targets,
                                                                               logprob, is_greedy, V);
  QUIP_LAUNCHED("token_logprobs_kernel");
  return QUIP_OK;
}
