// Continuation scoring: per-row log-probability of a target token and whether it is the row's argmax, from fp16
// logits (R, V) with row stride ld, without a full-vocab fp32 tensor.  The rule is stated in include/quip_b200.h
// (quip_token_logprobs); oracle/loglik.py restates it in float64.
//
// One CTA per row, one pass over the row: 16-byte loads for the aligned body, scalars for a head (up to the first
// 16-byte boundary) and a tail, so any V and ld work.  Each thread keeps an online (max m, sum s of exp(x - m)) in
// fp32 -- a group of 8 values rescales s once, by its own max -- and the (value, lowest index) of the largest value it
// saw.  Threads combine by a fixed xor-shuffle tree and then warp by warp in order, so every launch gives the same bits.
// Thread 0 reads the target logit (never dereferenced outside [0, V)).
#include <math.h>

#include "common.cuh"

namespace quip {

namespace {

constexpr int LP_THREADS = 512;
constexpr int LP_WARPS = LP_THREADS / 32;

struct RowStat {
  float m, s;      // running max and sum of exp(x - m); (-inf, 0) before any value
  float bv;        // largest value seen, and its lowest index (INT_MAX before any value)
  int bi;
  bool nan;
};

__device__ __forceinline__ void take_best(RowStat& a, float v, int i) {
  if (v > a.bv || (v == a.bv && i < a.bi)) {
    a.bv = v;
    a.bi = i;
  }
}

__device__ __forceinline__ void add_one(RowStat& a, float v, int i) {
  if (v != v) {
    a.nan = true;
    return;
  }
  take_best(a, v, i);
  if (v > a.m) {
    a.s = a.s * expf(a.m - v);
    a.m = v;
  }
  a.s += expf(v - a.m);
}

// 8 consecutive values starting at index i0: one rescale of s by the group's max
__device__ __forceinline__ void add_eight(RowStat& a, const uint4& raw, int i0) {
  const __half2* h = reinterpret_cast<const __half2*>(&raw);
  float v[8];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float2 f = __half22float2(h[j]);
    v[2 * j] = f.x;
    v[2 * j + 1] = f.y;
  }
  float gm = v[0];
  bool nan = false;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    nan |= v[j] != v[j];
    gm = fmaxf(gm, v[j]);
  }
  if (nan) {
    a.nan = true;
    return;
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) take_best(a, v[j], i0 + j);
  if (gm > a.m) {
    a.s = a.s * expf(a.m - gm);
    a.m = gm;
  }
  float t = 0.f;
#pragma unroll
  for (int j = 0; j < 8; ++j) t += expf(v[j] - a.m);
  a.s += t;
}

__device__ __forceinline__ void merge(RowStat& a, const RowStat& b) {
  a.nan |= b.nan;
  take_best(a, b.bv, b.bi);
  const float m = fmaxf(a.m, b.m);
  const float sa = a.s > 0.f ? a.s * expf(a.m - m) : 0.f;
  const float sb = b.s > 0.f ? b.s * expf(b.m - m) : 0.f;
  a.m = m;
  a.s = sa + sb;
}

__device__ __forceinline__ RowStat shfl_xor(const RowStat& a, int o) {
  RowStat b;
  b.m = __shfl_xor_sync(0xFFFFFFFFu, a.m, o);
  b.s = __shfl_xor_sync(0xFFFFFFFFu, a.s, o);
  b.bv = __shfl_xor_sync(0xFFFFFFFFu, a.bv, o);
  b.bi = __shfl_xor_sync(0xFFFFFFFFu, a.bi, o);
  b.nan = __shfl_xor_sync(0xFFFFFFFFu, (int)a.nan, o) != 0;
  return b;
}

__global__ void __launch_bounds__(LP_THREADS) token_logprobs_kernel(const __half* __restrict__ logits, int64_t ld,
                                                                    const int64_t* __restrict__ targets,
                                                                    float* __restrict__ logprob,
                                                                    uint8_t* __restrict__ is_greedy, int V) {
  __shared__ RowStat part[LP_WARPS];
  const int r = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const __half* x = logits + (size_t)r * (size_t)ld;
  RowStat a{-INFINITY, 0.f, -INFINITY, 0x7FFFFFFF, false};

  // head: scalars up to the first 16-byte boundary; body: 8 values per load; tail: scalars
  const int mis = (int)(((uintptr_t)x >> 1) & 7);
  const int head = min(V, (8 - mis) & 7);
  const int nvec = (V - head) >> 3;
  const int body_end = head + 8 * nvec;
  if (tid < head) add_one(a, __half2float(x[tid]), tid);
  const uint4* xv = reinterpret_cast<const uint4*>(x + head);
  int k = tid;
  for (; k + LP_THREADS < nvec; k += 2 * LP_THREADS) {           // two loads in flight
    const uint4 u0 = __ldg(xv + k), u1 = __ldg(xv + k + LP_THREADS);
    add_eight(a, u0, head + 8 * k);
    add_eight(a, u1, head + 8 * (k + LP_THREADS));
  }
  if (k < nvec) add_eight(a, __ldg(xv + k), head + 8 * k);
  if (body_end + tid < V) add_one(a, __half2float(x[body_end + tid]), body_end + tid);

#pragma unroll
  for (int o = 16; o; o >>= 1) merge(a, shfl_xor(a, o));
  if (lane == 0) part[warp] = a;
  __syncthreads();
  if (tid != 0) return;
  RowStat t = part[0];
  for (int w = 1; w < LP_WARPS; ++w) merge(t, part[w]);
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
