// The row pass of the log-probability kernels (csrc/logprob.cu, csrc/topk_logprobs.cu): the max m and the sum s of
// exp(x - m) over one fp16 logits row, and the (value, lowest index) of its largest value, in a fixed order.
//
// One CTA of LP_THREADS threads per row: 16-byte loads for the aligned body, scalars for a head (up to the first
// 16-byte boundary) and a tail, so any V and row address work.  Each thread keeps an online (m, s) in fp32 -- a group
// of 8 values rescales s once, by its own max -- and threads combine by a fixed xor-shuffle tree and then warp by warp
// in order.  Both kernels run this same code, so a logprob (x_t - m) - log(s) has the same bits from either.
#pragma once

#include <math.h>

#include "common.cuh"

namespace quip {

constexpr int LP_THREADS = 512;
constexpr int LP_WARPS = LP_THREADS / 32;

struct RowStat {
  float m, s;      // running max and sum of exp(x - m); (-inf, 0) before any finite value
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
  if (a.m == -INFINITY) return;                  // only -inf so far: adds nothing (expf(-inf - -inf) would be NaN)
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
  if (a.m == -INFINITY) return;                  // a group of -inf before any finite value adds nothing
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

// The split of a row at x into scalars [0, head), 16-byte vectors [head, body_end) and scalars [body_end, V).
struct RowSplit {
  int head, nvec, body_end;
};

__device__ __forceinline__ RowSplit row_split(const __half* x, int V) {
  const int mis = (int)(((uintptr_t)x >> 1) & 7);
  const int head = min(V, (8 - mis) & 7);
  const int nvec = (V - head) >> 3;
  return RowSplit{head, nvec, head + 8 * nvec};
}

// The statistics of row x (V values), by every thread of the CTA (a barrier inside; part: LP_WARPS shared slots).
__device__ __forceinline__ RowStat row_stat(const __half* x, int V, RowStat* part) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  RowStat a{-INFINITY, 0.f, -INFINITY, 0x7FFFFFFF, false};
  const RowSplit sp = row_split(x, V);
  if (tid < sp.head) add_one(a, __half2float(x[tid]), tid);
  const uint4* xv = reinterpret_cast<const uint4*>(x + sp.head);
  int k = tid;
  for (; k + LP_THREADS < sp.nvec; k += 2 * LP_THREADS) {        // two loads in flight
    const uint4 u0 = __ldg(xv + k), u1 = __ldg(xv + k + LP_THREADS);
    add_eight(a, u0, sp.head + 8 * k);
    add_eight(a, u1, sp.head + 8 * (k + LP_THREADS));
  }
  if (k < sp.nvec) add_eight(a, __ldg(xv + k), sp.head + 8 * k);
  if (sp.body_end + tid < V) add_one(a, __half2float(x[sp.body_end + tid]), sp.body_end + tid);

#pragma unroll
  for (int o = 16; o; o >>= 1) merge(a, shfl_xor(a, o));
  if (lane == 0) part[warp] = a;
  __syncthreads();
  RowStat t = part[0];
  for (int w = 1; w < LP_WARPS; ++w) merge(t, part[w]);
  return t;
}

}  // namespace quip
