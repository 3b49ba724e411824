// Constrained generation: a token automaton's allowed-token mask on fp16 logits rows, and the advance of each row's
// state over the tokens a step commits.  The rule is stated in include/quip_b200.h (quip_constrain_mask,
// quip_constrain_advance); oracle/constrain.py restates it in numpy.
//
// Mask: one CTA per logits row.  Thread 0 walks the row's drafts (one binary search over a state's sorted ids per
// draft), the CTA sets the V-bit shared-memory bitmap of the final state's allowed ids (one atomicOr per word a warp
// touches, so any table is safe), and after a barrier rewrites the whole row as x + (allowed ? +0 : -inf) with __hadd2,
// 16-byte vectors over the aligned body and scalars for the head and tail (rows need only 2-byte alignment).  Every
// write is a function of the row, its state, its drafts and the table only, so launches are bit-identical.
#include "common.cuh"

namespace quip {

namespace {

constexpr int CM_THREADS = 512;
constexpr int CM_MAX_V = 1 << 18;
constexpr int CM_MAX_T = 8;
constexpr int CA_THREADS = 128;

struct Table {
  const int32_t* offsets;  // (S + 1)
  const int32_t* ids;      // (nnz), strictly increasing within a state
  const int32_t* next;     // (nnz)
  int S, nnz;

  // state s's entries [lo, hi), clamped into the table whatever offsets holds; s must lie in [0, S)
  __device__ __forceinline__ void range(int s, int& lo, int& hi) const {
    lo = min(max(offsets[s], 0), nnz);
    hi = min(max(offsets[s + 1], lo), nnz);
  }

  __device__ __forceinline__ int delta(int s, int64_t v) const {
    if (s < 0 || s >= S) return s;
    int lo, hi;
    range(s, lo, hi);
    int a = lo, b = hi;  // first k in [lo, hi) with ids[k] >= v
    while (a < b) {
      const int m = (a + b) >> 1;
      if ((int64_t)ids[m] < v) a = m + 1;
      else b = m;
    }
    return a < hi && (int64_t)ids[a] == v ? next[a] : s;
  }
};

// +0 where bit j of m is set (allowed), -inf elsewhere, for the two values j = 2p, 2p + 1
__device__ __forceinline__ __half2 bias2(uint32_t m, int p) {
  const uint16_t lo = (m >> (2 * p)) & 1u ? 0 : 0xFC00u;
  const uint16_t hi = (m >> (2 * p + 1)) & 1u ? 0 : 0xFC00u;
  return __halves2half2(__ushort_as_half(lo), __ushort_as_half(hi));
}

__device__ __forceinline__ __half bias1(const uint32_t* bits, int v) {
  return __ushort_as_half((bits[v >> 5] >> (v & 31)) & 1u ? (uint16_t)0 : (uint16_t)0xFC00u);
}

__global__ void __launch_bounds__(CM_THREADS) constrain_mask_kernel(__half* __restrict__ logits, int64_t ld, int T,
                                                                    int V, const int64_t* __restrict__ rows,
                                                                    const int64_t* __restrict__ tokens,
                                                                    const int32_t* __restrict__ state, int B, Table tb) {
  extern __shared__ uint32_t cm_bits[];
  __shared__ int cm_state;
  const int r = blockIdx.x, tid = threadIdx.x;
  const int64_t b = rows ? rows[r / T] : (int64_t)(r / T);
  if (b < 0 || b >= B) return;
  if (tid == 0) {
    int s = state[b];
    const int i = r % T;
    for (int j = 1; j <= i; ++j) s = tb.delta(s, tokens[(size_t)b * T + j]);
    cm_state = s;
  }
  __syncthreads();
  const int s = cm_state;
  if (s < 0 || s >= tb.S) return;

  const int W = (V + 31) >> 5;
  for (int w = tid; w < W; w += CM_THREADS) cm_bits[w] = 0u;
  __syncthreads();
  int lo, hi;
  tb.range(s, lo, hi);
  // sorted ids put a warp's 32 ids in one or two words: the lanes of a word combine their bits and one of them ORs
  // them in
  const int lane = tid & 31;
  for (int k0 = lo + (tid & ~31); k0 < hi; k0 += CM_THREADS) {
    const int k = k0 + lane;
    const int v = k < hi ? tb.ids[k] : -1;
    const int w = v >= 0 && v < V ? v >> 5 : -1;
    const unsigned same = __match_any_sync(0xFFFFFFFFu, w);
    const uint32_t word = __reduce_or_sync(same, w >= 0 ? 1u << (v & 31) : 0u);
    if (w >= 0 && lane == __ffs(same) - 1) atomicOr(cm_bits + w, word);
  }
  __syncthreads();

  __half* x = logits + (size_t)r * (size_t)ld;
  const int mis = (int)(((uintptr_t)x >> 1) & 7);
  const int head = min(V, (8 - mis) & 7);
  const int nvec = (V - head) >> 3;
  const int body_end = head + 8 * nvec;
  if (tid < head) x[tid] = __hadd(x[tid], bias1(cm_bits, tid));
  uint4* xv = reinterpret_cast<uint4*>(x + head);
  for (int k = tid; k < nvec; k += CM_THREADS) {
    const int v0 = head + 8 * k, w = v0 >> 5, o = v0 & 31;
    // v0 + 7 < V, so a group crossing into word w + 1 stays inside the bitmap
    const uint32_t m = (cm_bits[w] >> o) | (o > 24 ? cm_bits[w + 1] << (32 - o) : 0u);
    uint4 u = xv[k];
    __half2* h = reinterpret_cast<__half2*>(&u);
#pragma unroll
    for (int p = 0; p < 4; ++p) h[p] = __hadd2(h[p], bias2(m, p));
    xv[k] = u;
  }
  if (body_end + tid < V) x[body_end + tid] = __hadd(x[body_end + tid], bias1(cm_bits, body_end + tid));
}

__global__ void __launch_bounds__(CA_THREADS) constrain_advance_kernel(int32_t* __restrict__ state, int B,
                                                                       const int64_t* __restrict__ tok, int64_t ld,
                                                                       int N, int T, const int64_t* __restrict__ rows,
                                                                       const int64_t* __restrict__ counts, Table tb) {
  const int n = blockIdx.x * CA_THREADS + threadIdx.x;
  if (n >= N) return;
  const int64_t b = rows ? rows[n] : (int64_t)n;
  if (b < 0 || b >= B) return;
  const int64_t c = counts ? min(max(counts[n], (int64_t)0), (int64_t)T) : (int64_t)T;
  int s = state[b];
  for (int64_t j = 0; j < c; ++j) s = tb.delta(s, tok[(size_t)n * (size_t)ld + j]);
  state[b] = s;
}

bool al(const void* p, int a) { return ((uintptr_t)p & (uintptr_t)(a - 1)) == 0; }

}  // namespace

}  // namespace quip

using namespace quip;

extern "C" int quip_constrain_mask(void* logits, int64_t ld, int32_t R, int32_t T, int32_t V, const int64_t* rows,
                                   const int64_t* tokens, const int32_t* state, int32_t B, const int32_t* offsets,
                                   const int32_t* ids, const int32_t* next, int32_t S, int32_t nnz, void* stream) {
  QUIP_CHECK_ARG(R >= 0 && T >= 1 && T <= CM_MAX_T && R % T == 0 && V >= 1 && V <= CM_MAX_V && ld >= V && B >= 1 &&
                     S >= 0 && nnz >= 0,
                 "quip_constrain_mask: bad sizes (R %d, T %d, V %d, ld %lld, B %d, S %d, nnz %d): need 1 <= T <= %d "
                 "dividing R, 1 <= V <= %d, ld >= V, B >= 1, S >= 0 and nnz >= 0", R, T, V, (long long)ld, B, S, nnz,
                 CM_MAX_T, CM_MAX_V);
  QUIP_CHECK_ARG(logits && state && offsets && (tokens || T == 1) && ((ids && next) || nnz == 0),
                 "quip_constrain_mask: null pointer");
  QUIP_CHECK_ARG(al(logits, 2) && al(rows, 8) && al(tokens, 8) && al(state, 4) && al(offsets, 4) && al(ids, 4) &&
                     al(next, 4),
                 "quip_constrain_mask: logits must be 2-byte, int64 arrays 8-byte and int32 arrays 4-byte aligned");
  if (R == 0) return QUIP_OK;
  const size_t smem = (size_t)((V + 31) / 32) * sizeof(uint32_t);
  constrain_mask_kernel<<<(unsigned)R, CM_THREADS, smem, (cudaStream_t)stream>>>(
      (__half*)logits, ld, T, V, rows, tokens, state, B, Table{offsets, ids, next, S, nnz});
  QUIP_LAUNCHED("constrain_mask_kernel");
  return QUIP_OK;
}

extern "C" int quip_constrain_advance(int32_t* state, int32_t B, const int64_t* tok, int64_t ld, int32_t N, int32_t T,
                                      const int64_t* rows, const int64_t* counts, const int32_t* offsets,
                                      const int32_t* ids, const int32_t* next, int32_t S, int32_t nnz, void* stream) {
  QUIP_CHECK_ARG(N >= 0 && T >= 1 && T <= CM_MAX_T && ld >= T && B >= 1 && S >= 0 && nnz >= 0,
                 "quip_constrain_advance: bad sizes (N %d, T %d, ld %lld, B %d, S %d, nnz %d): need N >= 0, "
                 "1 <= T <= %d, ld >= T, B >= 1, S >= 0 and nnz >= 0", N, T, (long long)ld, B, S, nnz, CM_MAX_T);
  QUIP_CHECK_ARG(state && tok && offsets && ((ids && next) || nnz == 0), "quip_constrain_advance: null pointer");
  QUIP_CHECK_ARG(al(tok, 8) && al(rows, 8) && al(counts, 8) && al(state, 4) && al(offsets, 4) && al(ids, 4) &&
                     al(next, 4),
                 "quip_constrain_advance: int64 arrays must be 8-byte and int32 arrays 4-byte aligned");
  if (N == 0) return QUIP_OK;
  constrain_advance_kernel<<<(unsigned)ceil_div(N, CA_THREADS), CA_THREADS, 0, (cudaStream_t)stream>>>(
      state, B, tok, ld, N, T, rows, counts, Table{offsets, ids, next, S, nnz});
  QUIP_LAUNCHED("constrain_advance_kernel");
  return QUIP_OK;
}
