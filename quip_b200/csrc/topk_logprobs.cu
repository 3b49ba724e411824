// Log-probabilities of generation: for each fp16 logits row, the logprob of the chosen token and the top-n tokens
// with their logprobs, written at the row's output column.  The rule is stated in include/quip_b200.h
// (quip_token_topk_logprobs); oracle/topk_logprobs.py restates it in numpy.
//
// One CTA per row.  The row pass of logprob_row.cuh gives (m, s), so every logprob (x - m) - log(s) has the bits
// quip_token_logprobs gives for that id.  The top n are found on 16-bit order-preserving keys of the fp16 values
// (-0 == +0): a 256-bin histogram of the high byte picks the byte holding the n-th largest key, a second one of the low
// byte among the values with that high byte picks the threshold key k*.  A third pass collects the (at most n - 1)
// values above k* and the values equal to k*, of which the lowest ids are taken: by rank when at most TK_TIE_CAP are
// tied, else by an in-order scan of 16 contiguous segments, one per warp.  The n entries are ranked in shared memory
// by (key descending, id ascending).  Each pass re-reads the row, mostly from L2.
#include "logprob_row.cuh"

namespace quip {

namespace {

constexpr int TK_MAX_N = 20;
constexpr int TK_MAX_T = 8;
constexpr int TK_MAX_V = 1 << 24;
constexpr int TK_TIE_CAP = 64;

// fp16 bits (not NaN) -> a key that orders like the value, -0 and +0 alike
__device__ __forceinline__ uint32_t order_key(uint32_t u) {
  u = u == 0x8000u ? 0u : u;
  return (u & 0x8000u) ? (~u & 0xFFFFu) : (u | 0x8000u);
}

// f(key, index) for each value of this thread's share of row x (the split of row_stat)
template <class F>
__device__ __forceinline__ void for_each_key(const __half* x, int V, F&& f) {
  const int tid = threadIdx.x;
  const uint16_t* xs = reinterpret_cast<const uint16_t*>(x);
  const RowSplit sp = row_split(x, V);
  if (tid < sp.head) f(order_key(xs[tid]), tid);
  const uint4* xv = reinterpret_cast<const uint4*>(x + sp.head);
  for (int k = tid; k < sp.nvec; k += LP_THREADS) {
    const uint4 u = __ldg(xv + k);
    const uint32_t w[4] = {u.x, u.y, u.z, u.w};
    const int i0 = sp.head + 8 * k;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      f(order_key(w[j] & 0xFFFFu), i0 + 2 * j);
      f(order_key(w[j] >> 16), i0 + 2 * j + 1);
    }
  }
  if (sp.body_end + tid < V) f(order_key(xs[sp.body_end + tid]), sp.body_end + tid);
}

// Warp 0: the bin of hist (256 counts) holding the need-th entry counted from the top bin (1 <= need <= total),
// into sel[0], and the count of the bins above it into sel[1].
__device__ __forceinline__ void pick_bin(const int* hist, int need, int* sel) {
  const int lane = threadIdx.x & 31, hi = 255 - 8 * lane;
  int s = 0;
#pragma unroll
  for (int j = 0; j < 8; ++j) s += hist[hi - j];
  int p = s;                                                       // inclusive prefix, lane 0 holding the top bins
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int v = __shfl_up_sync(0xFFFFFFFFu, p, o);
    if (lane >= o) p += v;
  }
  const unsigned hit = __ballot_sync(0xFFFFFFFFu, p >= need);
  if (lane != __ffs(hit) - 1) return;
  int run = p - s;
  for (int j = 0; j < 8; ++j) {
    const int c = hist[hi - j];
    if (run + c >= need) {
      sel[0] = hi - j;
      sel[1] = run;
      return;
    }
    run += c;
  }
}

__global__ void __launch_bounds__(LP_THREADS) topk_logprobs_kernel(
    const __half* __restrict__ logits, int64_t ld, int T, int V, const int64_t* __restrict__ rows,
    const int64_t* __restrict__ tokens, const int64_t* __restrict__ cols, int cols_stride, float* __restrict__ lp,
    int64_t* __restrict__ top_ids, float* __restrict__ top_lp, int n, int B, int gen_cols) {
  __shared__ RowStat part[LP_WARPS];
  __shared__ int hist[256];
  __shared__ int sel[2];
  __shared__ int n_gt, n_tie;
  __shared__ uint32_t gt_key[TK_MAX_N];
  __shared__ int gt_id[TK_MAX_N];
  __shared__ int tie_id[TK_TIE_CAP];
  __shared__ int warp_n[LP_WARPS];
  __shared__ int warp_tie[LP_WARPS][TK_MAX_N];
  __shared__ int out_id[TK_MAX_N];

  const int r = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int64_t b = rows ? rows[r / T] : (int64_t)(r / T);
  if (b < 0 || b >= B) return;
  const int64_t c = cols[b * cols_stride] + r % T;
  if (c < 0 || c >= gen_cols) return;                            // a done row's last entry stays as it is
  const __half* x = logits + (size_t)r * (size_t)ld;
  const RowStat t = row_stat(x, V, part);
  const size_t o = (size_t)b * (size_t)gen_cols + (size_t)c;
  if (tid == 0) {
    const int64_t tg = tokens[r];
    lp[o] = t.nan || tg < 0 || tg >= V ? __int_as_float(0x7FC00000) : (__half2float(x[tg]) - t.m) - logf(t.s);
  }
  if (n == 0) return;
  int64_t* ids = top_ids + o * (size_t)n;
  float* vals = top_lp + o * (size_t)n;
  const int need = t.nan ? 0 : min(n, V);
  if (tid >= need && tid < n) {
    ids[tid] = -1;
    vals[tid] = __int_as_float(0x7FC00000);
  }
  if (need == 0) return;

  // the threshold key: high byte, then low byte among the values with that high byte
  for (int i = tid; i < 256; i += LP_THREADS) hist[i] = 0;
  __syncthreads();
  for_each_key(x, V, [&](uint32_t k, int) { atomicAdd(&hist[k >> 8], 1); });
  __syncthreads();
  if (tid < 32) pick_bin(hist, need, sel);
  __syncthreads();
  const uint32_t hb = (uint32_t)sel[0];
  const int above_hb = sel[1];
  __syncthreads();
  for (int i = tid; i < 256; i += LP_THREADS) hist[i] = 0;
  __syncthreads();
  for_each_key(x, V, [&](uint32_t k, int) {
    if ((k >> 8) == hb) atomicAdd(&hist[k & 0xFFu], 1);
  });
  __syncthreads();
  if (tid < 32) pick_bin(hist, need - above_hb, sel);
  if (tid == 0) n_gt = n_tie = 0;
  __syncthreads();
  const uint32_t kth = (hb << 8) | (uint32_t)sel[0];
  const int n_above = above_hb + sel[1];                          // entries ranked above every value equal to kth
  const int ties = hist[sel[0]];
  const int take = need - n_above;                                // 1 <= take <= ties: the lowest ids among them
  const bool few = ties <= TK_TIE_CAP;

  for_each_key(x, V, [&](uint32_t k, int i) {
    if (k > kth) {
      const int s = atomicAdd(&n_gt, 1);
      gt_key[s] = k;
      gt_id[s] = i;
    } else if (few && k == kth) {
      tie_id[atomicAdd(&n_tie, 1)] = i;
    }
  });
  if (!few) {                                                     // warp w scans its segment in index order
    const uint16_t* xs = reinterpret_cast<const uint16_t*>(x);
    const int seg = (V + LP_WARPS - 1) / LP_WARPS;
    const int lo = warp * seg, hi = min(V, lo + seg);
    int found = 0;
    for (int base = lo; base < hi && found < take; base += 32) {
      const int i = base + lane;
      const bool hit = i < hi && order_key(xs[i]) == kth;
      const unsigned m = __ballot_sync(0xFFFFFFFFu, hit);
      const int pos = found + __popc(m & ((1u << lane) - 1u));
      if (hit && pos < take) warp_tie[warp][pos] = i;
      found += __popc(m);
    }
    if (lane == 0) warp_n[warp] = min(found, take);
  }
  __syncthreads();

  if (tid < n_above) {
    const uint32_t k = gt_key[tid];
    const int i = gt_id[tid];
    int rank = 0;
    for (int j = 0; j < n_above; ++j) rank += gt_key[j] > k || (gt_key[j] == k && gt_id[j] < i);
    out_id[rank] = i;
  }
  if (few) {
    if (tid < ties) {
      const int i = tie_id[tid];
      int rank = 0;
      for (int j = 0; j < ties; ++j) rank += tie_id[j] < i;
      if (rank < take) out_id[n_above + rank] = i;
    }
  } else if (tid == 0) {
    int q = n_above;
    for (int w = 0; w < LP_WARPS; ++w)
      for (int j = 0; j < warp_n[w] && q < need; ++j) out_id[q++] = warp_tie[w][j];
  }
  __syncthreads();
  if (tid < need) {
    const int i = out_id[tid];
    ids[tid] = i;
    vals[tid] = (__half2float(x[i]) - t.m) - logf(t.s);
  }
}

}  // namespace

}  // namespace quip

using namespace quip;

extern "C" int quip_token_topk_logprobs(const void* logits, int64_t ld, int32_t R, int32_t T, int32_t V,
                                        const int64_t* rows, const int64_t* tokens, const int64_t* cols,
                                        int32_t cols_per_row, float* lp, int64_t* top_ids, float* top_lp, int32_t n,
                                        int32_t B, int32_t gen_cols, void* stream) {
  QUIP_CHECK_ARG(R >= 0 && T >= 1 && T <= TK_MAX_T && R % T == 0 && V >= 1 && V <= TK_MAX_V && ld >= V && n >= 0 &&
                     n <= TK_MAX_N && B >= 1 && gen_cols >= 1 && (cols_per_row == 0 || cols_per_row == 1),
                 "quip_token_topk_logprobs: bad sizes (R %d, T %d, V %d, ld %lld, n %d, B %d, gen_cols %d, "
                 "cols_per_row %d): need 1 <= T <= %d dividing R, 1 <= V <= %d, ld >= V, 0 <= n <= %d, B >= 1, "
                 "gen_cols >= 1 and cols_per_row 0 or 1", R, T, V, (long long)ld, n, B, gen_cols, cols_per_row,
                 TK_MAX_T, TK_MAX_V, TK_MAX_N);
  QUIP_CHECK_ARG(logits && tokens && cols && lp && ((top_ids && top_lp) || n == 0),
                 "quip_token_topk_logprobs: null pointer");
  QUIP_CHECK_ARG(((uintptr_t)logits & 1) == 0 && ((uintptr_t)rows & 7) == 0 && ((uintptr_t)tokens & 7) == 0 &&
                     ((uintptr_t)cols & 7) == 0 && ((uintptr_t)top_ids & 7) == 0 && ((uintptr_t)lp & 3) == 0 &&
                     ((uintptr_t)top_lp & 3) == 0,
                 "quip_token_topk_logprobs: logits must be 2-byte, int64 arrays 8-byte and fp32 arrays 4-byte aligned");
  if (R == 0) return QUIP_OK;
  topk_logprobs_kernel<<<(unsigned)R, LP_THREADS, 0, (cudaStream_t)stream>>>(
      (const __half*)logits, ld, T, V, rows, tokens, cols, cols_per_row, lp, top_ids, top_lp, n, B, gen_cols);
  QUIP_LAUNCHED("topk_logprobs_kernel");
  return QUIP_OK;
}
