// Speculative generation: prompt-lookup drafts (quip_ngram_draft) and the acceptance of a verified step
// (quip_spec_accept).  The rules are stated in include/quip_b200.h; oracle/speculative.py restates them as numpy loops.
// Both read their counters from device memory and write them back, so a captured decode graph needs no host round trip.
#include "common.cuh"

namespace quip {

namespace {

constexpr int ND_THREADS = 256;
constexpr int SA_THREADS = 128;

// One CTA per row.  Thread t scores the candidate ends e = t, t + ND_THREADS, ... < c by the length of the common suffix
// of hist[..e] and hist[..c] (capped at n_max); the key (L << 32) | (e + 1) orders longest first, then most recent.
__global__ void __launch_bounds__(ND_THREADS)
ngram_draft_kernel(const int64_t* __restrict__ hist, const int64_t* __restrict__ positions, int64_t* __restrict__ tokens,
                   int max_len, int k, int n_min, int n_max) {
  __shared__ unsigned long long wbest[ND_THREADS / 32];
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int64_t* h = hist + (int64_t)b * max_len;
  int64_t* out = tokens + (int64_t)b * (k + 1);
  const int64_t c64 = positions[b];
  if (c64 < 0 || c64 >= max_len) {            // no current token in the history: zeros
    for (int i = tid; i <= k; i += ND_THREADS) out[i] = 0;
    return;
  }
  const int c = (int)c64;
  unsigned long long best = 0;
  for (int e = tid; e < c; e += ND_THREADS) {
    int L = 0;
    while (L < n_max && L <= e && h[e - L] == h[c - L]) ++L;
    if (L >= n_min) {
      const unsigned long long key = ((unsigned long long)L << 32) | (unsigned)(e + 1);
      best = key > best ? key : best;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const unsigned long long y = __shfl_xor_sync(0xffffffffu, best, o);
    best = y > best ? y : best;
  }
  if (lane == 0) wbest[warp] = best;
  __syncthreads();
  if (tid != 0) return;
  for (int w = 0; w < ND_THREADS / 32; ++w) best = wbest[w] > best ? wbest[w] : best;
  const int64_t cur = h[c];
  out[0] = cur;
  const int e = (int)(best & 0xFFFFFFFFull) - 1;   // -1: no match
  for (int i = 1; i <= k; ++i) {
    const int u = e + i;                           // u <= c: the history; past c: the drafts written so far
    out[i] = e < 0 ? cur : (u <= c ? h[u] : out[u - c]);
  }
}

__global__ void __launch_bounds__(SA_THREADS)
spec_accept_kernel(const int64_t* __restrict__ tokens, const int64_t* __restrict__ targets, int64_t* __restrict__ generated,
                   int64_t* __restrict__ hist, int64_t* __restrict__ positions, int64_t* __restrict__ n_gen,
                   int64_t* __restrict__ accepted, int B, int T, int max_new, int gen_cols, int max_len) {
  const int b = blockIdx.x * SA_THREADS + threadIdx.x;
  if (b >= B) return;
  const int64_t g = n_gen[b];
  if (g < 0 || g >= max_new) return;            // finished: no advance
  const int64_t* d = tokens + (int64_t)b * T;
  const int64_t* y = targets + (int64_t)b * T;
  int a = 0;
  while (a < T - 1 && d[a + 1] == y[a]) ++a;
  const int64_t e = min((int64_t)a + 1, (int64_t)max_new - g);
  const int64_t c = positions[b];
  for (int64_t j = 0; j < e; ++j) {
    generated[(int64_t)b * gen_cols + g + j] = y[j];
    if (c + 1 + j >= 0 && c + 1 + j < max_len) hist[(int64_t)b * max_len + c + 1 + j] = y[j];
  }
  positions[b] = c + e;
  n_gen[b] = g + e;
  accepted[b] += e - 1;
}

}  // namespace

}  // namespace quip

using namespace quip;

extern "C" int quip_ngram_draft(const int64_t* hist, const int64_t* positions, int64_t* tokens, int32_t B,
                                int32_t max_len, int32_t k, int32_t n_min, int32_t n_max, void* stream) {
  QUIP_CHECK_ARG(hist && positions && tokens, "quip_ngram_draft: null pointer");
  QUIP_CHECK_ARG(B >= 0 && B <= 0x7FFFFFFF && max_len > 0 && k >= 0,
                 "quip_ngram_draft: bad sizes (B %d, max_len %d, k %d)", B, max_len, k);
  QUIP_CHECK_ARG(n_min >= 1 && n_max >= n_min, "quip_ngram_draft: need 1 <= n_min <= n_max, got n_min %d, n_max %d",
                 n_min, n_max);
  if (B == 0) return QUIP_OK;
  ngram_draft_kernel<<<(unsigned)B, ND_THREADS, 0, (cudaStream_t)stream>>>(hist, positions, tokens, max_len, k, n_min,
                                                                           n_max);
  QUIP_LAUNCHED("ngram_draft_kernel");
  return QUIP_OK;
}

extern "C" int quip_spec_accept(const int64_t* tokens, const int64_t* targets, int64_t* generated, int64_t* hist,
                                int64_t* positions, int64_t* n_gen, int64_t* accepted, int32_t B, int32_t T,
                                int32_t max_new, int32_t gen_cols, int32_t max_len, void* stream) {
  QUIP_CHECK_ARG(tokens && targets && generated && hist && positions && n_gen && accepted, "quip_spec_accept: null pointer");
  QUIP_CHECK_ARG(B >= 0 && T >= 1 && max_len > 0 && max_new >= 0 && max_new <= gen_cols,
                 "quip_spec_accept: bad sizes (B %d, T %d, max_new %d, gen_cols %d, max_len %d): need max_new <= gen_cols",
                 B, T, max_new, gen_cols, max_len);
  if (B == 0) return QUIP_OK;
  spec_accept_kernel<<<(unsigned)ceil_div(B, SA_THREADS), SA_THREADS, 0, (cudaStream_t)stream>>>(
      tokens, targets, generated, hist, positions, n_gen, accepted, B, T, max_new, gen_cols, max_len);
  QUIP_LAUNCHED("spec_accept_kernel");
  return QUIP_OK;
}
