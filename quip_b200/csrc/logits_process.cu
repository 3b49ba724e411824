// Logits processors of generation: repetition penalty, no-repeat n-gram, bad words and min_new_tokens, in place on
// fp16 logits rows.  The rule is stated in include/quip_b200.h (quip_logits_process); oracle/logits_process.py restates
// it in numpy.
//
// One CTA per logits row.  Three V-bit shared-memory bitmaps: `seen` (the penalty's distinct history tokens), `hard`
// (n-gram and min_new bans: -inf) and `bias` (bad-word bans: + -inf).  Phase 1 walks the history: the thread whose
// atomicOr first sets a token's `seen` bit penalises that token, so each token is penalised once whatever the
// interleaving; the same phase tests every n-gram start e and every bad-word sequence and sets ban bits.  After a
// barrier, phase 2 scans the ban bitmaps word by word and writes the banned entries.  With bad words, phase 3 turns the
// row's -0 entries into +0 (the +0 of HF's bias row), 16-byte vectors over the aligned body.  Every write is a function
// of the row's data and settings only, so launches are bit-identical.
#include <math.h>

#include "common.cuh"

namespace quip {

namespace {

constexpr int LPR_THREADS = 512;
constexpr int LPR_MAX_V = 1 << 18;
constexpr int LPR_MAX_EOS = 8;
constexpr int LPR_MAX_BAD = 256;
constexpr int LPR_BAD_LEN = 16;

struct History {
  const int64_t* hist;    // hist[b, 0 .. c]
  const int64_t* drafts;  // tokens[b, 0 ..]: position c + j is drafts[j], j >= 1
  int64_t c;
  __device__ __forceinline__ int64_t at(int64_t j) const { return j <= c ? hist[j] : drafts[j - c]; }
};

__device__ __forceinline__ bool in_vocab(int64_t v, int V) { return v >= 0 && v < V; }

__device__ __forceinline__ void set_bit(uint32_t* bits, int64_t v) {
  atomicOr(bits + (v >> 5), 1u << (v & 31));
}

__global__ void __launch_bounds__(LPR_THREADS) logits_process_kernel(
    __half* __restrict__ logits, int64_t ld, int T, int V, const int64_t* __restrict__ rows,
    const int64_t* __restrict__ hist, const int64_t* __restrict__ last, const int64_t* __restrict__ tokens,
    const int64_t* __restrict__ prompt_len, const float* __restrict__ penalty, const int32_t* __restrict__ ngram,
    const int32_t* __restrict__ min_new, const int64_t* __restrict__ eos, int n_eos, const int64_t* __restrict__ bad,
    const int32_t* __restrict__ bad_len, int n_bad, int B, int max_len) {
  extern __shared__ uint32_t lpr_bits[];
  const int r = blockIdx.x, tid = threadIdx.x;
  const int64_t b = rows ? rows[r / T] : (int64_t)(r / T);
  if (b < 0 || b >= B) return;
  const int64_t c = last[b];
  if (c < 0 || c >= max_len) return;
  const int i = r % T;
  const int64_t L = c + 1 + i;
  const float rho = penalty[b];
  const int n = ngram[b];
  const bool pen = rho != 1.f;
  const bool ng = n >= 1 && n <= L;
  const bool ban_eos = n_eos > 0 && L - prompt_len[b] < (int64_t)min_new[b];
  if (!pen && !ng && !ban_eos && n_bad == 0) return;

  const int W = (V + 31) >> 5;
  uint32_t* seen = lpr_bits;
  uint32_t* hard = lpr_bits + W;
  uint32_t* bias = lpr_bits + 2 * W;
  for (int w = tid; w < 3 * W; w += LPR_THREADS) lpr_bits[w] = 0u;
  __syncthreads();

  __half* x = logits + (size_t)r * (size_t)ld;
  const History h{hist + (size_t)b * (size_t)max_len, tokens ? tokens + (size_t)b * (size_t)T : nullptr, c};
  if (pen) {
    for (int64_t j = tid; j < L; j += LPR_THREADS) {
      const int64_t v = h.at(j);
      if (!in_vocab(v, V)) continue;
      const uint32_t bit = 1u << (v & 31);
      if (atomicOr(seen + (v >> 5), bit) & bit) continue;
      const float f = __half2float(x[v]);
      x[v] = __float2half_rn(f < 0.f ? __fmul_rn(f, rho) : __fdiv_rn(f, rho));
    }
  }
  if (ng) {
    const int64_t s0 = L - n + 1;  // the current (n-1)-token suffix starts here
    for (int64_t e = tid; e <= L - n; e += LPR_THREADS) {
      bool match = true;
      for (int k = 0; k < n - 1 && match; ++k) match = h.at(e + k) == h.at(s0 + k);
      if (!match) continue;
      const int64_t v = h.at(e + n - 1);
      if (in_vocab(v, V)) set_bit(hard, v);
    }
  }
  for (int s = tid; s < n_bad; s += LPR_THREADS) {
    const int l = bad_len[s];
    const int64_t* w = bad + (size_t)s * LPR_BAD_LEN;
    if (l < 1 || l > LPR_BAD_LEN || (l > 1 && (int64_t)l > L)) continue;
    bool match = true;
    if (l == 1) {
      for (int k = 0; k < n_eos; ++k) match &= w[0] != eos[k];
    } else {
      for (int k = 0; k < l - 1 && match; ++k) match = h.at(L - l + 1 + k) == w[k];
    }
    if (match && in_vocab(w[l - 1], V)) set_bit(bias, w[l - 1]);
  }
  if (ban_eos && tid < n_eos && in_vocab(eos[tid], V)) set_bit(hard, eos[tid]);
  __syncthreads();

  for (int wi = tid; wi < W; wi += LPR_THREADS) {
    const uint32_t hb = hard[wi], bb = bias[wi];
    uint32_t u = hb | bb;
    while (u) {
      const int k = __ffs(u) - 1;
      u &= u - 1;
      const int v = wi * 32 + k;
      x[v] = (hb >> k) & 1u ? __float2half_rn(-INFINITY) : __float2half_rn(__half2float(x[v]) + (-INFINITY));
    }
  }
  if (n_bad == 0) return;
  __syncthreads();

  // -0 -> +0 over the row: scalars up to the first 16-byte boundary, 8 values per load, scalars for the tail
  uint16_t* xs = reinterpret_cast<uint16_t*>(x);
  const int mis = (int)(((uintptr_t)x >> 1) & 7);
  const int head = min(V, (8 - mis) & 7);
  const int nvec = (V - head) >> 3;
  const int body_end = head + 8 * nvec;
  if (tid < head && xs[tid] == 0x8000u) xs[tid] = 0;
  uint4* xv = reinterpret_cast<uint4*>(x + head);
  for (int k = tid; k < nvec; k += LPR_THREADS) {
    uint4 u = xv[k];
    uint32_t* p = reinterpret_cast<uint32_t*>(&u);
    bool hit = false;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const uint32_t lo = (p[j] & 0xFFFFu) == 0x8000u ? 0xFFFF0000u : 0xFFFFFFFFu;
      const uint32_t hi = (p[j] >> 16) == 0x8000u ? 0x0000FFFFu : 0xFFFFFFFFu;
      hit |= (lo & hi) != 0xFFFFFFFFu;
      p[j] &= lo & hi;
    }
    if (hit) xv[k] = u;
  }
  if (body_end + tid < V && xs[body_end + tid] == 0x8000u) xs[body_end + tid] = 0;
}

}  // namespace

}  // namespace quip

using namespace quip;

extern "C" int quip_logits_process(void* logits, int64_t ld, int32_t R, int32_t T, int32_t V, const int64_t* rows,
                                   const int64_t* hist, const int64_t* last, const int64_t* tokens,
                                   const int64_t* prompt_len, const float* penalty, const int32_t* ngram,
                                   const int32_t* min_new, const int64_t* eos, int32_t n_eos, const int64_t* bad,
                                   const int32_t* bad_len, int32_t n_bad, int32_t B, int32_t max_len, void* stream) {
  QUIP_CHECK_ARG(R >= 0 && T >= 1 && R % T == 0 && V >= 1 && V <= LPR_MAX_V && ld >= V && B >= 1 && max_len >= 1,
                 "quip_logits_process: bad sizes (R %d, T %d, V %d, ld %lld, B %d, max_len %d): need R %% T == 0, "
                 "1 <= V <= %d, ld >= V, B >= 1 and max_len >= 1", R, T, V, (long long)ld, B, max_len, LPR_MAX_V);
  QUIP_CHECK_ARG(n_eos >= 0 && n_eos <= LPR_MAX_EOS && n_bad >= 0 && n_bad <= LPR_MAX_BAD,
                 "quip_logits_process: %d eos ids and %d bad words: at most %d and %d", n_eos, n_bad, LPR_MAX_EOS,
                 LPR_MAX_BAD);
  QUIP_CHECK_ARG(logits && hist && last && prompt_len && penalty && ngram && min_new && (tokens || T == 1) &&
                     (eos || n_eos == 0) && ((bad && bad_len) || n_bad == 0),
                 "quip_logits_process: null pointer");
  QUIP_CHECK_ARG(((uintptr_t)logits & 1) == 0 && ((uintptr_t)hist & 7) == 0 && ((uintptr_t)last & 7) == 0 &&
                     ((uintptr_t)tokens & 7) == 0 && ((uintptr_t)prompt_len & 7) == 0 && ((uintptr_t)rows & 7) == 0 &&
                     ((uintptr_t)eos & 7) == 0 && ((uintptr_t)bad & 7) == 0 && ((uintptr_t)penalty & 3) == 0 &&
                     ((uintptr_t)ngram & 3) == 0 && ((uintptr_t)min_new & 3) == 0 && ((uintptr_t)bad_len & 3) == 0,
                 "quip_logits_process: logits must be 2-byte, int64 arrays 8-byte and 4-byte arrays 4-byte aligned");
  if (R == 0) return QUIP_OK;
  const size_t smem = 3 * (size_t)((V + 31) / 32) * sizeof(uint32_t);
  if (smem > 48 * 1024)
    QUIP_CUDA(cudaFuncSetAttribute(logits_process_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  logits_process_kernel<<<(unsigned)R, LPR_THREADS, smem, (cudaStream_t)stream>>>(
      (__half*)logits, ld, T, V, rows, hist, last, tokens, prompt_len, penalty, ngram, min_new, eos, n_eos, bad,
      bad_len, n_bad, B, max_len);
  QUIP_LAUNCHED("logits_process_kernel");
  return QUIP_OK;
}
