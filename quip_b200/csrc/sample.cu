// Token selection for generation: temperature, top-k and top-p sampling with per-row Philox4x32-10 seeds, or greedy
// argmax, one CTA per row of fp16 logits (B, V).  The rule is stated in include/quip_b200.h; oracle/sampling.py restates it.
//
// Every decision is made on an order-preserving uint32 key of z = fp32(x) / T (greedy rows: z = fp32(x)): larger key =
// larger z, -0 and +0 share a key, NaN maps above +inf (so a greedy row with NaN picks its first NaN, as torch.argmax
// does).  Rank order is (key descending, index ascending).
//
//   pass 0        argmax (max key, lowest index) and, when K < V, the level-0 digit histogram of the keys;
//   top-k         radix select over 8-bit digits (levels 1..3 each one pass over the prefix-matching keys) for the K-th
//                 key tau_k; the candidates are key > tau_k plus the first m_k keys == tau_k in index order.  A level whose
//                 bin holds exactly the remaining count stops the descent early (every key >= the bin's lowest is in);
//   top-p         the same descent over weight-summed histograms of the candidates (4 passes) for the key tau_p at which
//                 the rank-order prefix mass reaches target = ceil(p * S_C); the ties at tau_p all have one weight w, so
//                 the number kept, m_p = ceil(remaining / w), needs no pass of its own;
//   select        per-warp totals of the kept weight over contiguous index segments, a serial prefix over the 16 warps,
//                 and one warp walking its segment with a warp scan for the first running sum > u * S.
//
// Weights are e = expf(z - zmax) in fixed point, floor(e * 2^40) as uint64 (sums < 2^64 for V <= 2^24; e < 2^-40
// counts 0): integer histograms and sums are exact in any order, so shared-memory atomics are deterministic and the
// running sum of the walk reaches exactly the S it is compared against; u * S is taken exactly (floor(w24 * S / 2^24)).
// The kept set always has the form {key > tau} + {the first m keys == tau in index order}.  Every pass recomputes z from
// the fp16 row (re-read from L2); nothing depends on V fitting shared memory.  The launch reads the settings and the step
// from device memory, so a captured graph serves every step and every setting written between replays.
#include <math.h>

#include "common.cuh"

namespace quip {

namespace {

constexpr int SP_THREADS = 512;
constexpr int SP_WARPS = SP_THREADS / 32;
constexpr uint32_t SP_ALL = 0xFFFFFFFFu;      // m: every key == tau is kept
constexpr float SP_FIX = 1099511627776.f;     // 2^40
constexpr int SP_MAX_V = 1 << 24;             // V * 2^40 < 2^64: the fixed-point sums cannot overflow

__device__ __forceinline__ uint32_t order_key(float z) {
  if (z != z) return 0xFFFFFFFFu;
  const uint32_t u = __float_as_uint(z == 0.f ? 0.f : z);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

__device__ __forceinline__ float key_value(uint32_t k) {
  return __uint_as_float((k & 0x80000000u) ? (k ^ 0x80000000u) : ~k);
}

__device__ __forceinline__ unsigned long long weight(uint32_t key, float zmax) {
  const float e = expf(key_value(key) - zmax);
  return e > 0.f ? __float2ull_rz(fminf(e, 1.f) * SP_FIX) : 0ull;
}

__device__ __forceinline__ uint32_t digit(uint32_t key, int level) { return (key >> (24 - 8 * level)) & 255u; }

// keys whose digits above `level` equal those of prefix
__device__ __forceinline__ bool matches(uint32_t key, uint32_t prefix, int level) {
  const uint32_t mask = level ? (0xFFFFFFFFu << (32 - 8 * level)) : 0u;
  return (key & mask) == prefix;
}

// Philox4x32-10 (Salmon et al., SC'11), first output word of counter (c0, c1, 0, 0) under key (k0, k1)
__device__ __forceinline__ uint32_t philox_word0(uint32_t c0, uint32_t c1, uint32_t k0, uint32_t k1) {
  uint32_t c2 = 0, c3 = 0;
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
    const uint32_t n0 = hi1 ^ c1 ^ k0, n2 = hi0 ^ c3 ^ k1;
    c0 = n0; c1 = lo1; c2 = n2; c3 = lo0;
    k0 += 0x9E3779B9u;
    k1 += 0xBB67AE85u;
  }
  return c0;
}

// f(i, x_i) for this thread's indices i = tid + j * SP_THREADS, SP_U loads in flight before any is used (the passes are
// bound by L2 latency, not bandwidth)
constexpr int SP_U = 8;
template <typename F>
__device__ __forceinline__ void for_each(const __half* x, int V, F&& f) {
  for (int base = threadIdx.x; base < V; base += SP_U * SP_THREADS) {
    __half v[SP_U];
#pragma unroll
    for (int j = 0; j < SP_U; ++j) v[j] = base + j * SP_THREADS < V ? x[base + j * SP_THREADS] : __half(0.f);
#pragma unroll
    for (int j = 0; j < SP_U; ++j)
      if (base + j * SP_THREADS < V) f(base + j * SP_THREADS, v[j]);
  }
}

// the same over one warp's segment [lo, hi): f(i, x_i) for i = lo + lane + 32 j
template <typename F>
__device__ __forceinline__ void for_each_seg(const __half* x, int lo, int hi, F&& f) {
  const int lane = threadIdx.x & 31;
  for (int base = lo + lane; base < hi; base += SP_U * 32) {
    __half v[SP_U];
#pragma unroll
    for (int j = 0; j < SP_U; ++j) v[j] = base + j * 32 < hi ? x[base + j * 32] : __half(0.f);
#pragma unroll
    for (int j = 0; j < SP_U; ++j)
      if (base + j * 32 < hi) f(base + j * 32, v[j]);
  }
}

struct SampleSmem {
  union {
    uint32_t cnt[SP_WARPS][256];
    unsigned long long wt[SP_WARPS][256];
  } h;
  unsigned long long own[256], incl[256];     // reduced bins and their inclusive prefix, in descending digit order
  unsigned long long part[SP_WARPS];
  unsigned long long wtot[SP_WARPS];
  uint32_t ntie[SP_WARPS];
  unsigned long long argmax, need, total, thr, cum;
  uint32_t sel, ties;
  int warp_sel;
};

template <typename T>
__device__ __forceinline__ T* hist(SampleSmem& s) {
  if constexpr (sizeof(T) == 4) return &s.h.cnt[0][0];
  else return &s.h.wt[0][0];
}

template <typename T>
__device__ __forceinline__ void zero_hist(SampleSmem& s) {
  T* h = hist<T>(s);
  for (int i = threadIdx.x; i < SP_WARPS * 256; i += SP_THREADS) h[i] = 0;
}

// Sum the per-warp histogram copies (plus `extra` in bin extra_bin, -1 for none) into own[] with their inclusive prefix
// in descending digit order (slot j = digit 255 - j), and the total.  Integer sums: the same in any order.  Called by
// every thread; ends synchronised.
template <typename T>
__device__ void reduce_bins(SampleSmem& s, int extra_bin, unsigned long long extra) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const T* h = hist<T>(s);
  __syncthreads();
  unsigned long long v = 0, inc = 0;
  if (tid < 256) {
    const int d = 255 - tid;
#pragma unroll
    for (int w = 0; w < SP_WARPS; ++w) v += h[w * 256 + d];
    if (d == extra_bin) v += extra;
    inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const unsigned long long y = __shfl_up_sync(0xFFFFFFFFu, inc, o);
      if (lane >= o) inc += y;
    }
    if (lane == 31) s.part[warp] = inc;
  }
  __syncthreads();
  if (tid < 256) {
    unsigned long long base = 0;
    for (int w = 0; w < warp; ++w) base += s.part[w];
    s.own[tid] = v;
    s.incl[tid] = base + inc;
    if (tid == 255) s.total = base + inc;
  }
  __syncthreads();
}

// The bin whose exclusive prefix is < need and inclusive prefix >= need (1 <= need <= total): s.sel = its digit, s.need =
// need minus the mass of the higher bins.  Ends synchronised.
__device__ void select_bin(SampleSmem& s, unsigned long long need) {
  const int tid = threadIdx.x;
  if (tid < 256) {
    const unsigned long long inc = s.incl[tid], exc = inc - s.own[tid];
    if (exc < need && need <= inc) {
      s.sel = 255 - tid;
      s.need = need - exc;
    }
  }
  __syncthreads();
}

__global__ void __launch_bounds__(SP_THREADS, 1) sample_kernel(const __half* __restrict__ logits,
                                                            const float* __restrict__ temperature,
                                                            const int32_t* __restrict__ top_k,
                                                            const float* __restrict__ top_p,
                                                            const uint64_t* __restrict__ seed,
                                                            const int64_t* __restrict__ step,
                                                            int64_t* __restrict__ tokens, int V) {
  __shared__ SampleSmem s;
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const __half* x = logits + (size_t)b * V;
  const float T = temperature[b];
  const int32_t k = top_k[b];
  const float p = top_p[b];
  const bool greedy = !(T > 0.f) || k == 1;
  const uint32_t K = (k > 0 && k < V) ? (uint32_t)k : (uint32_t)V;
  auto key_of = [&](__half h) {
    const float v = __half2float(h);
    return order_key(greedy ? v : __fdiv_rn(v, T));
  };
  auto key_at = [&](int i) { return key_of(x[i]); };

  // ---- pass 0: argmax; level-0 count histogram for top-k
  const bool do_topk = !greedy && K < (uint32_t)V;
  if (do_topk) zero_hist<uint32_t>(s);
  __syncthreads();
  unsigned long long best = 0;
  for_each(x, V, [&](int i, __half h) {
    const uint32_t key = key_of(h);
    const unsigned long long packed = ((unsigned long long)key << 32) | (uint32_t)~(uint32_t)i;
    best = packed > best ? packed : best;
    if (do_topk) atomicAdd(&s.h.cnt[warp][digit(key, 0)], 1u);
  });
#pragma unroll
  for (int o = 16; o; o >>= 1) {
    const unsigned long long y = __shfl_xor_sync(0xFFFFFFFFu, best, o);
    best = y > best ? y : best;
  }
  if (lane == 0) s.part[warp] = best;
  __syncthreads();
  if (tid == 0) {
    unsigned long long m = 0;
    for (int w = 0; w < SP_WARPS; ++w) m = s.part[w] > m ? s.part[w] : m;
    s.argmax = m;
  }
  __syncthreads();
  const unsigned long long am = s.argmax;
  const int top_index = (int)~(uint32_t)am;
  if (greedy || K == 1) {
    if (tid == 0) tokens[b] = top_index;
    return;
  }
  const float zmax = key_value((uint32_t)(am >> 32));

  // ---- top-k: tau_k, m_k
  uint32_t tau = 0, m = SP_ALL;                            // K == V: every key >= 0, i.e. all tokens
  if (do_topk) {
    uint32_t prefix = 0;
    unsigned long long need = K;
    for (int level = 0; level < 4; ++level) {
      if (level) {
        __syncthreads();
        zero_hist<uint32_t>(s);
        __syncthreads();
        for_each(x, V, [&](int, __half h) {
          const uint32_t key = key_of(h);
          if (matches(key, prefix, level)) atomicAdd(&s.h.cnt[warp][digit(key, level)], 1u);
        });
      }
      reduce_bins<uint32_t>(s, -1, 0);
      select_bin(s, need);
      const uint32_t d = s.sel;
      const unsigned long long c = s.own[255 - d];
      prefix |= d << (24 - 8 * level);
      need = s.need;
      __syncthreads();
      if (need == c) {
        tau = prefix;
        m = SP_ALL;
        break;
      }
      if (level == 3) {
        tau = prefix;
        m = (uint32_t)need;
      }
    }
  }

  // ---- top-p: tau_p, m_p over the candidates {key > tau_k} + m_k keys == tau_k (those all weigh weight(tau_k))
  if (!(p >= 1.f) && p == p) {
    const unsigned long long wk = weight(tau, zmax);
    const unsigned long long tie_mass = m == SP_ALL ? 0ull : (unsigned long long)m * wk;
    uint32_t prefix = 0;
    unsigned long long need = 0;
    bool ok = true;
    for (int level = 0; level < 4; ++level) {
      __syncthreads();
      zero_hist<unsigned long long>(s);
      __syncthreads();
      for_each(x, V, [&](int, __half h) {
        const uint32_t key = key_of(h);
        if ((key > tau || (key == tau && m == SP_ALL)) && matches(key, prefix, level)) {
          const unsigned long long w = weight(key, zmax);
          if (w) atomicAdd(&s.h.wt[warp][digit(key, level)], w);
        }
      });
      const int extra_bin = (tie_mass && matches(tau, prefix, level)) ? (int)digit(tau, level) : -1;
      reduce_bins<unsigned long long>(s, extra_bin, tie_mass);
      if (level == 0) {
        const unsigned long long S = s.total;
        if (S == 0) {                                      // non-finite row: no top-p
          ok = false;
          break;
        }
        const double tt = ceil((double)p * (double)S);
        need = tt < 1.0 ? 1ull : (tt >= (double)S ? S : (unsigned long long)tt);
      }
      select_bin(s, need);
      prefix |= s.sel << (24 - 8 * level);
      need = s.need;
      __syncthreads();
    }
    if (ok) {
      const unsigned long long wp = weight(prefix, zmax);  // > 0: the selected bin has mass
      const unsigned long long mp = (need + wp - 1) / wp;
      tau = prefix;
      m = (uint32_t)mp;
    }
  }

  // ---- select: kept = {key > tau} + the first m keys == tau in index order
  const int seg = ((V + SP_WARPS * 32 - 1) / (SP_WARPS * 32)) * 32;
  const int lo = warp * seg, hi = min(V, lo + seg);
  const unsigned long long wt = weight(tau, zmax);
  {
    unsigned long long sum = 0;
    uint32_t nt = 0;
    for_each_seg(x, lo, hi, [&](int, __half h) {
      const uint32_t key = key_of(h);
      if (key > tau) sum += weight(key, zmax);
      nt += key == tau;
    });
#pragma unroll
    for (int o = 16; o; o >>= 1) {
      sum += __shfl_xor_sync(0xFFFFFFFFu, sum, o);
      nt += __shfl_xor_sync(0xFFFFFFFFu, nt, o);
    }
    if (lane == 0) {
      s.wtot[warp] = sum;
      s.ntie[warp] = nt;
    }
  }
  __syncthreads();
  if (tid == 0) {
    unsigned long long tot[SP_WARPS], S = 0;
    uint32_t before = 0;
    uint32_t tb[SP_WARPS];
    for (int w = 0; w < SP_WARPS; ++w) {
      const uint32_t left = m > before ? m - before : 0u;
      const uint32_t kept = s.ntie[w] < left ? s.ntie[w] : left;
      tb[w] = before;
      before += s.ntie[w];
      tot[w] = s.wtot[w] + (unsigned long long)kept * wt;
      S += tot[w];
    }
    const int64_t t = *step;
    const uint64_t sd = seed[b];
    const uint32_t w24 = philox_word0((uint32_t)t, (uint32_t)((uint64_t)t >> 32), (uint32_t)sd, (uint32_t)(sd >> 32)) >> 8;
    // thr = floor(u * S), u = w24 / 2^24, exactly (S < 2^57)
    const unsigned long long lo64 = S * (unsigned long long)w24, hi64 = __umul64hi(S, (unsigned long long)w24);
    const unsigned long long thr = (hi64 << 40) | (lo64 >> 24);
    s.warp_sel = -1;
    unsigned long long cum = 0;
    for (int w = 0; w < SP_WARPS; ++w) {
      if (cum + tot[w] > thr) {
        s.warp_sel = w;
        s.cum = cum;
        s.ties = tb[w];
        break;
      }
      cum += tot[w];
    }
    s.thr = thr;
    if (s.warp_sel < 0) tokens[b] = top_index;             // S == 0: a row with non-finite logits
  }
  __syncthreads();
  if (warp != s.warp_sel) return;
  const unsigned long long thr = s.thr;
  unsigned long long cum = s.cum;
  uint32_t ties = s.ties;
  for (int base = lo; base < hi; base += 32) {
    const int i = base + lane;
    const bool valid = i < hi;
    const uint32_t key = valid ? key_at(i) : 0u;
    const bool tie = valid && key == tau;
    const uint32_t tmask = __ballot_sync(0xFFFFFFFFu, tie);
    const uint32_t ord = ties + __popc(tmask & ((1u << lane) - 1u));
    unsigned long long w = 0;
    if (valid && key > tau) w = weight(key, zmax);
    else if (tie && ord < m) w = wt;
    unsigned long long incl = w;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const unsigned long long y = __shfl_up_sync(0xFFFFFFFFu, incl, o);
      if (lane >= o) incl += y;
    }
    const uint32_t hit = __ballot_sync(0xFFFFFFFFu, cum + incl > thr);
    if (hit) {
      if (lane == 0) tokens[b] = base + __ffs(hit) - 1;
      return;
    }
    cum += __shfl_sync(0xFFFFFFFFu, incl, 31);
    ties += __popc(tmask);
  }
  if (lane == 0) tokens[b] = top_index;                    // not reached: the selected warp's mass exceeds thr
}

}  // namespace

}  // namespace quip

using namespace quip;

extern "C" int quip_sample(const void* logits, const float* temperature, const int32_t* top_k, const float* top_p,
                           const uint64_t* seed, const int64_t* step, int64_t* tokens, int32_t B, int32_t V,
                           void* stream) {
  QUIP_CHECK_ARG(B >= 0 && V >= 1 && V <= SP_MAX_V, "quip_sample: bad sizes (B %d, V %d): need B >= 0 and 1 <= V <= %d",
                 B, V, SP_MAX_V);
  QUIP_CHECK_ARG(logits && temperature && top_k && top_p && seed && step && tokens, "quip_sample: null pointer");
  if (B == 0) return QUIP_OK;
  sample_kernel<<<(unsigned)B, SP_THREADS, 0, (cudaStream_t)stream>>>((const __half*)logits, temperature, top_k, top_p,
                                                                      seed, step, tokens, V);
  QUIP_LAUNCHED("sample_kernel");
  return QUIP_OK;
}
