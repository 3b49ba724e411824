// Beam search inside the decode graph: per-row top-C candidates, the per-prompt merge with the finished-hypothesis
// bookkeeping, and the fork of a paged KV cache after each step.  The rules are stated in include/quip_b200.h;
// quip_b200/decode.py (_beam_*_torch) and oracle/beam.py restate them in torch.
//
// quip_beam_candidates, one CTA per row of fp16 logits:
//   lse      one pass, per-thread online (max, sum of exp) over 16-byte loads with a scalar head and tail (any V, any
//            row stride), combined by a fixed xor-shuffle tree and then warp by warp in order: bit-identical launches;
//   select   s = ((x - m) - log S) + score, ranked by an order-preserving uint32 key (NaN below -inf) and then by lower
//            index.  An 8-bit radix descent over the keys finds the C-th key tau (levels 1..3 each one pass over the
//            prefix-matching keys; a bin that holds exactly the remaining count stops the descent).  When only m of the
//            keys == tau are kept, the same descent over the complemented indices of those ties finds the m-th lowest
//            index, so the kept set is {key > tau} + {key == tau, index <= i_m};
//   collect  one pass drops the <= C survivors into shared memory in any order; their rank (key desc, index asc) is
//            computed by comparison, so the output order is exact.
// Every pass recomputes s from the fp16 row (re-read from L2); nothing depends on V fitting shared memory.
#include <math.h>

#include "common.cuh"
#include "kv_page.cuh"

namespace quip {

namespace {

constexpr int BC_THREADS = 512;
constexpr int BC_WARPS = BC_THREADS / 32;
constexpr int BEAM_MAX_C = 64;
constexpr int BEAM_MAX_K = 16;
constexpr int BEAM_MAX_EOS = 3;
constexpr int BEAM_MAX_V = 1 << 24;
constexpr float BEAM_NEG = -1.0e9f;

// larger key = larger z; -0 and +0 share a key; NaN maps to 0, below -inf (0x007FFFFF)
__device__ __forceinline__ uint32_t beam_key(float z) {
  if (z != z) return 0u;
  const uint32_t u = __float_as_uint(z == 0.f ? 0.f : z);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

struct Lse {
  float m, s;
  bool nan;
};

__device__ __forceinline__ void lse_one(Lse& a, float v) {
  if (v != v) {
    a.nan = true;
    return;
  }
  if (v > a.m) {
    a.s = a.s * expf(a.m - v);
    a.m = v;
  }
  if (a.m == -INFINITY) return;                           // only -inf so far: adds nothing
  a.s += expf(v - a.m);
}

__device__ __forceinline__ void lse_eight(Lse& a, const float* v) {
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
  if (gm > a.m) {
    a.s = a.s * expf(a.m - gm);
    a.m = gm;
  }
  if (a.m == -INFINITY) return;                           // a group of -inf before any finite value adds nothing
  float t = 0.f;
#pragma unroll
  for (int j = 0; j < 8; ++j) t += expf(v[j] - a.m);
  a.s += t;
}

__device__ __forceinline__ void lse_merge(Lse& a, const Lse& b) {
  a.nan |= b.nan;
  const float m = fmaxf(a.m, b.m);
  const float sa = a.s > 0.f ? a.s * expf(a.m - m) : 0.f;
  const float sb = b.s > 0.f ? b.s * expf(b.m - m) : 0.f;
  a.m = m;
  a.s = sa + sb;
}

// f(i, x_i) over row x (V values) for this thread: a scalar head up to the first 16-byte boundary, 8 values per
// 16-byte load, a scalar tail.  f8(i0, v[8]) takes the body's groups (default: f on each).
template <typename F1, typename F8>
__device__ __forceinline__ void sweep(const __half* x, int V, F1&& f, F8&& f8) {
  const int tid = threadIdx.x;
  const int mis = (int)(((uintptr_t)x >> 1) & 7);
  const int head = min(V, (8 - mis) & 7);
  const int nvec = (V - head) >> 3;
  const int body_end = head + 8 * nvec;
  if (tid < head) f(tid, __half2float(x[tid]));
  const uint4* xv = reinterpret_cast<const uint4*>(x + head);
  for (int k = tid; k < nvec; k += BC_THREADS) {
    const uint4 raw = __ldg(xv + k);
    const __half2* h = reinterpret_cast<const __half2*>(&raw);
    float v[8];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 p = __half22float2(h[j]);
      v[2 * j] = p.x;
      v[2 * j + 1] = p.y;
    }
    f8(head + 8 * k, v);
  }
  if (body_end + tid < V) f(body_end + tid, __half2float(x[body_end + tid]));
}

template <typename F1>
__device__ __forceinline__ void sweep(const __half* x, int V, F1&& f) {
  sweep(x, V, f, [&](int i0, const float* v) {
#pragma unroll
    for (int j = 0; j < 8; ++j) f(i0 + j, v[j]);
  });
}

struct CandSmem {
  uint32_t cnt[BC_WARPS][256];
  uint32_t part[BC_WARPS];
  Lse lse[BC_WARPS];
  float m, logS;
  uint32_t sel, need, bin;
  uint32_t n;
  float vs[BEAM_MAX_C];
  int vi[BEAM_MAX_C];
};

// The bin of the level-`level` digit histogram in which the `need`-th largest key lies: s.sel = its digit, s.need =
// need minus the count of the higher bins, s.bin = the bin's count.  Called by every thread; ends synchronised.
__device__ void pick_bin(CandSmem& s, uint32_t need) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  __syncthreads();
  uint32_t v = 0, inc = 0;
  if (tid < 256) {
    const int d = 255 - tid;                              // descending digit order
#pragma unroll
    for (int w = 0; w < BC_WARPS; ++w) v += s.cnt[w][d];
    inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t y = __shfl_up_sync(0xFFFFFFFFu, inc, o);
      if (lane >= o) inc += y;
    }
    if (lane == 31) s.part[warp] = inc;
  }
  __syncthreads();
  if (tid < 256) {
    uint32_t base = 0;
    for (int w = 0; w < warp; ++w) base += s.part[w];
    inc += base;
    const uint32_t exc = inc - v;
    if (exc < need && need <= inc) {
      s.sel = 255 - tid;
      s.need = need - exc;
      s.bin = v;
    }
  }
  __syncthreads();
}

// The `need`-th largest of key(i, v) over the elements with in(i, v) (1 <= need <= their count): returns tau and
// sets `all` when every element with key >= tau is among the need largest (otherwise exactly `m` of the keys == tau
// are, m < their count).
template <typename FK>
__device__ uint32_t radix_nth(CandSmem& s, const __half* x, int V, uint32_t need, FK&& key_in, bool& all,
                              uint32_t& m) {
  const int warp = threadIdx.x >> 5;
  uint32_t prefix = 0;
  for (int level = 0; level < 4; ++level) {
    for (int i = threadIdx.x; i < BC_WARPS * 256; i += BC_THREADS) (&s.cnt[0][0])[i] = 0;
    __syncthreads();
    const uint32_t mask = level ? (0xFFFFFFFFu << (32 - 8 * level)) : 0u;
    const int sh = 24 - 8 * level;
    sweep(x, V, [&](int i, float v) {
      uint32_t k;
      if (key_in(i, v, k) && (k & mask) == prefix) atomicAdd(&s.cnt[warp][(k >> sh) & 255u], 1u);
    });
    pick_bin(s, need);
    prefix |= s.sel << sh;
    const uint32_t c = s.bin;
    need = s.need;
    __syncthreads();
    if (need == c) {                                      // the whole bin is in: every key >= prefix
      all = true;
      m = 0;
      return prefix;
    }
  }
  all = false;
  m = need;
  return prefix;
}

__global__ void __launch_bounds__(BC_THREADS, 1) beam_candidates_kernel(const __half* __restrict__ logits, int64_t ld,
                                                                        const float* __restrict__ scores,
                                                                        float* __restrict__ out_s,
                                                                        int32_t* __restrict__ out_i, int V, int K,
                                                                        int C) {
  __shared__ CandSmem s;
  const int r = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const __half* x = logits + (size_t)r * (size_t)ld;

  // ---- lse
  Lse a{-INFINITY, 0.f, false};
  sweep(x, V, [&](int, float v) { lse_one(a, v); }, [&](int, const float* v) { lse_eight(a, v); });
#pragma unroll
  for (int o = 16; o; o >>= 1) {
    Lse b;
    b.m = __shfl_xor_sync(0xFFFFFFFFu, a.m, o);
    b.s = __shfl_xor_sync(0xFFFFFFFFu, a.s, o);
    b.nan = __shfl_xor_sync(0xFFFFFFFFu, (int)a.nan, o) != 0;
    lse_merge(a, b);
  }
  if (lane == 0) s.lse[warp] = a;
  if (tid == 0) s.n = 0;
  __syncthreads();
  if (tid == 0) {
    Lse t = s.lse[0];
    for (int w = 1; w < BC_WARPS; ++w) lse_merge(t, s.lse[w]);
    s.m = t.nan ? __int_as_float(0x7FC00000) : t.m;
    s.logS = logf(t.s);
  }
  __syncthreads();
  const float m = s.m, logS = s.logS, score = scores[r];
  const bool ninf = m == -INFINITY;                       // a row of -inf: every s is -inf
  auto s_of = [&](float v) { return ninf ? -INFINITY : __fadd_rn(__fsub_rn(__fsub_rn(v, m), logS), score); };

  // ---- the C-th key, and the index bound of its kept ties
  const int want = min(C, V);
  uint32_t tau = 0, ilim = 0xFFFFFFFFu;
  bool all = true;
  if (V > C) {
    uint32_t mt;
    tau = radix_nth(s, x, V, (uint32_t)C, [&](int, float v, uint32_t& k) { k = beam_key(s_of(v)); return true; },
                    all, mt);
    if (!all) {
      bool all2;
      uint32_t m2;
      const uint32_t t2 = radix_nth(s, x, V, mt, [&](int i, float v, uint32_t& k) {
        k = ~(uint32_t)i;
        return beam_key(s_of(v)) == tau;
      }, all2, m2);
      ilim = ~t2;                                         // indices are unique: the descent ends with all2
    }
  }

  // ---- collect, then rank
  sweep(x, V, [&](int i, float v) {
    const float z = s_of(v);
    const uint32_t k = beam_key(z);
    if (V <= C || (all ? k >= tau : (k > tau || (k == tau && (uint32_t)i <= ilim)))) {
      const uint32_t j = atomicAdd(&s.n, 1u);
      if (j < BEAM_MAX_C) {
        s.vs[j] = z;
        s.vi[j] = i;
      }
    }
  });
  __syncthreads();
  const int n = min((int)s.n, want);
  const int beam = r % K;
  if (tid < C) {
    float* os = out_s + (size_t)r * C;
    int32_t* oi = out_i + (size_t)r * C;
    if (tid < n) {
      const uint32_t k = beam_key(s.vs[tid]);
      const int i = s.vi[tid];
      int rank = 0;
      for (int u = 0; u < n; ++u) {
        const uint32_t ku = beam_key(s.vs[u]);
        rank += ku > k || (ku == k && s.vi[u] < i);
      }
      os[rank] = s.vs[tid];
      oi[rank] = beam * V + i;
    } else {                                              // V < C: padding, ranked after every candidate
      os[tid] = __int_as_float(0x7FC00000);
      oi[tid] = -1;
    }
  }
}

// ---- quip_beam_select: one CTA per prompt

constexpr int BS_THREADS = 256;

struct SelSmem {
  float es[BEAM_MAX_K * BEAM_MAX_C];
  int ei[BEAM_MAX_K * BEAM_MAX_C];
  float cs[BEAM_MAX_C], r[BEAM_MAX_C], fv[BEAM_MAX_K + BEAM_MAX_C];
  int ci[BEAM_MAX_C];
  uint8_t hit[BEAM_MAX_C];
  int run_src[BEAM_MAX_K], fin_src[BEAM_MAX_K];
  float old_fs[BEAM_MAX_K];
  int64_t old_len[BEAM_MAX_K];
  uint8_t old_filled[BEAM_MAX_K], new_filled[BEAM_MAX_K];
  int all_hit;
};

// strict total order of the K x C entries: key desc, then index asc (padding -1 last), then (row, position)
__device__ __forceinline__ bool ent_before(float s1, int i1, int e1, float s2, int i2, int e2) {
  const uint32_t k1 = beam_key(s1), k2 = beam_key(s2);
  if (k1 != k2) return k1 > k2;
  const uint32_t j1 = i1 < 0 ? 0xFFFFFFFFu : (uint32_t)i1, j2 = i2 < 0 ? 0xFFFFFFFFu : (uint32_t)i2;
  if (j1 != j2) return j1 < j2;
  return e1 < e2;
}

__global__ void __launch_bounds__(BS_THREADS) beam_select_kernel(
    const float* __restrict__ cand_s, const int32_t* __restrict__ cand_i, const int64_t* __restrict__ eos, int n_eos,
    const int64_t* __restrict__ budget, const int64_t* __restrict__ step, const float* __restrict__ pen,
    float* __restrict__ score, int64_t* __restrict__ hist, int64_t* __restrict__ hist_tmp,
    float* __restrict__ fin_score, int64_t* __restrict__ fin_len, int64_t* __restrict__ fin_tok,
    int64_t* __restrict__ fin_tmp, uint8_t* __restrict__ fin_filled, uint8_t* __restrict__ heur,
    uint8_t* __restrict__ done, int64_t* __restrict__ tokens, int64_t* __restrict__ parents, int64_t* __restrict__ adv,
    int K, int C, int V, int max_new, int es_mode, int never_long) {
  __shared__ SelSmem s;
  const int b = blockIdx.x, tid = threadIdx.x;
  const int64_t row0 = (int64_t)b * K;
  if (done[b]) {                                          // frozen: identity parents, nothing advances
    if (tid < K) {
      parents[row0 + tid] = row0 + tid;
      adv[row0 + tid] = 0;
    }
    return;
  }
  const int64_t t = *step;
  const int64_t n_new = t + 1;
  const int64_t bud = budget[b];
  if (t < 0 || t >= max_new) {                            // outside the buffers: identity, no state change
    if (tid < K) {
      parents[row0 + tid] = row0 + tid;
      adv[row0 + tid] = 0;
    }
    return;
  }
  const int KC = K * C;
  for (int e = tid; e < KC; e += BS_THREADS) {
    s.es[e] = cand_s[row0 * C + e];
    s.ei[e] = cand_i[row0 * C + e];
  }
  if (tid == 0) s.all_hit = 1;
  __syncthreads();
  // merge: rank of each entry = its position in its own sorted list + the entries of every other list before it
  for (int e = tid; e < KC; e += BS_THREADS) {
    const int a = e / C, p = e % C;
    const float se = s.es[e];
    const int ie = s.ei[e];
    int rank = p;
    for (int o = 0; o < K && rank < C; ++o) {
      if (o == a) continue;
      int lo = 0, hi = C;                                 // entries of list o before e: a prefix of the list
      while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (ent_before(s.es[o * C + mid], s.ei[o * C + mid], o * C + mid, se, ie, e)) lo = mid + 1;
        else hi = mid;
      }
      rank += lo;
    }
    if (rank < C) {
      s.cs[rank] = se;
      s.ci[rank] = ie;
    }
  }
  __syncthreads();
  // hits and the running values
  if (tid < C) {
    const int ix = s.ci[tid];
    const int64_t tok = ix >= 0 ? ix % V : 0;
    bool h = n_new >= bud;
    for (int q = 0; q < n_eos; ++q) h |= tok == eos[q];
    s.hit[tid] = h;
    s.r[tid] = __fadd_rn(s.cs[tid], h ? BEAM_NEG : 0.f);
    if (!h) atomicAnd(&s.all_hit, 0);
  }
  if (tid < K) {
    s.old_fs[tid] = fin_score[row0 + tid];
    s.old_len[tid] = fin_len[row0 + tid];
    s.old_filled[tid] = fin_filled[row0 + tid];
  }
  __syncthreads();
  if (tid < C) {                                          // running beams: top K of r, ties by lower rank
    const uint32_t k = beam_key(s.r[tid]);
    int rank = 0;
    for (int u = 0; u < C; ++u) {
      const uint32_t ku = beam_key(s.r[u]);
      rank += ku > k || (ku == k && u < tid);
    }
    if (rank < K) s.run_src[rank] = tid;
  }
  // offered values: s / n_new^lambda, then HF's -1e9 penalties in HF's order
  bool full = true;
  for (int j = 0; j < K; ++j) full &= s.old_filled[j] != 0;
  full &= es_mode == 1;
  const bool h_ok = heur[b] != 0;
  if (tid < C) {
    const bool did = s.hit[tid] && tid < K;
    float v = __fdiv_rn(s.cs[tid], pen[n_new]);
    v = __fadd_rn(v, full ? BEAM_NEG : 0.f);
    v = __fadd_rn(v, h_ok ? 0.f : BEAM_NEG);
    v = __fadd_rn(v, did ? 0.f : BEAM_NEG);
    s.fv[K + tid] = v;
  }
  if (tid < K) s.fv[tid] = s.old_fs[tid];
  __syncthreads();
  if (tid < K + C) {                                      // finished slots: top K of old + offered, old first on ties
    const uint32_t k = beam_key(s.fv[tid]);
    int rank = 0;
    for (int u = 0; u < K + C; ++u) {
      const uint32_t ku = beam_key(s.fv[u]);
      rank += ku > k || (ku == k && u < tid);
    }
    if (rank < K) s.fin_src[rank] = tid;
  }
  // snapshots of the histories and finished tokens the gathers read
  int64_t* ht = hist_tmp + row0 * max_new;
  int64_t* ft = fin_tmp + row0 * max_new;
  const int64_t* hb = hist + row0 * max_new;
  const int64_t* fb = fin_tok + row0 * max_new;
  for (int e = tid; e < K * max_new; e += BS_THREADS) {
    ht[e] = hb[e];
    ft[e] = fb[e];
  }
  __syncthreads();
  // write the running beams
  for (int e = tid; e < K * (int)n_new; e += BS_THREADS) {
    const int k = e / (int)n_new, c = e % (int)n_new;
    const int src = s.run_src[k];
    const int ix = s.ci[src];
    const int pj = ix >= 0 ? ix / V : 0;
    hist[(row0 + k) * max_new + c] = c < t ? ht[(int64_t)pj * max_new + c] : (ix >= 0 ? ix % V : 0);
  }
  if (tid < K) {
    const int src = s.run_src[tid];
    const int ix = s.ci[src];
    const int pj = ix >= 0 ? ix / V : 0;
    tokens[row0 + tid] = ix >= 0 ? ix % V : 0;
    parents[row0 + tid] = row0 + pj;
    score[row0 + tid] = s.r[src];
    adv[row0 + tid] = 1;
  }
  // write the finished slots
  for (int e = tid; e < K * max_new; e += BS_THREADS) {
    const int k = e / max_new, c = e % max_new;
    const int src = s.fin_src[k];
    int64_t v;
    if (src < K) {
      v = ft[(int64_t)src * max_new + c];
    } else {
      const int ix = s.ci[src - K];
      const int pj = ix >= 0 ? ix / V : 0;
      v = c < t ? ht[(int64_t)pj * max_new + c] : (c == t ? (ix >= 0 ? ix % V : 0) : 0);
    }
    fin_tok[(row0 + k) * max_new + c] = v;
  }
  if (tid == 0) {
    float mn = INFINITY;
    bool all_filled = true;
    for (int k = 0; k < K; ++k) {
      const int src = s.fin_src[k];
      const float v = s.fv[src];
      const bool f = src < K ? s.old_filled[src] != 0 : (s.hit[src - K] && src - K < K);
      fin_score[row0 + k] = v;
      fin_len[row0 + k] = src < K ? s.old_len[src] : n_new;
      fin_filled[row0 + k] = f;
      mn = fminf(mn, v);
      all_filled &= f;
      s.new_filled[k] = f;
    }
    // HF's min propagates NaN
    for (int k = 0; k < K; ++k) {
      const float v = s.fv[s.fin_src[k]];
      if (v != v) mn = v;
    }
    const float best = __fdiv_rn(s.r[s.run_src[0]], pen[never_long ? min(bud, (int64_t)max_new) : n_new]);
    bool any = false;
    for (int k = 0; k < K; ++k) any |= best > (s.new_filled[k] ? mn : BEAM_NEG);
    const bool h = h_ok && any;
    heur[b] = h;
    done[b] = !h || (es_mode == 1 && all_filled) || s.all_hit;
  }
}

// ---- quip_kv_beam_fork: phase 0 gathers, phase 1 scatters.  Grid (rows, layers, 2 * nkv: k or v, head), so each CTA
// copies one head's slots of one layer (up to 64 * hd elements) and the copy spreads over many SMs.

template <typename T, bool SCALES>
__global__ void __launch_bounds__(128) beam_fork_kernel(int phase, T* __restrict__ k_pool, T* __restrict__ v_pool,
                                                        float* __restrict__ k_scale, float* __restrict__ v_scale,
                                                        int32_t* __restrict__ table, int32_t* __restrict__ table_tmp,
                                                        const int64_t* __restrict__ parents,
                                                        const int64_t* __restrict__ lens, int R, int n_pages, int nkv,
                                                        int hd, int max_pages, int scratch0) {
  const int j = blockIdx.x, l = blockIdx.y, w = blockIdx.z / nkv, h = blockIdx.z % nkv, tid = threadIdx.x;
  const bool first = l == 0 && blockIdx.z == 0;
  if (phase == 0 && first)
    for (int p = tid; p < max_pages; p += blockDim.x) table_tmp[(int64_t)j * max_pages + p] = table[(int64_t)j * max_pages + p];
  const int64_t par = parents[j], len = lens[j];
  if (par < 0 || par >= R || par == j || len < 1 || len > (int64_t)max_pages * KV_PAGE) return;
  const int pos = (int)(len - 1), cur = pos >> 6, nslot = (pos & 63) + 1;
  if (phase == 1 && first)
    for (int p = tid; p < cur; p += blockDim.x) table[(int64_t)j * max_pages + p] = table_tmp[par * max_pages + p];
  const int src = phase == 0 ? table[par * max_pages + cur] : scratch0 + j;
  const int dst = phase == 0 ? scratch0 + j : table[(int64_t)j * max_pages + cur];
  if (src < 0 || src >= n_pages || dst < 0 || dst >= n_pages || src == dst) return;
  T* pool = w ? v_pool : k_pool;
  const int64_t layer = (int64_t)l * n_pages;
  const int vecs = nslot * hd * (int)sizeof(T) / 16;      // 16-byte units (hd * sizeof(T) % 16 == 0)
  const uint4* sp = reinterpret_cast<const uint4*>(pool + ((layer + src) * nkv + h) * KV_PAGE * hd);
  uint4* dp = reinterpret_cast<uint4*>(pool + ((layer + dst) * nkv + h) * KV_PAGE * hd);
  for (int u = tid; u < vecs; u += blockDim.x) dp[u] = sp[u];
  if constexpr (SCALES) {
    float* sc = w ? v_scale : k_scale;
    const float* ss = sc + ((layer + src) * nkv + h) * KV_PAGE;
    float* ds = sc + ((layer + dst) * nkv + h) * KV_PAGE;
    for (int u = tid; u < nslot; u += blockDim.x) ds[u] = ss[u];
  }
}

// Checks and the two launches of quip_kv_beam_fork on pools of T (SCALES: e4m3 with scales); kv describes layer 0.
template <typename T, bool SCALES>
int launch_fork(const QuipKvCache& kv, KvPages pg, int32_t L, int32_t* table_tmp, const int64_t* parents,
                const int64_t* lens, int32_t R, int32_t scratch0, void* stream) {
  const int32_t nkv = kv.nkv, hd = kv.hd, max_pages = pg.max_pages, n_pages = pg.n_pages;
  QUIP_CHECK_ARG(R >= 0 && L >= 1 && L <= 65535 && nkv >= 1 && nkv <= 32767 && scratch0 >= 0 &&
                     (int64_t)scratch0 + R <= n_pages,
                 "quip_kv_beam_fork: bad sizes (R %d, L %d, n_pages %d, nkv %d, hd %d, max_pages %d, scratch0 %d)", R,
                 L, n_pages, nkv, hd, max_pages, scratch0);
  QUIP_CHECK_ARG(table_tmp && parents && lens, "quip_kv_beam_fork: null pointer");
  if (R == 0) return QUIP_OK;
  const dim3 grid((unsigned)R, (unsigned)L, 2u * (unsigned)nkv);
  for (int phase = 0; phase < 2; ++phase) {
    beam_fork_kernel<T, SCALES><<<grid, 128, 0, (cudaStream_t)stream>>>(phase, (T*)kv.k, (T*)kv.v, kv.k_scale,
                                                                         kv.v_scale, kv.page_table, table_tmp, parents,
                                                                         lens, R, n_pages, nkv, hd, max_pages,
                                                                         scratch0);
    QUIP_LAUNCHED("beam_fork_kernel");
  }
  return QUIP_OK;
}

}  // namespace

}  // namespace quip

using namespace quip;

extern "C" int quip_beam_candidates(const void* logits, int64_t ld, const float* scores, float* cand_s,
                                    int32_t* cand_i, int32_t R, int32_t V, int32_t K, int32_t C, void* stream) {
  QUIP_CHECK_ARG(R >= 0 && V >= 1 && V <= BEAM_MAX_V && ld >= V && K >= 1 && K <= BEAM_MAX_K && C >= 1 &&
                     C <= BEAM_MAX_C && (int64_t)K * V <= INT32_MAX,
                 "quip_beam_candidates: bad sizes (R %d, V %d, ld %lld, K %d, C %d)", R, V, (long long)ld, K, C);
  QUIP_CHECK_ARG(logits && scores && cand_s && cand_i, "quip_beam_candidates: null pointer");
  QUIP_CHECK_ARG(((uintptr_t)logits & 1) == 0, "quip_beam_candidates: logits must be 2-byte aligned");
  if (R == 0) return QUIP_OK;
  beam_candidates_kernel<<<(unsigned)R, BC_THREADS, 0, (cudaStream_t)stream>>>((const __half*)logits, ld, scores,
                                                                               cand_s, cand_i, V, K, C);
  QUIP_LAUNCHED("beam_candidates_kernel");
  return QUIP_OK;
}

extern "C" int quip_beam_select(const float* cand_s, const int32_t* cand_i, const int64_t* eos, int32_t n_eos,
                                const int64_t* budget, const int64_t* step, const float* pen, float* score,
                                int64_t* hist, int64_t* hist_tmp, float* fin_score, int64_t* fin_len, int64_t* fin_tok,
                                int64_t* fin_tmp, uint8_t* fin_filled, uint8_t* heur, uint8_t* done, int64_t* tokens,
                                int64_t* parents, int64_t* adv, int32_t B, int32_t K, int32_t C, int32_t V,
                                int32_t max_new, int32_t early_stopping, int32_t never_long, void* stream) {
  QUIP_CHECK_ARG(B >= 0 && K >= 1 && K <= BEAM_MAX_K && C >= K && C <= BEAM_MAX_C && V >= 1 &&
                     (int64_t)K * V <= INT32_MAX && max_new >= 1 && n_eos >= 0 && n_eos <= BEAM_MAX_EOS &&
                     early_stopping >= 0 && early_stopping <= 2,
                 "quip_beam_select: bad sizes (B %d, K %d, C %d, V %d, max_new %d, n_eos %d, early_stopping %d)", B,
                 K, C, V, max_new, n_eos, early_stopping);
  QUIP_CHECK_ARG(cand_s && cand_i && (eos || !n_eos) && budget && step && pen && score && hist && hist_tmp &&
                     fin_score && fin_len && fin_tok && fin_tmp && fin_filled && heur && done && tokens && parents && adv,
                 "quip_beam_select: null pointer");
  if (B == 0) return QUIP_OK;
  beam_select_kernel<<<(unsigned)B, BS_THREADS, 0, (cudaStream_t)stream>>>(
      cand_s, cand_i, eos, n_eos, budget, step, pen, score, hist, hist_tmp, fin_score, fin_len, fin_tok, fin_tmp,
      fin_filled, heur, done, tokens, parents, adv, K, C, V, max_new, early_stopping, never_long);
  QUIP_LAUNCHED("beam_select_kernel");
  return QUIP_OK;
}

extern "C" int quip_kv_beam_fork(const QuipKvCache* kv, int32_t L, int32_t* table_tmp, const int64_t* parents,
                                 const int64_t* lens, int32_t R, int32_t scratch0, void* stream) {
  const char* fn = "quip_kv_beam_fork";
  KvPages pg;
  int32_t max_len;
  if (const int e = kv_check(fn, kv, pg, max_len)) return e;
  QUIP_CHECK_ARG(kv->page_table, "%s: page_table is null: the fork is paged only", fn);
  return kv->format == QUIP_KV_E4M3
      ? launch_fork<uint8_t, true>(*kv, pg, L, table_tmp, parents, lens, R, scratch0, stream)
      : launch_fork<__half, false>(*kv, pg, L, table_tmp, parents, lens, R, scratch0, stream);
}
