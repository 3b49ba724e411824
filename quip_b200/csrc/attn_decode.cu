// Decode attention: one new token per sequence, each sequence at its own position, over the static KV cache of
// quip_b200/decode.py (one layer: k_cache / v_cache (B, nkv, max_len, hd), fp16 or e4m3 with per-slot fp32 scales).
//
//   o[b][h] = softmax_j(scale * q[b][h] . K[b][h/G][j]) V[b][h/G][j],   j = 0 .. positions[b],   G = nh / nkv
//
// with this step's k_new / v_new appended at slot positions[b] in the same launch.
//
// Split-KV.  The max_len slots of a row are cut into chunks of 128 slots, or 64 when that grid would hold fewer than
// two CTAs per SM (short caches, few rows: a shorter chain of dependent loads per CTA).  CTA (split, kv head, row) owns
// one chunk and all G query heads that share the kv head, so every cached byte of the valid prefix is read from HBM once per step (no
// repeat_interleave copies).  Chunks that start past positions[b] exit at once and slots past positions[b] inside the
// last chunk are never loaded: the cost is sum_b 2 * nkv * (positions[b] + 1) * hd * 2 bytes, whatever max_len is, and
// whatever an unused slot holds (NaN included) cannot reach the output.  The grid depends on (B, nkv, max_len) only, so a
// CUDA graph captured once serves every later step.
//
// The CTA whose chunk holds positions[b] writes k_new / v_new to that slot and computes with k_new / v_new directly; no
// other CTA of the launch touches the slot.
//
// Arithmetic is fp32 on the CUDA cores: at one query token per head (G <= 8 rows per kv head) a tensor-core tile would
// be at most 8 of its 64 rows full, and the kernel is bound by streaming K and V anyway (2 fp32 FMA per loaded fp16
// element and head).  Each CTA leaves its unnormalised partial (m, l, o) in fp32 workspace; a combine kernel merges the
// chunks of a row in ascending order and rounds once to fp16.  Fixed orders everywhere: bit-identical from run to run,
// and row b's result does not depend on the other rows.
//
// A position outside [0, max_len) is not looked at by the main kernel (no slot is written) and gives a NaN output row.
//
// e4m3 cache (quip_decode_attention_fp8, the same kernel instantiated for FP8).  Each cached head vector x (the hd
// values of one layer, row, kv head and slot; fp32 from fp16) is stored as hd e4m3fn bytes q plus one fp32 scale s:
//
//   amax = max_i |x_i|;   s = amax / 448 (IEEE fp32 division), s = 1 when amax == 0;   q_i = e4m3fn_rn(x_i / s)
//
// round to nearest even, subnormals kept, IEEE division (the build has no fast-math).  |x_i / s| < 464, so the saturating
// cvt.rn.satfinite.e4m3x2.f32 and a non-saturating conversion (torch's .to(torch.float8_e4m3fn)) give the same bytes.  The
// value of a slot is float(q_i) * s.  The appending CTA quantizes k_new / v_new (one warp each) and attends over the
// quantized values of its own slot too, so a step's result equals what every later step reads back.  Scores are
// s_k[j] * scale * sum_i q_i k8_i, P.V weights are p_j * s_v[j]: one multiply per slot, not per element.  The lanes of a
// slot are the fp16 kernel's (8 elements each), with 8-byte loads and AD_U8 = 8 loads in flight per lane, so a lane has
// the same 64 bytes in flight and the same q registers.  A cached slot costs hd + 4 bytes instead of 2 * hd.
#include <cuda_fp8.h>
#include <math.h>

#include <type_traits>

#include "common.cuh"
#include "kv_fp8.cuh"
#include "kv_page.cuh"

namespace quip {

namespace {

constexpr int AD_CHUNK = 128;        // KV slots per CTA (at most)
constexpr int AD_SMALL_CHUNK = 64;   // when B * nkv * ceil(max_len / AD_CHUNK) < AD_SMALL_GRID
constexpr int AD_SMALL_GRID = 2 * 132;
constexpr int AD_U = 4;              // slots per slot group whose loads are in flight together
constexpr int AD_U8 = 8;             // the same for the e4m3 cache (8-byte loads)
constexpr int AD_THREADS = 128;
constexpr int AD_MAXG = 8;           // query heads per kv head

__device__ __forceinline__ void h8_to_f(const uint4& u, float (&f)[8]) {
  AH8 t;
  t.v = u;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 p = __half22float2(t.h2[i]);
    f[2 * i] = p.x;
    f[2 * i + 1] = p.y;
  }
}

// 8 e4m3 bytes (element i in byte i) -> fp32, through cvt.rn.f16x2.e4m3x2 (exact: every e4m3 value is an fp16 value)
__device__ __forceinline__ void e4m3x8_to_f(const uint2& u, float (&f)[8]) {
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const uint32_t w = i < 2 ? u.x : u.y;
    const __half2_raw r = __nv_cvt_fp8x2_to_halfraw2((__nv_fp8x2_storage_t)((w >> (16 * (i & 1))) & 0xFFFFu), __NV_E4M3);
    const float2 p = __half22float2(__half2(r));
    f[2 * i] = p.x;
    f[2 * i + 1] = p.y;
  }
}

// Shared memory of the e4m3 instantiation: the chunk's slot scales and the appended slot (bytes and scale, k then v).
template <bool FP8, int HD>
struct AttnFp8Smem {
  float ks[AD_CHUNK], vs[AD_CHUNK];
  alignas(16) uint8_t q[2][HD];
  float qs[2];
};
template <int HD>
struct AttnFp8Smem<false, HD> {};

// Partials: o  [B][nh][nsplit][HD] fp32, then ml [B][nh][nsplit][2] fp32 (running max, sum of exp).
// FP8: kc / vc hold e4m3 bytes with one fp32 scale per slot in ksc / vsc (same (row, slot) index); fp16: ksc / vsc unused.
// PAGED: kc / vc (and ksc / vsc) are the page pools and pg the page table (kv_page.cuh); a chunk spans at most two pages.
template <bool FP8, bool PAGED, int HD, int G>
__global__ void __launch_bounds__(AD_THREADS)
attn_decode_split_kernel(const __half* __restrict__ q, const __half* __restrict__ k_new, const __half* __restrict__ v_new,
                         void* __restrict__ kc, void* __restrict__ vc, float* __restrict__ ksc, float* __restrict__ vsc,
                         const int64_t* __restrict__ positions, float* __restrict__ part_o, float* __restrict__ part_ml,
                         KvPages pg, int nh, int nkv, int max_len, int nsplit, int chunk, float scale) {
  using CT = std::conditional_t<FP8, uint8_t, __half>;   // cache element
  using LT = std::conditional_t<FP8, uint2, uint4>;      // a lane's 8 elements of a slot
  constexpr int U = FP8 ? AD_U8 : AD_U;
  constexpr int LPS = HD / 8;                 // lanes per slot: 8 elements (16 bytes fp16, 8 bytes e4m3) per lane
  constexpr int SG = AD_THREADS / LPS;        // slot groups of the CTA
  constexpr int NW = AD_THREADS / 32;
  __shared__ float sc[G][AD_CHUNK];           // scores, then exp(score - m) (times s_v for FP8)
  __shared__ float red[NW][G][HD];            // per-warp P.V partials
  __shared__ AttnFp8Smem<FP8, HD> f8;

  const int split = blockIdx.x, kvh = blockIdx.y, b = blockIdx.z;
  const int64_t pos = positions[b];
  const int start = split * chunk;
  if (pos < 0 || pos >= max_len || start > pos) return;
  const int n = (int)min((int64_t)chunk, pos - start + 1);
  const int rel = (int)(pos - start);         // the appended slot, when < chunk
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int sg = tid / LPS, sl = tid % LPS;

  // head-vector index of chunk slot j (kv_page.cuh): the chunk's pages are looked up once, here.  A page outside the
  // pool is not dereferenced: the chunk's partials are NaN, so the combine gives the row NaN, and nothing is written.
  const int64_t v0 = kv_vec<PAGED>(pg, b, kvh, nkv, max_len, start);
  const int64_t v1 = PAGED && n > KV_PAGE ? kv_vec<PAGED>(pg, b, kvh, nkv, max_len, start + KV_PAGE) : v0 + KV_PAGE;
  if (PAGED && (v0 < 0 || v1 < 0)) {
    if (tid < G) {
      float* ml = part_ml + (((int64_t)b * nh + (int64_t)kvh * G + tid) * nsplit + split) * 2;
      ml[0] = NAN;
      ml[1] = NAN;
    }
    return;
  }
  auto slot = [&](int j) -> int64_t {
    if constexpr (PAGED) return (j < KV_PAGE ? v0 : v1 - KV_PAGE) + j;
    else return v0 + j;
  };

  const int64_t row = (int64_t)b * nkv + kvh;
  const __half* kn = k_new + row * HD;
  const __half* vn = v_new + row * HD;
  CT* kr = reinterpret_cast<CT*>(kc);
  CT* vr = reinterpret_cast<CT*>(vc);
  float ks = 0.f, vs = 0.f;                   // FP8: the scales of slot start + tid, in flight during the scores
  if constexpr (FP8) {
    if (tid < n && tid != rel) {
      ks = ksc[slot(tid)];
      vs = vsc[slot(tid)];
    }
    if (rel < chunk) {                        // append: this CTA owns slot pos; warp 0 quantizes k_new, warp 1 v_new
      if (warp < 2) {
        float s;
        const uint32_t w = e4m3_quantize_warp<HD>(warp ? vn : kn, lane, s);
        e4m3_store_warp<HD>((warp ? vr : kr) + slot(rel) * HD, lane, w);
        e4m3_store_warp<HD>(f8.q[warp], lane, w);
        if (lane == 0) {
          (warp ? vsc : ksc)[slot(rel)] = s;
          f8.qs[warp] = s;
        }
      }
      __syncthreads();
    }
  } else if (rel < chunk && tid < 2 * LPS) {  // append: this CTA owns slot pos
    const int c = tid % LPS;
    if (tid < LPS) reinterpret_cast<uint4*>(kr + slot(rel) * HD)[c] = reinterpret_cast<const uint4*>(kn)[c];
    else reinterpret_cast<uint4*>(vr + slot(rel) * HD)[c] = reinterpret_cast<const uint4*>(vn)[c];
  }

  // q of the G heads sharing this kv head: the lane's 8 dims of each, in registers
  float qf[G][8];
  const __half* qh = q + ((int64_t)b * nh + (int64_t)kvh * G) * HD;
#pragma unroll
  for (int g = 0; g < G; ++g) h8_to_f(__ldg(reinterpret_cast<const uint4*>(qh + g * HD) + sl), qf[g]);

  // scores: slot group sg takes slots sg, sg + SG, ...; all lanes run the same trip count (the shuffles are warp-wide).
  // U loads are issued before any of them is used; a slot index past n loads slot n - 1 again (valid, discarded).
  // FP8: the appended slot is read from shared memory (its load goes to k_new, a valid address, and is discarded).
  for (int jb = 0; jb < n; jb += U * SG) {
    LT raw[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int j = min(jb + u * SG + sg, n - 1);
      if constexpr (FP8) {
        const void* src = j == rel ? (const void*)kn : (const void*)(kr + slot(j) * HD);
        raw[u] = ldg_nc_v2(reinterpret_cast<const uint2*>(src) + sl);
      } else {
        const __half* src = j == rel ? kn : kr + slot(j) * HD;
        raw[u] = ldg_nc_v4(reinterpret_cast<const uint4*>(src) + sl);
      }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int j = jb + u * SG + sg;
      float kf[8];
      if constexpr (FP8) {
        uint2 w = raw[u];
        if (min(j, n - 1) == rel) w = reinterpret_cast<const uint2*>(f8.q[0])[sl];
        e4m3x8_to_f(w, kf);
      } else {
        h8_to_f(raw[u], kf);
      }
#pragma unroll
      for (int g = 0; g < G; ++g) {
        float d = 0.f;
#pragma unroll
        for (int e = 0; e < 8; ++e) d = fmaf(qf[g][e], kf[e], d);
#pragma unroll
        for (int o = LPS / 2; o > 0; o >>= 1) d += __shfl_xor_sync(0xffffffffu, d, o);
        if (j < n && sl == 0) sc[g][j] = d * scale;
      }
    }
  }
  if constexpr (FP8) {
    if (tid < n) {
      f8.ks[tid] = tid == rel ? f8.qs[0] : ks;
      f8.vs[tid] = tid == rel ? f8.qs[1] : vs;
    }
  }
  __syncthreads();

  // chunk softmax per head: max, exp, sum (one warp per head, fixed order)
  for (int g = warp; g < G; g += NW) {
    float m = -INFINITY;
    for (int j = lane; j < n; j += 32) {
      float s = sc[g][j];
      if constexpr (FP8) {
        s *= f8.ks[j];
        sc[g][j] = s;
      }
      m = fmaxf(m, s);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    float l = 0.f;
    for (int j = lane; j < n; j += 32) {
      const float p = expf(sc[g][j] - m);
      if constexpr (FP8) sc[g][j] = p * f8.vs[j];
      else sc[g][j] = p;
      l += p;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) l += __shfl_xor_sync(0xffffffffu, l, o);
    if (lane == 0) {
      float* ml = part_ml + (((int64_t)b * nh + (int64_t)kvh * G + g) * nsplit + split) * 2;
      ml[0] = m;
      ml[1] = l;
    }
  }
  __syncthreads();

  // P.V: the lane's 8 dims of every head, summed over the group's slots
  float acc[G][8];
#pragma unroll
  for (int g = 0; g < G; ++g)
#pragma unroll
    for (int e = 0; e < 8; ++e) acc[g][e] = 0.f;
  for (int jb = 0; jb < n; jb += U * SG) {
    LT raw[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int j = min(jb + u * SG + sg, n - 1);
      if constexpr (FP8) {
        const void* src = j == rel ? (const void*)vn : (const void*)(vr + slot(j) * HD);
        raw[u] = ldg_nc_v2(reinterpret_cast<const uint2*>(src) + sl);
      } else {
        const __half* src = j == rel ? vn : vr + slot(j) * HD;
        raw[u] = ldg_nc_v4(reinterpret_cast<const uint4*>(src) + sl);
      }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int j = jb + u * SG + sg;
      if (j < n) {
        float vf[8];
        if constexpr (FP8) {
          uint2 w = raw[u];
          if (j == rel) w = reinterpret_cast<const uint2*>(f8.q[1])[sl];
          e4m3x8_to_f(w, vf);
        } else {
          h8_to_f(raw[u], vf);
        }
#pragma unroll
        for (int g = 0; g < G; ++g) {
          const float p = sc[g][j];
#pragma unroll
          for (int e = 0; e < 8; ++e) acc[g][e] = fmaf(p, vf[e], acc[g][e]);
        }
      }
    }
  }
  // across the slot groups of a warp, then across warps (fixed order)
#pragma unroll
  for (int o = LPS; o < 32; o <<= 1)
#pragma unroll
    for (int g = 0; g < G; ++g)
#pragma unroll
      for (int e = 0; e < 8; ++e) acc[g][e] += __shfl_xor_sync(0xffffffffu, acc[g][e], o);
  if (lane < LPS) {
#pragma unroll
    for (int g = 0; g < G; ++g)
#pragma unroll
      for (int e = 0; e < 8; ++e) red[warp][g][sl * 8 + e] = acc[g][e];
  }
  __syncthreads();
  for (int i = tid; i < G * HD; i += AD_THREADS) {
    const int g = i / HD, d = i % HD;
    float s = 0.f;
#pragma unroll
    for (int w = 0; w < NW; ++w) s += red[w][g][d];
    part_o[(((int64_t)b * nh + (int64_t)kvh * G + g) * nsplit + split) * HD + d] = s;
  }
}

// One CTA per (row, token, head), one thread per dim: merge the chunks 0 .. (positions[b] + i) / chunk of token i in
// ascending order.  T = 1 is the decode step; a row with positions[b] + T > max_len gets NaN.
__global__ void __launch_bounds__(128)
attn_decode_combine_kernel(const float* __restrict__ part_o, const float* __restrict__ part_ml,
                           const int64_t* __restrict__ positions, __half* __restrict__ out, int nh, int hd, int max_len,
                           int nsplit, int chunk, int T) {
  const int bh = blockIdx.x, d = threadIdx.x;
  const int bt = bh / nh, b = bt / T;
  const int64_t pos = positions[b];
  if (pos < 0 || pos > (int64_t)max_len - T) {
    out[(int64_t)bh * hd + d] = __float2half_rn(NAN);
    return;
  }
  const int ns = (int)((pos + bt % T) / chunk) + 1;
  const float* ml = part_ml + (int64_t)bh * nsplit * 2;
  const float* po = part_o + (int64_t)bh * nsplit * hd + d;
  float M = -INFINITY;
  for (int s = 0; s < ns; ++s) M = fmaxf(M, ml[2 * s]);
  float L = 0.f, O = 0.f;
  for (int s = 0; s < ns; ++s) {
    const float w = expf(ml[2 * s] - M);
    L = fmaf(ml[2 * s + 1], w, L);
    O = fmaf(po[(int64_t)s * hd], w, O);
  }
  out[(int64_t)bh * hd + d] = __float2half_rn(O / L);
}

// ---- Extend attention: T <= 8 new tokens per row (speculative verification), on tensor cores.
//
// CTA (split, kv head, row) owns one AX_CHUNK-slot chunk and the R = G * T query rows (token i, head g) -> r = i * G + g
// of its kv head, padded to MT = ceil(R / 16) m16 tiles.  The chunk's K and V (e4m3: converted exactly to fp16) and Q
// are staged in shared memory; S = Q.K^T and O = P.V run as mma.sync m16n8k16 (fp16 in, fp32 accumulate).  Token i
// sees slots j <= positions[b] + i.  Scores are fp32 (e4m3: times the slot's k scale), the chunk softmax is fp32 and P
// is rounded once to fp16 for the MMA; e4m3 folds the slot's v scale into p before that rounding, normalised by the
// largest v scale among the row's visible slots of the chunk (multiplied back into O) so that p * s_v keeps fp16's
// normal range and a token's result does not depend on the slots it cannot see.  New slot
// positions[b] + i is written by the CTA whose chunk holds it, which computes with the new (quantized) values directly.
constexpr int AX_CHUNK = 64;
constexpr int AX_THREADS = 128;
constexpr int AX_MAXT = 8;
constexpr int AX_ROWS = AD_MAXG * AX_MAXT;   // query rows per CTA at most

template <int HD>
struct AxLayout {
  static constexpr int QS = HD + 8;          // row stride (halves) of the Q, K and V tiles: conflict-free fragments
  static constexpr int PS = AX_CHUNK + 8;    // row stride (halves) of the P tile
  static constexpr int SS = AX_CHUNK + 4;    // row stride (floats) of the score tile (aliases the Q tile)
  static constexpr size_t QB = (size_t)AX_ROWS * QS * 2, SB = (size_t)AX_ROWS * SS * 4;
  static constexpr size_t K_OFF = ((QB > SB ? QB : SB) + 15) & ~(size_t)15;
  static constexpr size_t V_OFF = K_OFF + (size_t)AX_CHUNK * QS * 2;
  static constexpr size_t P_OFF = V_OFF + (size_t)AX_CHUNK * QS * 2;
  static constexpr size_t F_OFF = P_OFF + (size_t)AX_ROWS * PS * 2;   // k scales, v scales, each row's max v scale
  static constexpr size_t BYTES = F_OFF + (2 * AX_CHUNK + AX_ROWS) * sizeof(float);
};

__device__ __forceinline__ uint32_t h2_pack(__half lo, __half hi) {
  return (uint32_t)__half_as_ushort(lo) | ((uint32_t)__half_as_ushort(hi) << 16);
}

// Partials: o [B][T][nh][nsplit][HD], ml [B][T][nh][nsplit][2], the layout of the decode kernel with B * T rows.
// PAGED: kc / vc (and ksc / vsc) are the page pools and pg the page table; a chunk is one page.
template <bool FP8, bool PAGED, int HD, int G>
__global__ void __launch_bounds__(AX_THREADS)
attn_extend_split_kernel(const __half* __restrict__ q, const __half* __restrict__ k_new, const __half* __restrict__ v_new,
                         void* __restrict__ kc, void* __restrict__ vc, float* __restrict__ ksc, float* __restrict__ vsc,
                         const int64_t* __restrict__ positions, float* __restrict__ part_o, float* __restrict__ part_ml,
                         KvPages pg, int nh, int nkv, int max_len, int nsplit, int T, float scale) {
  using L = AxLayout<HD>;
  using CT = std::conditional_t<FP8, uint8_t, __half>;
  constexpr int QS = L::QS, PS = L::PS, SS = L::SS;
  constexpr int SEG = HD / 8;                 // 16-byte fp16 segments of a head vector
  constexpr int NT = HD / 32;                 // n8 tiles of a warp's quarter of the P.V output
  extern __shared__ __align__(16) unsigned char ax_smem[];
  __half* sq = reinterpret_cast<__half*>(ax_smem);
  float* ss = reinterpret_cast<float*>(ax_smem);
  __half* sk = reinterpret_cast<__half*>(ax_smem + L::K_OFF);
  __half* sv = reinterpret_cast<__half*>(ax_smem + L::V_OFF);
  __half* sp = reinterpret_cast<__half*>(ax_smem + L::P_OFF);
  float* sks = reinterpret_cast<float*>(ax_smem + L::F_OFF);
  float* svs = sks + AX_CHUNK;
  float* svmax = svs + AX_CHUNK;              // per query row

  const int split = blockIdx.x, kvh = blockIdx.y, b = blockIdx.z;
  const int64_t pos = positions[b];
  const int start = split * AX_CHUNK;
  if (pos < 0 || pos > (int64_t)max_len - T || start > pos + T - 1) return;
  const int n = (int)min((int64_t)AX_CHUNK, pos + T - start);          // slots start .. start + n - 1
  const int nold = (int)max((int64_t)0, min((int64_t)n, pos - start));  // of which cached (the rest are new)
  const int R = G * T, MT = (R + 15) / 16;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, gid = lane >> 2, tig = lane & 3;

  // head-vector index of chunk slot 0 (kv_page.cuh).  A page outside the pool is not dereferenced: every query row's
  // partial of this chunk is NaN (the combine reads it only for the tokens that see the chunk), nothing is written.
  const int64_t v0 = kv_vec<PAGED>(pg, b, kvh, nkv, max_len, start);
  if (PAGED && v0 < 0) {
    for (int r = tid; r < R; r += AX_THREADS) {
      float* ml = part_ml + ((((int64_t)b * T + r / G) * nh + (int64_t)kvh * G + r % G) * nsplit + split) * 2;
      ml[0] = NAN;
      ml[1] = NAN;
    }
    return;
  }
  CT* kr = reinterpret_cast<CT*>(kc) + v0 * HD;
  CT* vr = reinterpret_cast<CT*>(vc) + v0 * HD;
  float* ksr = ksc + v0;
  float* vsr = vsc + v0;
  auto new_vec = [&](const __half* x, int j) {  // the new key / value of chunk slot j
    return x + (((int64_t)b * T + (start + j - pos)) * nkv + kvh) * HD;
  };

  // ---- stage Q (rows >= R zero), the chunk's K / V (rows >= n zero) and, e4m3, the slot scales
  for (int i = tid; i < MT * 16 * SEG; i += AX_THREADS) {
    const int r = i / SEG, c = i % SEG;
    uint4 v = make_uint4(0, 0, 0, 0);
    if (r < R) v = __ldg(reinterpret_cast<const uint4*>(q + (((int64_t)b * T + r / G) * nh + (int64_t)kvh * G + r % G) * HD) + c);
    reinterpret_cast<uint4*>(sq + r * QS)[c] = v;
  }
  for (int i = tid; i < AX_CHUNK * SEG; i += AX_THREADS) {
    const int j = i / SEG, c = i % SEG;
    uint4 kv = make_uint4(0, 0, 0, 0), vv = kv;
    if (j < nold) {
      if constexpr (FP8) {
        kv = e4m3x8_to_h8(ldg_nc_v2(reinterpret_cast<const uint2*>(kr + (int64_t)j * HD) + c));
        vv = e4m3x8_to_h8(ldg_nc_v2(reinterpret_cast<const uint2*>(vr + (int64_t)j * HD) + c));
      } else {
        kv = ldg_nc_v4(reinterpret_cast<const uint4*>(kr + (int64_t)j * HD) + c);
        vv = ldg_nc_v4(reinterpret_cast<const uint4*>(vr + (int64_t)j * HD) + c);
      }
    } else if (j < n && !FP8) {               // append: this CTA owns slot start + j
      kv = reinterpret_cast<const uint4*>(new_vec(k_new, j))[c];
      vv = reinterpret_cast<const uint4*>(new_vec(v_new, j))[c];
      reinterpret_cast<uint4*>(kr + (int64_t)j * HD)[c] = kv;
      reinterpret_cast<uint4*>(vr + (int64_t)j * HD)[c] = vv;
    } else if (j < n) {
      continue;                               // e4m3 append below
    }
    reinterpret_cast<uint4*>(sk + j * QS)[c] = kv;
    reinterpret_cast<uint4*>(sv + j * QS)[c] = vv;
  }
  if constexpr (FP8) {
    for (int j = tid; j < nold; j += AX_THREADS) {
      sks[j] = ksr[j];
      svs[j] = vsr[j];
    }
    // append: one warp per new vector (k of slot j, then v), quantized, stored, and staged as fp16
    constexpr int E = HD / 32;
    for (int v = warp; v < 2 * (n - nold); v += AX_THREADS / 32) {
      const int isv = v & 1, j = nold + v / 2;
      float s;
      const uint32_t w = e4m3_quantize_warp<HD>(new_vec(isv ? v_new : k_new, j), lane, s);
      e4m3_store_warp<HD>((isv ? vr : kr) + (int64_t)j * HD, lane, w);
      __half* t = (isv ? sv : sk) + j * QS + lane * E;
#pragma unroll
      for (int e = 0; e < E / 2; ++e)
        reinterpret_cast<__half2*>(t)[e] =
            __half2(__nv_cvt_fp8x2_to_halfraw2((__nv_fp8x2_storage_t)((w >> (16 * e)) & 0xFFFFu), __NV_E4M3));
      if (lane == 0) {
        (isv ? vsr : ksr)[j] = s;
        (isv ? svs : sks)[j] = s;
      }
    }
  }
  __syncthreads();

  // ---- S = Q.K^T: warp w takes slots 16w .. 16w + 15 of every m tile
  float acc[4][2][4];
#pragma unroll
  for (int mt = 0; mt < 4; ++mt)
#pragma unroll
    for (int nt = 0; nt < 2; ++nt)
#pragma unroll
      for (int e = 0; e < 4; ++e) acc[mt][nt][e] = 0.f;
  if (warp * 16 < n) {
#pragma unroll
    for (int kk = 0; kk < HD; kk += 16) {
      uint32_t bf[2][2];
#pragma unroll
      for (int nt = 0; nt < 2; ++nt) {
        const __half* kp = sk + (warp * 16 + nt * 8 + gid) * QS + kk + tig * 2;
        bf[nt][0] = *reinterpret_cast<const uint32_t*>(kp);
        bf[nt][1] = *reinterpret_cast<const uint32_t*>(kp + 8);
      }
#pragma unroll
      for (int mt = 0; mt < 4; ++mt) {
        if (mt < MT) {
          const __half* qp = sq + (mt * 16 + gid) * QS + kk + tig * 2;
          const uint32_t a[4] = {*reinterpret_cast<const uint32_t*>(qp), *reinterpret_cast<const uint32_t*>(qp + 8 * QS),
                                 *reinterpret_cast<const uint32_t*>(qp + 8),
                                 *reinterpret_cast<const uint32_t*>(qp + 8 * QS + 8)};
#pragma unroll
          for (int nt = 0; nt < 2; ++nt) mma16816(acc[mt][nt], a, bf[nt]);
        }
      }
    }
  }
  __syncthreads();                            // the score tile overwrites the Q tile
#pragma unroll
  for (int mt = 0; mt < 4; ++mt) {
    if (mt < MT) {
#pragma unroll
      for (int nt = 0; nt < 2; ++nt)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int r = mt * 16 + gid + (e >> 1) * 8, j = warp * 16 + nt * 8 + tig * 2 + (e & 1);
          float s = acc[mt][nt][e] * scale;
          if constexpr (FP8) s = j < n ? s * sks[j] : s;
          const bool ok = r < R && j < n && (int64_t)start + j <= pos + r / G;
          ss[r * SS + j] = ok ? s : -INFINITY;
        }
    }
  }
  __syncthreads();

  // ---- chunk softmax per query row (one warp per row, fixed order); P (fp16) for the MMA
  for (int r = warp; r < MT * 16; r += AX_THREADS / 32) {
    float p0 = 0.f, p1 = 0.f;
    if (r < R) {
      const float s0 = ss[r * SS + lane], s1 = ss[r * SS + lane + 32];
      float m = fmaxf(s0, s1);
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
      if (m != -INFINITY) {
        p0 = expf(s0 - m);
        p1 = expf(s1 - m);
      }
      float l = p0 + p1;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) l += __shfl_xor_sync(0xffffffffu, l, o);
      if (lane == 0) {
        float* ml = part_ml + ((((int64_t)b * T + r / G) * nh + (int64_t)kvh * G + r % G) * nsplit + split) * 2;
        ml[0] = m;
        ml[1] = l;
      }
      if constexpr (FP8) {                    // p0 / p1 are 0 at the slots the row does not see
        const int64_t last = pos + r / G - start;
        float sm = fmaxf(lane <= last && lane < n ? svs[lane] : 0.f, lane + 32 <= last && lane + 32 < n ? svs[lane + 32] : 0.f);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) sm = fmaxf(sm, __shfl_xor_sync(0xffffffffu, sm, o));
        sm = sm > 0.f ? sm : 1.f;
        const float vnorm = 1.f / sm;
        p0 = p0 > 0.f ? p0 * (svs[lane] * vnorm) : 0.f;
        p1 = p1 > 0.f ? p1 * (svs[lane + 32] * vnorm) : 0.f;
        if (lane == 0) svmax[r] = sm;
      }
    }
    sp[r * PS + lane] = __float2half_rn(p0);
    sp[r * PS + lane + 32] = __float2half_rn(p1);
  }
  __syncthreads();

  // ---- O = P.V: warp w takes dims w * HD / 4 .. of every m tile; k steps past n hold P = V = 0 and are skipped
  float o[4][NT][4];
#pragma unroll
  for (int mt = 0; mt < 4; ++mt)
#pragma unroll
    for (int nt = 0; nt < NT; ++nt)
#pragma unroll
      for (int e = 0; e < 4; ++e) o[mt][nt][e] = 0.f;
#pragma unroll
  for (int kk = 0; kk < AX_CHUNK; kk += 16) {
    if (kk < n) {
      uint32_t bf[NT][2];
#pragma unroll
      for (int nt = 0; nt < NT; ++nt) {
        const __half* vp = sv + (kk + tig * 2) * QS + warp * (HD / 4) + nt * 8 + gid;
        bf[nt][0] = h2_pack(vp[0], vp[QS]);
        bf[nt][1] = h2_pack(vp[8 * QS], vp[9 * QS]);
      }
#pragma unroll
      for (int mt = 0; mt < 4; ++mt) {
        if (mt < MT) {
          const __half* pp = sp + (mt * 16 + gid) * PS + kk + tig * 2;
          const uint32_t a[4] = {*reinterpret_cast<const uint32_t*>(pp), *reinterpret_cast<const uint32_t*>(pp + 8 * PS),
                                 *reinterpret_cast<const uint32_t*>(pp + 8),
                                 *reinterpret_cast<const uint32_t*>(pp + 8 * PS + 8)};
#pragma unroll
          for (int nt = 0; nt < NT; ++nt) mma16816(o[mt][nt], a, bf[nt]);
        }
      }
    }
  }
#pragma unroll
  for (int mt = 0; mt < 4; ++mt) {
    if (mt < MT) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int r = mt * 16 + gid + 8 * h;
        if (r < R) {
          const float oscale = FP8 ? svmax[r] : 1.f;
          float* dst = part_o + ((((int64_t)b * T + r / G) * nh + (int64_t)kvh * G + r % G) * nsplit + split) * HD +
                       warp * (HD / 4) + tig * 2;
#pragma unroll
          for (int nt = 0; nt < NT; ++nt)
            *reinterpret_cast<float2*>(dst + nt * 8) = make_float2(o[mt][nt][2 * h] * oscale, o[mt][nt][2 * h + 1] * oscale);
        }
      }
    }
  }
}

// Prefill: one warp per head vector v = (row, p) of src (rows, P, HD) fp16 -> e4m3 slot p of cache (rows, max_len, HD)
// and its scale; slots >= P are not touched.
constexpr int KQ_WARPS = 8;

template <int HD>
__global__ void __launch_bounds__(KQ_WARPS * 32)
kv_quantize_fp8_kernel(const __half* __restrict__ src, uint8_t* __restrict__ cache, float* __restrict__ scales,
                       int64_t nvec, int P, int max_len) {
  const int64_t v = (int64_t)blockIdx.x * KQ_WARPS + threadIdx.x / 32;
  if (v >= nvec) return;                      // warp-uniform
  const int lane = threadIdx.x & 31;
  const int64_t slot = v / P * max_len + v % P;
  float s;
  const uint32_t w = e4m3_quantize_warp<HD>(src + v * HD, lane, s);
  e4m3_store_warp<HD>(cache + slot * HD, lane, w);
  if (lane == 0) scales[slot] = s;
}

template <bool FP8, bool PAGED, int HD, int G>
void launch_split(dim3 grid, cudaStream_t st, const void* q, const void* kn, const void* vn, void* kc, void* vc,
                  float* ksc, float* vsc, const int64_t* pos, float* po, float* pml, KvPages pg, int nh, int nkv,
                  int max_len, int nsplit, int chunk, float scale) {
  attn_decode_split_kernel<FP8, PAGED, HD, G><<<grid, AD_THREADS, 0, st>>>((const __half*)q, (const __half*)kn,
                                                                           (const __half*)vn, kc, vc, ksc, vsc, pos, po,
                                                                           pml, pg, nh, nkv, max_len, nsplit, chunk, scale);
}

template <bool FP8, bool PAGED, int HD>
void launch_split_g(int G, dim3 grid, cudaStream_t st, const void* q, const void* kn, const void* vn, void* kc, void* vc,
                    float* ksc, float* vsc, const int64_t* pos, float* po, float* pml, KvPages pg, int nh, int nkv,
                    int max_len, int nsplit, int chunk, float scale) {
#define AD_LAUNCH(g) \
  launch_split<FP8, PAGED, HD, g>(grid, st, q, kn, vn, kc, vc, ksc, vsc, pos, po, pml, pg, nh, nkv, max_len, nsplit, \
                                  chunk, scale)
  switch (G) {
    case 1: AD_LAUNCH(1); break;
    case 2: AD_LAUNCH(2); break;
    case 3: AD_LAUNCH(3); break;
    case 4: AD_LAUNCH(4); break;
    case 5: AD_LAUNCH(5); break;
    case 6: AD_LAUNCH(6); break;
    case 7: AD_LAUNCH(7); break;
    default: AD_LAUNCH(8); break;
  }
#undef AD_LAUNCH
}

size_t ws_bytes(int64_t B, int64_t nh, int64_t hd, int64_t nsplit) {
  const size_t o = (size_t)(B * nh * nsplit * hd) * sizeof(float);
  return ((o + 255) & ~(size_t)255) + (size_t)(B * nh * nsplit * 2) * sizeof(float);
}

// Argument checks and launches of quip_decode_attention on a cache kv_check accepted (FP8: e4m3; PAGED: the caches
// and scales are page pools behind pg, max_len = max_pages * 64); fn names the entry point in the messages.
template <bool FP8, bool PAGED>
int decode_attention(const char* fn, const QuipKvCache& kv, KvPages pg, int32_t max_len, const void* q,
                     const void* k_new, const void* v_new, const int64_t* positions, void* out, int32_t B, int32_t nh,
                     float scale, void* workspace, size_t workspace_bytes, void* stream) {
  const int32_t nkv = kv.nkv, hd = kv.hd;
  QUIP_CHECK_ARG(q && k_new && v_new && positions && out && workspace, "%s: null pointer", fn);
  QUIP_CHECK_ARG(B >= 0 && B <= 65535 && max_len > 0 && nkv > 0 && nkv <= 65535 && nh > 0,
                 "%s: bad sizes (B %d, nh %d, nkv %d, max_len %d)", fn, B, nh, nkv, max_len);
  QUIP_CHECK_ARG(nh % nkv == 0 && nh / nkv <= AD_MAXG,
                 "%s: %d query heads on %d kv heads: nh %% nkv must be 0 with at most %d per kv head",
                 fn, nh, nkv, AD_MAXG);
  QUIP_CHECK_ARG(al16(q) && al16(k_new) && al16(v_new) && al16(out) && al16(workspace),
                 "%s: pointers must be 16-byte aligned", fn);
  const int chunk = (int64_t)B * nkv * ceil_div(max_len, AD_CHUNK) < AD_SMALL_GRID ? AD_SMALL_CHUNK : AD_CHUNK;
  const int nsplit = ceil_div(max_len, chunk);
  const size_t need = ws_bytes(B, nh, hd, nsplit);
  QUIP_CHECK_ARG(workspace_bytes >= need, "%s: workspace of %zu bytes, %zu needed", fn, workspace_bytes, need);
  if (B == 0) return QUIP_OK;
  float* po = (float*)workspace;
  float* pml = (float*)((char*)workspace + (((size_t)B * nh * nsplit * hd * sizeof(float) + 255) & ~(size_t)255));
  const cudaStream_t st = (cudaStream_t)stream;
  const dim3 grid(nsplit, nkv, B);
  const int G = nh / nkv;
  if (hd == 64) launch_split_g<FP8, PAGED, 64>(G, grid, st, q, k_new, v_new, kv.k, kv.v, kv.k_scale, kv.v_scale, positions, po, pml, pg, nh, nkv, max_len, nsplit, chunk, scale);
  else launch_split_g<FP8, PAGED, 128>(G, grid, st, q, k_new, v_new, kv.k, kv.v, kv.k_scale, kv.v_scale, positions, po, pml, pg, nh, nkv, max_len, nsplit, chunk, scale);
  QUIP_LAUNCHED("attn_decode_split_kernel");
  attn_decode_combine_kernel<<<(unsigned)(B * nh), hd, 0, st>>>(po, pml, positions, (__half*)out, nh, hd, max_len, nsplit, chunk, 1);
  QUIP_LAUNCHED("attn_decode_combine_kernel");
  return QUIP_OK;
}

template <bool FP8, bool PAGED, int HD, int G>
int launch_extend(dim3 grid, cudaStream_t st, const void* q, const void* kn, const void* vn, void* kc, void* vc,
                  float* ksc, float* vsc, const int64_t* pos, float* po, float* pml, KvPages pg, int nh, int nkv,
                  int max_len, int nsplit, int T, float scale) {
  constexpr size_t smem = AxLayout<HD>::BYTES;
  auto kern = attn_extend_split_kernel<FP8, PAGED, HD, G>;
  if (smem > 48 * 1024) QUIP_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  kern<<<grid, AX_THREADS, smem, st>>>((const __half*)q, (const __half*)kn, (const __half*)vn, kc, vc, ksc, vsc, pos, po,
                                       pml, pg, nh, nkv, max_len, nsplit, T, scale);
  QUIP_LAUNCHED("attn_extend_split_kernel");
  return QUIP_OK;
}

template <bool FP8, bool PAGED, int HD>
int launch_extend_g(int G, dim3 grid, cudaStream_t st, const void* q, const void* kn, const void* vn, void* kc,
                    void* vc, float* ksc, float* vsc, const int64_t* pos, float* po, float* pml, KvPages pg, int nh,
                    int nkv, int max_len, int nsplit, int T, float scale) {
#define AX_LAUNCH(g) \
  return launch_extend<FP8, PAGED, HD, g>(grid, st, q, kn, vn, kc, vc, ksc, vsc, pos, po, pml, pg, nh, nkv, max_len, \
                                          nsplit, T, scale)
  switch (G) {
    case 1: AX_LAUNCH(1);
    case 2: AX_LAUNCH(2);
    case 3: AX_LAUNCH(3);
    case 4: AX_LAUNCH(4);
    case 5: AX_LAUNCH(5);
    case 6: AX_LAUNCH(6);
    case 7: AX_LAUNCH(7);
    default: AX_LAUNCH(8);
  }
#undef AX_LAUNCH
}

// Argument checks and launches of quip_extend_attention on a cache kv_check accepted, as decode_attention.
template <bool FP8, bool PAGED>
int extend_attention(const char* fn, const QuipKvCache& kv, KvPages pg, int32_t max_len, const void* q,
                     const void* k_new, const void* v_new, const int64_t* positions, void* out, int32_t B, int32_t T,
                     int32_t nh, float scale, void* workspace, size_t workspace_bytes, void* stream) {
  const int32_t nkv = kv.nkv, hd = kv.hd;
  QUIP_CHECK_ARG(q && k_new && v_new && positions && out && workspace, "%s: null pointer", fn);
  QUIP_CHECK_ARG(T >= 1 && T <= AX_MAXT, "%s: %d tokens per row: need 1 <= T <= %d", fn, T, AX_MAXT);
  QUIP_CHECK_ARG(B >= 0 && B <= 65535 && max_len > 0 && nkv > 0 && nkv <= 65535 && nh > 0,
                 "%s: bad sizes (B %d, nh %d, nkv %d, max_len %d)", fn, B, nh, nkv, max_len);
  QUIP_CHECK_ARG(nh % nkv == 0 && nh / nkv <= AD_MAXG,
                 "%s: %d query heads on %d kv heads: nh %% nkv must be 0 with at most %d per kv head",
                 fn, nh, nkv, AD_MAXG);
  QUIP_CHECK_ARG(al16(q) && al16(k_new) && al16(v_new) && al16(out) && al16(workspace),
                 "%s: pointers must be 16-byte aligned", fn);
  const int nsplit = ceil_div(max_len, AX_CHUNK);
  const size_t need = ws_bytes((int64_t)B * T, nh, hd, nsplit);
  QUIP_CHECK_ARG(workspace_bytes >= need, "%s: workspace of %zu bytes, %zu needed", fn, workspace_bytes, need);
  if (B == 0) return QUIP_OK;
  float* po = (float*)workspace;
  float* pml = (float*)((char*)workspace + (((size_t)B * T * nh * nsplit * hd * sizeof(float) + 255) & ~(size_t)255));
  const cudaStream_t st = (cudaStream_t)stream;
  const dim3 grid(nsplit, nkv, B);
  const int G = nh / nkv;
  const int e = hd == 64
      ? launch_extend_g<FP8, PAGED, 64>(G, grid, st, q, k_new, v_new, kv.k, kv.v, kv.k_scale, kv.v_scale, positions, po, pml, pg, nh, nkv, max_len, nsplit, T, scale)
      : launch_extend_g<FP8, PAGED, 128>(G, grid, st, q, k_new, v_new, kv.k, kv.v, kv.k_scale, kv.v_scale, positions, po, pml, pg, nh, nkv, max_len, nsplit, T, scale);
  if (e != QUIP_OK) return e;
  attn_decode_combine_kernel<<<(unsigned)((int64_t)B * T * nh), hd, 0, st>>>(po, pml, positions, (__half*)out, nh, hd,
                                                                             max_len, nsplit, AX_CHUNK, T);
  QUIP_LAUNCHED("attn_decode_combine_kernel");
  return QUIP_OK;
}

}  // namespace

}  // namespace quip

using namespace quip;

extern "C" int quip_decode_attention_workspace_bytes(int32_t B, int32_t nh, int32_t hd, int32_t max_len,
                                                     size_t* out_bytes) {
  QUIP_CHECK_ARG(out_bytes, "quip_decode_attention_workspace_bytes: null pointer");
  QUIP_CHECK_ARG(B >= 0 && nh > 0 && max_len > 0, "quip_decode_attention_workspace_bytes: bad sizes");
  QUIP_CHECK_ARG(hd == 64 || hd == 128, "quip_decode_attention_workspace_bytes: head_dim %d is not 64 or 128", hd);
  *out_bytes = ws_bytes(B, nh, hd, ceil_div(max_len, AD_SMALL_CHUNK));      // the larger of the two chunkings
  return QUIP_OK;
}

extern "C" int quip_decode_attention(const QuipKvCache* kv, const void* q, const void* k_new, const void* v_new,
                                     const int64_t* positions, void* out, int32_t B, int32_t nh, float scale,
                                     void* workspace, size_t workspace_bytes, void* stream) {
  const char* fn = "quip_decode_attention";
  KvPages pg;
  int32_t max_len;
  if (const int e = kv_check(fn, kv, pg, max_len)) return e;
  return kv_dispatch(*kv, [&](auto fp8, auto paged) {
    return decode_attention<decltype(fp8)::value, decltype(paged)::value>(fn, *kv, pg, max_len, q, k_new, v_new,
                                                                        positions, out, B, nh, scale, workspace,
                                                                        workspace_bytes, stream);
  });
}

extern "C" int quip_extend_attention_workspace_bytes(int32_t B, int32_t T, int32_t nh, int32_t hd, int32_t max_len,
                                                     size_t* out_bytes) {
  QUIP_CHECK_ARG(out_bytes, "quip_extend_attention_workspace_bytes: null pointer");
  QUIP_CHECK_ARG(B >= 0 && T >= 1 && T <= AX_MAXT && nh > 0 && max_len > 0,
                 "quip_extend_attention_workspace_bytes: bad sizes (B %d, T %d, nh %d, max_len %d)", B, T, nh, max_len);
  QUIP_CHECK_ARG(hd == 64 || hd == 128, "quip_extend_attention_workspace_bytes: head_dim %d is not 64 or 128", hd);
  *out_bytes = ws_bytes((int64_t)B * T, nh, hd, ceil_div(max_len, AX_CHUNK));
  return QUIP_OK;
}

extern "C" int quip_extend_attention(const QuipKvCache* kv, const void* q, const void* k_new, const void* v_new,
                                     const int64_t* positions, void* out, int32_t B, int32_t T, int32_t nh, float scale,
                                     void* workspace, size_t workspace_bytes, void* stream) {
  const char* fn = "quip_extend_attention";
  KvPages pg;
  int32_t max_len;
  if (const int e = kv_check(fn, kv, pg, max_len)) return e;
  return kv_dispatch(*kv, [&](auto fp8, auto paged) {
    return extend_attention<decltype(fp8)::value, decltype(paged)::value>(fn, *kv, pg, max_len, q, k_new, v_new,
                                                                        positions, out, B, T, nh, scale, workspace,
                                                                        workspace_bytes, stream);
  });
}

extern "C" int quip_kv_quantize_fp8(const void* src, void* cache, float* scales, int32_t B, int32_t nkv, int32_t P,
                                    int32_t max_len, int32_t hd, void* stream) {
  QUIP_CHECK_ARG(src && cache && scales, "quip_kv_quantize_fp8: null pointer");
  QUIP_CHECK_ARG(hd == 64 || hd == 128, "quip_kv_quantize_fp8: head_dim %d is not 64 or 128", hd);
  QUIP_CHECK_ARG(B >= 0 && nkv > 0 && P >= 0 && max_len > 0 && P <= max_len,
                 "quip_kv_quantize_fp8: bad sizes (B %d, nkv %d, P %d, max_len %d): need P <= max_len", B, nkv, P, max_len);
  QUIP_CHECK_ARG(al16(src) && al16(cache) && al4(scales),
                 "quip_kv_quantize_fp8: src and cache must be 16-byte aligned, scales 4-byte aligned");
  const int64_t nvec = (int64_t)B * nkv * P;
  if (nvec == 0) return QUIP_OK;
  const unsigned blocks = (unsigned)((nvec + KQ_WARPS - 1) / KQ_WARPS);
  const cudaStream_t st = (cudaStream_t)stream;
  if (hd == 64) kv_quantize_fp8_kernel<64><<<blocks, KQ_WARPS * 32, 0, st>>>((const __half*)src, (uint8_t*)cache, scales, nvec, P, max_len);
  else kv_quantize_fp8_kernel<128><<<blocks, KQ_WARPS * 32, 0, st>>>((const __half*)src, (uint8_t*)cache, scales, nvec, P, max_len);
  QUIP_LAUNCHED("kv_quantize_fp8_kernel");
  return QUIP_OK;
}
