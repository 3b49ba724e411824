// Decode attention: one new token per sequence, each sequence at its own position, over the static KV cache of
// quip_b200/decode.py (one layer: k_cache / v_cache (B, nkv, max_len, hd) fp16).
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
#include <math.h>

#include "common.cuh"

namespace quip {

namespace {

constexpr int AD_CHUNK = 128;        // KV slots per CTA (at most)
constexpr int AD_SMALL_CHUNK = 64;   // when B * nkv * ceil(max_len / AD_CHUNK) < AD_SMALL_GRID
constexpr int AD_SMALL_GRID = 2 * 132;
constexpr int AD_U = 4;              // slots per slot group whose loads are in flight together
constexpr int AD_THREADS = 128;
constexpr int AD_MAXG = 8;           // query heads per kv head

union AH8 {
  uint4 v;
  __half2 h2[4];
};

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

// Partials: o  [B][nh][nsplit][HD] fp32, then ml [B][nh][nsplit][2] fp32 (running max, sum of exp).
template <int HD, int G>
__global__ void __launch_bounds__(AD_THREADS)
attn_decode_split_kernel(const __half* __restrict__ q, const __half* __restrict__ k_new, const __half* __restrict__ v_new,
                         __half* __restrict__ kc, __half* __restrict__ vc, const int64_t* __restrict__ positions,
                         float* __restrict__ part_o, float* __restrict__ part_ml, int nh, int nkv, int max_len,
                         int nsplit, int chunk, float scale) {
  constexpr int LPS = HD / 8;                 // lanes per slot: 8 fp16 (16 bytes) per lane
  constexpr int SG = AD_THREADS / LPS;        // slot groups of the CTA
  constexpr int NW = AD_THREADS / 32;
  __shared__ float sc[G][AD_CHUNK];           // scores, then exp(score - m)
  __shared__ float red[NW][G][HD];            // per-warp P.V partials

  const int split = blockIdx.x, kvh = blockIdx.y, b = blockIdx.z;
  const int64_t pos = positions[b];
  const int start = split * chunk;
  if (pos < 0 || pos >= max_len || start > pos) return;
  const int n = (int)min((int64_t)chunk, pos - start + 1);
  const int rel = (int)(pos - start);         // the appended slot, when < chunk
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int sg = tid / LPS, sl = tid % LPS;

  const int64_t row = (int64_t)b * nkv + kvh;
  const __half* kn = k_new + row * HD;
  const __half* vn = v_new + row * HD;
  __half* kr = kc + row * (int64_t)max_len * HD;
  __half* vr = vc + row * (int64_t)max_len * HD;
  if (rel < chunk && tid < 2 * LPS) {      // append: this CTA owns slot pos
    const int c = tid % LPS;
    if (tid < LPS) reinterpret_cast<uint4*>(kr + pos * HD)[c] = reinterpret_cast<const uint4*>(kn)[c];
    else reinterpret_cast<uint4*>(vr + pos * HD)[c] = reinterpret_cast<const uint4*>(vn)[c];
  }

  // q of the G heads sharing this kv head: the lane's 8 dims of each, in registers
  float qf[G][8];
  const __half* qh = q + ((int64_t)b * nh + (int64_t)kvh * G) * HD;
#pragma unroll
  for (int g = 0; g < G; ++g) h8_to_f(__ldg(reinterpret_cast<const uint4*>(qh + g * HD) + sl), qf[g]);

  // scores: slot group sg takes slots sg, sg + SG, ...; all lanes run the same trip count (the shuffles are warp-wide).
  // AD_U loads are issued before any of them is used; a slot index past n loads slot n - 1 again (valid, discarded).
  for (int jb = 0; jb < n; jb += AD_U * SG) {
    uint4 raw[AD_U];
#pragma unroll
    for (int u = 0; u < AD_U; ++u) {
      const int j = min(jb + u * SG + sg, n - 1);
      const __half* src = j == rel ? kn : kr + (int64_t)(start + j) * HD;
      raw[u] = ldg_nc_v4(reinterpret_cast<const uint4*>(src) + sl);
    }
#pragma unroll
    for (int u = 0; u < AD_U; ++u) {
      const int j = jb + u * SG + sg;
      float kf[8];
      h8_to_f(raw[u], kf);
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
  __syncthreads();

  // chunk softmax per head: max, exp, sum (one warp per head, fixed order)
  for (int g = warp; g < G; g += NW) {
    float m = -INFINITY;
    for (int j = lane; j < n; j += 32) m = fmaxf(m, sc[g][j]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    float l = 0.f;
    for (int j = lane; j < n; j += 32) {
      const float p = expf(sc[g][j] - m);
      sc[g][j] = p;
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
  for (int jb = 0; jb < n; jb += AD_U * SG) {
    uint4 raw[AD_U];
#pragma unroll
    for (int u = 0; u < AD_U; ++u) {
      const int j = min(jb + u * SG + sg, n - 1);
      const __half* src = j == rel ? vn : vr + (int64_t)(start + j) * HD;
      raw[u] = ldg_nc_v4(reinterpret_cast<const uint4*>(src) + sl);
    }
#pragma unroll
    for (int u = 0; u < AD_U; ++u) {
      const int j = jb + u * SG + sg;
      if (j < n) {
        float vf[8];
        h8_to_f(raw[u], vf);
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

// One CTA per (row, head), one thread per dim: merge the chunks 0 .. positions[b] / chunk in ascending order.
__global__ void __launch_bounds__(128)
attn_decode_combine_kernel(const float* __restrict__ part_o, const float* __restrict__ part_ml,
                           const int64_t* __restrict__ positions, __half* __restrict__ out, int nh, int hd, int max_len,
                           int nsplit, int chunk) {
  const int bh = blockIdx.x, d = threadIdx.x;
  const int b = bh / nh;
  const int64_t pos = positions[b];
  if (pos < 0 || pos >= max_len) {
    out[(int64_t)bh * hd + d] = __float2half_rn(NAN);
    return;
  }
  const int ns = (int)(pos / chunk) + 1;
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

template <int HD, int G>
void launch_split(dim3 grid, cudaStream_t st, const void* q, const void* kn, const void* vn, void* kc, void* vc,
                  const int64_t* pos, float* po, float* pml, int nh, int nkv, int max_len, int nsplit, int chunk, float scale) {
  attn_decode_split_kernel<HD, G><<<grid, AD_THREADS, 0, st>>>((const __half*)q, (const __half*)kn, (const __half*)vn,
                                                               (__half*)kc, (__half*)vc, pos, po, pml, nh, nkv, max_len,
                                                               nsplit, chunk, scale);
}

template <int HD>
void launch_split_g(int G, dim3 grid, cudaStream_t st, const void* q, const void* kn, const void* vn, void* kc, void* vc,
                    const int64_t* pos, float* po, float* pml, int nh, int nkv, int max_len, int nsplit, int chunk, float scale) {
  switch (G) {
    case 1: launch_split<HD, 1>(grid, st, q, kn, vn, kc, vc, pos, po, pml, nh, nkv, max_len, nsplit, chunk, scale); break;
    case 2: launch_split<HD, 2>(grid, st, q, kn, vn, kc, vc, pos, po, pml, nh, nkv, max_len, nsplit, chunk, scale); break;
    case 3: launch_split<HD, 3>(grid, st, q, kn, vn, kc, vc, pos, po, pml, nh, nkv, max_len, nsplit, chunk, scale); break;
    case 4: launch_split<HD, 4>(grid, st, q, kn, vn, kc, vc, pos, po, pml, nh, nkv, max_len, nsplit, chunk, scale); break;
    case 5: launch_split<HD, 5>(grid, st, q, kn, vn, kc, vc, pos, po, pml, nh, nkv, max_len, nsplit, chunk, scale); break;
    case 6: launch_split<HD, 6>(grid, st, q, kn, vn, kc, vc, pos, po, pml, nh, nkv, max_len, nsplit, chunk, scale); break;
    case 7: launch_split<HD, 7>(grid, st, q, kn, vn, kc, vc, pos, po, pml, nh, nkv, max_len, nsplit, chunk, scale); break;
    default: launch_split<HD, 8>(grid, st, q, kn, vn, kc, vc, pos, po, pml, nh, nkv, max_len, nsplit, chunk, scale); break;
  }
}

bool al16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

size_t ws_bytes(int64_t B, int64_t nh, int64_t hd, int64_t nsplit) {
  const size_t o = (size_t)(B * nh * nsplit * hd) * sizeof(float);
  return ((o + 255) & ~(size_t)255) + (size_t)(B * nh * nsplit * 2) * sizeof(float);
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

extern "C" int quip_decode_attention(const void* q, const void* k_new, const void* v_new, void* k_cache, void* v_cache,
                                     const int64_t* positions, void* out, int32_t B, int32_t nh, int32_t nkv, int32_t hd,
                                     int32_t max_len, float scale, void* workspace, size_t workspace_bytes,
                                     void* stream) {
  QUIP_CHECK_ARG(q && k_new && v_new && k_cache && v_cache && positions && out && workspace,
                 "quip_decode_attention: null pointer");
  QUIP_CHECK_ARG(hd == 64 || hd == 128, "quip_decode_attention: head_dim %d is not 64 or 128", hd);
  QUIP_CHECK_ARG(B >= 0 && B <= 65535 && max_len > 0 && nkv > 0 && nkv <= 65535 && nh > 0,
                 "quip_decode_attention: bad sizes (B %d, nh %d, nkv %d, max_len %d)", B, nh, nkv, max_len);
  QUIP_CHECK_ARG(nh % nkv == 0 && nh / nkv <= AD_MAXG,
                 "quip_decode_attention: %d query heads on %d kv heads: nh %% nkv must be 0 with at most %d per kv head",
                 nh, nkv, AD_MAXG);
  QUIP_CHECK_ARG(al16(q) && al16(k_new) && al16(v_new) && al16(k_cache) && al16(v_cache) && al16(out) && al16(workspace),
                 "quip_decode_attention: pointers must be 16-byte aligned");
  const int chunk = (int64_t)B * nkv * ceil_div(max_len, AD_CHUNK) < AD_SMALL_GRID ? AD_SMALL_CHUNK : AD_CHUNK;
  const int nsplit = ceil_div(max_len, chunk);
  const size_t need = ws_bytes(B, nh, hd, nsplit);
  QUIP_CHECK_ARG(workspace_bytes >= need, "quip_decode_attention: workspace of %zu bytes, %zu needed", workspace_bytes, need);
  if (B == 0) return QUIP_OK;
  float* po = (float*)workspace;
  float* pml = (float*)((char*)workspace + (((size_t)B * nh * nsplit * hd * sizeof(float) + 255) & ~(size_t)255));
  const cudaStream_t st = (cudaStream_t)stream;
  const dim3 grid(nsplit, nkv, B);
  const int G = nh / nkv;
  if (hd == 64) launch_split_g<64>(G, grid, st, q, k_new, v_new, k_cache, v_cache, positions, po, pml, nh, nkv, max_len, nsplit, chunk, scale);
  else launch_split_g<128>(G, grid, st, q, k_new, v_new, k_cache, v_cache, positions, po, pml, nh, nkv, max_len, nsplit, chunk, scale);
  QUIP_LAUNCHED("attn_decode_split_kernel");
  attn_decode_combine_kernel<<<(unsigned)(B * nh), hd, 0, st>>>(po, pml, positions, (__half*)out, nh, hd, max_len, nsplit, chunk);
  QUIP_LAUNCHED("attn_decode_combine_kernel");
  return QUIP_OK;
}
