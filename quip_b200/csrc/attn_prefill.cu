// Chunked prefill into the static KV cache of quip_b200/decode.py: many new tokens per row, each row at its own
// position, attending causally over the cache itself (one layer: k_cache / v_cache (B, nkv, max_len, hd), fp16 or e4m3
// with per-slot fp32 scales).  Two launches per layer:
//
//   quip_kv_append(_fp8)          token i < counts[b] of row b to slot positions[b] + i (e4m3: quantized on the way);
//   quip_prefill_attention(_fp8)  out[b][i][h] = softmax_j(scale * q[b][i][h] . K[b][h/G][j]) V[b][h/G][j],
//                                 j = 0 .. positions[b] + i, over the cache as the append left it.
//
// Appending first means no CTA of the attention writes what another one reads, and with an e4m3 cache the new tokens
// attend over their own quantized keys and values, which is what every later decode step reads back.
//
// Attention is flash-attention-2 style, no split-KV and no workspace.  CTA (query tile, kv head, row) owns 64 query
// rows r = i * G + g (token i, head g of the kv head), so every K / V byte staged serves the G heads that share it; warp
// w owns rows 16w .. 16w + 15 of the tile.  The tile walks the 64-slot KV blocks 0 .. (positions[b] + its last token) /
// 64 through a two-stage cp.async ring (block kb + 1 loads while block kb is multiplied); slots past the tile's last
// causal slot are zero-filled, never read.  S = Q.K^T and O = P.V run on mma.sync m16n8k16 (fp16 operands from ldmatrix,
// fp32 accumulation), Q held in registers, S and O in registers.  The softmax is online in fp32 (running max and sum per
// row); the causal mask is applied only on the blocks that reach past the tile's first token; P is rounded to fp16 once
// per block.  One fp16 rounding of the output.  Tiles are issued longest first (the last query tile has the most blocks).
//
// e4m3: each stage also holds the block's slot scales; the bytes are converted exactly to fp16 in shared memory after
// they land.  As in the extend kernel, a slot's k scale multiplies its score column, and s_v[j] / max s_v (the largest v
// scale among the row's visible slots of the block) is folded into p before its fp16 rounding; max s_v multiplies the
// block's P.V.  That factor rides on the accumulator: O is kept as O' * c with c the last block's max s_v, so adding a
// block rescales O' by alpha * c / max s_v once instead of keeping a second accumulator.
//
// Fixed orders everywhere: bit-identical from run to run; a row's result depends on its own q, cache and counts only.
#include <math.h>

#include <type_traits>

#include "common.cuh"
#include "kv_fp8.cuh"

namespace quip {

namespace {

constexpr int PF_BM = 64;        // query rows per CTA
constexpr int PF_BN = 64;        // KV slots per block
constexpr int PF_THREADS = 128;
constexpr int PF_STAGES = 2;
constexpr int PF_MAXG = 8;
constexpr int KA_WARPS = 8;      // head vectors per append CTA

template <bool FP8, int HD>
struct PfLayout {
  static constexpr int KS = HD + 8;                  // row stride (halves) of an fp16 K / V tile: conflict-free ldmatrix
  static constexpr int BS = HD + 16;                 // row stride (bytes) of an e4m3 K / V tile
  static constexpr size_t TILE16 = (size_t)PF_BN * KS * 2;
  static constexpr size_t TILE8 = (size_t)PF_BN * BS;
  // a stage: fp16 K, V; e4m3 K, V bytes and the k, v scales of the block's slots
  static constexpr size_t STAGE = FP8 ? 2 * TILE8 + 2 * PF_BN * sizeof(float) : 2 * TILE16;
  static constexpr size_t CONV = PF_STAGES * STAGE;  // e4m3: the block's K and V converted to fp16
  static constexpr size_t BYTES = CONV + (FP8 ? 2 * TILE16 : 0);
};

__device__ __forceinline__ void cp_async16(void* dst, const void* src, int bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_u32(dst)), "l"(src), "r"(bytes) : "memory");
}
__device__ __forceinline__ void cp_async4(void* dst, const void* src, int bytes) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(smem_u32(dst)), "l"(src), "r"(bytes) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

__device__ __forceinline__ void ldsm_x4(uint32_t (&r)[4], const void* p) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(smem_u32(p))
               : "memory");
}
__device__ __forceinline__ void ldsm_x4_trans(uint32_t (&r)[4], const void* p) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(smem_u32(p))
               : "memory");
}

__device__ __forceinline__ uint32_t f2_to_h2(float lo, float hi) {
  const __half2 h = __floats2half2_rn(lo, hi);
  return *reinterpret_cast<const uint32_t*>(&h);
}

// a row with positions / counts outside the cache or outside [0, T] is not looked at: no slot written, NaN outputs
__device__ __forceinline__ bool row_ok(int64_t pos, int64_t cnt, int T, int max_len) {
  return pos >= 0 && cnt >= 0 && cnt <= T && pos + cnt <= max_len;
}

// One warp per new head vector v = (b, i, h) of k_new / v_new (B, T, nkv, HD): slot positions[b] + i of both caches
// when i < counts[b].
template <bool FP8, int HD>
__global__ void __launch_bounds__(KA_WARPS * 32)
kv_append_kernel(const __half* __restrict__ k_new, const __half* __restrict__ v_new, void* __restrict__ kc,
                 void* __restrict__ vc, float* __restrict__ ksc, float* __restrict__ vsc,
                 const int64_t* __restrict__ positions, const int64_t* __restrict__ counts, int64_t nvec, int T, int nkv,
                 int max_len) {
  const int64_t v = (int64_t)blockIdx.x * KA_WARPS + threadIdx.x / 32;
  if (v >= nvec) return;                      // warp-uniform
  const int lane = threadIdx.x & 31;
  const int64_t b = v / ((int64_t)T * nkv);
  const int i = (int)(v / nkv % T), h = (int)(v % nkv);
  const int64_t pos = positions[b], cnt = counts[b];
  if (!row_ok(pos, cnt, T, max_len) || i >= cnt) return;
  const int64_t slot = (b * nkv + h) * max_len + pos + i;
  if constexpr (FP8) {
#pragma unroll
    for (int t = 0; t < 2; ++t) {
      float s;
      const uint32_t w = e4m3_quantize_warp<HD>((t ? v_new : k_new) + v * HD, lane, s);
      e4m3_store_warp<HD>(reinterpret_cast<uint8_t*>(t ? vc : kc) + slot * HD, lane, w);
      if (lane == 0) (t ? vsc : ksc)[slot] = s;
    }
  } else {
    constexpr int SEG = HD / 8;
    if (lane < 2 * SEG) {
      const int c = lane % SEG;
      const __half* src = (lane < SEG ? k_new : v_new) + v * HD;
      __half* dst = reinterpret_cast<__half*>(lane < SEG ? kc : vc) + slot * HD;
      reinterpret_cast<uint4*>(dst)[c] = reinterpret_cast<const uint4*>(src)[c];
    }
  }
}

template <bool FP8, int HD, int G>
__global__ void __launch_bounds__(PF_THREADS)
attn_prefill_kernel(const __half* __restrict__ q, const void* __restrict__ kc, const void* __restrict__ vc,
                    const float* __restrict__ ksc, const float* __restrict__ vsc, const int64_t* __restrict__ positions,
                    const int64_t* __restrict__ counts, __half* __restrict__ out, int T, int nh, int nkv, int max_len,
                    float scale) {
  using L = PfLayout<FP8, HD>;
  using CT = std::conditional_t<FP8, uint8_t, __half>;
  constexpr int KS = L::KS, BS = L::BS;
  constexpr int KT = HD / 16;                 // k16 steps of Q.K^T, n16 pairs of P.V
  constexpr int SEG = HD / 8;                 // 8-element segments of a head vector
  extern __shared__ __align__(16) unsigned char pf_smem[];

  const int tile = gridDim.x - 1 - blockIdx.x, kvh = blockIdx.y, b = blockIdx.z;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, gid = lane >> 2, tig = lane & 3;
  const int R = G * T, r_lo = tile * PF_BM;
  const int64_t pos = positions[b], cnt64 = counts[b];
  const bool ok = row_ok(pos, cnt64, T, max_len);
  const int cnt = ok ? (int)cnt64 : 0;
  const int i_lo = r_lo / G;                  // the tile's first token
  auto out_row = [&](int r) { return out + (((int64_t)b * T + r / G) * nh + (int64_t)kvh * G + r % G) * HD; };

  if (i_lo >= cnt) {                          // nothing to attend: zero rows (NaN for a row that is not looked at)
    const uint4 z = ok ? make_uint4(0, 0, 0, 0) : make_uint4(0x7E007E00u, 0x7E007E00u, 0x7E007E00u, 0x7E007E00u);
    for (int x = tid; x < PF_BM * SEG; x += PF_THREADS) {
      const int r = r_lo + x / SEG;
      if (r < R) reinterpret_cast<uint4*>(out_row(r))[x % SEG] = z;
    }
    return;
  }
  const int i_hi = min(min(r_lo + PF_BM - 1, R - 1) / G, cnt - 1);   // the tile's last token with an output
  const int64_t last = pos + i_hi;            // the last slot the tile reads
  const int64_t diag0 = pos + i_lo;           // blocks reaching past this slot need the mask
  const int nblk = (int)(last / PF_BN) + 1;

  const int64_t row = (int64_t)b * nkv + kvh;
  const CT* kr = reinterpret_cast<const CT*>(kc) + row * max_len * HD;
  const CT* vr = reinterpret_cast<const CT*>(vc) + row * max_len * HD;

  // the thread's two query rows (gid, gid + 8 of the warp's 16) and the last slot each sees
  int rr[2];
  int64_t lim[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    rr[h] = r_lo + warp * 16 + gid + 8 * h;
    lim[h] = pos + min(rr[h] / G, i_hi);
  }

  // Q fragments (A of m16n8k16) for every k16 step; rows past R or past the count are zero
  uint32_t qa[KT][4];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const bool live = rr[h] < R && rr[h] / G < cnt;
    const __half* qp = q + (((int64_t)b * T + rr[h] / G) * nh + (int64_t)kvh * G + rr[h] % G) * HD + 2 * tig;
#pragma unroll
    for (int kk = 0; kk < KT; ++kk) {
      qa[kk][h] = live ? __ldg(reinterpret_cast<const unsigned int*>(qp + 16 * kk)) : 0u;
      qa[kk][2 + h] = live ? __ldg(reinterpret_cast<const unsigned int*>(qp + 16 * kk + 8)) : 0u;
    }
  }

  auto load_block = [&](int kb, int st) {
    unsigned char* base = pf_smem + st * L::STAGE;
    const int64_t start = (int64_t)kb * PF_BN;
    if constexpr (FP8) {
      constexpr int S8 = HD / 16;             // 16-byte segments of an e4m3 head vector
      for (int x = tid; x < PF_BN * S8; x += PF_THREADS) {
        const int j = x / S8, c = x % S8;
        const bool in = start + j <= last;
        const int64_t off = (in ? start + j : 0) * HD + c * 16;
        cp_async16(base + j * BS + c * 16, kr + off, in ? 16 : 0);
        cp_async16(base + L::TILE8 + j * BS + c * 16, vr + off, in ? 16 : 0);
      }
      float* sc = reinterpret_cast<float*>(base + 2 * L::TILE8);
      const int j = tid % PF_BN;
      const bool in = start + j <= last;
      cp_async4(sc + tid, (tid < PF_BN ? ksc : vsc) + row * max_len + (in ? start + j : 0), in ? 4 : 0);
    } else {
      for (int x = tid; x < PF_BN * SEG; x += PF_THREADS) {
        const int j = x / SEG, c = x % SEG;
        const bool in = start + j <= last;
        const int64_t off = (in ? start + j : 0) * HD + c * 8;
        cp_async16(base + (j * KS + c * 8) * 2, kr + off, in ? 16 : 0);
        cp_async16(base + L::TILE16 + (j * KS + c * 8) * 2, vr + off, in ? 16 : 0);
      }
    }
  };

  float o[2 * KT][4];
#pragma unroll
  for (int n = 0; n < 2 * KT; ++n)
#pragma unroll
    for (int e = 0; e < 4; ++e) o[n][e] = 0.f;
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f}, c[2] = {1.f, 1.f};

  load_block(0, 0);
  cp_async_commit();
  for (int kb = 0; kb < nblk; ++kb) {
    const int st = kb & 1;
    if (kb + 1 < nblk) load_block(kb + 1, st ^ 1);
    cp_async_commit();
    cp_async_wait<1>();
    __syncthreads();

    const unsigned char* base = pf_smem + st * L::STAGE;
    const __half* sk;
    const __half* sv;
    const float* sks = nullptr;
    const float* svs = nullptr;
    if constexpr (FP8) {
      __half* k16 = reinterpret_cast<__half*>(pf_smem + L::CONV);
      __half* v16 = reinterpret_cast<__half*>(pf_smem + L::CONV + L::TILE16);
      for (int x = tid; x < PF_BN * SEG; x += PF_THREADS) {
        const int j = x / SEG, s = x % SEG;
        reinterpret_cast<uint4*>(k16 + j * KS)[s] = e4m3x8_to_h8(*reinterpret_cast<const uint2*>(base + j * BS + s * 8));
        reinterpret_cast<uint4*>(v16 + j * KS)[s] =
            e4m3x8_to_h8(*reinterpret_cast<const uint2*>(base + L::TILE8 + j * BS + s * 8));
      }
      sks = reinterpret_cast<const float*>(base + 2 * L::TILE8);
      svs = sks + PF_BN;
      __syncthreads();
      sk = k16;
      sv = v16;
    } else {
      sk = reinterpret_cast<const __half*>(base);
      sv = reinterpret_cast<const __half*>(base + L::TILE16);
    }
    const int64_t start = (int64_t)kb * PF_BN;
    const bool diag = start + PF_BN - 1 > diag0;

    // ---- S = Q.K^T over the block's 64 slots (16-slot groups past the tile's last slot stay 0: masked below)
    float s[8][4];
#pragma unroll
    for (int n = 0; n < 8; ++n)
#pragma unroll
      for (int e = 0; e < 4; ++e) s[n][e] = 0.f;
#pragma unroll
    for (int np = 0; np < 4; ++np) {
      if (start + 16 * np <= last) {
        const int mi = lane >> 3;
        const __half* kp = sk + (16 * np + (mi >> 1) * 8 + (lane & 7)) * KS + (mi & 1) * 8;
#pragma unroll
        for (int kk = 0; kk < KT; ++kk) {
          uint32_t r[4];
          ldsm_x4(r, kp + 16 * kk);
          const uint32_t b0[2] = {r[0], r[1]}, b1[2] = {r[2], r[3]};
          mma16816(s[2 * np], qa[kk], b0);
          mma16816(s[2 * np + 1], qa[kk], b1);
        }
      }
    }

    // ---- scale (e4m3: times the slot's k scale), causal mask on the diagonal blocks, online softmax
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float mx = -INFINITY;
#pragma unroll
      for (int n = 0; n < 8; ++n)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int j = 8 * n + 2 * tig + e;
          float x = s[n][2 * h + e] * scale;
          if constexpr (FP8) x = x * sks[j];
          if (diag && start + j > lim[h]) x = -INFINITY;
          s[n][2 * h + e] = x;
          mx = fmaxf(mx, x);
        }
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      const float mn = fmaxf(m[h], mx);       // finite: slot 0 (block 0) is visible to every row
      const float alpha = expf(m[h] - mn);
      m[h] = mn;
      float ps = 0.f;
#pragma unroll
      for (int n = 0; n < 8; ++n)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const float p = expf(s[n][2 * h + e] - mn);
          s[n][2 * h + e] = p;
          ps += p;
        }
      l[h] = l[h] * alpha + ps;
      float f = alpha;
      if constexpr (FP8) {                    // p is 0 at the slots the row does not see
        float sm = 0.f;
#pragma unroll
        for (int n = 0; n < 8; ++n)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int j = 8 * n + 2 * tig + e;
            if (start + j <= lim[h]) sm = fmaxf(sm, svs[j]);
          }
        sm = fmaxf(sm, __shfl_xor_sync(0xffffffffu, sm, 1));
        sm = fmaxf(sm, __shfl_xor_sync(0xffffffffu, sm, 2));
        if (sm > 0.f) {                       // a block the row sees none of leaves O' and c alone
          f = alpha * c[h] / sm;
          c[h] = sm;
          const float vnorm = 1.f / sm;
#pragma unroll
          for (int n = 0; n < 8; ++n)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const float p = s[n][2 * h + e];
              s[n][2 * h + e] = p > 0.f ? p * (svs[8 * n + 2 * tig + e] * vnorm) : 0.f;
            }
        }
      }
#pragma unroll
      for (int n = 0; n < 2 * KT; ++n) {
        o[n][2 * h] *= f;
        o[n][2 * h + 1] *= f;
      }
    }

    // ---- O += P.V: P (fp16) straight from the score registers
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      if (start + 16 * kk <= last) {
        const uint32_t a[4] = {f2_to_h2(s[2 * kk][0], s[2 * kk][1]), f2_to_h2(s[2 * kk][2], s[2 * kk][3]),
                               f2_to_h2(s[2 * kk + 1][0], s[2 * kk + 1][1]),
                               f2_to_h2(s[2 * kk + 1][2], s[2 * kk + 1][3])};
        const int mi = lane >> 3;
        const __half* vp = sv + (16 * kk + (mi & 1) * 8 + (lane & 7)) * KS + (mi >> 1) * 8;
#pragma unroll
        for (int np = 0; np < KT; ++np) {
          uint32_t r[4];
          ldsm_x4_trans(r, vp + 16 * np);
          const uint32_t b0[2] = {r[0], r[1]}, b1[2] = {r[2], r[3]};
          mma16816(o[2 * np], a, b0);
          mma16816(o[2 * np + 1], a, b1);
        }
      }
    }
    __syncthreads();                          // the stage (and the converted tiles) are free for the next loads
  }
  cp_async_wait<0>();

  // ---- epilogue: O / l (e4m3: O' * c / l), one fp16 rounding; rows past the count are zero
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    float sum = l[h];
    sum += __shfl_xor_sync(0xffffffffu, sum, 1);
    sum += __shfl_xor_sync(0xffffffffu, sum, 2);
    const int r = rr[h];
    if (r < R) {
      const bool live = r / G < cnt;
      __half* dst = out_row(r) + 2 * tig;
#pragma unroll
      for (int n = 0; n < 2 * KT; ++n) {
        float x0 = o[n][2 * h], x1 = o[n][2 * h + 1];
        if constexpr (FP8) {
          x0 *= c[h];
          x1 *= c[h];
        }
        *reinterpret_cast<uint32_t*>(dst + 8 * n) = live ? f2_to_h2(x0 / sum, x1 / sum) : 0u;
      }
    }
  }
}

bool al16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }
bool al4(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 3) == 0; }

template <bool FP8, int HD, int G>
int launch_prefill(dim3 grid, cudaStream_t st, const void* q, const void* kc, const void* vc, const float* ksc,
                   const float* vsc, const int64_t* pos, const int64_t* cnt, void* out, int T, int nh, int nkv,
                   int max_len, float scale) {
  constexpr size_t smem = PfLayout<FP8, HD>::BYTES;
  auto kern = attn_prefill_kernel<FP8, HD, G>;
  if (smem > 48 * 1024) QUIP_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  kern<<<grid, PF_THREADS, smem, st>>>((const __half*)q, kc, vc, ksc, vsc, pos, cnt, (__half*)out, T, nh, nkv, max_len,
                                       scale);
  QUIP_LAUNCHED("attn_prefill_kernel");
  return QUIP_OK;
}

template <bool FP8, int HD>
int launch_prefill_g(int G, dim3 grid, cudaStream_t st, const void* q, const void* kc, const void* vc, const float* ksc,
                     const float* vsc, const int64_t* pos, const int64_t* cnt, void* out, int T, int nh, int nkv,
                     int max_len, float scale) {
#define PF_LAUNCH(g) return launch_prefill<FP8, HD, g>(grid, st, q, kc, vc, ksc, vsc, pos, cnt, out, T, nh, nkv, max_len, scale)
  switch (G) {
    case 1: PF_LAUNCH(1);
    case 2: PF_LAUNCH(2);
    case 3: PF_LAUNCH(3);
    case 4: PF_LAUNCH(4);
    case 5: PF_LAUNCH(5);
    case 6: PF_LAUNCH(6);
    case 7: PF_LAUNCH(7);
    default: PF_LAUNCH(8);
  }
#undef PF_LAUNCH
}

// Argument checks and launches of quip_prefill_attention (FP8 false) and quip_prefill_attention_fp8 (FP8 true).
template <bool FP8>
int prefill_attention(const char* fn, const void* q, const void* k_cache, const void* v_cache, const float* k_scale,
                      const float* v_scale, const int64_t* positions, const int64_t* counts, void* out, int32_t B,
                      int32_t T, int32_t nh, int32_t nkv, int32_t hd, int32_t max_len, float scale, void* stream) {
  QUIP_CHECK_ARG(q && k_cache && v_cache && positions && counts && out && (!FP8 || (k_scale && v_scale)),
                 "%s: null pointer", fn);
  QUIP_CHECK_ARG(hd == 64 || hd == 128, "%s: head_dim %d is not 64 or 128", fn, hd);
  QUIP_CHECK_ARG(B >= 0 && B <= 65535 && max_len > 0 && nkv > 0 && nkv <= 65535 && nh > 0,
                 "%s: bad sizes (B %d, nh %d, nkv %d, max_len %d)", fn, B, nh, nkv, max_len);
  QUIP_CHECK_ARG(T >= 1 && T <= max_len, "%s: %d tokens per row: need 1 <= T <= max_len %d", fn, T, max_len);
  QUIP_CHECK_ARG(nh % nkv == 0 && nh / nkv <= PF_MAXG,
                 "%s: %d query heads on %d kv heads: nh %% nkv must be 0 with at most %d per kv head", fn, nh, nkv,
                 PF_MAXG);
  QUIP_CHECK_ARG(al16(q) && al16(k_cache) && al16(v_cache) && al16(out), "%s: pointers must be 16-byte aligned", fn);
  QUIP_CHECK_ARG(!FP8 || (al4(k_scale) && al4(v_scale)), "%s: scale pointers must be 4-byte aligned", fn);
  if (B == 0) return QUIP_OK;
  const int G = nh / nkv;
  const dim3 grid(ceil_div((int64_t)G * T, PF_BM), nkv, B);
  const cudaStream_t st = (cudaStream_t)stream;
  return hd == 64 ? launch_prefill_g<FP8, 64>(G, grid, st, q, k_cache, v_cache, k_scale, v_scale, positions, counts, out,
                                              T, nh, nkv, max_len, scale)
                  : launch_prefill_g<FP8, 128>(G, grid, st, q, k_cache, v_cache, k_scale, v_scale, positions, counts,
                                               out, T, nh, nkv, max_len, scale);
}

// Argument checks and launches of quip_kv_append (FP8 false) and quip_kv_append_fp8 (FP8 true).
template <bool FP8>
int kv_append(const char* fn, const void* k_new, const void* v_new, void* k_cache, void* v_cache, float* k_scale,
              float* v_scale, const int64_t* positions, const int64_t* counts, int32_t B, int32_t T, int32_t nkv,
              int32_t hd, int32_t max_len, void* stream) {
  QUIP_CHECK_ARG(k_new && v_new && k_cache && v_cache && positions && counts && (!FP8 || (k_scale && v_scale)),
                 "%s: null pointer", fn);
  QUIP_CHECK_ARG(hd == 64 || hd == 128, "%s: head_dim %d is not 64 or 128", fn, hd);
  QUIP_CHECK_ARG(B >= 0 && max_len > 0 && nkv > 0, "%s: bad sizes (B %d, nkv %d, max_len %d)", fn, B, nkv, max_len);
  QUIP_CHECK_ARG(T >= 1 && T <= max_len, "%s: %d tokens per row: need 1 <= T <= max_len %d", fn, T, max_len);
  QUIP_CHECK_ARG(al16(k_new) && al16(v_new) && al16(k_cache) && al16(v_cache), "%s: pointers must be 16-byte aligned",
                 fn);
  QUIP_CHECK_ARG(!FP8 || (al4(k_scale) && al4(v_scale)), "%s: scale pointers must be 4-byte aligned", fn);
  const int64_t nvec = (int64_t)B * T * nkv;
  if (nvec == 0) return QUIP_OK;
  const unsigned blocks = (unsigned)((nvec + KA_WARPS - 1) / KA_WARPS);
  const cudaStream_t st = (cudaStream_t)stream;
  const __half* kn = (const __half*)k_new;
  const __half* vn = (const __half*)v_new;
  if (hd == 64)
    kv_append_kernel<FP8, 64><<<blocks, KA_WARPS * 32, 0, st>>>(kn, vn, k_cache, v_cache, k_scale, v_scale, positions,
                                                                counts, nvec, T, nkv, max_len);
  else
    kv_append_kernel<FP8, 128><<<blocks, KA_WARPS * 32, 0, st>>>(kn, vn, k_cache, v_cache, k_scale, v_scale, positions,
                                                                 counts, nvec, T, nkv, max_len);
  QUIP_LAUNCHED("kv_append_kernel");
  return QUIP_OK;
}

}  // namespace

}  // namespace quip

using namespace quip;

extern "C" int quip_kv_append(const void* k_new, const void* v_new, void* k_cache, void* v_cache,
                              const int64_t* positions, const int64_t* counts, int32_t B, int32_t T, int32_t nkv,
                              int32_t hd, int32_t max_len, void* stream) {
  return kv_append<false>("quip_kv_append", k_new, v_new, k_cache, v_cache, nullptr, nullptr, positions, counts, B, T,
                          nkv, hd, max_len, stream);
}

extern "C" int quip_kv_append_fp8(const void* k_new, const void* v_new, void* k_cache, void* v_cache, float* k_scale,
                                  float* v_scale, const int64_t* positions, const int64_t* counts, int32_t B, int32_t T,
                                  int32_t nkv, int32_t hd, int32_t max_len, void* stream) {
  return kv_append<true>("quip_kv_append_fp8", k_new, v_new, k_cache, v_cache, k_scale, v_scale, positions, counts, B,
                         T, nkv, hd, max_len, stream);
}

extern "C" int quip_prefill_attention(const void* q, const void* k_cache, const void* v_cache, const int64_t* positions,
                                      const int64_t* counts, void* out, int32_t B, int32_t T, int32_t nh, int32_t nkv,
                                      int32_t hd, int32_t max_len, float scale, void* stream) {
  return prefill_attention<false>("quip_prefill_attention", q, k_cache, v_cache, nullptr, nullptr, positions, counts,
                                  out, B, T, nh, nkv, hd, max_len, scale, stream);
}

extern "C" int quip_prefill_attention_fp8(const void* q, const void* k_cache, const void* v_cache, const float* k_scale,
                                          const float* v_scale, const int64_t* positions, const int64_t* counts,
                                          void* out, int32_t B, int32_t T, int32_t nh, int32_t nkv, int32_t hd,
                                          int32_t max_len, float scale, void* stream) {
  return prefill_attention<true>("quip_prefill_attention_fp8", q, k_cache, v_cache, k_scale, v_scale, positions,
                                 counts, out, B, T, nh, nkv, hd, max_len, scale, stream);
}
