// Packed-integer x fp16 GEMM on the Hopper tensor cores (wgmma + TMA), for many tokens
// (the reference's eval loop calls every Linear with M = 2048: opt.py:262-264, llama.py:226-227).
//
//   D[n][m] (registers, fp32) = sum_k A[n][k] * B[m][k]
//     A = packed weights, 128 output rows per tile.  The packed words of a k super-block are staged in shared
//         memory by TMA, and each consumer warp expands its own 16 rows to fp16 d=(c-cbar)/2^bits directly
//         into the wgmma A registers (the packed layout is the m16n8k16 A fragment with k relabelled, see
//         frag_natural), so A never exists as fp16 in shared memory or HBM;
//     B = activations x2 (M,K) fp16, BN tokens per tile, staged by TMA (cp.async.bulk.tensor, 128B
//         swizzle, out-of-bounds rows zero-filled so ragged M needs no special case);
//   epilogue: z[m][n] = P_n * D + R_n * xsum[m] (+ bias_n) -> fp16, transposed through shared memory so
//   that every store is 16 contiguous bytes of one token row.
//
// Warp roles (288 threads, one persistent CTA per SM, static tile schedule):
//   warps 0-7   two consumer warpgroups: warpgroup w issues wgmma.m64nBNk16 (A from registers, B from shared
//               memory) for rows 64w..64w+63 of the tile, then runs the epilogue of those rows
//   warp 8      TMA producer: activation tile of every 64-k stage, packed words of every 128-k super-block
// Pipeline: smem ring full[s]/empty[s] (TMA -> 8 consumer warps).  The TMA warp keeps filling the ring while the
// consumers run a tile's epilogue.  Per SM clock at full tensor rate the shared-memory traffic is the wgmma B reads
// (64 B) + the TMA writes of B (32 B) + the packed words (about 4 B), under the 128 B/clk the SM can serve.
// 2-bit tiles of 256 rows (RB = 2, when they alone fill every SM): each warpgroup owns 128 rows in two 64-row halves,
// so an activation tile fetched from L2 feeds twice the rows and the TMA writes of B per flop halve.  384 threads
// (warps 8-11 the producer warpgroup, registers moved to the consumers by setmaxnreg), 7-stage ring of 24 KB.
#include <type_traits>

#include "tc_common.cuh"

namespace quip {

constexpr int TC_SMEM_MAX = 227 * 1024;                      // opt-in dynamic shared memory per block

template <int BITS, int BN, bool DENSE, int RB = 1>
struct TcCfg {
  static constexpr int BM = TC_BM * RB;                        // weight rows (packed GEMM) or tokens (dense) per tile
  // A region of a stage: the fp16 A tile (dense), or the packed words of the tile's BM / 16 row blocks for one k
  // super-block (packed; written on even stages only, the odd stage of the same super-block reads its words from
  // registers (RB = 1) or from the even stage's slot (RB = 2))
  static constexpr int A_BYTES = DENSE ? BM * TC_BK * 2 : (BM / SB_ROWS) * sb_words(BITS) * 4;   // 16 / 4, 6, 8 KB (x RB)
  static constexpr int B_BYTES = BN * TC_BK * 2;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;        // multiple of 1024: B stays aligned for its swizzle
  // epilogue transpose buffer of one consumer warpgroup: BN token rows x 64 n (packed) or 64 token rows x BN
  // columns (dense), rows padded by 16 bytes against bank conflicts
  static constexpr int EPI_HALVES = BN * 72 > 64 * (BN + 8) ? BN * 72 : 64 * (BN + 8);
  static constexpr int EPI_BYTES = 2 * EPI_HALVES * 2;
  static constexpr int STAGES_FIT = (TC_SMEM_MAX - EPI_BYTES - 1024 - 256) / STAGE_BYTES;
  static constexpr int STAGES = STAGES_FIT < 16 ? STAGES_FIT : 16;       // 2 x 16 barriers fill the 256-byte area
  static constexpr size_t SMEM = (size_t)STAGES * STAGE_BYTES + 1024 /*align*/ + 256 /*barriers*/ + EPI_BYTES;
  static_assert(STAGE_BYTES % 1024 == 0 && 2 * STAGES * 8 <= 256, "stage layout");
  static_assert(RB == 1 || DENSE || BN == 128, "256-row packed tiles: BN = 128 only");
  static_assert(RB == 1 || STAGES >= 3, "256-row tiles: at least 3 stages in flight");
};

// DENSE = false: A is the packed matrix (N rows, K columns); its words are staged by TMA and expanded in registers.
// DENSE = true : block-diagonal pass with big blocks -- `nblk` independent GEMMs out_b = in_b . F_b^T, A = the
//                block's p contiguous activation columns (128 * RB tokens per tile), B = BN rows of the fp16 factor F_b
//                (N = K = p) fetched by TMA (3-D map, rows/cols beyond p zero-filled), output written to the same
//                columns.  RB = 2: each consumer warpgroup owns 128 tokens in two 64-token halves, so a factor tile
//                fetched from L2 feeds twice the tokens; BN is then sized to the block (dense_cols), not fixed at 128.
// tmap_a: packed words (DENSE = false; 2-D, one row of KSB * sb_words words per 16-row block) or the factors.
// RB: 64-row blocks per consumer warpgroup (packed GEMM).  RB = 2 makes 256-row tiles: warpgroup w owns rows
// 128w..128w+127 in two halves of 64 (one accumulator set each), and every activation tile fetched from L2 feeds
// twice the weight rows.  Each output element sees the same wgmma k16 steps in the same order and the same epilogue
// arithmetic as at RB = 1, so the two produce identical bits (dense pass: at any BN, too).
template <int BITS, int BN, bool DENSE, int RB = 1>
__global__ void __launch_bounds__(RB == 1 ? TC_THREADS : TC_THREADS_TALL, 1)
qgemm_tc_kernel(const __grid_constant__ CUtensorMap tmap_x, const __grid_constant__ CUtensorMap tmap_a,
                const float* __restrict__ scales, const float* __restrict__ zeros, const __half* __restrict__ bias,
                const float* __restrict__ xsum, __half* __restrict__ z, int M, int K, int N, int symmetric, int nblk,
                int shared_factor) {
  using C = TcCfg<BITS, BN, DENSE, RB>;
  extern __shared__ unsigned char smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  unsigned char* smem_gen = smem_raw + (smem_base - smem_u32(smem_raw));
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem_gen + (size_t)C::STAGES * C::STAGE_BYTES);
  uint64_t* full = bars;                       // [STAGES]
  uint64_t* empty = bars + C::STAGES;          // [STAGES]
  __half* epi = reinterpret_cast<__half*>(smem_gen + (size_t)C::STAGES * C::STAGE_BYTES + 256);   // 2 x EPI_HALVES

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // packed GEMM: 128 * RB output rows (wgmma M) x BN tokens (wgmma N).  DENSE pass: 128 * RB TOKENS (wgmma M) x BN
  // factor rows (wgmma N).
  const int tiles_n = DENSE ? (N + BN - 1) / BN : (N + C::BM - 1) / C::BM;
  const int tiles_m = DENSE ? (M + C::BM - 1) / C::BM : (M + BN - 1) / BN;
  const int per_blk = tiles_n * tiles_m;
  const int num_tiles = per_blk * nblk;
  const int KB = (K + TC_BK - 1) / TC_BK;
  const int64_t ldz = (int64_t)N * nblk;       // output row pitch (== N for the packed GEMM)
  constexpr int TMA_WARP = TC_CONSUMER_WARPS;

  if (warp == TMA_WARP && lane == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmap_x) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmap_a) : "memory");
    for (int s = 0; s < C::STAGES; ++s) {
      mbar_init(&full[s], 1);                  // TMA producer
      mbar_init(&empty[s], TC_CONSUMER_WARPS); // one arrival per consumer warp
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (RB == 1 ? warp == TMA_WARP : warp >= TMA_WARP) {
    // ================= TMA producer: activation tiles (+ packed words, one super-block per even stage) ==========
    // RB = 2: a whole producer warpgroup (warps 8-11, only warp 8 works) hands its registers to the consumers
    if constexpr (RB == 2) asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(TC_TALL_PRODUCER_REGS));
    if (lane == 0 && (RB == 1 || warp == TMA_WARP)) {
      int s = 0;
      uint32_t ph = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int blk = tile / per_blk, rr = tile % per_blk;
        const int m0 = (rr / tiles_n) * (DENSE ? C::BM : BN), n0 = (rr % tiles_n) * (DENSE ? BN : C::BM);
        for (int kb = 0; kb < KB; ++kb) {
          mbar_wait(&empty[s], ph ^ 1u);
          unsigned char* stage = smem_gen + (size_t)s * C::STAGE_BYTES;
          if (DENSE) {
            mbar_arrive_expect_tx(&full[s], C::STAGE_BYTES);
            tma_load_2d(stage, &tmap_x, &full[s], blk * K + kb * TC_BK, m0);                     // A: 128 * RB tokens
            tma_load_3d(stage + C::A_BYTES, &tmap_a, &full[s], kb * TC_BK, n0, shared_factor ? 0 : blk);   // B: BN factor rows
          } else {
            // row blocks beyond N are zero-filled; their output rows are never stored
            const bool words = (kb & 1) == 0;
            mbar_arrive_expect_tx(&full[s], C::B_BYTES + (words ? C::A_BYTES : 0));
            if (words) tma_load_2d(stage, &tmap_a, &full[s], (kb >> 1) * sb_words(BITS), n0 / SB_ROWS);
            tma_load_2d(stage + C::A_BYTES, &tmap_x, &full[s], kb * TC_BK, m0);
          }
          if (++s == C::STAGES) { s = 0; ph ^= 1u; }
        }
      }
    }
  } else {
    // ================= consumers: wgmma over the ring, then the epilogue of 64 * RB rows (dense: tokens) =========
    if constexpr (RB == 2) asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(TC_TALL_CONSUMER_REGS));
    const int wg = warp >> 2, wtid = threadIdx.x & 127;
    const int frow = (warp & 3) * 16 + (lane >> 2);        // accumulator row of d[j] for (j & 2) == 0; +8 otherwise
    const int fcol = (lane & 3) * 2;                       // accumulator column of d[j] is 8 * (j >> 2) + fcol + (j & 1)
    __half* eb = epi + wg * C::EPI_HALVES;
    float acc[RB][BN / 2];                                 // acc[hf]: rows 64 hf.. of the warpgroup's 64 * RB
#pragma unroll
    for (int j = 0; j < BN / 2; ++j) acc[0][j] = 0.f;
    int s = 0;
    uint32_t ph = 0;
    auto advance = [&]() { if (++s == C::STAGES) { s = 0; ph ^= 1u; } };
    auto release = [&](int st) {
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[st]);
    };
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      const int blk = tile / per_blk, rr = tile % per_blk;
      int prev = 0;
      // packed epilogue operands, fetched before the k loop so that their latency is hidden behind it: P_n, R_n,
      // bias_n of rows frow / frow + 8 of each half in registers, the tile's BN xsum values into L1
      const int n_base = (rr % tiles_n) * C::BM + wg * 64 * RB, m0 = (rr / tiles_n) * BN;
      float Pn[RB][2], Rn[RB][2], bn[RB][2];
      if constexpr (!DENSE) {
#pragma unroll
        for (int hf = 0; hf < RB; ++hf)
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int n = n_base + 64 * hf + frow + 8 * h;
            Pn[hf][h] = 1.f; Rn[hf][h] = 0.f; bn[hf][h] = 0.f;
            if (n < N) {
              const float sc = scales[n];
              Pn[hf][h] = sc * (float)(1 << BITS);
              if (!symmetric) Rn[hf][h] = sc * (0.5f * (float)((1 << BITS) - 1)) - zeros[n];
              if (bias) bn[hf][h] = __half2float(bias[n]);
            }
          }
        if (!symmetric && wtid < BN / 32 && m0 + 32 * wtid < M)
          asm volatile("prefetch.global.L1 [%0];" ::"l"(xsum + m0 + 32 * wtid));
      }
      if constexpr (DENSE) {
        for (int kb = 0; kb < KB; ++kb) {
          mbar_wait(&full[s], ph);
          const uint32_t a_addr = smem_base + (uint32_t)(s * C::STAGE_BYTES);
          const uint64_t bdesc = make_sw128_desc(a_addr + C::A_BYTES);
          wgmma_fence();
#pragma unroll
          for (int hf = 0; hf < RB; ++hf) {        // token rows 64 (RB wg + hf).. of the tile
            const uint64_t adesc = make_sw128_desc(a_addr + (uint32_t)((wg * RB + hf) * 64 * 128));
#pragma unroll
            for (int k = 0; k < TC_BK / 16; ++k)   // +32 bytes along K inside the swizzle atom = +2 encoded
              wgmma_f16_ss<BN>(acc[hf], adesc + (uint64_t)(2 * k), bdesc + (uint64_t)(2 * k), (kb | k) ? 1 : 0);
          }
          wgmma_commit();
          wgmma_wait<1>();                         // the previous stage's wgmma have read their operands
          if (kb > 0) release(prev);
          prev = s;
          advance();
        }
      } else if constexpr (RB == 1) {
        // Warp w owns row block w of the tile (rows 16w..16w+15 = the wgmma A rows of its warpgroup).  Each super-block
        // (two stages) is read from shared memory once, at its even stage; the A fragments of a stage are built while
        // the previous stage's wgmma run, into the other of two register sets (wgmma reads them asynchronously).
        const int g = lane >> 2, t = lane & 3;
        const uint32_t row_off = (uint32_t)(warp * sb_words(BITS) * 4);
        uint32_t w[row_words(BITS)];
        uint32_t fa[2][16];                        // A fragments of the even / odd stage: 4 k16 steps x a0..a3
        auto issue = [&](const uint32_t (&f)[16], int first) {
          const uint64_t bdesc = make_sw128_desc(smem_base + (uint32_t)(s * C::STAGE_BYTES) + C::A_BYTES);
          wgmma_fence();
#pragma unroll
          for (int k = 0; k < TC_BK / 16; ++k)
            wgmma_f16_rs<BN>(acc[0], &f[4 * k], bdesc + (uint64_t)(2 * k), (first && k == 0) ? 0 : 1);
          wgmma_commit();
        };
        auto load_words = [&]() {
          mbar_wait(&full[s], ph);
          tc_load_row_words<BITS>(smem_base + (uint32_t)(s * C::STAGE_BYTES) + row_off, g, w);
        };
        load_words();
        frag_natural<BITS, 0, 0>(w, t, &fa[0][0]);
        frag_natural<BITS, 0, 1>(w, t, &fa[0][4]);
        frag_natural<BITS, 1, 0>(w, t, &fa[0][8]);
        frag_natural<BITS, 1, 1>(w, t, &fa[0][12]);
        const int KSB = KB >> 1;
        for (int ksb = 0; ksb < KSB; ++ksb) {
          // even stage: chunks 0-1 of the super-block
          const int se = s;
          issue(fa[0], ksb == 0);
          wgmma_wait<1>();                         // the odd stage of the previous super-block is done with fa[1]
          if (ksb > 0) release(prev);
          advance();
          // odd stage: chunks 2-3, words already in registers
          mbar_wait(&full[s], ph);
          frag_natural<BITS, 2, 0>(w, t, &fa[1][0]);
          frag_natural<BITS, 2, 1>(w, t, &fa[1][4]);
          frag_natural<BITS, 3, 0>(w, t, &fa[1][8]);
          frag_natural<BITS, 3, 1>(w, t, &fa[1][12]);
          issue(fa[1], 0);
          wgmma_wait<1>();                         // the even stage is done with fa[0] and its shared memory
          release(se);
          prev = s;
          advance();
          if (ksb + 1 < KSB) {
            load_words();
            frag_natural<BITS, 0, 0>(w, t, &fa[0][0]);
            frag_natural<BITS, 0, 1>(w, t, &fa[0][4]);
            frag_natural<BITS, 1, 0>(w, t, &fa[0][8]);
            frag_natural<BITS, 1, 1>(w, t, &fa[0][12]);
          }
        }
      } else {
        // RB = 2: warp j of warpgroup w owns row blocks 8w + j (half 0) and 8w + 4 + j (half 1) of the tile's 16.  Per
        // stage the warpgroup issues one commit group per half (4 x k16 each, same B descriptor): the groups run
        // (even, half 0), (even, half 1), (odd, half 0), (odd, half 1).  Two fragment sets alternate between the groups
        // (set = half); a group's fragments are built while the previous group's wgmma run, one wgmma.wait_group 1
        // behind, from the words of one row block reloaded from the even stage's slot (16 registers, not 32).  The
        // even slot is released once the last group of the super-block has its fragments and both even groups are
        // done; the odd slot once its second group is.
        const int g = lane >> 2, t = lane & 3;
        const uint32_t row_off0 = (uint32_t)((wg * 8 + (warp & 3)) * sb_words(BITS) * 4);
        const uint32_t row_off1 = row_off0 + (uint32_t)(4 * sb_words(BITS) * 4);
        uint32_t w[row_words(BITS)];
        uint32_t fa[2][16];                        // A fragments of half 0 / half 1: 4 k16 steps x a0..a3
        auto issue = [&](const uint32_t (&f)[16], float (&d)[BN / 2], int first) {
          const uint64_t bdesc = make_sw128_desc(smem_base + (uint32_t)(s * C::STAGE_BYTES) + C::A_BYTES);
          wgmma_fence();
#pragma unroll
          for (int k = 0; k < TC_BK / 16; ++k)
            wgmma_f16_rs<BN>(d, &f[4 * k], bdesc + (uint64_t)(2 * k), (first && k == 0) ? 0 : 1);
          wgmma_commit();
        };
        // fragments of chunks 0-1 (ODD = false) or 2-3 (ODD = true) of one row block, words from the even slot se
        auto build = [&](auto odd, int se, uint32_t off, uint32_t (&f)[16]) {
          tc_load_row_words<BITS>(smem_base + (uint32_t)(se * C::STAGE_BYTES) + off, g, w);
          constexpr int c0 = decltype(odd)::value ? 2 : 0;
          frag_natural<BITS, c0, 0>(w, t, &f[0]);
          frag_natural<BITS, c0, 1>(w, t, &f[4]);
          frag_natural<BITS, c0 + 1, 0>(w, t, &f[8]);
          frag_natural<BITS, c0 + 1, 1>(w, t, &f[12]);
        };
        using Even = std::false_type;
        using Odd = std::true_type;
        mbar_wait(&full[s], ph);
        build(Even{}, s, row_off0, fa[0]);
        const int KSB = KB >> 1;
        for (int ksb = 0; ksb < KSB; ++ksb) {
          const int se = s;
          issue(fa[0], acc[0], ksb == 0);          // (even, half 0)
          wgmma_wait<1>();                         // the previous super-block's last group is done with fa[1], its slot
          if (ksb > 0) release(prev);
          build(Even{}, se, row_off1, fa[1]);
          issue(fa[1], acc[1], ksb == 0);          // (even, half 1)
          wgmma_wait<1>();                         // (even, half 0) is done with fa[0]
          build(Odd{}, se, row_off0, fa[0]);
          advance();
          mbar_wait(&full[s], ph);
          issue(fa[0], acc[0], 0);                 // (odd, half 0)
          wgmma_wait<1>();                         // (even, half 1) is done with fa[1]: both even groups are
          build(Odd{}, se, row_off1, fa[1]);
          release(se);                             // the even slot's activations and words are no longer read
          issue(fa[1], acc[1], 0);                 // (odd, half 1)
          wgmma_wait<1>();                         // (odd, half 0) is done with fa[0]
          prev = s;
          advance();
          if (ksb + 1 < KSB) {
            mbar_wait(&full[s], ph);
            build(Even{}, s, row_off0, fa[0]);
          }
        }
      }
      wgmma_wait<0>();
      wgmma_fence_regs(acc[0]);
      if constexpr (RB == 2) wgmma_fence_regs(acc[RB - 1]);
      release(prev);

      if constexpr (DENSE) {
        // eb[token row r][column c], pitch BN + 8; one 64-token half at a time
        constexpr int EP = BN + 8;
        const int i0 = (rr % tiles_n) * BN;
#pragma unroll
        for (int hf = 0; hf < RB; ++hf) {
#pragma unroll
          for (int j = 0; j < BN / 2; j += 2) {
            const int r = frow + ((j & 2) ? 8 : 0), c = 8 * (j >> 2) + fcol;
            *reinterpret_cast<__half2*>(&eb[r * EP + c]) = __floats2half2_rn(acc[hf][j], acc[hf][j + 1]);
          }
          asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory");
          const int m_base = (rr / tiles_n) * C::BM + (wg * RB + hf) * 64;
          for (int idx = wtid; idx < 64 * (BN / 8); idx += 128) {
            const int r = idx / (BN / 8), v = idx % (BN / 8);
            const int m = m_base + r, i = i0 + 8 * v;
            if (m < M && i < N)
              *reinterpret_cast<uint4*>(z + (int64_t)m * ldz + (int64_t)blk * N + i) =
                  *reinterpret_cast<const uint4*>(&eb[r * EP + 8 * v]);
          }
          if (hf + 1 < RB) asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory");   // eb is free for the next half
        }
      } else {
        // eb[token c][row r], pitch 72; one 64-row half at a time
        constexpr int EP = 72;
#pragma unroll
        for (int hf = 0; hf < RB; ++hf) {
#pragma unroll
          for (int j = 0; j < BN / 2; ++j) {
            const int h = (j >> 1) & 1, c = 8 * (j >> 2) + fcol + (j & 1), m = m0 + c;
            float v = Pn[hf][h] * acc[hf][j] + bn[hf][h];
            if (!symmetric) v += Rn[hf][h] * (m < M ? __ldg(&xsum[m]) : 0.f);
            eb[c * EP + frow + 8 * h] = __float2half_rn(v);
          }
          asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory");
          for (int idx = wtid; idx < BN * 8; idx += 128) {
            const int c = idx >> 3, v = idx & 7;
            const int m = m0 + c, n = n_base + 64 * hf + 8 * v;
            if (m < M && n < N)
              *reinterpret_cast<uint4*>(z + (int64_t)m * ldz + n) = *reinterpret_cast<const uint4*>(&eb[c * EP + 8 * v]);
          }
          if (hf + 1 < RB) asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory");   // eb is free for the next half
        }
      }
      asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory");   // eb is free for the next tile
    }
  }
}

// ---- host side ---------------------------------------------------------------------------------
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode() {
  static PFN_encodeTiled fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = (PFN_encodeTiled)p;
  }
  return fn;
}

static int g_num_sms = 0;

int num_sms() {
  if (!g_num_sms) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess ||
        cudaDeviceGetAttribute(&g_num_sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess)
      g_num_sms = 132;
  }
  return g_num_sms;
}

// activations (rows, cols) fp16 row-major -> 2-D map, box {64 cols, box_rows}, 128B swizzle, zero OOB fill
int make_act_map(CUtensorMap* tmap, const void* x, int64_t rows, int64_t cols, int box_rows) {
  PFN_encodeTiled enc = get_encode();
  if (!enc) {
    set_error("cuTensorMapEncodeTiled is not available from the driver");
    return QUIP_ERR_CUDA;
  }
  cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)cols * sizeof(__half)};
  cuuint32_t box[2] = {(cuuint32_t)TC_BK, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(tmap, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, (void*)x, dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed with CUresult %d (ptr=%p rows=%lld cols=%lld)", (int)r, x,
              (long long)rows, (long long)cols);
    return QUIP_ERR_CUDA;
  }
  return QUIP_OK;
}

// packed words -> 2-D map: one row of KSB * sb_words words per 16-row block, box {sb_words, rows / 16} = one k
// super-block of a tile's row blocks; row blocks beyond N are zero-filled
static int make_words_map(CUtensorMap* tmap, const QuipLinearDesc* d, int rows) {
  PFN_encodeTiled enc = get_encode();
  if (!enc) {
    set_error("cuTensorMapEncodeTiled is not available from the driver");
    return QUIP_ERR_CUDA;
  }
  const int sbw = sb_words(d->bits);
  cuuint64_t dims[2] = {(cuuint64_t)(d->K / SB_K) * sbw, (cuuint64_t)(d->N / SB_ROWS)};
  cuuint64_t strides[1] = {dims[0] * sizeof(uint32_t)};
  cuuint32_t box[2] = {(cuuint32_t)sbw, (cuuint32_t)(rows / SB_ROWS)};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(tmap, CU_TENSOR_MAP_DATA_TYPE_UINT32, 2, (void*)d->qweight, dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled (packed words) failed with CUresult %d (N=%d K=%d bits=%d)", (int)r, d->N, d->K,
              d->bits);
    return QUIP_ERR_CUDA;
  }
  return QUIP_OK;
}

template <int BITS, int BN, int RB = 1>
static int launch_tc(const QuipLinearDesc* d, const __half* x, const float* xsum, const __half* bias, __half* z,
                     int M, cudaStream_t s) {
  using C = TcCfg<BITS, BN, false, RB>;
  CUtensorMap tmx, tmq;
  if (int e = make_act_map(&tmx, x, M, d->K, BN)) return e;
  if (int e = make_words_map(&tmq, d, C::BM)) return e;
  auto kern = qgemm_tc_kernel<BITS, BN, false, RB>;
  QUIP_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)C::SMEM));
  int tiles = ceil_div(d->N, C::BM) * ceil_div(M, BN);
  int grid = tiles < num_sms() ? tiles : num_sms();
  kern<<<grid, RB == 1 ? TC_THREADS : TC_THREADS_TALL, C::SMEM, s>>>(tmx, tmq, d->scales, d->zeros, bias, xsum, z, M, d->K, d->N,
                                         (d->flags & QUIP_FLAG_SYMMETRIC) ? 1 : 0, 1, 0);
  QUIP_LAUNCHED("qgemm_tc_kernel");
  return QUIP_OK;
}

// block-diagonal pass with big contiguous blocks on the tensor cores (see DENSE in the kernel)
template <int BN, int RB = 1>
static int launch_tc_dense(const QuipPass* ps, const __half* in, __half* out, int M, int n, cudaStream_t s) {
  using C = TcCfg<2, BN, true, RB>;
  PFN_encodeTiled enc = get_encode();
  CUtensorMap tmx, tma;
  if (int e = make_act_map(&tmx, in, M, n, C::BM)) return e;       // 128 * RB tokens per tile (MMA M)
  const int p = ps->p;
  cuuint64_t dims[3] = {(cuuint64_t)p, (cuuint64_t)p, (cuuint64_t)(ps->shared ? 1 : ps->nblk)};
  cuuint64_t strides[2] = {(cuuint64_t)p * sizeof(__half), (cuuint64_t)p * p * sizeof(__half)};
  cuuint32_t box[3] = {(cuuint32_t)TC_BK, (cuuint32_t)BN, 1};       // BN factor rows per tile (MMA N)
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = enc(&tma, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 3, (void*)ps->factors, dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled (factors) failed with CUresult %d (p=%d nblk=%d)", (int)r, p, ps->nblk);
    return QUIP_ERR_CUDA;
  }
  auto kern = qgemm_tc_kernel<2, BN, true, RB>;
  QUIP_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)C::SMEM));
  int tiles = ceil_div(p, BN) * ceil_div(M, C::BM) * ps->nblk;
  int grid = tiles < num_sms() ? tiles : num_sms();
  kern<<<grid, RB == 1 ? TC_THREADS : TC_THREADS_TALL, C::SMEM, s>>>(tmx, tma, nullptr, nullptr, nullptr, nullptr, out, M,
                                                                     p, p, 1, ps->nblk, ps->shared ? 1 : 0);
  QUIP_LAUNCHED("qgemm_tc_kernel<dense>");
  return QUIP_OK;
}

// Tokens per tile of the dense pass (quip_config "dense_tile"): 0 = by shape (256 when the 256-token tiles alone fill
// every SM and their column width is instantiated, else 128), 128 or 256 = forced.
int g_dense_tile = 0;

// Factor columns per 256-token tile: the block split into ceil(p / 184) equal tiles, rounded up to 8 columns (688 ->
// 4 x 176).  At most 184 columns keeps the two 64-token halves' accumulators (2 x 92 per thread) within the consumers'
// 232 registers.
static int dense_cols(int p) { return 8 * ceil_div(p, 8 * ceil_div(p, 184)); }

int pass_big_tc(const QuipPass* ps, const __half* in, __half* out, int64_t M, int n, cudaStream_t s) {
  QUIP_CHECK_ARG(!ps->strided && ps->p % 8 == 0 && n % 8 == 0, "tensor-core pass needs contiguous blocks, p %% 8 == 0");
  QUIP_CHECK_ARG((((uintptr_t)in | (uintptr_t)out | (uintptr_t)ps->factors) & 15) == 0, "tensor-core pass: unaligned pointer");
  const int w = dense_cols(ps->p);
  // the widths of the supported models' blocks: 96, 128, 144, 160 (one tile), 224 -> 2 x 112, 448 -> 3 x 152, 688 -> 4 x 176
  const bool have = w == 96 || w == 112 || w == 128 || w == 144 || w == 152 || w == 160 || w == 176;
  bool tall = g_dense_tile == 256;
  if (g_dense_tile == 0)     // 256-token tiles halve the factor traffic from L2 per flop, but must fill every SM
    tall = have && (int64_t)ceil_div(ps->p, w) * ceil_div(M, (int64_t)2 * TC_BM) * ps->nblk >= num_sms();
  if (!tall) return launch_tc_dense<128>(ps, in, out, (int)M, n, s);
  switch (w) {
    case 96: return launch_tc_dense<96, 2>(ps, in, out, (int)M, n, s);
    case 112: return launch_tc_dense<112, 2>(ps, in, out, (int)M, n, s);
    case 128: return launch_tc_dense<128, 2>(ps, in, out, (int)M, n, s);
    case 144: return launch_tc_dense<144, 2>(ps, in, out, (int)M, n, s);
    case 152: return launch_tc_dense<152, 2>(ps, in, out, (int)M, n, s);
    case 160: return launch_tc_dense<160, 2>(ps, in, out, (int)M, n, s);
    case 176: return launch_tc_dense<176, 2>(ps, in, out, (int)M, n, s);
  }
  set_error("dense pass: no 256-token kernel for %d-column tiles (p=%d)", w, ps->p);
  return QUIP_ERR_UNSUPPORTED;
}

// Weight rows per tile of the 2-bit kernel above 64 tokens (quip_config "tc_rows"): 0 = by shape (256 when the
// 256-row tiles alone fill every SM, else 128), 128 or 256 = forced.  3- and 4-bit tiles are always 128 rows.
int g_tc_rows = 0;

int qgemm_tc(const QuipLinearDesc* d, const __half* x, const float* xsum, const __half* bias, __half* z, int M,
             cudaStream_t s) {
  QUIP_CHECK_ARG((((uintptr_t)x | (uintptr_t)d->qweight) & 15) == 0,
                 "tensor-core path needs 16-byte aligned activations and packed words");
  const bool wide = M > 64;
  if (d->bits == 2 && wide) {
    // 256-row tiles halve the activation traffic from L2 per flop, but at fewer tiles than SMs they leave SMs idle
    const bool tall = g_tc_rows == 0 ? ceil_div(d->N, 2 * TC_BM) * ceil_div(M, 128) >= num_sms() : g_tc_rows == 256;
    return tall ? launch_tc<2, 128, 2>(d, x, xsum, bias, z, M, s) : launch_tc<2, 128>(d, x, xsum, bias, z, M, s);
  }
#define QUIP_TC(B)                                                            \
  if (d->bits == B)                                                           \
    return wide ? launch_tc<B, 128>(d, x, xsum, bias, z, M, s) : launch_tc<B, 64>(d, x, xsum, bias, z, M, s);
  QUIP_TC(2) QUIP_TC(3) QUIP_TC(4)
#undef QUIP_TC
  set_error("tensor-core kernel: unsupported bits=%d", d->bits);
  return QUIP_ERR_UNSUPPORTED;
}

}  // namespace quip
