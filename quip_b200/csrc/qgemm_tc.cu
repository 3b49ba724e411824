// Packed-integer x fp16 GEMM on the Hopper tensor cores (wgmma + TMA), for many tokens
// (the reference's eval loop calls every Linear with M = 2048: opt.py:262-264, llama.py:226-227).
//
//   D[n][m] (registers, fp32) = sum_k A[n][k] * B[m][k]
//     A = packed weights, 128 output rows per tile, expanded to fp16 d=(c-cbar)/2^bits by the
//         producer warps and written straight into the 128B-swizzled K-major operand layout
//         (generic-proxy st.shared + fence.proxy.async), never touching HBM as fp16;
//     B = activations x2 (M,K) fp16, BN tokens per tile, staged by TMA (cp.async.bulk.tensor, 128B
//         swizzle, out-of-bounds rows zero-filled so ragged M needs no special case);
//   epilogue: z[m][n] = P_n * D + R_n * xsum[m] (+ bias_n) -> fp16, transposed through shared memory so
//   that every store is 16 contiguous bytes of one token row.
//
// Warp roles (544 threads, one persistent CTA per SM, static tile schedule):
//   warps 0-7   two consumer warpgroups: warpgroup w issues wgmma.m64nBNk16 for rows 64w..64w+63 of the
//               tile, then runs the epilogue of those rows
//   warps 8-15  weight producers (2 groups of 4 alternating k super-blocks): 128-bit loads of packed
//               words -> registers -> fp16 -> smem
//   warp 16     TMA producer
// Pipeline: smem ring full[s]/empty[s] (TMA + 4 producer warps -> 8 consumer warps).  The producers keep
// filling the ring while the consumers run a tile's epilogue.
#include "tc_common.cuh"

namespace quip {

constexpr int TC_SMEM_MAX = 227 * 1024;                      // opt-in dynamic shared memory per block

template <int BN>
struct TcCfg {
  static constexpr int A_BYTES = TC_BM * TC_BK * 2;            // 16 KB
  static constexpr int B_BYTES = BN * TC_BK * 2;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  // epilogue transpose buffer of one consumer warpgroup: BN token rows x 64 n (packed) or 64 token rows x BN
  // columns (dense), rows padded by 16 bytes against bank conflicts
  static constexpr int EPI_HALVES = BN * 72 > 64 * (BN + 8) ? BN * 72 : 64 * (BN + 8);
  static constexpr int EPI_BYTES = 2 * EPI_HALVES * 2;
  static constexpr int STAGES = (TC_SMEM_MAX - EPI_BYTES - 1024 - 256) / STAGE_BYTES;   // 128 -> 5, 64 -> 8
  static constexpr size_t SMEM = (size_t)STAGES * STAGE_BYTES + 1024 /*align*/ + 256 /*barriers*/ + EPI_BYTES;
};

// DENSE = false: A is the packed matrix (N rows, K columns), expanded by the producer warps.
// DENSE = true : block-diagonal pass with big blocks -- `nblk` independent GEMMs out_b = in_b . F_b^T, A = the
//                block's p contiguous activation columns (128 tokens per tile), B = fp16 factor F_b (N = K = p)
//                fetched by TMA (3-D map, rows/cols beyond p zero-filled), output written to the same columns.
template <int BITS, int BN, bool DENSE>
__global__ void __launch_bounds__(TC_THREADS, 1)
qgemm_tc_kernel(const __grid_constant__ CUtensorMap tmap_x, const __grid_constant__ CUtensorMap tmap_a,
                const uint32_t* __restrict__ q, const float* __restrict__ scales, const float* __restrict__ zeros,
                const __half* __restrict__ bias, const float* __restrict__ xsum, __half* __restrict__ z, int M, int K,
                int N, int symmetric, int nblk, int shared_factor) {
  using C = TcCfg<BN>;
  extern __shared__ unsigned char smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  unsigned char* smem_gen = smem_raw + (smem_base - smem_u32(smem_raw));
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem_gen + (size_t)C::STAGES * C::STAGE_BYTES);
  uint64_t* full = bars;                       // [STAGES]
  uint64_t* empty = bars + C::STAGES;          // [STAGES]
  __half* epi = reinterpret_cast<__half*>(smem_gen + (size_t)C::STAGES * C::STAGE_BYTES + 256);   // 2 x EPI_HALVES

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // packed GEMM: 128 output rows (wgmma M) x BN tokens (wgmma N).  DENSE pass: 128 TOKENS (wgmma M) x BN factor
  // rows (wgmma N).
  const int tiles_n = DENSE ? (N + BN - 1) / BN : (N + TC_BM - 1) / TC_BM;
  const int tiles_m = DENSE ? (M + TC_BM - 1) / TC_BM : (M + BN - 1) / BN;
  const int per_blk = tiles_n * tiles_m;
  const int num_tiles = per_blk * nblk;
  const int KB = (K + TC_BK - 1) / TC_BK;
  const int KSB = K >> 7;
  const int64_t ldz = (int64_t)N * nblk;       // output row pitch (== N for the packed GEMM)
  constexpr int TMA_WARP = TC_CONSUMER_WARPS + 4 * TC_PROD_GROUPS;

  if (warp == TMA_WARP && lane == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmap_x) : "memory");
    if (DENSE) asm volatile("prefetch.tensormap [%0];" ::"l"(&tmap_a) : "memory");
    for (int s = 0; s < C::STAGES; ++s) {
      mbar_init(&full[s], DENSE ? 1 : 1 + 4);  // TMA producer (+ 4 weight-producer warps)
      mbar_init(&empty[s], TC_CONSUMER_WARPS); // one arrival per consumer warp
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp == TMA_WARP) {
    // ================= TMA producer: activation tiles =================
    if (lane == 0) {
      int s = 0;
      uint32_t ph = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int blk = tile / per_blk, rr = tile % per_blk;
        const int m0 = (rr / tiles_n) * (DENSE ? TC_BM : BN), n0 = (rr % tiles_n) * (DENSE ? BN : TC_BM);
        for (int kb = 0; kb < KB; ++kb) {
          mbar_wait(&empty[s], ph ^ 1u);
          mbar_arrive_expect_tx(&full[s], DENSE ? C::STAGE_BYTES : C::B_BYTES);
          unsigned char* stage = smem_gen + (size_t)s * C::STAGE_BYTES;
          if (DENSE) {
            tma_load_2d(stage, &tmap_x, &full[s], blk * K + kb * TC_BK, m0);                     // A: 128 tokens
            tma_load_3d(stage + C::A_BYTES, &tmap_a, &full[s], kb * TC_BK, n0, shared_factor ? 0 : blk);   // B: BN factor rows
          } else {
            tma_load_2d(stage + C::A_BYTES, &tmap_x, &full[s], kb * TC_BK, m0);
          }
          if (++s == C::STAGES) { s = 0; ph ^= 1u; }
        }
      }
    }
  } else if (warp < TC_CONSUMER_WARPS) {
    // ================= consumers: wgmma over the ring, then the epilogue of 64 rows =================
    const int wg = warp >> 2, wtid = threadIdx.x & 127;
    const int frow = (warp & 3) * 16 + (lane >> 2);        // accumulator row of d[j] for (j & 2) == 0; +8 otherwise
    const int fcol = (lane & 3) * 2;                       // accumulator column of d[j] is 8 * (j >> 2) + fcol + (j & 1)
    __half* eb = epi + wg * C::EPI_HALVES;
    float acc[BN / 2];
#pragma unroll
    for (int j = 0; j < BN / 2; ++j) acc[j] = 0.f;
    int s = 0;
    uint32_t ph = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      const int blk = tile / per_blk, rr = tile % per_blk;
      int prev = 0;
      for (int kb = 0; kb < KB; ++kb) {
        mbar_wait(&full[s], ph);
        const uint32_t a_addr = smem_base + (uint32_t)(s * C::STAGE_BYTES);
        const uint64_t adesc = make_sw128_desc(a_addr + (uint32_t)(wg * 64 * 128));
        const uint64_t bdesc = make_sw128_desc(a_addr + C::A_BYTES);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < TC_BK / 16; ++k)     // +32 bytes along K inside the swizzle atom = +2 encoded
          wgmma_f16_ss<BN>(acc, adesc + (uint64_t)(2 * k), bdesc + (uint64_t)(2 * k), (kb | k) ? 1 : 0);
        wgmma_commit();
        wgmma_wait<1>();                         // the previous stage's wgmma have read their operands
        if (kb > 0) {
          __syncwarp();
          if (lane == 0) mbar_arrive(&empty[prev]);
        }
        prev = s;
        if (++s == C::STAGES) { s = 0; ph ^= 1u; }
      }
      wgmma_wait<0>();
      wgmma_fence_regs(acc);
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[prev]);

      if constexpr (DENSE) {
        // eb[token row r][column c], pitch BN + 8
        constexpr int EP = BN + 8;
#pragma unroll
        for (int j = 0; j < BN / 2; j += 2) {
          const int r = frow + ((j & 2) ? 8 : 0), c = 8 * (j >> 2) + fcol;
          *reinterpret_cast<__half2*>(&eb[r * EP + c]) = __floats2half2_rn(acc[j], acc[j + 1]);
        }
        asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory");
        const int m_base = (rr / tiles_n) * TC_BM + wg * 64, i0 = (rr % tiles_n) * BN;
        for (int idx = wtid; idx < 64 * (BN / 8); idx += 128) {
          const int r = idx / (BN / 8), v = idx % (BN / 8);
          const int m = m_base + r, i = i0 + 8 * v;
          if (m < M && i < N)
            *reinterpret_cast<uint4*>(z + (int64_t)m * ldz + (int64_t)blk * N + i) =
                *reinterpret_cast<const uint4*>(&eb[r * EP + 8 * v]);
        }
      } else {
        // eb[token c][row r], pitch 72
        constexpr int EP = 72;
        const int n_base = (rr % tiles_n) * TC_BM + wg * 64, m0 = (rr / tiles_n) * BN;
        float Pn[2], Rn[2], bn[2];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int n = n_base + frow + 8 * h;
          Pn[h] = 1.f; Rn[h] = 0.f; bn[h] = 0.f;
          if (n < N) {
            const float sc = scales[n];
            Pn[h] = sc * (float)(1 << BITS);
            if (!symmetric) Rn[h] = sc * (0.5f * (float)((1 << BITS) - 1)) - zeros[n];
            if (bias) bn[h] = __half2float(bias[n]);
          }
        }
#pragma unroll
        for (int j = 0; j < BN / 2; ++j) {
          const int h = (j >> 1) & 1, c = 8 * (j >> 2) + fcol + (j & 1), m = m0 + c;
          float v = Pn[h] * acc[j] + bn[h];
          if (!symmetric) v += Rn[h] * (m < M ? __ldg(&xsum[m]) : 0.f);
          eb[c * EP + frow + 8 * h] = __float2half_rn(v);
        }
        asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory");
        for (int idx = wtid; idx < BN * 8; idx += 128) {
          const int c = idx >> 3, v = idx & 7;
          const int m = m0 + c, n = n_base + 8 * v;
          if (m < M && n < N)
            *reinterpret_cast<uint4*>(z + (int64_t)m * ldz + n) = *reinterpret_cast<const uint4*>(&eb[c * EP + 8 * v]);
        }
      }
      asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory");   // eb is free for the next tile
    }
  } else if (!DENSE) {
    // ================= weight producers: packed words -> fp16 operand tile =================
    const int pw = (warp - TC_CONSUMER_WARPS) & 3, grp = (warp - TC_CONSUMER_WARPS) >> 2;
    weight_producer_loop<BITS, C::STAGES, C::STAGE_BYTES>(
        pw, grp, lane, q, KSB, N, empty, smem_base, (int)blockIdx.x, (int)gridDim.x, num_tiles,
        [&](int tile) { return ((tile % per_blk) % tiles_n) * (TC_BM / 16); },
        [&](int s) { mbar_arrive(&full[s]); });
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

template <int BITS, int BN>
static int launch_tc(const QuipLinearDesc* d, const __half* x, const float* xsum, const __half* bias, __half* z,
                     int M, cudaStream_t s) {
  using C = TcCfg<BN>;
  CUtensorMap tmap;
  if (int e = make_act_map(&tmap, x, M, d->K, BN)) return e;
  auto kern = qgemm_tc_kernel<BITS, BN, false>;
  QUIP_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)C::SMEM));
  int tiles = ceil_div(d->N, TC_BM) * ceil_div(M, BN);
  int grid = tiles < num_sms() ? tiles : num_sms();
  kern<<<grid, TC_THREADS, C::SMEM, s>>>(tmap, tmap, reinterpret_cast<const uint32_t*>(d->qweight), d->scales, d->zeros,
                                         bias, xsum, z, M, d->K, d->N, (d->flags & QUIP_FLAG_SYMMETRIC) ? 1 : 0, 1, 0);
  QUIP_LAUNCHED("qgemm_tc_kernel");
  return QUIP_OK;
}

// block-diagonal pass with big contiguous blocks on the tensor cores (see DENSE in the kernel)
template <int BN>
static int launch_tc_dense(const QuipPass* ps, const __half* in, __half* out, int M, int n, cudaStream_t s) {
  using C = TcCfg<BN>;
  PFN_encodeTiled enc = get_encode();
  CUtensorMap tmx, tma;
  if (int e = make_act_map(&tmx, in, M, n, TC_BM)) return e;       // 128 tokens per tile (MMA M)
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
  auto kern = qgemm_tc_kernel<2, BN, true>;
  QUIP_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)C::SMEM));
  int tiles = ceil_div(p, BN) * ceil_div(M, TC_BM) * ps->nblk;
  int grid = tiles < num_sms() ? tiles : num_sms();
  kern<<<grid, TC_THREADS, C::SMEM, s>>>(tmx, tma, nullptr, nullptr, nullptr, nullptr, nullptr, out, M, p, p, 1,
                                         ps->nblk, ps->shared ? 1 : 0);
  QUIP_LAUNCHED("qgemm_tc_kernel<dense>");
  return QUIP_OK;
}

int pass_big_tc(const QuipPass* ps, const __half* in, __half* out, int64_t M, int n, cudaStream_t s) {
  QUIP_CHECK_ARG(!ps->strided && ps->p % 8 == 0 && n % 8 == 0, "tensor-core pass needs contiguous blocks, p %% 8 == 0");
  QUIP_CHECK_ARG((((uintptr_t)in | (uintptr_t)out | (uintptr_t)ps->factors) & 15) == 0, "tensor-core pass: unaligned pointer");
  return launch_tc_dense<128>(ps, in, out, (int)M, n, s);
}

int qgemm_tc(const QuipLinearDesc* d, const __half* x, const float* xsum, const __half* bias, __half* z, int M,
             cudaStream_t s) {
  QUIP_CHECK_ARG(((uintptr_t)x & 15) == 0, "tensor-core path needs 16-byte aligned activations");
  const bool wide = M > 64;
#define QUIP_TC(B)                                                            \
  if (d->bits == B)                                                           \
    return wide ? launch_tc<B, 128>(d, x, xsum, bias, z, M, s) : launch_tc<B, 64>(d, x, xsum, bias, z, M, s);
  QUIP_TC(2) QUIP_TC(3) QUIP_TC(4)
#undef QUIP_TC
  set_error("tensor-core kernel: unsupported bits=%d", d->bits);
  return QUIP_ERR_UNSUPPORTED;
}

}  // namespace quip
