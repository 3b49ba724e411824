// Device helpers shared by the tensor-core kernels: mbarrier / TMA / wgmma PTX wrappers, the 128B-swizzle
// operand descriptor, and the packed-word -> fp16 operand-tile producer.
#pragma once
#include <cuda.h>

#include "common.cuh"

namespace quip {

constexpr int TC_BM = 128;            // output rows per tile: two consumer warpgroups of 64 (wgmma M)
constexpr int TC_BK = 64;             // k per stage = one 128-byte swizzle atom of fp16
constexpr int TC_PROD_GROUPS = 2;     // producer groups of 4 warps alternate k super-blocks
constexpr int TC_CONSUMER_WARPS = 8;  // warps 0-7: two consumer warpgroups (wgmma + epilogue)
constexpr int TC_THREADS = 32 * TC_CONSUMER_WARPS + 128 * TC_PROD_GROUPS + 32;   // + one TMA warp
constexpr uint32_t TC_WATCHDOG = 1u << 28;

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t addr = smem_u32(bar), done = 0, spins = 0;
  while (true) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done)
        : "r"(addr), "r"(parity)
        : "memory");
    if (done) break;
    if (++spins > TC_WATCHDOG) __trap();      // a protocol bug must not hang the GPU
  }
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// K-major, SWIZZLE_128B operand tile: rows of 128 bytes, 8-row groups 1024 bytes apart (sm_90 wgmma descriptor).
__device__ __forceinline__ uint64_t make_sw128_desc(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr & 0x3FFFFu) >> 4);        // start address, bits [0,14)
  d |= (uint64_t)1 << 16;                              // leading byte offset (unused for swizzled K-major)
  d |= (uint64_t)(1024 >> 4) << 32;                    // stride byte offset: 8 rows * 128 B
  d |= (uint64_t)1 << 62;                              // SWIZZLE_128B
  return d;
}

// D (registers, fp32, 64 x N per warpgroup) (+)= A[smem desc] (64 x 16) * B[smem desc]^T (N x 16), both K-major
template <int N>
__device__ __forceinline__ void wgmma_f16_ss(float (&d)[N / 2], uint64_t adesc, uint64_t bdesc, int scale_d);
template <>
__device__ __forceinline__ void wgmma_f16_ss<64>(float (&d)[32], uint64_t adesc, uint64_t bdesc, int scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
      "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, "
      "%32, %33, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(adesc), "l"(bdesc), "r"(scale_d));
}

template <>
__device__ __forceinline__ void wgmma_f16_ss<128>(float (&d)[64], uint64_t adesc, uint64_t bdesc, int scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
      "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, "
      "%64, %65, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(adesc), "l"(bdesc), "r"(scale_d));
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int PENDING>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(PENDING) : "memory"); }
// keeps the compiler from moving accumulator reads or writes across a wgmma fence / wait
template <int R>
__device__ __forceinline__ void wgmma_fence_regs(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// packed words one producer thread needs for one (row block, lane) over one k super-block (128 k)
template <int BITS>
struct TcWords {
  uint32_t w[BITS == 2 ? 4 : (BITS == 3 ? 6 : 8)];
};
template <int BITS>
__device__ __forceinline__ void tc_load_words(const uint32_t* __restrict__ sb, int l, TcWords<BITS>& r, bool valid) {
  if (!valid) {
#pragma unroll
    for (int i = 0; i < (int)(sizeof(r.w) / 4); ++i) r.w[i] = 0;
    return;
  }
  if constexpr (BITS == 2) {
    uint4 v = *reinterpret_cast<const uint4*>(sb + l * 4);
    r.w[0] = v.x; r.w[1] = v.y; r.w[2] = v.z; r.w[3] = v.w;
  } else if constexpr (BITS == 4) {
    uint4 a = *reinterpret_cast<const uint4*>(sb + l * 4), b = *reinterpret_cast<const uint4*>(sb + 128 + l * 4);
    r.w[0] = a.x; r.w[1] = a.y; r.w[2] = a.z; r.w[3] = a.w;
    r.w[4] = b.x; r.w[5] = b.y; r.w[6] = b.z; r.w[7] = b.w;
  } else {
    uint4 a = *reinterpret_cast<const uint4*>(sb + l * 4);
    uint2 b = *reinterpret_cast<const uint2*>(sb + 128 + l * 2);
    r.w[0] = a.x; r.w[1] = a.y; r.w[2] = a.z; r.w[3] = a.w;
    r.w[4] = b.x; r.w[5] = b.y;
  }
}
// expand chunk CH (0..3) of a super-block and store rows g / g+8 of row block `rbl` into the stage's A tile
template <int BITS, int CH>
__device__ __forceinline__ void tc_store_chunk(const TcWords<BITS>& r, uint32_t a_tile, int rbl, int g, int t,
                                               bool valid) {
  uint32_t h[8];
  if (valid) {
    if constexpr (BITS == 2) expand_chunk<2>(r.w[CH], 0u, h);
    else if constexpr (BITS == 4) expand_chunk<4>(r.w[2 * CH], r.w[2 * CH + 1], h);
    else expand_chunk<3, (CH & 1)>(r.w[CH], r.w[4 + (CH >> 1)], h);
  } else {
#pragma unroll
    for (int i = 0; i < 8; ++i) h[i] = 0;     // rows beyond N contribute exact zeros
  }
  const int cidx = (CH & 1) * 4 + t;          // 16-byte chunk inside the 128-byte row of this stage
  const uint32_t off = (uint32_t)(rbl * 16 + g) * 128u + (uint32_t)((cidx ^ g) << 4);
  asm volatile("st.shared.v4.b32 [%0], {%1,%2,%3,%4};" ::"r"(a_tile + off), "r"(h[0]), "r"(h[2]), "r"(h[4]), "r"(h[6])
               : "memory");
  asm volatile("st.shared.v4.b32 [%0], {%1,%2,%3,%4};" ::"r"(a_tile + off + 8u * 128u), "r"(h[1]), "r"(h[3]),
               "r"(h[5]), "r"(h[7])
               : "memory");
}


// Weight-producer loop of the packed GEMM.  Group `grp` (4 warps) expands the k
// super-blocks grp, grp+G, ... of every tile into stages 2*ksb and 2*ksb+1 of the global stage sequence.
// Two groups are needed because fence.proxy.async compiles to MEMBAR.ALL.CTA, which also waits for the
// thread's outstanding prefetch loads: with one group the ~1 us global-load latency would be exposed once
// per super-block; alternating groups give each load two super-block periods to land.
template <int BITS, int STAGES, int STAGE_BYTES, class RbBaseFn, class ArriveFn>
__device__ __forceinline__ void weight_producer_loop(int pw, int grp, int lane, const uint32_t* __restrict__ q, int KSB,
                                                     int N, uint64_t* empty, uint32_t smem_base, int first_tile,
                                                     int tile_step, int num_tiles, RbBaseFn rb_base_of,
                                                     ArriveFn arrive_full) {
  const int g = lane & 7, t = lane >> 3;         // 8 consecutive lanes = 8 rows g: conflict-free st.shared.v4
  const int l = 4 * g + t;                       // "lane" index of the native layout
  const int NRB = N >> 4;
  uint32_t it_base = 0;                          // stages consumed by earlier tiles
  const int rbl0 = pw, rbl1 = pw + 4;            // this thread serves row blocks pw and pw+4 of every tile
  TcWords<BITS> c0, c1, n0, n1;
  // the first super-block of a tile is fetched while the previous tile is still being expanded, so the
  // ~1 us global-load latency is not exposed at every tile boundary
  auto fetch_first = [&](int tile, TcWords<BITS>& a, TcWords<BITS>& b) {
    const bool in_range = tile < num_tiles && grp < KSB;
    const int rb_base = in_range ? rb_base_of(tile) : 0;
    tc_load_words<BITS>(q + ((int64_t)(rb_base + rbl0) * KSB + grp) * sb_words(BITS), l, a, in_range && rb_base + rbl0 < NRB);
    tc_load_words<BITS>(q + ((int64_t)(rb_base + rbl1) * KSB + grp) * sb_words(BITS), l, b, in_range && rb_base + rbl1 < NRB);
  };
  fetch_first(first_tile, c0, c1);
  for (int tile = first_tile; tile < num_tiles; tile += tile_step, it_base += 2u * (uint32_t)KSB) {
    const int rb_base = rb_base_of(tile);
    const bool v0 = rb_base + rbl0 < NRB, v1 = rb_base + rbl1 < NRB;
    const uint32_t* q0 = q + (int64_t)(rb_base + rbl0) * KSB * sb_words(BITS);
    const uint32_t* q1 = q + (int64_t)(rb_base + rbl1) * KSB * sb_words(BITS);
    for (int ksb = grp; ksb < KSB; ksb += TC_PROD_GROUPS) {
      const bool more = ksb + TC_PROD_GROUPS < KSB;
      if (more) {
        tc_load_words<BITS>(q0 + (int64_t)(ksb + TC_PROD_GROUPS) * sb_words(BITS), l, n0, v0);
        tc_load_words<BITS>(q1 + (int64_t)(ksb + TC_PROD_GROUPS) * sb_words(BITS), l, n1, v1);
      } else {
        fetch_first(tile + tile_step, n0, n1);
      }
#pragma unroll
      for (int half = 0; half < 2; ++half) {     // two 64-k stages per 128-k super-block
        const uint32_t it = it_base + 2u * (uint32_t)ksb + (uint32_t)half;
        const int s = (int)(it % (uint32_t)STAGES);
        const uint32_t ph = (it / (uint32_t)STAGES) & 1u;
        mbar_wait(&empty[s], ph ^ 1u);
        const uint32_t a_tile = smem_base + (uint32_t)(s * STAGE_BYTES);
        if (half == 0) {
          tc_store_chunk<BITS, 0>(c0, a_tile, rbl0, g, t, v0);
          tc_store_chunk<BITS, 1>(c0, a_tile, rbl0, g, t, v0);
          tc_store_chunk<BITS, 0>(c1, a_tile, rbl1, g, t, v1);
          tc_store_chunk<BITS, 1>(c1, a_tile, rbl1, g, t, v1);
        } else {
          tc_store_chunk<BITS, 2>(c0, a_tile, rbl0, g, t, v0);
          tc_store_chunk<BITS, 3>(c0, a_tile, rbl0, g, t, v0);
          tc_store_chunk<BITS, 2>(c1, a_tile, rbl1, g, t, v1);
          tc_store_chunk<BITS, 3>(c1, a_tile, rbl1, g, t, v1);
        }
        fence_proxy_async();                     // generic-proxy writes -> visible to the tensor core
        __syncwarp();
        if (lane == 0) arrive_full(s);
      }
      c0 = n0;
      c1 = n1;
    }
  }
}

}  // namespace quip
