// Shared helpers for the quip_b200 sm_90a kernels.
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include <atomic>

#include "../../include/quip_b200.h"

namespace quip {

// ---- error plumbing (thread-local message, C ABI returns codes) -------------
void set_error(const char* fmt, ...);
extern std::atomic<int64_t> g_launches;

#define QUIP_CHECK_ARG(cond, ...)            \
  do {                                       \
    if (!(cond)) {                           \
      quip::set_error(__VA_ARGS__);          \
      return QUIP_ERR_ARG;                   \
    }                                        \
  } while (0)

#define QUIP_CUDA(expr)                                                                  \
  do {                                                                                   \
    cudaError_t _e = (expr);                                                             \
    if (_e != cudaSuccess) {                                                             \
      quip::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__,  \
                      __LINE__);                                                         \
      return QUIP_ERR_CUDA;                                                              \
    }                                                                                    \
  } while (0)

// call right after a <<<>>> launch
#define QUIP_LAUNCHED(name)                                                                   \
  do {                                                                                        \
    quip::g_launches.fetch_add(1, std::memory_order_relaxed);                                 \
    cudaError_t _e = cudaPeekAtLastError();                                                   \
    if (_e != cudaSuccess) {                                                                  \
      cudaGetLastError();                                                                     \
      quip::set_error("launch of %s failed: %s", name, cudaGetErrorString(_e));               \
      return QUIP_ERR_CUDA;                                                                   \
    }                                                                                         \
  } while (0)

constexpr int SB_ROWS = 16;   // super-block: 16 rows x 128 k  (oracle/packing.py)
constexpr int SB_K = 128;
__host__ __device__ constexpr int sb_words(int bits) { return bits == 2 ? 128 : (bits == 3 ? 192 : 256); }

static inline int ceil_div(int64_t a, int64_t b) { return (int)((a + b - 1) / b); }

// ---- device helpers ---------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return (uint32_t)__cvta_generic_to_shared(p);
}

__device__ __forceinline__ uint4 ldg_nc_v4(const void* p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p));
  return r;
}
__device__ __forceinline__ uint2 ldg_nc_v2(const void* p) {
  uint2 r;
  asm volatile("ld.global.nc.L1::no_allocate.v2.u32 {%0,%1}, [%2];" : "=r"(r.x), "=r"(r.y) : "l"(p));
  return r;
}

// mma.sync m16n8k16, fp16 inputs, fp32 accumulate (legacy tensor path; used by the
// HBM-bound skinny kernel and the small block-diagonal rotation passes)
__device__ __forceinline__ void mma16816(float (&d)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, "
      "{%0,%1,%2,%3};"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}

// ---- code -> fp16 "d = (c - cbar) / 2^bits" expansion ------------------------------
// A pair of codes sits at bits [lo, lo+q) and [16+lo, 16+lo+q) of a word.  One shift moves
// them to the top of the two fp16 mantissas, one LOP3 masks and ORs the exponent of 1.0, so the
// halves read 1 + c/2^q; one HADD2 recentres.  (c - cbar)/2^q is exact in fp16 for q <= 4.
template <int BITS>
struct Dq {
  static constexpr uint32_t kMask = BITS == 2 ? 0x03000300u : (BITS == 3 ? 0x03800380u : 0x03C003C0u);
  static constexpr uint32_t kOne = 0x3C003C00u;
  // -(1 + cbar/2^bits): 2-bit -1.375, 3-bit -1.4375, 4-bit -1.46875
  static constexpr uint32_t kNegCenter = BITS == 2 ? 0xBD80BD80u : (BITS == 3 ? 0xBDC0BDC0u : 0xBDE0BDE0u);
};

__device__ __forceinline__ uint32_t hadd2_u32(uint32_t a, uint32_t b) {
  uint32_t r;
  asm("add.rn.f16x2 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b));
  return r;
}

// pair at field offset `lo` (compile-time) of a plane with Q bits per code, destination mantissa bit DST
template <int LO, int DST>
__device__ __forceinline__ uint32_t shift_to(uint32_t w) {
  if constexpr (LO < DST) return w << (DST - LO);
  else if constexpr (LO > DST) return w >> (LO - DST);
  else return w;
}

// 2-bit word (8 pairs j at bits 2j / 16+2j) -> pair j as fp16x2 of d
template <int J>
__device__ __forceinline__ uint32_t dq2(uint32_t w) {
  uint32_t v = (shift_to<2 * J, 8>(w) & Dq<2>::kMask) | Dq<2>::kOne;
  return hadd2_u32(v, Dq<2>::kNegCenter);
}
// 4-bit word (4 pairs j at bits 4j / 16+4j)
template <int J>
__device__ __forceinline__ uint32_t dq4(uint32_t w) {
  uint32_t v = (shift_to<4 * J, 6>(w) & Dq<4>::kMask) | Dq<4>::kOne;
  return hadd2_u32(v, Dq<4>::kNegCenter);
}
// 3-bit: hi word as 2-bit (pair J), lo word holds pair JJ at bits JJ / 16+JJ
template <int J, int JJ>
__device__ __forceinline__ uint32_t dq3(uint32_t whi, uint32_t wlo) {
  uint32_t v = (shift_to<2 * J, 8>(whi) & 0x03000300u) | Dq<3>::kOne;
  v |= shift_to<JJ, 7>(wlo) & 0x00800080u;
  return hadd2_u32(v, Dq<3>::kNegCenter);
}

// Bit layout of one (lane, chunk) word group: 16 codes = rows {g, g+8} x the lane's 8 consecutive k.
// Three consumers read the same bits, each with the cheapest extraction its datapath allows:
//   * IMMA.16832 (qgemv.cu, 1-5 tokens): the four A registers are  w & 0x03030303, w & 0x0C0C0C0C,
//     (w>>4) & 0x03030303, (w>>4) & 0x0C0C0C0C  -- byte j of the word holds "slot" j (bits 0-1 row g,
//     2-3 row g+8) and slot 4+j (bits 4-5, 6-7);
//   * HMMA.16816 / wgmma (fp16): a register is a pair of codes of one row at the same offset of the low
//     and high half-word -- slots (j, j+2) -- so slot s stands for k offset {0,2,1,3,4,6,5,7}[s] and every
//     fp16x2 register holds two consecutive k.
// In half-word terms: pair (u = pos/2, row half r) sits at bit 2*slot2(u,r) of each half.  4-bit: word
// pos/4, nibble slot4(u%2, r) of each half (byte j: low nibble row g, high nibble row g+8).
__host__ __device__ constexpr int slot2(int u, int r) { return 2 * ((u & 1) * 2 + (u >> 1)) + r; }
__host__ __device__ constexpr int slot4(int uw, int r) { return 2 * uw + r; }

// Expand one (lane, chunk): 16 codes -> 8 fp16x2 registers h[2u + r] (k pair u, row half r).
// MMA step s (k positions 4s..4s+3) uses a0..a3 = h[4s..4s+3].
// words: bits=2 -> w[0]; bits=4 -> w[0] (pos 0-3), w[1] (pos 4-7); bits=3 -> w[0] hi, w[1] lo with LOSEL
template <int BITS, int LOSEL = 0>
__device__ __forceinline__ void expand_chunk(uint32_t w0, uint32_t w1, uint32_t (&h)[8]) {
  if constexpr (BITS == 2) {
    h[0] = dq2<slot2(0, 0)>(w0); h[1] = dq2<slot2(0, 1)>(w0); h[2] = dq2<slot2(1, 0)>(w0); h[3] = dq2<slot2(1, 1)>(w0);
    h[4] = dq2<slot2(2, 0)>(w0); h[5] = dq2<slot2(2, 1)>(w0); h[6] = dq2<slot2(3, 0)>(w0); h[7] = dq2<slot2(3, 1)>(w0);
  } else if constexpr (BITS == 4) {
    h[0] = dq4<slot4(0, 0)>(w0); h[1] = dq4<slot4(0, 1)>(w0); h[2] = dq4<slot4(1, 0)>(w0); h[3] = dq4<slot4(1, 1)>(w0);
    h[4] = dq4<slot4(0, 0)>(w1); h[5] = dq4<slot4(0, 1)>(w1); h[6] = dq4<slot4(1, 0)>(w1); h[7] = dq4<slot4(1, 1)>(w1);
  } else {
    constexpr int B = 8 * LOSEL;
    h[0] = dq3<slot2(0, 0), B + slot2(0, 0)>(w0, w1); h[1] = dq3<slot2(0, 1), B + slot2(0, 1)>(w0, w1);
    h[2] = dq3<slot2(1, 0), B + slot2(1, 0)>(w0, w1); h[3] = dq3<slot2(1, 1), B + slot2(1, 1)>(w0, w1);
    h[4] = dq3<slot2(2, 0), B + slot2(2, 0)>(w0, w1); h[5] = dq3<slot2(2, 1), B + slot2(2, 1)>(w0, w1);
    h[6] = dq3<slot2(3, 0), B + slot2(3, 0)>(w0, w1); h[7] = dq3<slot2(3, 1), B + slot2(3, 1)>(w0, w1);
  }
}

// The A fragment of mma.sync m16n8k16 / wgmma m64nNk16 (per warp: 16 rows) in NATURAL k order, straight from the
// packed words.  Lane (g, t) needs, for k16 step S (0, 1) of chunk CH, rows g / g+8 (row half r = 0 / 1) at chunk k
//   a0 / a1: 16S + 2t, +1        a2 / a3: 16S + 8 + 2t, +1.
// In the native layout chunk k = 8t' + pos belongs to lane 4g + t' (same g), pos = 2u + e, so those are pair u = t of
// lanes 4g + 2S (a0, a1) and 4g + 2S + 1 (a2, a3): every fragment of a row group comes from the words of its lanes
// 4g..4g+3, held as RowWords w[row_words(BITS)]:
//   bits 2: w[4t' + ch]                      = word ch of lane 4g + t'          (super-block words 16g + [0,16))
//   bits 3: as bits 2 (hi plane), w[16 + 2t' + ch/2] = lo-plane word of lane 4g + t'   (words 128 + 8g + [0,8))
//   bits 4: w[16(ch/2) + 4t' + 2(ch%2) + pos/4]                                  (words 128(ch/2) + 16g + [0,16))
// Pair u = t of row half r sits at field slot2(t, r) = slot2(t, 0) + r (bits 4: word pos/4 = t/2, slot4(t%2, r)), so
// one runtime shift per word, by the lane's own field offset, moves row half 0 to field 0 and row half 1 to field 1;
// the compile-time dq helpers then finish as in expand_chunk.  The fp16 values are the ones expand_chunk makes.
__host__ __device__ constexpr int row_words(int bits) { return bits == 2 ? 16 : (bits == 3 ? 24 : 32); }

template <int BITS, int CH, int S>
__device__ __forceinline__ void frag_natural(const uint32_t (&w)[row_words(BITS)], int t, uint32_t* a) {
  if constexpr (BITS == 2 || BITS == 3) {
    const uint32_t sh = 2u * (uint32_t)slot2(t, 0);
    const uint32_t x0 = w[4 * (2 * S) + CH] >> sh, x1 = w[4 * (2 * S + 1) + CH] >> sh;
    if constexpr (BITS == 2) {
      a[0] = dq2<0>(x0); a[1] = dq2<1>(x0); a[2] = dq2<0>(x1); a[3] = dq2<1>(x1);
    } else {
      // lo plane: pair 8 (CH % 2) + slot of word CH / 2
      const uint32_t shl = 8u * (CH & 1) + (uint32_t)slot2(t, 0);
      const uint32_t y0 = w[16 + 2 * (2 * S) + (CH >> 1)] >> shl, y1 = w[16 + 2 * (2 * S + 1) + (CH >> 1)] >> shl;
      a[0] = dq3<0, 0>(x0, y0); a[1] = dq3<1, 1>(x0, y0); a[2] = dq3<0, 0>(x1, y1); a[3] = dq3<1, 1>(x1, y1);
    }
  } else {
    const uint32_t sh = 4u * (uint32_t)slot4(t & 1, 0);
    constexpr int i0 = 16 * (CH >> 1) + 4 * (2 * S) + 2 * (CH & 1), i1 = i0 + 4;
    const uint32_t x0 = ((t & 2) ? w[i0 + 1] : w[i0]) >> sh, x1 = ((t & 2) ? w[i1 + 1] : w[i1]) >> sh;
    a[0] = dq4<0>(x0); a[1] = dq4<1>(x0); a[2] = dq4<0>(x1); a[3] = dq4<1>(x1);
  }
}

}  // namespace quip
