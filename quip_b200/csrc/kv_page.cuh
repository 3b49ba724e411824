// Where a cached slot lives: the contiguous KV cache (B, nkv, max_len, hd) or the paged one (include/quip_b200.h: a
// (n_pages, nkv, 64, hd) pool per layer behind page_table (B, max_pages) int32).  Every attention kernel walks the cache
// in 64-slot blocks aligned to 64, so a block lies in one page and a kernel looks up each page once per block.  One
// helper serves both layouts; the contiguous instantiation is the index arithmetic the kernels always had.
#pragma once
#include <stdint.h>

namespace quip {

constexpr int KV_PAGE = 64;   // slots per page

// The page table of a paged launch (unused by the contiguous one).
struct KvPages {
  const int32_t* table;       // (B, max_pages)
  int max_pages, n_pages;
};

// Head-vector index of slot j of (row b, kv head h) -- element offset index * hd, scale offset index -- or -1 when the
// slot's page id lies outside [0, n_pages) (paged only; such a page is never dereferenced).  Contiguous: max_len slots
// per (row, kv head).  Consecutive slots of one 64-slot block have consecutive indices in both layouts.
template <bool PAGED>
__device__ __forceinline__ int64_t kv_vec(const KvPages& pg, int64_t b, int h, int nkv, int max_len, int64_t j) {
  if constexpr (PAGED) {
    const int p = pg.table[b * pg.max_pages + (j >> 6)];
    return p >= 0 && p < pg.n_pages ? ((int64_t)p * nkv + h) * KV_PAGE + (j & (KV_PAGE - 1)) : -1;
  } else {
    return (b * nkv + h) * (int64_t)max_len + j;
  }
}

// The checks of a paged launch's table: 4-byte aligned, max_len = max_pages * 64 an int32, a non-empty pool.
inline bool pages_ok(const KvPages& pg) {
  return pg.table && (reinterpret_cast<uintptr_t>(pg.table) & 3) == 0 && pg.max_pages > 0 &&
         pg.max_pages <= INT32_MAX / KV_PAGE && pg.n_pages > 0;
}
// max_len of a paged launch; 1 for a max_pages that pages_ok refuses (the launch then fails on the table)
inline int32_t paged_len(int32_t max_pages) {
  return max_pages > 0 && max_pages <= INT32_MAX / KV_PAGE ? max_pages * KV_PAGE : 1;
}

}  // namespace quip
