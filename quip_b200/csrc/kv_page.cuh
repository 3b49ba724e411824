// Where a cached slot lives: the contiguous KV cache (B, nkv, max_len, hd) or the paged one (include/quip_b200.h: a
// (n_pages, nkv, 64, hd) pool per layer behind page_table (B, max_pages) int32).  Every attention kernel walks the cache
// in 64-slot blocks aligned to 64, so a block lies in one page and a kernel looks up each page once per block.  One
// helper serves both layouts; the contiguous instantiation is the index arithmetic the kernels always had.  The entry
// points take a layer's cache as one QuipKvCache, which kv_check validates and resolves for the kernels.
#pragma once
#include <stdint.h>

#include <type_traits>

#include "common.cuh"

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

inline bool al16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }
inline bool al4(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 3) == 0; }

// The host check of a cache descriptor, shared by every entry point that takes one (fn names it in the messages).  On
// success pg is the page table (empty when contiguous) and max_len the slots per row the kernels take: the
// descriptor's max_len, or max_pages * 64 when paged.
inline int kv_check(const char* fn, const QuipKvCache* kv, KvPages& pg, int32_t& max_len) {
  QUIP_CHECK_ARG(kv, "%s: null cache descriptor", fn);
  QUIP_CHECK_ARG(kv->format == QUIP_KV_FP16 || kv->format == QUIP_KV_E4M3,
                 "%s: format %d is neither QUIP_KV_FP16 nor QUIP_KV_E4M3", fn, kv->format);
  const bool fp8 = kv->format == QUIP_KV_E4M3;
  QUIP_CHECK_ARG(kv->k && kv->v, "%s: null pointer (k / v)", fn);
  QUIP_CHECK_ARG(!fp8 || (kv->k_scale && kv->v_scale), "%s: null pointer (k_scale / v_scale of an e4m3 cache)", fn);
  QUIP_CHECK_ARG(fp8 || (!kv->k_scale && !kv->v_scale), "%s: k_scale / v_scale given for an fp16 cache", fn);
  QUIP_CHECK_ARG(al16(kv->k) && al16(kv->v), "%s: k and v must be 16-byte aligned", fn);
  QUIP_CHECK_ARG(!fp8 || (al4(kv->k_scale) && al4(kv->v_scale)), "%s: k_scale and v_scale must be 4-byte aligned", fn);
  QUIP_CHECK_ARG(kv->hd == 64 || kv->hd == 128, "%s: head_dim %d is not 64 or 128", fn, kv->hd);
  if (!kv->page_table) {
    pg = KvPages{};
    max_len = kv->max_len;
    return QUIP_OK;
  }
  pg = KvPages{kv->page_table, kv->max_pages, kv->n_pages};
  QUIP_CHECK_ARG(al4(pg.table) && pg.max_pages > 0 && pg.max_pages <= INT32_MAX / KV_PAGE && pg.n_pages > 0,
                 "%s: page_table must be 4-byte aligned, 0 < max_pages <= %d, n_pages > 0 (got %d, %d)", fn,
                 INT32_MAX / KV_PAGE, pg.max_pages, pg.n_pages);
  max_len = pg.max_pages * KV_PAGE;
  return QUIP_OK;
}

// Calls f(fp8, paged), two std::bool_constant tags, for the format and layout of a checked descriptor, so an entry
// point instantiates its host template once per cache kind.
template <class F>
int kv_dispatch(const QuipKvCache& kv, F&& f) {
  if (kv.format == QUIP_KV_E4M3)
    return kv.page_table ? f(std::true_type{}, std::true_type{}) : f(std::true_type{}, std::false_type{});
  return kv.page_table ? f(std::false_type{}, std::true_type{}) : f(std::false_type{}, std::false_type{});
}

}  // namespace quip
