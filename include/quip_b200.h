/*
 * quip_b200 -- C ABI of the H100-native packed QuantLinear path.
 *
 * This is the boundary the reference's FFI for this path would bind.  The
 * reference (Cornell-RelaxML/QuIP) has exactly one native call site on the
 * path, the absent `quant_cuda` extension:
 *
 *     quant_cuda.vecquant3matmul(x, qweight, y, scales, zeros)   quant.py:229-230
 *     quant_cuda.vecquant4matmul(x, qweight, y, scales, zeros)   zeroShot/models/quant.py:207-208
 *
 * i.e. "y += (scales*code - zeros) . x" on a packed-integer matrix, called from
 * Quant3Linear.forward (quant.py:222-233).  quip_qlinear_forward() replaces that
 * call and, in the same launch sequence, the work the reference folds into its
 * dense fp16 weight at quantization time (method.py:195-214): the scaleWH
 * rescale and the U / V incoherence un-projection.  quip_pack_codes() replaces
 * the CPU/numpy packer Quant3Linear.pack (quant.py:185-220, TODO at opt.py:302);
 * quip_convert_ref() reads the reference's own 3-/4-bit layouts.
 *
 * Conventions: plain pointers and sizes, no torch types.  All data pointers are
 * DEVICE pointers unless a parameter says "host"; the caller owns every buffer;
 * calls are asynchronous on the `stream` handle (a cudaStream_t cast to void*);
 * no internal allocation -- scratch comes from the caller-provided workspace.
 * Every function returns 0 on success and a non-zero code on error, with a
 * human-readable message available from quip_last_error() (thread-local).
 * There is no CPU fallback: on a machine without an sm_90 device the launch
 * entry points return QUIP_ERR_CUDA.
 */
#ifndef QUIP_B200_H_
#define QUIP_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define QUIP_ABI_VERSION 2

enum {
  QUIP_OK = 0,
  QUIP_ERR_ARG = 1,        /* bad shape / null pointer / unsupported bits */
  QUIP_ERR_WORKSPACE = 2,  /* workspace too small */
  QUIP_ERR_CUDA = 3,       /* CUDA runtime / driver error (message has the detail) */
  QUIP_ERR_UNSUPPORTED = 4
};

/* One block-diagonal pass of a butterfly (reference method.py:58-63).
 * A side of size n is viewed as nblk blocks of p elements; block b is
 * multiplied by its own (or the shared) p x p factor:
 *     out[pos(b,i)] = sum_j factors[b or 0][i][j] * in[pos(b,j)]
 * pos(b,j) = b*p + j (strided == 0) or j*nblk + b (strided == 1). */
typedef struct {
  int32_t p;
  int32_t nblk;
  int32_t strided;
  int32_t shared;          /* 1: a single factor for every block (method.py:38-39, "noblock") */
  const void* factors;     /* fp16 [shared ? 1 : nblk][p][p], row-major */
  const void* factors_frag;/* optional copy of the same factors in tensor-core fragment order, or NULL.  Only read by
                              the one-kernel sides of the many-token forward (p in {32, 64}); without it those sides run
                              as separate gather / pass kernels with the same result.  Word
                              (((blk*(p/8) + nt)*(p/32) + j)*32 + lane)*4 + q  holds  F[blk][8nt + lane/4][k0], [k0+1]
                              with k0 = 32j + 16(q/2) + 8(q%2) + 2(lane%4): one 128-bit load per lane is two k-steps
                              of mma.m16n8k16 B fragments. */
} QuipPass;

/* One incoherence side: V acts on the K input features, U on the N outputs.
 * n == 0 means the side is absent (no --pre_proj). */
typedef struct {
  int32_t n;
  int32_t npass;           /* 0..2 */
  QuipPass pass[2];        /* execution order */
  const int32_t* idx;      /* gather index, length n, or NULL for identity:
                              V: layout[l] = x[idx[l]] ; U: y[j] = layout[idx[j]] */
  const int32_t* inv_idx;  /* optional inverse of idx (inv_idx[idx[j]] = j), or NULL.  With it the few-token
                              forward (M <= 8) writes the last U pass straight to y (one launch fewer); the
                              result is the same without it. */
} QuipSide;

/* A packed linear layer  y = ((x * inv_scale) V^T) Q^T U + bias,
 * Q[n][k] = scales[n]*code[n][k] - zeros[n]  (Quant3Linear convention, quant.py:186-191).
 * qweight is in the native fragment-major layout (DESIGN.md, oracle/packing.py), rows
 * and columns already in the U / V layout order, scales/zeros in the same row order. */
typedef struct {
  int32_t K, N, bits;      /* bits in {2,3,4}; K % 128 == 0; N % 16 == 0 */
  int32_t flags;           /* QUIP_FLAG_* */
  const int32_t* qweight;
  const float* scales;     /* (N) */
  const float* zeros;      /* (N) */
  const void* bias;        /* fp16 (N) in output-feature order, or NULL */
  const float* inv_scale;  /* fp32 (K) = 1/scaleWH in input-feature order, or NULL */
  QuipSide V, U;
} QuipLinearDesc;

#define QUIP_FLAG_SYMMETRIC 1   /* scales*cbar == zeros for every row: the row-sum term vanishes (qfn 'b') */

/* y (M,N) fp16 = forward of x (M,K) fp16.  Replaces Quant3Linear.forward's
 * vecquant3matmul call (quant.py:222-233) for any M >= 1. */
int quip_qlinear_forward(const QuipLinearDesc* d, const void* x, void* y, int64_t M,
                         void* workspace, size_t workspace_bytes, void* stream);
int quip_qlinear_workspace_bytes(const QuipLinearDesc* d, int64_t M, size_t* out_bytes);

/* Building blocks (also exported for tests and micro-benchmarks). */
/* z (M,N) fp16 = x2 (M,K) fp16 contracted with the packed matrix + affine epilogue (+bias if given).
 * xsum (M) fp32 row sums of x2, required unless QUIP_FLAG_SYMMETRIC.  path: 0 auto, 1 few-token kernels (32-token
 * chunks; needs the workspace), 2 wgmma kernel. */
int quip_qgemm(const QuipLinearDesc* d, const void* x2, const float* xsum, const void* bias,
               void* z, int64_t M, int path, void* workspace, size_t workspace_bytes, void* stream);
int quip_rowsum(const void* x, float* xsum, int64_t M, int32_t K, void* stream);
/* out[m][l] = in[m][idx[l]] * scale[idx[l]] (+ bias[l]);  idx / scale / bias may be NULL. */
int quip_gather(const void* in, void* out, int64_t M, int32_t n, const int32_t* idx,
                const float* scale, const void* bias, void* stream);
/* impl: 0 auto, 1 generic CUDA-core kernel, 2 tensor-core kernels only */
int quip_rot_pass(const QuipPass* pass, const void* in, void* out, int64_t M, int32_t n, int impl,
                  void* stream);

/* Glue of a Llama decoder layer between its packed linears: what the reference's eval loop gets from the HF layer it
 * calls (llama.py:227 `layer(inps[j].unsqueeze(0), attention_mask=..., position_ids=...)`: LlamaRMSNorm, the residual
 * adds, apply_rotary_pos_emb, SiLU(gate)*up), each as one HBM pass with the HF modules' fp16 rounding points.  All
 * tensors fp16, contiguous, 16-byte aligned.
 *   quip_rmsnorm   s = x (+ residual);  y = weight * fp16(s * rsqrt(mean(s^2) + eps));  s is written to sum_out when
 *                  given (residual and sum_out may be NULL; sum_out may alias x or residual).  d % 8 == 0, d <= 32768.
 *   quip_rope      in place on q (rows, n_q_heads*head_dim) and k (rows, n_kv_heads*head_dim) with cos/sin
 *                  (rows, head_dim): out = x*cos + rotate_half(x)*sin.  head_dim % 16 == 0; k may be NULL with 0 heads.
 *   quip_silu_mul  out = silu(gate) * up over n elements (n % 8 == 0); out may alias gate or up. */
int quip_rmsnorm(const void* x, const void* residual, const void* weight, void* sum_out, void* y,
                 int64_t rows, int32_t d, float eps, void* stream);
int quip_rope(void* q, void* k, const void* cos, const void* sin, int64_t rows, int32_t n_q_heads,
              int32_t n_kv_heads, int32_t head_dim, void* stream);
int quip_silu_mul(const void* gate, const void* up, void* out, int64_t n, void* stream);
/*   quip_silu_mul_gather  the same product with the permutations of the surrounding incoherence sides folded in:
 *                  out[r][l] = silu(gate[r][idx[l] & 0xFFFF]) * up[r][idx[l] >> 16] for rows of n < 65536 features; gate / up
 *                  are the projections in their N-side layout order (quip_qlinear_forward with U.idx = NULL), out feeds a
 *                  forward with V.idx = NULL: idx[l] = u_idx_gate[v_idx_down[l]] | u_idx_up[v_idx_down[l]] << 16. */
int quip_silu_mul_gather(const void* gate, const void* up, const uint32_t* idx, void* out, int64_t rows, int32_t n,
                         void* stream);

/* One decode-attention step for B sequences, each at its own position, on one layer of the static KV cache.
 *   q (B, nh, hd) fp16 with rotary applied; k_new / v_new (B, nkv, hd) fp16: this step's key / value;
 *   k_cache / v_cache (B, nkv, max_len, hd) fp16; positions (B) int64 on the device; out (B, nh, hd) fp16.
 * Writes k_new / v_new at slot positions[b] and returns
 *   out[b][h] = softmax_j(scale * q[b][h] . k[b][h / G][j]) v[b][h / G][j],  j = 0 .. positions[b],  G = nh / nkv,
 * reading no slot past positions[b].  fp32 scores, softmax and P.V; one fp16 rounding of the output.  The launch grid
 * depends on (B, nkv, max_len) only, so one captured graph serves every position.  hd in {64, 128}, nh % nkv == 0,
 * nh / nkv <= 8; all pointers 16-byte aligned; fp32 scratch from quip_decode_attention_workspace_bytes.  A position
 * outside [0, max_len) leaves the cache untouched and gives a NaN output row.  Deterministic: bit-identical results from
 * run to run and for every other content of the other rows. */
int quip_decode_attention(const void* q, const void* k_new, const void* v_new, void* k_cache, void* v_cache,
                          const int64_t* positions, void* out, int32_t B, int32_t nh, int32_t nkv, int32_t hd,
                          int32_t max_len, float scale, void* workspace, size_t workspace_bytes, void* stream);
int quip_decode_attention_workspace_bytes(int32_t B, int32_t nh, int32_t hd, int32_t max_len, size_t* out_bytes);

/* The same step on an e4m3 KV cache: k_cache / v_cache (B, nkv, max_len, hd) e4m3fn bytes, k_scale / v_scale
 * (B, nkv, max_len) fp32, one scale per cached head vector x (hd values):
 *   amax = max_i |x_i|;  s = amax / 448 (IEEE fp32 division; s = 1 when amax == 0);  q_i = e4m3fn(x_i / s), round to
 *   nearest even, subnormals kept;  the vector's value is float(q_i) * s.
 * k_new / v_new (fp16) are quantized so, written with their scales at slot positions[b], and attended over as quantized
 * values like every other slot 0 .. positions[b].  No slot or scale past positions[b] is read.  Same grid, workspace
 * (quip_decode_attention_workspace_bytes) and determinism as quip_decode_attention; the scale pointers 4-byte aligned.
 * Non-finite inputs may give a NaN output row. */
int quip_decode_attention_fp8(const void* q, const void* k_new, const void* v_new, void* k_cache, void* v_cache,
                              float* k_scale, float* v_scale, const int64_t* positions, void* out, int32_t B,
                              int32_t nh, int32_t nkv, int32_t hd, int32_t max_len, float scale, void* workspace,
                              size_t workspace_bytes, void* stream);
/* One attention step with T new tokens per row (speculative verification), each row at its own position, on one layer
 * of the static KV cache.  q (B, T, nh, hd) fp16 token-major, rotary applied; k_new / v_new (B, T, nkv, hd) fp16;
 * caches (B, nkv, max_len, hd); positions (B) int64 on the device; out (B, T, nh, hd) fp16.  Token i of row b is written
 * at slot positions[b] + i, and
 *   out[b][i][h] = softmax_j(scale * q[b][i][h] . k[b][h / G][j]) v[b][h / G][j],  j = 0 .. positions[b] + i,
 * causal inside the new tokens.  No slot past positions[b] + T - 1 is read.  Scores and softmax in fp32; Q.K^T and P.V
 * on tensor cores (fp16 operands, fp32 accumulation; p rounded once to fp16); one fp16 rounding of the output.  1 <= T
 * <= 8, hd in {64, 128}, nh % nkv == 0, nh / nkv <= 8; pointers 16-byte aligned; fp32 scratch from
 * quip_extend_attention_workspace_bytes.  The grid depends on (B, T, nkv, max_len) only.  A row with positions[b] < 0
 * or positions[b] + T > max_len writes nothing and gets NaN outputs.  Deterministic, and a row's result does not depend
 * on the other rows.  T = 1 computes what quip_decode_attention does, to within its rounding of p. */
int quip_extend_attention(const void* q, const void* k_new, const void* v_new, void* k_cache, void* v_cache,
                          const int64_t* positions, void* out, int32_t B, int32_t T, int32_t nh, int32_t nkv, int32_t hd,
                          int32_t max_len, float scale, void* workspace, size_t workspace_bytes, void* stream);
int quip_extend_attention_workspace_bytes(int32_t B, int32_t T, int32_t nh, int32_t hd, int32_t max_len,
                                          size_t* out_bytes);
/* The same on an e4m3 cache with per-slot scales (the format of quip_decode_attention_fp8): the new keys and values are
 * quantized on append and attended over as quantized values.  A slot's k scale multiplies its score column; its v scale
 * multiplies p before p is rounded to fp16 (normalised by the chunk's largest v scale, which multiplies the chunk's
 * P.V). */
int quip_extend_attention_fp8(const void* q, const void* k_new, const void* v_new, void* k_cache, void* v_cache,
                              float* k_scale, float* v_scale, const int64_t* positions, void* out, int32_t B, int32_t T,
                              int32_t nh, int32_t nkv, int32_t hd, int32_t max_len, float scale, void* workspace,
                              size_t workspace_bytes, void* stream);

/* Prompt-lookup drafts.  hist (B, max_len) int64 holds each row's tokens by position; the current token is at
 * c = positions[b].  For e < c let L(e) be the length of the common suffix of hist[b, ..e] and hist[b, ..c], capped at
 * n_max.  The match is the e with the largest L(e) >= n_min, the largest such e on ties (longest n-gram first, then the
 * most recent).  tokens (B, 1 + k): column 0 is hist[b, c]; the drafts d_i = u[e + i], i = 1..k, with u = hist[b, 0..c]
 * followed by d itself (an overlapping copy, so a period shorter than k still fills k drafts).  No match: every d_i is
 * the current token.  A row with c outside [0, max_len) gets zeros.  1 <= n_min <= n_max; O(c * n_max) reads. */
int quip_ngram_draft(const int64_t* hist, const int64_t* positions, int64_t* tokens, int32_t B, int32_t max_len,
                     int32_t k, int32_t n_min, int32_t n_max, void* stream);
/* Acceptance of a verified speculative step.  tokens (B, T) are the step's inputs (the current token, then T - 1 drafts),
 * targets (B, T) the tokens selected from the step's logits.  For each row with n_gen[b] < max_new: a = the length of the
 * longest prefix with tokens[b][i] == targets[b][i - 1] (i = 1 ..); e = min(a + 1, max_new - n_gen[b]); targets[b][0 ..
 * e-1] are written to generated[b][n_gen ..] (rows of gen_cols >= max_new) and hist[b][positions + 1 ..] (slots below
 * max_len); positions and n_gen advance by e, accepted by e - 1.  Finished rows are left alone. */
int quip_spec_accept(const int64_t* tokens, const int64_t* targets, int64_t* generated, int64_t* hist,
                     int64_t* positions, int64_t* n_gen, int64_t* accepted, int32_t B, int32_t T, int32_t max_new,
                     int32_t gen_cols, int32_t max_len, void* stream);

/* Prefill of an e4m3 cache: src (B, nkv, P, hd) fp16 quantized as above into slots 0 .. P-1 of cache
 * (B, nkv, max_len, hd) e4m3fn and scales (B, nkv, max_len) fp32; slots >= P are not touched.  hd in {64, 128},
 * P <= max_len; src and cache 16-byte aligned, scales 4-byte aligned. */
int quip_kv_quantize_fp8(const void* src, void* cache, float* scales, int32_t B, int32_t nkv, int32_t P,
                         int32_t max_len, int32_t hd, void* stream);

/* Chunked prefill, part 1: append a chunk of new keys and values to one layer of the static KV cache.  k_new / v_new
 * (B, T, nkv, hd) fp16 token-major; caches (B, nkv, max_len, hd) fp16; positions, counts (B) int64 on the device.  Token
 * i of row b goes to slot positions[b] + i for i < counts[b]; no other slot, and nothing of a row with counts[b] == 0, is
 * touched.  A row with positions[b] < 0, counts[b] outside [0, T] or positions[b] + counts[b] > max_len writes nothing.
 * 1 <= T <= max_len, hd in {64, 128}; pointers 16-byte aligned. */
int quip_kv_append(const void* k_new, const void* v_new, void* k_cache, void* v_cache, const int64_t* positions,
                   const int64_t* counts, int32_t B, int32_t T, int32_t nkv, int32_t hd, int32_t max_len, void* stream);
/* The same into an e4m3 cache: each new head vector is quantized by the rule of quip_decode_attention_fp8 (amax / 448,
 * round to nearest even, subnormals kept) and stored with its fp32 scale in k_scale / v_scale (B, nkv, max_len). */
int quip_kv_append_fp8(const void* k_new, const void* v_new, void* k_cache, void* v_cache, float* k_scale,
                       float* v_scale, const int64_t* positions, const int64_t* counts, int32_t B, int32_t T,
                       int32_t nkv, int32_t hd, int32_t max_len, void* stream);
/* Chunked prefill, part 2: causal attention of a chunk of T query tokens per row over the cache that already holds the
 * chunk (quip_kv_append first).  q (B, T, nh, hd) fp16 token-major, rotary applied; out (B, T, nh, hd) fp16.  For
 * i < counts[b]
 *   out[b][i][h] = softmax_j(scale * q[b][i][h] . k[b][h / G][j]) v[b][h / G][j],  j = 0 .. positions[b] + i,
 * and out[b][i] = 0 for counts[b] <= i < T.  No slot past positions[b] + counts[b] - 1 is read.  Flash-attention style:
 * Q.K^T and P.V on tensor cores (fp16 operands, fp32 accumulation), online softmax in fp32, p rounded once to fp16 per
 * 64-slot block, one fp16 rounding of the output; no workspace.  1 <= T <= max_len, hd in {64, 128}, nh % nkv == 0,
 * nh / nkv <= 8; pointers 16-byte aligned.  A row with positions[b] < 0, counts[b] outside [0, T] or positions[b] +
 * counts[b] > max_len gets NaN outputs.  Deterministic, and a row's result does not depend on the other rows.  At T <= 8
 * it computes what quip_extend_attention does, to within the rounding of p. */
int quip_prefill_attention(const void* q, const void* k_cache, const void* v_cache, const int64_t* positions,
                           const int64_t* counts, void* out, int32_t B, int32_t T, int32_t nh, int32_t nkv, int32_t hd,
                           int32_t max_len, float scale, void* stream);
/* The same over an e4m3 cache with per-slot scales (scale pointers 4-byte aligned).  A chunk attends over the quantized
 * values the cache holds, its own keys and values included (quip_kv_append_fp8 wrote them): the values every later
 * decode step reads back, the rule of quip_decode_attention_fp8 and quip_extend_attention_fp8.  (Filling the cache by
 * quip_kv_quantize_fp8 after an fp16 forward instead attends in fp16 and rounds afterwards.)  Per 64-slot block, a
 * slot's k scale multiplies its score column; its v scale multiplies p before p is rounded to fp16, normalised by the
 * largest v scale among the query row's visible slots of the block, which multiplies the block's P.V. */
int quip_prefill_attention_fp8(const void* q, const void* k_cache, const void* v_cache, const float* k_scale,
                               const float* v_scale, const int64_t* positions, const int64_t* counts, void* out,
                               int32_t B, int32_t T, int32_t nh, int32_t nkv, int32_t hd, int32_t max_len, float scale,
                               void* stream);

/* Paged KV cache.  Per layer, k_pool / v_pool (n_pages, nkv, 64, hd) hold fp16 or e4m3fn values (e4m3: with k_scale /
 * v_scale (n_pages, nkv, 64) fp32, the format of quip_decode_attention_fp8); a page holds 64 slots of every kv head.
 * page_table (B, max_pages) int32 on the device, shared by all layers: slot j of row b lives at slot j % 64 of page
 * page_table[b][j / 64].  Rows may map the same page (a shared prompt prefix).  A page id outside [0, n_pages) -- the
 * -1 of an unmapped entry, say -- follows the rule of a position outside the cache: it is never dereferenced, nothing
 * is written through it, and every output of a token that would read or write a slot on that page is NaN.  Pages past
 * the slots a launch reads or writes are not looked up.
 *
 * Each entry point below takes the arguments of its contiguous twin with the caches replaced by the pools and max_len by
 * (page_table, max_pages, n_pages); max_len = max_pages * 64 everywhere it mattered (decode chunking, grids, the
 * workspace sizes of quip_decode_attention_workspace_bytes / quip_extend_attention_workspace_bytes), so a paged launch
 * runs the contiguous launch's blocks and arithmetic: its results are bit-identical to the contiguous launch over the
 * same cached bytes.  page_table 4-byte aligned, 0 < max_pages <= 2^31 / 64, n_pages > 0. */
int quip_decode_attention_paged(const void* q, const void* k_new, const void* v_new, void* k_pool, void* v_pool,
                                const int64_t* positions, void* out, int32_t B, int32_t nh, int32_t nkv, int32_t hd,
                                float scale, void* workspace, size_t workspace_bytes, const int32_t* page_table,
                                int32_t max_pages, int32_t n_pages, void* stream);
int quip_decode_attention_paged_fp8(const void* q, const void* k_new, const void* v_new, void* k_pool, void* v_pool,
                                    float* k_scale, float* v_scale, const int64_t* positions, void* out, int32_t B,
                                    int32_t nh, int32_t nkv, int32_t hd, float scale, void* workspace,
                                    size_t workspace_bytes, const int32_t* page_table, int32_t max_pages,
                                    int32_t n_pages, void* stream);
int quip_extend_attention_paged(const void* q, const void* k_new, const void* v_new, void* k_pool, void* v_pool,
                                const int64_t* positions, void* out, int32_t B, int32_t T, int32_t nh, int32_t nkv,
                                int32_t hd, float scale, void* workspace, size_t workspace_bytes,
                                const int32_t* page_table, int32_t max_pages, int32_t n_pages, void* stream);
int quip_extend_attention_paged_fp8(const void* q, const void* k_new, const void* v_new, void* k_pool, void* v_pool,
                                    float* k_scale, float* v_scale, const int64_t* positions, void* out, int32_t B,
                                    int32_t T, int32_t nh, int32_t nkv, int32_t hd, float scale, void* workspace,
                                    size_t workspace_bytes, const int32_t* page_table, int32_t max_pages,
                                    int32_t n_pages, void* stream);
int quip_kv_append_paged(const void* k_new, const void* v_new, void* k_pool, void* v_pool, const int64_t* positions,
                         const int64_t* counts, int32_t B, int32_t T, int32_t nkv, int32_t hd,
                         const int32_t* page_table, int32_t max_pages, int32_t n_pages, void* stream);
int quip_kv_append_paged_fp8(const void* k_new, const void* v_new, void* k_pool, void* v_pool, float* k_scale,
                             float* v_scale, const int64_t* positions, const int64_t* counts, int32_t B, int32_t T,
                             int32_t nkv, int32_t hd, const int32_t* page_table, int32_t max_pages, int32_t n_pages,
                             void* stream);
int quip_prefill_attention_paged(const void* q, const void* k_pool, const void* v_pool, const int64_t* positions,
                                 const int64_t* counts, void* out, int32_t B, int32_t T, int32_t nh, int32_t nkv,
                                 int32_t hd, float scale, const int32_t* page_table, int32_t max_pages, int32_t n_pages,
                                 void* stream);
int quip_prefill_attention_paged_fp8(const void* q, const void* k_pool, const void* v_pool, const float* k_scale,
                                     const float* v_scale, const int64_t* positions, const int64_t* counts, void* out,
                                     int32_t B, int32_t T, int32_t nh, int32_t nkv, int32_t hd, float scale,
                                     const int32_t* page_table, int32_t max_pages, int32_t n_pages, void* stream);

/* Token selection of one generation step: for each row b of logits (B, V) fp16 contiguous (rows need no alignment),
 * with T = temperature[b], k = top_k[b], p = top_p[b] and s = seed[b] (each (B), device) and t = *step (device; the
 * index of the token being chosen, 0 for the one after the prompt), tokens[b] (int64) is:
 *   1. greedy rows (T <= 0, T NaN, or k == 1): the smallest i with x_i = max x (torch.argmax; a NaN counts as the max);
 *   2. z_i = fp32(x_i) / T, IEEE division;
 *   3. rank: z descending, equal z by lower index first;
 *   4. top-k: K = min(k, V) if k > 0, else V; the candidates are the first K tokens in rank order (exactly K);
 *   5. e_i = exp(z_i - max z);
 *   6. top-p, if p < 1 (not NaN): keep the shortest rank-order prefix of the candidates whose sum of e is >= p times
 *      their total; at least one token (p <= 0 keeps the top one);
 *   7. u = (w >> 8) * 2^-24, w the first word of Philox4x32-10 with key (s low word, s high word) and counter
 *      (t low word, t high word, 0, 0);
 *   8. S = sum of e over the kept tokens; walking them in INDEX order, the first whose running sum of e exceeds u * S.
 * e is fp32 expf, then floor(e * 2^40) as an integer: every sum and comparison after that is exact and independent of
 * order (u * S exactly), so a token depends only on (row, settings, seed, t) -- not on the batch, the row index or the
 * launch -- and is bit-identical from run to run.  A row with non-finite logits still gets an index in [0, V).  The
 * launch depends on (B, V) only: one captured graph serves every step and any settings written between replays.
 * No workspace.  B >= 0 (0: nothing to do), 1 <= V <= 2^24. */
int quip_sample(const void* logits, const float* temperature, const int32_t* top_k, const float* top_p,
                const uint64_t* seed, const int64_t* step, int64_t* tokens, int32_t B, int32_t V, void* stream);
/* The same rule over logits (B * T, V): row b * T + i takes the settings and seed of row b (each (B)) and
 * t = steps[b] + i, steps (B) int64 on the device.  Row b * T + i's token is what quip_sample gives for that logits row
 * with those settings at step t. */
int quip_sample_at(const void* logits, const float* temperature, const int32_t* top_k, const float* top_p,
                   const uint64_t* seed, const int64_t* steps, int64_t* tokens, int32_t B, int32_t T, int32_t V,
                   void* stream);

/* Continuation scoring: for each row r of fp16 logits (R, V) with row stride ld (elements; rows need only 2-byte
 * alignment) and t = targets[r] (int64):
 *   logprob[r]   = (x_t - m) - log(sum_j exp(x_j - m)),  m = max_j x_j,  in fp32 (fp32 expf / logf);
 *   is_greedy[r] = 1 if t is the lowest index holding the row's largest value (torch.argmax's tie rule), else 0 (uint8).
 * A NaN anywhere in the row gives logprob NaN and is_greedy 0.  A target outside [0, V) is never dereferenced and gives
 * NaN and 0 (the guard rule of the paged kernels).  One pass over the row; no workspace.  The per-thread partial sums
 * are combined in a fixed order, so repeated launches are bit-identical, and a row's result does not depend on the
 * other rows.  R >= 0 (0: nothing to do), V >= 1, ld >= V; targets 8-byte and logprob 4-byte aligned. */
int quip_token_logprobs(const void* logits, int64_t ld, const int64_t* targets, float* logprob, uint8_t* is_greedy,
                        int32_t R, int32_t V, void* stream);

/* Signature-compatible replacement of the reference's own native call (quant_cuda.vecquant3matmul quant.py:229-230,
 * vecquant4matmul zeroShot/models/quant.py:207-208): ONE token, fp32, on the REFERENCE's packed layout
 * (bits 3: int32 (K*3/32, N) as Quant3Linear.pack writes it; bits 4: (K/8, N); bits 2: (K/16, N)):
 *     mul[n] += sum_k (scales[n] * code[k][n] - zeros[n]) * vec[k]        (in-place accumulate, like the reference's call)
 * so a checkpoint packed by the reference runs without conversion.  K % 32 == 0.  quip_qlinear_forward on the native
 * layout is the fast path; this one is a plain HBM-streaming kernel. */
int quip_vecquant_matmul(const float* vec, const int32_t* mat, float* mul, const float* scales, const float* zeros,
                         int32_t K, int32_t N, int32_t bits, void* stream);

/* codes (N,K) uint8 row-major <-> native packed layout.  Replaces Quant3Linear.pack (quant.py:185-220). */
int quip_pack_codes(const uint8_t* codes_nk, int32_t N, int32_t K, int32_t bits, int32_t* qweight,
                    void* stream);
int quip_unpack_codes(const int32_t* qweight, int32_t N, int32_t K, int32_t bits, uint8_t* codes_nk,
                      void* stream);
/* Reference layouts -> codes (N,K): bits=3 quant.py:192-220 [(K*3/32, N) int32], bits=4
 * zeroShot/models/quant.py:193-199 [(K/8, N)], bits=2 the natural extension [(K/16, N)]. */
int quip_convert_ref(const int32_t* ref_qweight, int32_t K, int32_t N, int32_t bits,
                     uint8_t* codes_nk, void* stream);
size_t quip_packed_words(int32_t N, int32_t K, int32_t bits);

/* Quantisation-time hot loop (SURVEY section 8f rank 1): the column-sequential part of LDLQ rounding for one block of
 * <= 128 columns, all rows in one launch (reference: the Python column loops of round_ldl / round_ldl_block,
 * vector_balance.py:155-199, :218-257).  All matrices fp32, column-major over rows ("transposed": element (row r,
 * column j) at [j*ld + r]); the feedback of the finished blocks is the caller's GEMM (quip_b200/quantize.py).
 *   quip_ldlq_block    q[:, j] = clamp(floor(base[:, j] + sum_{j' > j} err[:, j'] * Lb[j'][j] + 1/2), 0, 2^bits - 1),
 *                      err[:, j] = w[:, j] - q[:, j], for j = cnt-1 .. 0.  base = w[:, blk] + err[:, done] @ L[done, blk];
 *                      Lb (cnt, cnt) row-major = L[blk, blk] - I (unit-lower LDL factor of H, strictly lower part read).
 *   quip_greedy_block  one coordinate-descent sweep over the block (vector_balance.py:267-283): for i = cnt-1 .. 0,
 *                      move = wr_i - rint(wr_i - (pre_i + sum_j s_j Hb[j][i]) / Hb[i][i]); wr_i -= move; s_i -= move.
 *                      pre = s[:, outside blk] @ Hn[outside, blk]; Hb = Hn[blk, blk]; wr, s updated in place. */
int quip_ldlq_block(const float* baseT, const float* wT, const float* Lb, float* qT, float* errT, int64_t m, int64_t ld,
                    int32_t cnt, int32_t bits, void* stream);
int quip_greedy_block(const float* preT, const float* Hb, float* wrT, float* sT, int64_t m, int64_t ld, int32_t cnt,
                      void* stream);

/* Calibration Hessian (SURVEY section 8f rank 2; reference QuantMethod.add_batch, method.py:98-120): H += X^T X for
 * X (tokens, K) fp16 row-major, H (K, K) float64 row-major.  Products on the fp16 tensor cores (exact in float32), float32
 * sums over 256 tokens, float64 carry in H.  Only the upper BLOCK triangle of 128 x 128 tiles is updated (tile row <= tile
 * column, diagonal tiles whole): mirror it once after the last batch.  K % 8 == 0. */
int quip_hessian_accumulate(const void* x, double* H, int64_t tokens, int32_t K, void* stream);

/* Optional per-launch timing of the contraction kernels with CUDA events recorded on the launch stream
 * (bench.py's roofline leg).  path: 1 = mma.sync skinny kernel, 2 = wgmma kernel.  quip_timing_read
 * waits for the recorded events and returns the totals since the last reset: device milliseconds,
 * launches, algorithmic flops (2*M*N*K) and algorithmic bytes (packed codes + fp16 activations in + out). */
int quip_timing_enable(int on);
int quip_timing_reset(void);
int quip_timing_read(int path, double* total_ms, int64_t* launches, double* flops, double* bytes);

/* Routing switches for ablations, tests and micro-benchmarks (defaults in parentheses); results do not depend on them.
 *   "side_fused" (1)  M > 8: a whole incoherence side in one kernel when both blocks are 32/64 wide and factors_frag is set
 *   "fewtok" (1)      M <= 8: few-token pass / gather kernels (fused input gather, output scatter + bias)
 *   "fewtok_max_m" (32) 8..32: token count up to which the few-token passes run (batched decode)
 *   "side_fewtok" (0) M <= 8: both passes of a side (+ gather / scatter, bias) in one launch: side, contraction, side
 *                     (ablation: measured slower than the two-pass route, see profiles/README.md)
 *   "pdl" (1)         programmatic dependent launch along the few-token chain
 *   "gemv" (1)        M <= 8: whole-K qgemv kernels (0: split-K mma.sync kernel)
 *   "gv_int" (1)      qgemv: int8 tensor-core path for 2-/4-bit and <= 5 tokens (0: fp16 path)
 *   "gv_tma" (1), "gv_cw" (16), "gv_rbc" (0 = auto), "gv_persist" (1)   variants of the cooperative int8 kernel
 *   "gv_stream" (32)  streaming int8 kernel when N/16 >= value * SMs (0: never)
 *   "sk_ksplit" (0)   split-K kernel (9..32 tokens): cap on the number of K splits, only ever lowering the heuristic's choice
 *                     (the workspace is sized for that); 0 = the heuristic
 *   "gather_rows", "pass_min_tiles"   tune the many-token un-projection kernels */
int quip_config(const char* key, int value);

const char* quip_last_error(void);
int quip_abi_version(void);
/* Number of kernels this library has launched on behalf of the calling process (for bench gpu_launches). */
int64_t quip_launch_count(void);

#ifdef __cplusplus
}
#endif
#endif /* QUIP_B200_H_ */
