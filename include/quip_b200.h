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

#define QUIP_ABI_VERSION 3

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

/* The KV cache of one layer, as every cache operation below takes it (decode, extend and prefill attention, the
 * appends and the beam fork).  The format is stated once here; the operations add only their own rules.
 *
 * Format.  QUIP_KV_FP16: k / v hold fp16 values and k_scale / v_scale are NULL.  QUIP_KV_E4M3: k / v hold e4m3fn
 * bytes and k_scale / v_scale fp32, one scale per cached head vector x (hd values):
 *   amax = max_i |x_i|;  s = amax / 448 (IEEE fp32 division; s = 1 when amax == 0);  q_i = e4m3fn(x_i / s), round to
 *   nearest even, subnormals kept;  the vector's value is float(q_i) * s.
 * New keys and values (fp16) are quantized so when they are appended, written with their scales, and attended over as
 * quantized values like every other slot; no scale past the slots a launch reads is read.  Non-finite inputs may give
 * NaN outputs.  The format is never inferred from the scales: they must be non-NULL exactly when it is QUIP_KV_E4M3, so
 * a NULL scale pointer is an error, never e4m3 bytes read as fp16.
 *
 * Layout.  page_table NULL: the contiguous cache, k / v (B, nkv, max_len, hd) and scales (B, nkv, max_len);
 * max_pages and n_pages are not read.  page_table non-NULL: the paged cache, k / v pools (n_pages, nkv, 64, hd) and
 * scales (n_pages, nkv, 64); a page holds 64 slots of every kv head.  page_table (B, max_pages) int32 on the device,
 * shared by all layers: slot j of row b lives at slot j % 64 of page page_table[b][j / 64].  Rows may map the same page
 * (a shared prompt prefix).  A page id outside [0, n_pages) -- the -1 of an unmapped entry, say -- follows the rule of a
 * position outside the cache: it is never dereferenced, nothing is written through it, and every output of a token that
 * would read or write a slot on that page is NaN.  Pages past the slots a launch reads or writes are not looked up.
 * max_len is not read: it is max_pages * 64 everywhere it matters (decode chunking, grids, the workspace sizes of
 * quip_decode_attention_workspace_bytes / quip_extend_attention_workspace_bytes), so a paged launch runs the contiguous
 * launch's blocks and arithmetic: its results are bit-identical to the contiguous launch over the same cached bytes.
 *
 * Every operation checks the descriptor before it launches: k and v non-NULL and 16-byte aligned, the scales 4-byte
 * aligned, hd in {64, 128}; paged: page_table 4-byte aligned, 0 < max_pages <= 2^31 / 64, n_pages > 0.  B below is the
 * number of rows of the contiguous cache or of page_table. */
typedef struct {
  void* k;                 /* keys: the cache or the page pool */
  void* v;                 /* values, of the same shape */
  float* k_scale;          /* QUIP_KV_E4M3 only, else NULL */
  float* v_scale;
  int32_t* page_table;     /* NULL: contiguous.  Only quip_kv_beam_fork writes through it */
  int32_t format;          /* QUIP_KV_FP16 or QUIP_KV_E4M3 */
  int32_t nkv, hd;         /* kv heads, head dim */
  int32_t max_len;         /* contiguous only: slots per row */
  int32_t max_pages;       /* paged only: columns of page_table */
  int32_t n_pages;         /* paged only: pages in each pool */
} QuipKvCache;

#define QUIP_KV_FP16 1
#define QUIP_KV_E4M3 2

/* One decode-attention step for B sequences, each at its own position, on one layer's KV cache kv.
 *   q (B, nh, hd) fp16 with rotary applied; k_new / v_new (B, nkv, hd) fp16: this step's key / value; positions (B)
 *   int64 on the device; out (B, nh, hd) fp16.
 * Writes k_new / v_new at slot positions[b] and returns
 *   out[b][h] = softmax_j(scale * q[b][h] . k[b][h / G][j]) v[b][h / G][j],  j = 0 .. positions[b],  G = nh / nkv,
 * reading no slot past positions[b].  fp32 scores, softmax and P.V; one fp16 rounding of the output.  The launch grid
 * depends on (B, nkv, max_len) only, so one captured graph serves every position.  nh % nkv == 0, nh / nkv <= 8; q,
 * k_new, v_new, out and workspace 16-byte aligned; fp32 scratch from quip_decode_attention_workspace_bytes.  A position
 * outside [0, max_len) leaves the cache untouched and gives a NaN output row.  Deterministic: bit-identical results from
 * run to run and for every other content of the other rows. */
int quip_decode_attention(const QuipKvCache* kv, const void* q, const void* k_new, const void* v_new,
                          const int64_t* positions, void* out, int32_t B, int32_t nh, float scale, void* workspace,
                          size_t workspace_bytes, void* stream);
int quip_decode_attention_workspace_bytes(int32_t B, int32_t nh, int32_t hd, int32_t max_len, size_t* out_bytes);

/* One attention step with T new tokens per row (speculative verification), each row at its own position, on one layer's
 * KV cache kv.  q (B, T, nh, hd) fp16 token-major, rotary applied; k_new / v_new (B, T, nkv, hd) fp16; positions (B)
 * int64 on the device; out (B, T, nh, hd) fp16.  Token i of row b is written at slot positions[b] + i, and
 *   out[b][i][h] = softmax_j(scale * q[b][i][h] . k[b][h / G][j]) v[b][h / G][j],  j = 0 .. positions[b] + i,
 * causal inside the new tokens.  No slot past positions[b] + T - 1 is read.  Scores and softmax in fp32; Q.K^T and P.V
 * on tensor cores (fp16 operands, fp32 accumulation; p rounded once to fp16); one fp16 rounding of the output.  1 <= T
 * <= 8, nh % nkv == 0, nh / nkv <= 8; pointers 16-byte aligned; fp32 scratch from
 * quip_extend_attention_workspace_bytes.  The grid depends on (B, T, nkv, max_len) only.  A row with positions[b] < 0
 * or positions[b] + T > max_len writes nothing and gets NaN outputs.  Deterministic, and a row's result does not depend
 * on the other rows.  T = 1 computes what quip_decode_attention does, to within its rounding of p.  e4m3: a slot's k
 * scale multiplies its score column; its v scale multiplies p before p is rounded to fp16 (normalised by the chunk's
 * largest v scale, which multiplies the chunk's P.V). */
int quip_extend_attention(const QuipKvCache* kv, const void* q, const void* k_new, const void* v_new,
                          const int64_t* positions, void* out, int32_t B, int32_t T, int32_t nh, float scale,
                          void* workspace, size_t workspace_bytes, void* stream);
int quip_extend_attention_workspace_bytes(int32_t B, int32_t T, int32_t nh, int32_t hd, int32_t max_len,
                                          size_t* out_bytes);

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

/* Prefill of an e4m3 cache: src (B, nkv, P, hd) fp16 quantized by the rule of QuipKvCache into slots 0 .. P-1 of
 * cache (B, nkv, max_len, hd) e4m3fn and scales (B, nkv, max_len) fp32; slots >= P are not touched.  hd in {64, 128},
 * P <= max_len; src and cache 16-byte aligned, scales 4-byte aligned. */
int quip_kv_quantize_fp8(const void* src, void* cache, float* scales, int32_t B, int32_t nkv, int32_t P,
                         int32_t max_len, int32_t hd, void* stream);

/* Chunked prefill, part 1: append a chunk of new keys and values to one layer's KV cache kv.  k_new / v_new
 * (B, T, nkv, hd) fp16 token-major; positions, counts (B) int64 on the device.  Token i of row b goes to slot
 * positions[b] + i for i < counts[b]; no other slot, and nothing of a row with counts[b] == 0, is touched.  A row with
 * positions[b] < 0, counts[b] outside [0, T] or positions[b] + counts[b] > max_len writes nothing.  1 <= T <= max_len;
 * pointers 16-byte aligned. */
int quip_kv_append(const QuipKvCache* kv, const void* k_new, const void* v_new, const int64_t* positions,
                   const int64_t* counts, int32_t B, int32_t T, void* stream);
/* Chunked prefill, part 2: causal attention of a chunk of T query tokens per row over the cache that already holds the
 * chunk (quip_kv_append first).  q (B, T, nh, hd) fp16 token-major, rotary applied; out (B, T, nh, hd) fp16.  For
 * i < counts[b]
 *   out[b][i][h] = softmax_j(scale * q[b][i][h] . k[b][h / G][j]) v[b][h / G][j],  j = 0 .. positions[b] + i,
 * and out[b][i] = 0 for counts[b] <= i < T.  No slot past positions[b] + counts[b] - 1 is read.  Flash-attention style:
 * Q.K^T and P.V on tensor cores (fp16 operands, fp32 accumulation), online softmax in fp32, p rounded once to fp16 per
 * 64-slot block, one fp16 rounding of the output; no workspace.  1 <= T <= max_len, nh % nkv == 0, nh / nkv <= 8;
 * pointers 16-byte aligned.  A row with positions[b] < 0, counts[b] outside [0, T] or positions[b] + counts[b] > max_len
 * gets NaN outputs.  Deterministic, and a row's result does not depend on the other rows.  At T <= 8 it computes what
 * quip_extend_attention does, to within the rounding of p.
 * e4m3: a chunk attends over the quantized values the cache holds, its own keys and values included (quip_kv_append
 * wrote them): the values every later decode step reads back, the rule of quip_decode_attention and
 * quip_extend_attention.  (Filling the cache by quip_kv_quantize_fp8 after an fp16 forward instead attends in fp16 and
 * rounds afterwards.)  Per 64-slot block, a slot's k scale multiplies its score column; its v scale multiplies p before
 * p is rounded to fp16, normalised by the largest v scale among the query row's visible slots of the block, which
 * multiplies the block's P.V. */
int quip_prefill_attention(const QuipKvCache* kv, const void* q, const int64_t* positions, const int64_t* counts,
                           void* out, int32_t B, int32_t T, int32_t nh, float scale, void* stream);

/* Ragged (packed) chunks over a paged cache (kv must have a page_table): S sequences of different lengths back to back
 * in N token rows, so a step that mixes decode rows (one token each) and prompt chunks feeds no padding.  seq_start
 * (S + 1) int64 on the device holds offsets 0 <= seq_start[0] <= ... <= seq_start[S] <= N: token i of sequence s is
 * packed row seq_start[s] + i, at slot positions[s] + i (positions (S) int64) of row s of page_table (S, max_pages) --
 * the table rows of the S sequences.  k_new / v_new are (N, nkv, hd), q / out (N, nh, hd), fp16 token-major.
 * max_count >= 1 bounds every sequence's length (the attention grid is (query tile, kv head, sequence) with
 * ceil(G * max_count / 64) tiles; a tile past its sequence's length exits at once).
 *
 * Guards: a sequence with positions[s] < 0, positions[s] + its length > max_pages * 64 or a length above max_count
 * writes nothing and its outputs are NaN (as far as max_count reaches); a page outside the pool follows the paged rule.
 * A sequence whose offsets break the order above or leave [0, N] is not looked at: nothing is read or written for it.
 * There are no padding rows: out rows outside every sequence are not written.
 *
 * The rule: per sequence s, the ragged launch is bit-identical to the padded launch (quip_kv_append,
 * quip_prefill_attention) on the same paged cache with B = S, T = max_count, counts[s] = seq_start[s + 1] - seq_start[s]
 * and row s of the padded q / k_new / v_new holding the sequence's tokens, over the same cached bytes: each sequence runs
 * the same query tiles, 64-slot blocks and arithmetic, and only the addressing of the packed rows differs. */
int quip_kv_append_ragged(const QuipKvCache* kv, const void* k_new, const void* v_new, const int64_t* seq_start,
                          const int64_t* positions, int32_t S, int32_t N, int32_t max_count, void* stream);
int quip_prefill_attention_ragged(const QuipKvCache* kv, const void* q, const int64_t* seq_start,
                                  const int64_t* positions, void* out, int32_t S, int32_t N, int32_t max_count,
                                  int32_t nh, float scale, void* stream);

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
 * No workspace.  B >= 0 (0: nothing to do), 1 <= V <= 2^24 - 1 (V weights of at most 2^40 sum below 2^64). */
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
/* Log-probabilities of generation, from the raw fp16 logits (R, V) with row stride ld (elements; rows need only
 * 2-byte alignment).  Logits row r is offset i = r % T of decoder row b = rows[r / T] (rows (R / T) int64; null:
 * b = r / T), its chosen token tokens[r] (int64), and its results go to column c = cols[b * cols_per_row] + i (cols
 * int64 on the device: one counter per decoder row, cols_per_row = 1, or one shared by every row, 0) of the outputs
 * lp (B, gen_cols) fp32, top_ids (B, gen_cols, n) int64 and top_lp (B, gen_cols, n) fp32.  A row with b outside
 * [0, B) or c outside [0, gen_cols) writes nothing (c is not clamped: a done row's last entry is kept).  Otherwise
 *   lp[b, c]        = what quip_token_logprobs gives for the row and target tokens[r], bit for bit (NaN for a row
 *                     holding a NaN or a token outside [0, V));
 *   top_ids[b, c, j], top_lp[b, c, j], j < min(n, V): the row's ids ranked by fp16 logit descending, equal values
 *                     (-0 == +0) by lower id, and for each the logprob quip_token_logprobs gives with that id as the
 *                     target, bit for bit (the same row pass: logprob_row.cuh).  The order agrees with the logprob
 *                     order, as both subtract the same constants;
 *   j >= min(n, V), and every j of a row holding a NaN: (-1, NaN).
 * top_ids and top_lp may be null when n = 0.  The launch depends on (R, T, V, n, B, gen_cols) only, so one captured
 * graph serves every step.  One CTA per row; no workspace.  Bounds: 1 <= T <= 8 dividing R, 1 <= V <= 2^24, ld >= V,
 * 0 <= n <= 20; int64 arrays 8-byte and fp32 arrays 4-byte aligned. */
int quip_token_topk_logprobs(const void* logits, int64_t ld, int32_t R, int32_t T, int32_t V, const int64_t* rows,
                             const int64_t* tokens, const int64_t* cols, int32_t cols_per_row, float* lp,
                             int64_t* top_ids, float* top_lp, int32_t n, int32_t B, int32_t gen_cols, void* stream);

/* Logits processors of generation (HF's RepetitionPenalty, NoRepeatNGram, NoBadWords and MinNewTokensLength, in that
 * order), in place on fp16 logits (R, V) with row stride ld (elements; rows need only 2-byte alignment).  Logits row r
 * is offset i = r % T of decoder row b = rows[r / T] (rows (R / T) int64; null: b = r / T); T = 1 except in speculative
 * steps.  Its history h is hist[b, 0 .. c] (hist (B, max_len) int64, c = last[b]) followed by the drafts
 * tokens[b, 1 .. i] (tokens (B, T) int64; may be null when T = 1); L = c + 1 + i, n_new = L - prompt_len[b].  Per decoder
 * row (device): penalty rho (fp32), ngram size n (int32, 0 = off), min_new m (int32).  For the call: eos (n_eos int64)
 * and the bad-word sequences bad (n_bad, 16) int64 with lengths bad_len (n_bad) int32.
 *   1. repetition penalty (rho != 1): for each distinct v of h, x_v <- x_v < 0 ? x_v * rho : x_v / rho in fp32 (IEEE),
 *      rounded once to fp16 (NaN stays NaN, -0 -> -0 / rho);
 *   2. no-repeat n-gram (n >= 1): for every 0 <= e <= L - n with h[e .. e+n-2] == h[L-n+1 .. L-1], x_{h[e+n-1]} <- -inf
 *      (n = 1 bans every token of h);
 *   3. bad words: the sequences of length 1 equal to an eos id are dropped.  A sequence w of length l bans w[l-1] when
 *      l == 1, or l <= L and the last l - 1 tokens of h equal w[0 .. l-2].  HF adds a bias row b (-inf at banned
 *      tokens, +0 elsewhere), so with n_bad > 0 a banned x becomes x + (-inf) (NaN for +inf and NaN) and every -0 of the
 *      row becomes +0;
 *   4. min_new_tokens: if n_new < m, every eos id gets -inf.
 * Steps 2 and 4 assign -inf and step 3 adds it, so a token banned by 2 or 4 ends at -inf whatever 3 does.  A token id
 * outside [0, V) (in h, eos or bad) is never dereferenced; a row with b outside [0, B) or c outside [0, max_len) is not
 * touched, nor is a row with rho == 1, n == 0, no eos ban due and n_bad == 0 (bit for bit).  Only the penalised and
 * banned entries (and, with bad words, the -0 entries) are written.  The launch depends on (R, T, V, B, max_len, n_eos,
 * n_bad) only, so one captured graph serves any settings written between replays.  One CTA per row; no workspace.
 * Bounds: 1 <= V <= 2^18, 0 <= n_eos <= 8, 0 <= n_bad <= 256, 1 <= bad_len <= 16 (a longer or empty sequence is
 * ignored), R % T == 0; hist, last, tokens, prompt_len, eos and bad 8-byte aligned. */
int quip_logits_process(void* logits, int64_t ld, int32_t R, int32_t T, int32_t V, const int64_t* rows,
                        const int64_t* hist, const int64_t* last, const int64_t* tokens, const int64_t* prompt_len,
                        const float* penalty, const int32_t* ngram, const int32_t* min_new, const int64_t* eos,
                        int32_t n_eos, const int64_t* bad, const int32_t* bad_len, int32_t n_bad, int32_t B,
                        int32_t max_len, void* stream);

/* Constrained generation (HF's PrefixConstrainedLogitsProcessor, which runs right after the processors above) by a
 * token automaton on the device.  The table packs S states: offsets (S + 1) int32, ids (nnz) int32 and next (nnz)
 * int32; state s allows ids[k] and leads to next[k] for k in [lo_s, hi_s), lo_s = clamp(offsets[s], 0, nnz),
 * hi_s = clamp(offsets[s + 1], lo_s, nnz).  Several automata (one per prompt) share one table with disjoint state
 * ranges.  The host validates the table (offsets[0] = 0 and non-decreasing, ids strictly increasing within a state,
 * next in [0, S), every state non-empty); the kernels never read outside it whatever it holds.
 *   delta(s, v) = next[k] if ids[k] == v for some k in [lo_s, hi_s), else s: a token without a transition (possible
 *   only when the masked row had no finite allowed entry, e.g. min_new_tokens banning an EOS-only state) leaves the
 *   state unchanged.  For s outside [0, S), delta(s, v) = s.
 *
 * quip_constrain_mask, in place on fp16 logits (R, V) with row stride ld (elements; rows need only 2-byte alignment):
 * logits row r is offset i = r % T of decoder row b = rows[r / T] (rows (R / T) int64; null: b = r / T), with
 * s_0 = state[b] (state (B) int32; -1 marks an unconstrained row) and s_j = delta(s_{j-1}, tokens[b, j]) for
 * j = 1 .. i (tokens (B, T) int64, the speculative step's current token and drafts; may be null when T = 1).  A row
 * with b outside [0, B) or s_i outside [0, S) is not touched, bit for bit.  Otherwise every x_v, v in [0, V), becomes
 * x_v + (v allowed in s_i ? +0 : -inf) in fp16: HF's scores + mask, so an allowed -0 becomes +0 and a disallowed +inf or
 * NaN becomes NaN (each sum is exact).  Table ids outside [0, V) allow nothing.
 *
 * quip_constrain_advance moves the state over the tokens a step commits: for n in [0, N), b = rows[n] (rows (N) int64,
 * distinct; null: b = n), skipped when outside [0, B); c = counts[n] (counts (N) int64; null: T) clamped to [0, T];
 * state[b] <- delta(... delta(state[b], tok[n * ld + 0]) ..., tok[n * ld + c - 1]) (tok int64, row stride ld >= T).
 * A plain step passes its selected tokens (T = 1), a speculative step the targets (B, T) with counts = the tokens
 * quip_spec_accept appended, a continuous step its rows with counts = 1 for live rows and 0 otherwise.
 *
 * Both launches depend on (R, T, V, B, S, nnz) and (N, T, B, S, nnz) only, so one captured graph serves every step.
 * Mask: one CTA per logits row, a V-bit shared-memory bitmap of the allowed ids, no workspace.  Advance: one thread
 * per entry.  Bounds: 1 <= V <= 2^18, 1 <= T <= 8 dividing R, ld >= V, S >= 0, nnz >= 0; int64 arrays 8-byte and int32
 * arrays 4-byte aligned. */
int quip_constrain_mask(void* logits, int64_t ld, int32_t R, int32_t T, int32_t V, const int64_t* rows,
                        const int64_t* tokens, const int32_t* state, int32_t B, const int32_t* offsets,
                        const int32_t* ids, const int32_t* next, int32_t S, int32_t nnz, void* stream);
int quip_constrain_advance(int32_t* state, int32_t B, const int64_t* tok, int64_t ld, int32_t N, int32_t T,
                           const int64_t* rows, const int64_t* counts, const int32_t* offsets, const int32_t* ids,
                           const int32_t* next, int32_t S, int32_t nnz, void* stream);

/* Beam search (HF's GenerationMixin._beam_search, prompt by prompt).  B prompts of K beams each are the rows
 * r = b * K + j (2 <= K <= 16 in generate).  C = max(2, 1 + n_eos) * K <= 64 candidates per prompt.
 *
 * quip_beam_candidates: for each row r of fp16 logits (R, V), row stride ld (rows need only 2-byte alignment), with
 * j = r % K and score = scores[r] (fp32, device):
 *   s_v = ((x_v - m) - log(sum exp(x - m))) + score, m = max x, in fp32 (expf / logf; the per-thread sums are combined
 *         in a fixed order, so launches are bit-identical).  A NaN anywhere in the row makes every s NaN; a row whose
 *         maximum is -inf gives s = -inf throughout;
 *   rank: s descending, then the lower flat index j * V + v.  NaN ranks below every number (-inf included), -0 == +0;
 *   cand_s[r, :], cand_i[r, :] (fp32, int32) = the first min(C, V) entries in rank order as (s, j * V + v); when
 *   V < C the rest are (NaN, -1), ranked after every entry.  The K lists of a prompt hold its top C over all K * V.
 *
 * quip_beam_select: one prompt b at step t = *step (device; n = t + 1 tokens after this step) with n_b = budget[b]:
 *   0. done[b] set: parents[r] = r and adv[r] = 0 for its rows; nothing else is read or written (likewise t outside
 *      [0, max_new));
 *   1. merge its K candidate lists into the top C by the rank above (ties across lists: lower flat index, then row);
 *   2. a candidate hits when its token (index % V) is one of the n_eos <= 3 ids eos[] or n >= n_b;
 *   3. running beams: the top K of r_i = s_i + (hit ? -1e9 : 0) (ties: lower rank).  Beam k gets parent j_i, token,
 *      score[b*K+k] = r_i, history hist[b, k, :t] = hist[b, j_i, :t] with hist[b, k, t] = token (gathered from the copy
 *      hist_tmp); tokens[r] = token (the next input), parents[r] = b * K + j_i, adv[r] = 1;
 *   4. finished slots (fin_score, fin_len, fin_tok, fin_filled; K per prompt, kept sorted): every candidate i < C is
 *      offered with v_i = s_i / pen[n] (IEEE division; pen[n] = fp32(n ** length_penalty), n = 0 .. max_new) plus, in
 *      this order, -1e9 when early_stopping == 1 (True) and every slot is filled, -1e9 when heur[b] is 0, and -1e9
 *      unless i < K and i hits.  The slots keep the top K of (old slots, offered) by value (ties: the lower merged
 *      index, old slots first); an offered candidate's slot holds (v_i, n, its history and token, filled = i < K and
 *      hit);
 *   5. heur[b] &= any over slots k of best > (filled_k ? min of the slot values : -1e9), best = the top running score
 *      / pen[never_long ? n_b : n] (never_long: early_stopping 'never' with length_penalty > 0);
 *   6. done[b] = !heur[b] || (early_stopping == 1 && every slot filled) || every one of the C candidates hits.
 * early_stopping: 0 False, 1 True, 2 'never'.  Histories are (B, K, max_new) int64, fin_tmp / hist_tmp scratch of
 * that shape.  One CTA per prompt; everything is read from device memory, so one captured graph serves every step.
 *
 * quip_kv_beam_fork: after a select, with len = lens[r] (the slots row r has filled, the last at pos = len - 1,
 * cur = pos / 64) and p = parents[r] != r: table[r, :cur] = the old table[p, :cur] (read from table_tmp, a copy made by
 * the first phase, so rows may swap); slots 64 * cur .. pos of row p's current page are copied (every layer, k and v,
 * and on e4m3 pools their scales) into row r's current page, through scratch page scratch0 + r in two phases (gather
 * every parent, then scatter), so cycles and fan-out are safe.  kv describes layer 0 of L layers of paged pools
 * (L, n_pages, nkv, 64, hd) (scales (L, n_pages, nkv, 64)); table is its page_table (R, max_pages), which the fork
 * writes, and table_tmp scratch of that shape.  scratch0 + R <= n_pages.  A page id outside [0, n_pages) is never
 * dereferenced; rows with p == r or p outside [0, R) change nothing.  Two launches. */
int quip_beam_candidates(const void* logits, int64_t ld, const float* scores, float* cand_s, int32_t* cand_i,
                         int32_t R, int32_t V, int32_t K, int32_t C, void* stream);
int quip_beam_select(const float* cand_s, const int32_t* cand_i, const int64_t* eos, int32_t n_eos,
                     const int64_t* budget, const int64_t* step, const float* pen, float* score, int64_t* hist,
                     int64_t* hist_tmp, float* fin_score, int64_t* fin_len, int64_t* fin_tok, int64_t* fin_tmp,
                     uint8_t* fin_filled, uint8_t* heur, uint8_t* done, int64_t* tokens, int64_t* parents,
                     int64_t* adv, int32_t B, int32_t K, int32_t C, int32_t V, int32_t max_new,
                     int32_t early_stopping, int32_t never_long, void* stream);
int quip_kv_beam_fork(const QuipKvCache* kv, int32_t L, int32_t* table_tmp, const int64_t* parents,
                      const int64_t* lens, int32_t R, int32_t scratch0, void* stream);

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
