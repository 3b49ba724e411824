"""Llama decoder layers of the eval loop with the glue between the packed linears fused (csrc/glue.cu).

The reference's eval loop calls the HF decoder layer (llama.py:227); around the seven linears that layer issues ~25
elementwise / reduction launches (LlamaRMSNorm 8, apply_rotary_pos_emb 9 for q and k, residual adds, SiLU and the gate
product), a large share of a 2048-token step once the linears are packed.  `llama_stack`
runs the same layers -- the layer's own modules for every linear and its own weights for the norms -- with that glue as
four kernel launches per layer:

    x        = rmsnorm(h)                                   first layer only
    q, k, v  = q_proj(x), k_proj(x), v_proj(x);  rope_(q, k)           in place, token-major layout
    o        = o_proj(SDPA(q, k, v))                        torch SDPA (cuDNN / flash), strided head views, no copies
    h, x     = add_rmsnorm(h, o)                            residual add + post-attention norm
    d        = down_proj(silu_mul(gate_proj(x), up_proj(x)))
    h, x     = add_rmsnorm(h, d)                            residual add + the NEXT layer's input norm

Every fp16 rounding point of the HF modules is kept (see glue.cu), so the hidden states differ from the HF layer's only
through the summation order of the norms' fp32 mean.

`ops` is the provider of the three glue kernels: `CudaGlue` (the product: the C ABI, CUDA only, raises without the
extension) or, in the CPU tests, the torch restatement under oracle/ -- which this module never imports.
"""
import ctypes as C
import os

import torch
import torch.nn.functional as F

from . import _lib


class CudaGlue:
    """quip_rmsnorm / quip_rope / quip_silu_mul of the C ABI on torch tensors (fp16, CUDA, contiguous)."""

    @staticmethod
    def _check(*ts):
        for t in ts:
            if t is None:
                continue
            if not t.is_cuda:
                raise RuntimeError('the fused glue kernels run on a CUDA device only (there is no CPU fallback)')
            if t.dtype != torch.float16 or not t.is_contiguous():
                raise ValueError('fused glue kernels take contiguous fp16 tensors')

    @staticmethod
    def _stream(t):
        return torch.cuda.current_stream(t.device).cuda_stream

    def rmsnorm(self, x, weight, eps, residual=None):
        """y = weight * norm(x [+ residual]).  Returns y, or (x + residual, y) when a residual is given."""
        self._check(x, weight, residual)
        d = x.shape[-1]
        rows = x.numel() // d
        y = torch.empty_like(x)
        s = torch.empty_like(x) if residual is not None else None
        with torch.cuda.device(x.device):
            _lib.check(_lib.load().quip_rmsnorm(x.data_ptr(), residual.data_ptr() if residual is not None else None,
                                                weight.data_ptr(), s.data_ptr() if s is not None else None, y.data_ptr(),
                                                rows, d, C.c_float(eps), self._stream(x)))
        return y if residual is None else (s, y)

    def rope_(self, q, k, cos, sin, head_dim):
        """In place: q (..., nq*hd), k (..., nkv*hd) token-major; cos, sin (rows, hd)."""
        self._check(q, k, cos, sin)
        rows = q.numel() // q.shape[-1]
        if cos.numel() != rows * head_dim or sin.numel() != rows * head_dim:
            raise ValueError(f'cos/sin must hold one row of {head_dim} per token ({rows} tokens), got {tuple(cos.shape)}')
        with torch.cuda.device(q.device):
            _lib.check(_lib.load().quip_rope(q.data_ptr(), k.data_ptr(), cos.data_ptr(), sin.data_ptr(), rows,
                                             q.shape[-1] // head_dim, k.shape[-1] // head_dim, head_dim, self._stream(q)))

    def silu_mul(self, gate, up):
        self._check(gate, up)
        out = torch.empty_like(gate)
        with torch.cuda.device(gate.device):
            _lib.check(_lib.load().quip_silu_mul(gate.data_ptr(), up.data_ptr(), out.data_ptr(), gate.numel(),
                                                 self._stream(gate)))
        return out


    def silu_mul_gather(self, gate, up, idx):
        """silu(gate[..., ig]) * up[..., iu] with idx = ig | iu << 16 per output feature (int32 tensor): quip_silu_mul_gather."""
        self._check(gate, up)
        n = gate.shape[-1]
        out = torch.empty_like(gate)
        with torch.cuda.device(gate.device):
            _lib.check(_lib.load().quip_silu_mul_gather(gate.data_ptr(), up.data_ptr(), idx.data_ptr(), out.data_ptr(),
                                                        gate.numel() // n, n, self._stream(gate)))
        return out


KV_PAGE = 64


def _kv_format(fn, k_cache, v_cache, k_scale, v_scale):
    """Whether one layer's caches are e4m3: fp16 caches take no scales, float8_e4m3fn caches fp32 k_scale / v_scale."""
    fp8 = k_cache.dtype == torch.float8_e4m3fn
    if not fp8 and (k_scale is not None or v_scale is not None):
        raise ValueError(f'{fn}: k_scale / v_scale go with float8_e4m3fn caches only')
    if fp8 and (k_scale is None or v_scale is None):
        raise ValueError(f'{fn}: float8_e4m3fn caches need k_scale and v_scale')
    cdt = torch.float8_e4m3fn if fp8 else torch.float16
    if (k_cache.dtype != cdt or v_cache.dtype != cdt or
            (fp8 and (k_scale.dtype != torch.float32 or v_scale.dtype != torch.float32))):
        raise ValueError(f'{fn} takes fp16 or float8_e4m3fn caches (fp32 scales), got {k_cache.dtype} / '
                         f'{v_cache.dtype}')
    return fp8


def _kv_cache(fn, k_cache, v_cache, k_scale, v_scale, page_table, rows):
    """The checked QuipKvCache of one layer's cache (include/quip_b200.h has the rule): fp16 caches, or float8_e4m3fn
    caches with fp32 k_scale / v_scale, one per slot.  Without a page table the caches are (rows, nkv, max_len, hd);
    with page_table (rows, max_pages) int32 they are pools (n_pages, nkv, 64, hd) and max_len = max_pages * 64, which
    the descriptor's max_len holds in both layouts.  Checks the table's dtype, shape, device and alignment and the
    pools' alignment; the callers check that the caches and scales are contiguous CUDA tensors with their operands."""
    fp8 = _kv_format(fn, k_cache, v_cache, k_scale, v_scale)
    if k_cache.dim() != 4:
        raise ValueError(f'{fn}: the caches must be (B, nkv, max_len, hd), got {tuple(k_cache.shape)}')
    n, nkv, slots, hd = k_cache.shape
    kv = _lib.QuipKvCache(k=k_cache.data_ptr(), v=v_cache.data_ptr(), nkv=nkv, hd=hd,
                          format=_lib.QUIP_KV_E4M3 if fp8 else _lib.QUIP_KV_FP16)
    if page_table is None:
        kv.max_len = slots
        if n != rows:
            raise ValueError(f'{fn}: caches {tuple(k_cache.shape)} do not agree with {rows} rows')
    else:
        if (page_table.dtype != torch.int32 or page_table.dim() != 2 or page_table.shape[0] != rows or
                page_table.shape[1] < 1):
            raise ValueError(f'{fn}: page_table must be (B={rows}, max_pages >= 1) int32, got '
                             f'{tuple(page_table.shape)} {page_table.dtype}')
        if slots != KV_PAGE or n < 1:
            raise ValueError(f'{fn}: with a page table the caches are pools (n_pages, nkv, {KV_PAGE}, hd), got '
                             f'{tuple(k_cache.shape)}')
        if page_table.shape[1] > (2 ** 31 - 1) // KV_PAGE:
            raise ValueError(f'{fn}: {page_table.shape[1]} pages per row: max_pages * {KV_PAGE} must fit int32')
        if not page_table.is_cuda or page_table.device != k_cache.device or not page_table.is_contiguous():
            raise ValueError(f'{fn}: page_table must be a contiguous CUDA tensor on the caches\' device')
        if page_table.data_ptr() % 4 or k_cache.data_ptr() % 16 or v_cache.data_ptr() % 16:
            raise ValueError(f'{fn}: page_table must be 4-byte aligned and the pools 16-byte aligned')
        kv.page_table, kv.max_pages, kv.n_pages = page_table.data_ptr(), page_table.shape[1], n
        kv.max_len = page_table.shape[1] * KV_PAGE
    if v_cache.shape != k_cache.shape or (fp8 and (tuple(k_scale.shape) != (n, nkv, slots) or
                                                    v_scale.shape != k_scale.shape)):
        raise ValueError(f'{fn}: shapes caches {tuple(k_cache.shape)} / {tuple(v_cache.shape)}, scales '
                         f'{None if k_scale is None else tuple(k_scale.shape)} / '
                         f'{None if v_scale is None else tuple(v_scale.shape)} do not agree')
    if fp8:
        kv.k_scale, kv.v_scale = k_scale.data_ptr(), v_scale.data_ptr()
    return kv


def _check_cuda(fn, ts, dev):
    for t in ts:
        if t is None:
            continue
        if not t.is_cuda:
            raise RuntimeError(f'{fn} runs on a CUDA device only (there is no CPU fallback)')
        if t.device != dev:
            raise ValueError(f'{fn}: all tensors must be on one device')
        if not t.is_contiguous():
            raise ValueError(f'{fn} takes contiguous tensors')


def decode_attention(q, k_new, v_new, k_cache, v_cache, positions, scale, k_scale=None, v_scale=None, page_table=None):
    """quip_decode_attention on torch tensors: append k_new / v_new (B, nkv, hd) at slot positions[b] of one layer's
    k_cache / v_cache (B, nkv, max_len, hd) and attend q (B, nh, hd) over slots 0 .. positions[b].  fp16, CUDA,
    contiguous; positions (B,) int64 on the same device.  Returns (B, nh, hd) fp16, on the current stream.

    Caches of dtype torch.float8_e4m3fn need their per-slot fp32 scales k_scale / v_scale (B, nkv, max_len): k_new /
    v_new are quantized on append (include/quip_b200.h has the format).

    page_table (B, max_pages) int32: the caches are page pools (n_pages, nkv, 64, hd), scales (n_pages, nkv, 64), and
    slot j of row b lives at slot j % 64 of page page_table[b, j // 64]; a row that would touch a page id outside
    [0, n_pages) writes nothing there and gets NaN."""
    if q.dim() != 3:
        raise ValueError(f'decode_attention: q must be (B, nh, hd), got {tuple(q.shape)}')
    B, nh, hd = q.shape
    kv = _kv_cache('decode_attention', k_cache, v_cache, k_scale, v_scale, page_table, B)
    if any(t.dtype != torch.float16 for t in (q, k_new, v_new)) or positions.dtype != torch.int64:
        raise ValueError('decode_attention takes fp16 q / k / v and int64 positions')
    if (kv.hd != hd or tuple(k_new.shape) != (B, kv.nkv, hd) or v_new.shape != k_new.shape or
            tuple(positions.shape) != (B,)):
        raise ValueError(f'decode_attention: shapes q {tuple(q.shape)}, k_new {tuple(k_new.shape)}, v_new '
                         f'{tuple(v_new.shape)}, caches {tuple(k_cache.shape)}, positions {tuple(positions.shape)} do '
                         'not agree')
    _check_cuda('decode_attention', (q, k_new, v_new, k_cache, v_cache, k_scale, v_scale, positions), q.device)
    lib = _lib.load()
    need = C.c_size_t(0)
    _lib.check(lib.quip_decode_attention_workspace_bytes(B, nh, hd, kv.max_len, C.byref(need)))
    ws = torch.empty(max(int(need.value), 16), dtype=torch.uint8, device=q.device)
    out = torch.empty_like(q)
    st = torch.cuda.current_stream(q.device).cuda_stream
    with torch.cuda.device(q.device):
        _lib.check(lib.quip_decode_attention(C.byref(kv), q.data_ptr(), k_new.data_ptr(), v_new.data_ptr(),
                                             positions.data_ptr(), out.data_ptr(), B, nh, C.c_float(scale),
                                             ws.data_ptr(), ws.numel(), st))
    return out


def kv_quantize(src, cache, scales):
    """quip_kv_quantize_fp8 on torch tensors: quantize src (B, nkv, P, hd) fp16 into slots 0 .. P-1 of cache
    (B, nkv, max_len, hd) float8_e4m3fn and scales (B, nkv, max_len) fp32; slots >= P are not touched.  CUDA, one
    device, contiguous; on the current stream.  Dtypes and shapes are checked before the device."""
    if src.dtype != torch.float16 or cache.dtype != torch.float8_e4m3fn or scales.dtype != torch.float32:
        raise ValueError('kv_quantize takes fp16 src, a float8_e4m3fn cache and fp32 scales')
    if src.dim() != 4 or cache.dim() != 4:
        raise ValueError(f'kv_quantize: src must be (B, nkv, P, hd) and the cache (B, nkv, max_len, hd), got '
                         f'{tuple(src.shape)} and {tuple(cache.shape)}')
    B, nkv, P, hd = src.shape
    max_len = cache.shape[2]
    if tuple(cache.shape) != (B, nkv, max_len, hd) or tuple(scales.shape) != (B, nkv, max_len) or P > max_len:
        raise ValueError(f'kv_quantize: shapes src {tuple(src.shape)}, cache {tuple(cache.shape)}, scales '
                         f'{tuple(scales.shape)} do not agree')
    _check_cuda('kv_quantize', (src, cache, scales), src.device)
    with torch.cuda.device(src.device):
        _lib.check(_lib.load().quip_kv_quantize_fp8(src.data_ptr(), cache.data_ptr(), scales.data_ptr(), B, nkv, P,
                                                    max_len, hd, torch.cuda.current_stream(src.device).cuda_stream))


SAMPLE_MAX_V = 2 ** 24 - 1


def sample(logits, temperature, top_k, top_p, seed, step, out):
    """quip_sample on torch tensors: one token per row of logits (B, V) fp16 into out (B,) int64, by the rule of
    include/quip_b200.h (greedy rows T <= 0 or k == 1; else temperature, top-k, top-p and a Philox draw of (seed, step)).
    temperature / top_p (B,) fp32, top_k (B,) int32, seed (B,) int64 (the seeds' two's-complement bits, read as uint64)
    or uint64, step (1,) int64.  CUDA, one device, contiguous; on the current stream.  Returns out."""
    B = logits.shape[0] if logits.dim() == 2 else -1
    if logits.dim() != 2 or logits.dtype != torch.float16:
        raise ValueError(f'sample: logits must be (B, V) fp16, got {tuple(logits.shape)} {logits.dtype}')
    for name, t, dts in (('temperature', temperature, (torch.float32,)), ('top_k', top_k, (torch.int32,)),
                         ('top_p', top_p, (torch.float32,)), ('seed', seed, (torch.int64, torch.uint64)),
                         ('out', out, (torch.int64,))):
        if t.dtype not in dts or tuple(t.shape) != (B,):
            raise ValueError(f'sample: {name} must be ({B},) {" or ".join(str(d) for d in dts)}, got '
                             f'{tuple(t.shape)} {t.dtype}')
    if step.dtype != torch.int64 or step.numel() != 1:
        raise ValueError(f'sample: step must be one int64, got {tuple(step.shape)} {step.dtype}')
    if not 1 <= logits.shape[1] <= SAMPLE_MAX_V:
        raise ValueError(f'sample: need 1 <= V <= {SAMPLE_MAX_V} (the fixed-point sum of V weights), got V {logits.shape[1]}')
    _check_cuda('sample', (logits, temperature, top_k, top_p, seed, step, out), logits.device)
    with torch.cuda.device(logits.device):
        _lib.check(_lib.load().quip_sample(logits.data_ptr(), temperature.data_ptr(), top_k.data_ptr(), top_p.data_ptr(),
                                           seed.data_ptr(), step.data_ptr(), out.data_ptr(), B, logits.shape[1],
                                           torch.cuda.current_stream(logits.device).cuda_stream))
    return out


def token_logprobs(logits, targets, logprob_out, greedy_out):
    """quip_token_logprobs on torch tensors: for each row r of logits (R, V) fp16 (rows may be strided: stride(1) == 1,
    any stride(0) >= V) and targets (R,) int64, logprob_out[r] (fp32) = log_softmax(logits[r])[targets[r]] and
    greedy_out[r] (uint8) = 1 when targets[r] is the lowest index of the row's largest value (the rule of
    include/quip_b200.h: NaN rows and targets outside [0, V) give NaN and 0).  CUDA, one device; targets and the
    outputs contiguous.  Everything is checked before the launch, which runs on the current stream.  Returns
    (logprob_out, greedy_out)."""
    if logits.dim() != 2 or logits.dtype != torch.float16:
        raise ValueError(f'token_logprobs: logits must be (R, V) fp16, got {tuple(logits.shape)} {logits.dtype}')
    R, V = logits.shape
    if V < 1 or (R > 1 and logits.stride(0) < V) or (V > 1 and logits.stride(1) != 1):
        raise ValueError(f'token_logprobs: logits rows must be unit-stride and not overlap, got shape {tuple(logits.shape)}'
                         f' strides {tuple(logits.stride())}')
    if R > 2 ** 31 - 1:
        raise ValueError(f'token_logprobs: {R} rows exceed the launch limit of 2^31 - 1')
    for name, t, dt in (('targets', targets, torch.int64), ('logprob_out', logprob_out, torch.float32),
                        ('greedy_out', greedy_out, torch.uint8)):
        if t.dtype != dt or tuple(t.shape) != (R,):
            raise ValueError(f'token_logprobs: {name} must be ({R},) {dt}, got {tuple(t.shape)} {t.dtype}')
    for t in (logits, targets, logprob_out, greedy_out):
        if not t.is_cuda:
            raise RuntimeError('token_logprobs runs on a CUDA device only (there is no CPU fallback)')
        if t.device != logits.device:
            raise ValueError('token_logprobs: all tensors must be on one device')
    _check_cuda('token_logprobs', (targets, logprob_out, greedy_out), logits.device)
    ld = logits.stride(0) if R > 1 else V
    with torch.cuda.device(logits.device):
        _lib.check(_lib.load().quip_token_logprobs(logits.data_ptr(), ld, targets.data_ptr(), logprob_out.data_ptr(),
                                                   greedy_out.data_ptr(), R, V,
                                                   torch.cuda.current_stream(logits.device).cuda_stream))
    return logprob_out, greedy_out


TOPK_MAX_N, TOPK_MAX_T, TOPK_MAX_V = 20, 8, 2 ** 24


def token_topk_logprobs(logits, tokens, cols, lp, top_ids=None, top_lp=None, T=1, rows=None):
    """quip_token_topk_logprobs: for each row r of raw logits (R, V) fp16 (stride(1) == 1, any stride(0) >= V), offset
    r % T of decoder row b = rows[r // T] (rows (R // T,) int64; default r // T), writes at column
    c = cols[b] + r % T (cols (B,) int64, or (1,) shared by every row) lp[b, c] = log_softmax(logits[r])[tokens[r]]
    and the row's top n ids and logprobs into top_ids[b, c, :] / top_lp[b, c, :] (the rule of include/quip_b200.h;
    nothing is written when c is outside [0, gen_cols)).  tokens (R,) int64; lp (B, gen_cols) fp32; top_ids
    (B, gen_cols, n) int64 and top_lp (B, gen_cols, n) fp32 with 1 <= n <= 20, or both None.  CUDA, one device,
    outputs contiguous; everything is checked before the launch, which runs on the current stream.  Returns lp."""
    if logits.dim() != 2 or logits.dtype != torch.float16:
        raise ValueError(f'token_topk_logprobs: logits must be (R, V) fp16, got {tuple(logits.shape)} {logits.dtype}')
    R, V = logits.shape
    if not 1 <= V <= TOPK_MAX_V or (R > 1 and logits.stride(0) < V) or (V > 1 and logits.stride(1) != 1):
        raise ValueError(f'token_topk_logprobs: logits rows must be unit-stride, not overlap and hold 1 .. {TOPK_MAX_V}'
                         f' values, got shape {tuple(logits.shape)} strides {tuple(logits.stride())}')
    if isinstance(T, bool) or int(T) != T or not 1 <= T <= TOPK_MAX_T or R % T:
        raise ValueError(f'token_topk_logprobs: T must be an integer in [1, {TOPK_MAX_T}] dividing R = {R}, got {T!r}')
    if R > 2 ** 31 - 1:
        raise ValueError(f'token_topk_logprobs: {R} rows exceed the launch limit of 2^31 - 1')
    if lp.dim() != 2:
        raise ValueError(f'token_topk_logprobs: lp must be (B, gen_cols), got {tuple(lp.shape)}')
    B, G = lp.shape
    if (top_ids is None) != (top_lp is None):
        raise ValueError('token_topk_logprobs: pass top_ids and top_lp together, or neither')
    n = 0 if top_ids is None else (top_ids.shape[-1] if top_ids.dim() == 3 else -1)
    if top_ids is not None and not 1 <= n <= TOPK_MAX_N:
        raise ValueError(f'token_topk_logprobs: top_ids must be (B, gen_cols, n) with 1 <= n <= {TOPK_MAX_N}, got '
                         f'{tuple(top_ids.shape)}')
    if rows is None and R // T != B:
        raise ValueError(f'token_topk_logprobs: {R // T} logits rows of T = {T} for {B} output rows: pass rows')
    checks = [('tokens', tokens, torch.int64, (R,)), ('lp', lp, torch.float32, (B, G))]
    if cols.dtype != torch.int64 or tuple(cols.shape) not in ((B,), (1,)):
        raise ValueError(f'token_topk_logprobs: cols must be ({B},) or (1,) int64, got {tuple(cols.shape)} {cols.dtype}')
    checks.append(('cols', cols, torch.int64, tuple(cols.shape)))
    if top_ids is not None:
        checks += [('top_ids', top_ids, torch.int64, (B, G, n)), ('top_lp', top_lp, torch.float32, (B, G, n))]
    if rows is not None:
        checks.append(('rows', rows, torch.int64, (R // T,)))
    for name, t, dt, shape in checks:
        if t.dtype != dt or tuple(t.shape) != shape:
            raise ValueError(f'token_topk_logprobs: {name} must be {shape} {dt}, got {tuple(t.shape)} {t.dtype}')
    if not logits.is_cuda:
        raise RuntimeError('token_topk_logprobs runs on a CUDA device only (there is no CPU fallback)')
    _check_cuda('token_topk_logprobs', [t for _, t, _, _ in checks], logits.device)
    ld = logits.stride(0) if R > 1 else V
    p = lambda t: None if t is None else t.data_ptr()
    with torch.cuda.device(logits.device):
        _lib.check(_lib.load().quip_token_topk_logprobs(logits.data_ptr(), ld, R, int(T), V, p(rows), tokens.data_ptr(),
                                                        cols.data_ptr(), int(cols.numel() == B), lp.data_ptr(),
                                                        p(top_ids), p(top_lp),
                                                        n, B, G, torch.cuda.current_stream(logits.device).cuda_stream))
    return lp


def extend_attention(q, k_new, v_new, k_cache, v_cache, positions, scale, k_scale=None, v_scale=None, page_table=None):
    """quip_extend_attention on torch tensors: append token i of k_new / v_new (B, T, nkv, hd) at slot positions[b] + i
    of one layer's caches (B, nkv, max_len, hd) and attend q (B, T, nh, hd) causally over slots 0 .. positions[b] + i.
    fp16 q / k / v; fp16 caches, or float8_e4m3fn caches with fp32 k_scale / v_scale (B, nkv, max_len).  CUDA, one
    device, contiguous; positions (B,) int64.  Returns (B, T, nh, hd) fp16.  page_table: page pools as in
    decode_attention."""
    if q.dim() != 4:
        raise ValueError(f'extend_attention: q must be (B, T, nh, hd), got {tuple(q.shape)}')
    B, T, nh, hd = q.shape
    kv = _kv_cache('extend_attention', k_cache, v_cache, k_scale, v_scale, page_table, B)
    if any(t.dtype != torch.float16 for t in (q, k_new, v_new)) or positions.dtype != torch.int64:
        raise ValueError('extend_attention takes fp16 q / k / v and int64 positions')
    if (kv.hd != hd or tuple(k_new.shape) != (B, T, kv.nkv, hd) or v_new.shape != k_new.shape or
            tuple(positions.shape) != (B,)):
        raise ValueError(f'extend_attention: shapes q {tuple(q.shape)}, k_new {tuple(k_new.shape)}, v_new '
                         f'{tuple(v_new.shape)}, caches {tuple(k_cache.shape)}, positions {tuple(positions.shape)} do '
                         'not agree')
    _check_cuda('extend_attention', (q, k_new, v_new, k_cache, v_cache, k_scale, v_scale, positions), q.device)
    lib = _lib.load()
    need = C.c_size_t(0)
    _lib.check(lib.quip_extend_attention_workspace_bytes(B, T, nh, hd, kv.max_len, C.byref(need)))
    ws = torch.empty(max(int(need.value), 16), dtype=torch.uint8, device=q.device)
    out = torch.empty_like(q)
    st = torch.cuda.current_stream(q.device).cuda_stream
    with torch.cuda.device(q.device):
        _lib.check(lib.quip_extend_attention(C.byref(kv), q.data_ptr(), k_new.data_ptr(), v_new.data_ptr(),
                                             positions.data_ptr(), out.data_ptr(), B, T, nh, C.c_float(scale),
                                             ws.data_ptr(), ws.numel(), st))
    return out


def _check_chunk(fn, positions, counts):
    """The operand checks kv_append and prefill_attention share: positions and counts (B,) int64.  Returns B."""
    if positions.dtype != torch.int64 or counts.dtype != torch.int64:
        raise ValueError(f'{fn} takes int64 positions and counts')
    if positions.dim() != 1 or counts.shape != positions.shape:
        raise ValueError(f'{fn}: shapes positions {tuple(positions.shape)}, counts {tuple(counts.shape)} do not agree')
    return positions.shape[0]


def kv_append(k_new, v_new, k_cache, v_cache, positions, counts, k_scale=None, v_scale=None, page_table=None):
    """quip_kv_append on torch tensors: token i of k_new / v_new (B, T, nkv, hd) fp16 to slot positions[b] + i of one
    layer's caches (B, nkv, max_len, hd) for i < counts[b]; nothing else is written.  fp16 caches, or float8_e4m3fn
    caches with fp32 k_scale / v_scale (B, nkv, max_len), quantized on the way.  CUDA, one device, contiguous;
    positions / counts (B,) int64.  On the current stream.  page_table: page pools as in decode_attention; a slot whose
    page id lies outside the pool is not written."""
    B = _check_chunk('kv_append', positions, counts)
    kv = _kv_cache('kv_append', k_cache, v_cache, k_scale, v_scale, page_table, B)
    if k_new.dtype != torch.float16 or v_new.dtype != torch.float16:
        raise ValueError('kv_append takes fp16 k_new / v_new')
    if (k_new.dim() != 4 or k_new.shape[0] != B or tuple(k_new.shape[2:]) != (kv.nkv, kv.hd) or
            v_new.shape != k_new.shape):
        raise ValueError(f'kv_append: k_new {tuple(k_new.shape)} / v_new {tuple(v_new.shape)} must be (B, T, nkv, hd) '
                         f'for caches {tuple(k_cache.shape)}')
    _check_cuda('kv_append', (k_new, v_new, k_cache, v_cache, k_scale, v_scale, positions, counts), k_new.device)
    with torch.cuda.device(k_new.device):
        _lib.check(_lib.load().quip_kv_append(C.byref(kv), k_new.data_ptr(), v_new.data_ptr(), positions.data_ptr(),
                                              counts.data_ptr(), B, k_new.shape[1],
                                              torch.cuda.current_stream(k_new.device).cuda_stream))


def prefill_attention(q, k_cache, v_cache, positions, counts, scale, k_scale=None, v_scale=None, page_table=None):
    """quip_prefill_attention on torch tensors: q (B, T, nh, hd) fp16 attends causally over one layer's caches
    (B, nkv, max_len, hd), which already hold the chunk (kv_append): token i of row b over slots 0 .. positions[b] + i
    for i < counts[b]; rows i >= counts[b] are zero.  fp16 caches, or float8_e4m3fn caches with fp32 k_scale / v_scale.
    CUDA, one device, contiguous; positions / counts (B,) int64.  Returns (B, T, nh, hd) fp16, on the current stream.
    page_table: page pools as in decode_attention."""
    B = _check_chunk('prefill_attention', positions, counts)
    kv = _kv_cache('prefill_attention', k_cache, v_cache, k_scale, v_scale, page_table, B)
    if q.dtype != torch.float16 or q.dim() != 4:
        raise ValueError(f'prefill_attention: q must be (B, T, nh, hd) fp16, got {tuple(q.shape)} {q.dtype}')
    T, nh, hd = q.shape[1:]
    if q.shape[0] != B or kv.hd != hd:
        raise ValueError(f'prefill_attention: q {tuple(q.shape)} and caches {tuple(k_cache.shape)} do not agree')
    _check_cuda('prefill_attention', (q, k_cache, v_cache, k_scale, v_scale, positions, counts), q.device)
    out = torch.empty_like(q)
    with torch.cuda.device(q.device):
        _lib.check(_lib.load().quip_prefill_attention(C.byref(kv), q.data_ptr(), positions.data_ptr(),
                                                      counts.data_ptr(), out.data_ptr(), B, T, nh, C.c_float(scale),
                                                      torch.cuda.current_stream(q.device).cuda_stream))
    return out


class RaggedChunk:
    """The sequences of a ragged (packed) chunk: seq_start, S + 1 offsets with 0 = seq_start[0] <= ... <= seq_start[S]
    = N, so sequence s is the packed token rows seq_start[s] .. seq_start[s + 1] - 1 and every row belongs to one
    sequence.  The offsets are checked on the host when the chunk is made; `seq_start` is their device copy, which every
    layer's ragged launches read, so a step checks and copies them once."""

    def __init__(self, seq_start, device):
        offs = seq_start.tolist() if torch.is_tensor(seq_start) else list(seq_start)
        if len(offs) < 2 or any(int(x) != x for x in offs):
            raise ValueError(f'seq_start must hold S + 1 >= 2 integer offsets, got {offs}')
        offs = [int(x) for x in offs]
        if offs[0] != 0 or any(b < a for a, b in zip(offs, offs[1:])):
            raise ValueError(f'seq_start must rise monotonically from 0, got {offs}')
        if len(offs) - 1 > 65535 or offs[-1] > 2 ** 31 - 1:
            raise ValueError(f'{len(offs) - 1} sequences of {offs[-1]} tokens: at most 65535 sequences and 2^31 - 1 '
                             'tokens')
        self.offsets = offs
        self.S, self.N = len(offs) - 1, offs[-1]
        self.max_count = max(1, max(b - a for a, b in zip(offs, offs[1:])))
        self.seq_start = torch.tensor(offs, dtype=torch.int64).to(device)


def _check_ragged(fn, seqs, positions, page_table, dev):
    """The operand checks kv_append_ragged and prefill_attention_ragged share: the chunk, on the pools' device dev,
    positions (S,) int64 and a page table."""
    if not isinstance(seqs, RaggedChunk):
        raise ValueError(f'{fn}: seqs must be a RaggedChunk (its offsets are checked when it is made)')
    if page_table is None:
        raise ValueError(f'{fn}: a ragged chunk is paged only: pass the page_table')
    if positions.dtype != torch.int64 or tuple(positions.shape) != (seqs.S,):
        raise ValueError(f'{fn}: positions must be ({seqs.S},) int64 for {seqs.S} sequences, got '
                         f'{tuple(positions.shape)} {positions.dtype}')
    if seqs.seq_start.device != dev:
        raise ValueError(f'{fn}: the chunk\'s offsets live on {seqs.seq_start.device}, the pools on {dev}')


def kv_append_ragged(k_new, v_new, k_pool, v_pool, seqs, positions, page_table, k_scale=None, v_scale=None):
    """quip_kv_append_ragged on torch tensors: packed row seq_start[s] + i of k_new / v_new (N, nkv, hd) fp16 -- token
    i of sequence s (seqs: a RaggedChunk) -- to slot positions[s] + i of row s of page_table (S, max_pages) int32, in
    one layer's pools (n_pages, nkv, 64, hd): fp16, or float8_e4m3fn with fp32 k_scale / v_scale (n_pages, nkv, 64),
    quantized on the way.  A sequence whose slots leave the cache, or a slot whose page id lies outside the pool, writes
    nothing.  CUDA, one device, contiguous; positions (S,) int64.  Everything is checked before the launch, which runs on
    the current stream."""
    _check_ragged('kv_append_ragged', seqs, positions, page_table, k_pool.device)
    kv = _kv_cache('kv_append_ragged', k_pool, v_pool, k_scale, v_scale, page_table, seqs.S)
    if k_new.dtype != torch.float16 or v_new.dtype != torch.float16:
        raise ValueError('kv_append_ragged takes fp16 k_new / v_new')
    if tuple(k_new.shape) != (seqs.N, kv.nkv, kv.hd) or v_new.shape != k_new.shape:
        raise ValueError(f'kv_append_ragged: k_new {tuple(k_new.shape)} / v_new {tuple(v_new.shape)} must be '
                         f'(N={seqs.N}, nkv={kv.nkv}, hd={kv.hd})')
    _check_cuda('kv_append_ragged', (k_new, v_new, k_pool, v_pool, k_scale, v_scale, positions), k_new.device)
    with torch.cuda.device(k_new.device):
        _lib.check(_lib.load().quip_kv_append_ragged(C.byref(kv), k_new.data_ptr(), v_new.data_ptr(),
                                                     seqs.seq_start.data_ptr(), positions.data_ptr(), seqs.S, seqs.N,
                                                     seqs.max_count,
                                                     torch.cuda.current_stream(k_new.device).cuda_stream))


def prefill_attention_ragged(q, k_pool, v_pool, seqs, positions, page_table, scale, k_scale=None, v_scale=None):
    """quip_prefill_attention_ragged on torch tensors: packed row seq_start[s] + i of q (N, nh, hd) fp16 -- token i of
    sequence s (seqs: a RaggedChunk) -- attends causally over slots 0 .. positions[s] + i of row s of page_table
    (S, max_pages), in one layer's pools that already hold the chunk (kv_append_ragged).  Returns (N, nh, hd) fp16, on
    the current stream.  Per sequence the result is bit-identical to prefill_attention with page_table, B = S,
    T = seqs.max_count and counts = the sequence lengths (include/quip_b200.h); a sequence that would read a slot
    outside the cache or a page outside the pool gets NaN.  Pools, scales and checks as kv_append_ragged."""
    _check_ragged('prefill_attention_ragged', seqs, positions, page_table, k_pool.device)
    kv = _kv_cache('prefill_attention_ragged', k_pool, v_pool, k_scale, v_scale, page_table, seqs.S)
    if q.dtype != torch.float16 or q.dim() != 3 or q.shape[0] != seqs.N or q.shape[2] != kv.hd:
        raise ValueError(f'prefill_attention_ragged: q must be (N={seqs.N}, nh, hd={kv.hd}) fp16, got '
                         f'{tuple(q.shape)} {q.dtype}')
    _check_cuda('prefill_attention_ragged', (q, k_pool, v_pool, k_scale, v_scale, positions), q.device)
    out = torch.empty_like(q)
    with torch.cuda.device(q.device):
        _lib.check(_lib.load().quip_prefill_attention_ragged(C.byref(kv), q.data_ptr(), seqs.seq_start.data_ptr(),
                                                             positions.data_ptr(), out.data_ptr(), seqs.S, seqs.N,
                                                             seqs.max_count, q.shape[1], C.c_float(scale),
                                                             torch.cuda.current_stream(q.device).cuda_stream))
    return out


def sample_at(logits, temperature, top_k, top_p, seed, steps, out):
    """quip_sample_at: logits (B, T, V) fp16 -> out (B, T) int64, token i of row b by the rule of quip_sample with row b's
    settings and seed at step steps[b] + i (steps (B,) int64).  CUDA, one device, contiguous; on the current stream."""
    if logits.dim() != 3 or logits.dtype != torch.float16:
        raise ValueError(f'sample_at: logits must be (B, T, V) fp16, got {tuple(logits.shape)} {logits.dtype}')
    B, T, V = logits.shape
    for name, t, dts, shape in (('temperature', temperature, (torch.float32,), (B,)),
                                ('top_k', top_k, (torch.int32,), (B,)), ('top_p', top_p, (torch.float32,), (B,)),
                                ('seed', seed, (torch.int64, torch.uint64), (B,)), ('steps', steps, (torch.int64,), (B,)),
                                ('out', out, (torch.int64,), (B, T))):
        if t.dtype not in dts or tuple(t.shape) != shape:
            raise ValueError(f'sample_at: {name} must be {shape} {" or ".join(str(d) for d in dts)}, got '
                             f'{tuple(t.shape)} {t.dtype}')
    if not 1 <= V <= SAMPLE_MAX_V:
        raise ValueError(f'sample_at: need 1 <= V <= {SAMPLE_MAX_V} (the fixed-point sum of V weights), got V {V}')
    _check_cuda('sample_at', (logits, temperature, top_k, top_p, seed, steps, out), logits.device)
    with torch.cuda.device(logits.device):
        _lib.check(_lib.load().quip_sample_at(logits.data_ptr(), temperature.data_ptr(), top_k.data_ptr(),
                                              top_p.data_ptr(), seed.data_ptr(), steps.data_ptr(), out.data_ptr(), B, T, V,
                                              torch.cuda.current_stream(logits.device).cuda_stream))
    return out


def _check_i64(fn, **ts):
    for name, (t, shape) in ts.items():
        if t.dtype != torch.int64 or tuple(t.shape) != tuple(shape):
            raise ValueError(f'{fn}: {name} must be {tuple(shape)} int64, got {tuple(t.shape)} {t.dtype}')


def ngram_draft(hist, positions, tokens, n_min, n_max):
    """quip_ngram_draft: tokens (B, 1 + k) = the current token hist[b, positions[b]] and k prompt-lookup drafts from
    hist (B, max_len) (the rule is in include/quip_b200.h).  int64, CUDA, contiguous.  Returns tokens."""
    B, max_len = hist.shape
    _check_i64('ngram_draft', hist=(hist, (B, max_len)), positions=(positions, (B,)),
               tokens=(tokens, (B, tokens.shape[-1] if tokens.dim() == 2 else -1)))
    _check_cuda('ngram_draft', (hist, positions, tokens), hist.device)
    with torch.cuda.device(hist.device):
        _lib.check(_lib.load().quip_ngram_draft(hist.data_ptr(), positions.data_ptr(), tokens.data_ptr(), B, max_len,
                                                tokens.shape[1] - 1, n_min, n_max,
                                                torch.cuda.current_stream(hist.device).cuda_stream))
    return tokens


def spec_accept(tokens, targets, generated, hist, positions, n_gen, accepted, max_new):
    """quip_spec_accept: accept the longest matching prefix of drafts plus one token per unfinished row (the rule is in
    include/quip_b200.h), writing generated (B, >= max_new) and hist (B, max_len) and advancing positions, n_gen and
    accepted (B,).  int64, CUDA, contiguous."""
    B, T = tokens.shape
    _check_i64('spec_accept', tokens=(tokens, (B, T)), targets=(targets, (B, T)),
               generated=(generated, (B, generated.shape[-1])), hist=(hist, (B, hist.shape[-1])),
               positions=(positions, (B,)), n_gen=(n_gen, (B,)), accepted=(accepted, (B,)))
    _check_cuda('spec_accept', (tokens, targets, generated, hist, positions, n_gen, accepted), tokens.device)
    with torch.cuda.device(tokens.device):
        _lib.check(_lib.load().quip_spec_accept(tokens.data_ptr(), targets.data_ptr(), generated.data_ptr(),
                                                hist.data_ptr(), positions.data_ptr(), n_gen.data_ptr(),
                                                accepted.data_ptr(), B, T, max_new, generated.shape[1], hist.shape[1],
                                                torch.cuda.current_stream(tokens.device).cuda_stream))


def mlp_layout_plan(mlp):
    """The combined index of the three permutations around SiLU(gate) * up of a packed Llama MLP -- the output gathers of
    gate_proj / up_proj (y[j] = layout[u_idx[j]]) and the input gather of down_proj (layout[l] = x[v_idx[l]]) -- so that one
    kernel (quip_silu_mul_gather) replaces three gather launches and silu_mul: for an 11008-wide side the gather is a kernel of
    its own.  None when the layers are not packed, have a bias /
    unfolded 1/s at those gathers, or are too wide for 16-bit positions.  Cached on the module."""
    from .quant import QuantLinear
    gate, up, down = mlp.gate_proj, mlp.up_proj, mlp.down_proj
    if not all(isinstance(m, QuantLinear) for m in (gate, up, down)):
        return None
    dev = gate.qweight.device
    cached = getattr(mlp, '_quip_layout_plan', None)
    if cached is not None and cached[0] == dev:
        return cached[1]
    plan = None
    n = gate.outfeatures
    if (dev.type == 'cuda' and n == up.outfeatures == down.infeatures and n % 8 == 0 and n < 65536 and
            gate.layout_variant_ok(skip_out=True) and up.layout_variant_ok(skip_out=True) and down.layout_variant_ok(skip_in=True)):
        ar = torch.arange(n, device=dev)
        ig, iu, idn = (i if i is not None else ar for i in (gate.gather_index('u'), up.gather_index('u'), down.gather_index('v')))
        comb = ig[idn] | (iu[idn] << 16)                                     # int64, < 2^32
        plan = torch.where(comb >= 2 ** 31, comb - 2 ** 32, comb).to(torch.int32).contiguous()
    mlp._quip_layout_plan = (dev, plan)
    return plan


def enabled():
    """The fused stack is opt-in (QUIP_FUSED_LAYER=1): the library default is the HF modules' own glue, the reference's; bench.py
    and GraphDecoder switch it on after checking it against the HF layers in the run (bit-exact ops, one-ulp norms)."""
    return os.environ.get('QUIP_FUSED_LAYER') == '1'


def supports(model, h, kwargs):
    """Llama-family model, one fp16 sample, SiLU MLP, HF default rotary application, SDPA attention."""
    cfg = getattr(model, 'config', None)
    if cfg is None or getattr(cfg, 'model_type', None) != 'llama':
        return False
    if getattr(cfg, 'hidden_act', 'silu') != 'silu' or getattr(cfg, '_attn_implementation', 'sdpa') not in ('sdpa', None):
        return False
    if h.dim() != 3 or h.shape[0] != 1 or h.dtype != torch.float16:
        return False
    pe = kwargs.get('position_embeddings')
    if pe is None or pe[0].shape[0] != 1 or pe[0].dtype != torch.float16:
        return False
    hd = getattr(cfg, 'head_dim', None) or cfg.hidden_size // cfg.num_attention_heads
    return hd % 16 == 0 and cfg.hidden_size % 8 == 0 and cfg.intermediate_size % 8 == 0


def llama_stack(layers, h, kwargs, ops=None, trace=None, fold_gathers=None):
    """`for layer in layers: h = layer(h, **kwargs)` for LlamaDecoderLayers on one sample h (1, S, hidden).  `trace`: an optional
    list that receives (layer index, stage name, tensor) for tools/glue_bisect.py."""
    ops = ops or CudaGlue()
    if fold_gathers is None:
        fold_gathers = trace is None and os.environ.get('QUIP_FOLD_GATHERS', '1') == '1'
    cos, sin = kwargs['position_embeddings']
    cos, sin = cos[0].contiguous(), sin[0].contiguous()                     # (S, head_dim)
    mask = kwargs.get('attention_mask')
    S = h.shape[1]
    pend = None                        # previous layer's MLP output, not yet added to h
    x = None
    h = h.contiguous()

    def rec(li, name, t):
        if trace is not None:
            trace.append((li, name, t.clone()))

    for li, layer in enumerate(layers):
        a, mlp = layer.self_attn, layer.mlp
        n1, n2 = layer.input_layernorm, layer.post_attention_layernorm
        hd = a.head_dim
        if pend is None:
            x = ops.rmsnorm(h, n1.weight, n1.variance_epsilon)
        else:
            h, x = ops.rmsnorm(h, n1.weight, n1.variance_epsilon, residual=pend)
        rec(li, 'h_in', h)
        rec(li, 'x_attn', x)
        q, k, v = a.q_proj(x), a.k_proj(x), a.v_proj(x)                     # sibling groups launch these concurrently
        for nm, t in (('q_lin', q), ('k_lin', k), ('v_lin', v)):
            rec(li, nm, t)
        ops.rope_(q, k, cos, sin, hd)
        rec(li, 'q_rope', q)
        rec(li, 'k_rope', k)
        nq, nkv = q.shape[-1] // hd, k.shape[-1] // hd
        qh = q.view(1, S, nq, hd).transpose(1, 2)
        kh = k.view(1, S, nkv, hd).transpose(1, 2)
        vh = v.view(1, S, nkv, hd).transpose(1, 2)
        extra = {}
        # the same call transformers' sdpa_attention_forward makes (enable_gqa whenever there is no mask, also for
        # nkv == nq), so that torch picks the same SDPA backend for both glues
        if mask is None:
            extra['enable_gqa'] = True
        elif nkv != nq:
            kh = kh.repeat_interleave(nq // nkv, dim=1)
            vh = vh.repeat_interleave(nq // nkv, dim=1)
        o = F.scaled_dot_product_attention(qh, kh, vh, attn_mask=mask, dropout_p=0.0, scale=a.scaling,
                                           is_causal=(mask is None and S > 1), **extra)
        o = o.transpose(1, 2).reshape(1, S, nq * hd).contiguous()
        rec(li, 'attn_out', o)
        ao = a.o_proj(o)
        rec(li, 'o_lin', ao)
        h, x = ops.rmsnorm(h, n2.weight, n2.variance_epsilon, residual=ao)
        rec(li, 'h_mid', h)
        rec(li, 'x_mlp', x)
        plan = mlp_layout_plan(mlp) if (fold_gathers and hasattr(ops, 'silu_mul_gather')) else None
        if plan is not None:
            # gate / up stay in their N-side layout order, the product lands in down_proj's K-side layout order: one kernel
            # instead of three gathers + silu_mul (same arithmetic per element, only the data movement differs)
            g, u = mlp.gate_proj.forward_layout(x, skip_out=True), mlp.up_proj.forward_layout(x, skip_out=True)
            act = ops.silu_mul_gather(g, u, plan)
            pend = mlp.down_proj.forward_layout(act, skip_in=True)
        else:
            g, u = mlp.gate_proj(x), mlp.up_proj(x)
            rec(li, 'gate', g)
            rec(li, 'up', u)
            act = ops.silu_mul(g, u)
            rec(li, 'act', act)
            pend = mlp.down_proj(act)
        rec(li, 'down', pend)
    return h if pend is None else h + pend


BEAM_MAX_K, BEAM_MAX_C, BEAM_MAX_EOS = 16, 64, 3


def beam_candidates(logits, scores, K, C, cand_s, cand_i):
    """quip_beam_candidates: for each row r of logits (R, V) fp16 (stride(1) == 1, any stride(0) >= V) with score
    scores[r] (fp32), the top C of s = log_softmax(row) + score in rank order (s descending, then lower flat index
    (r % K) * V + v; NaN last) into cand_s (R, C) fp32 and cand_i (R, C) int32 (include/quip_b200.h has the rule; rows
    with V < C are padded with (NaN, -1)).  CUDA, one device; everything is checked before the launch, which runs on
    the current stream.  Returns (cand_s, cand_i)."""
    if logits.dim() != 2 or logits.dtype != torch.float16:
        raise ValueError(f'beam_candidates: logits must be (R, V) fp16, got {tuple(logits.shape)} {logits.dtype}')
    R, V = logits.shape
    if V < 1 or (R > 1 and logits.stride(0) < V) or (V > 1 and logits.stride(1) != 1):
        raise ValueError(f'beam_candidates: logits rows must be unit-stride and not overlap, got shape '
                         f'{tuple(logits.shape)} strides {tuple(logits.stride())}')
    if not (1 <= K <= BEAM_MAX_K and 1 <= C <= BEAM_MAX_C) or V > 2 ** 24 or K * V > 2 ** 31 - 1:
        raise ValueError(f'beam_candidates: need 1 <= K <= {BEAM_MAX_K}, 1 <= C <= {BEAM_MAX_C}, V <= 2^24, got K {K}, '
                         f'C {C}, V {V}')
    for name, t, dt, shape in (('scores', scores, torch.float32, (R,)), ('cand_s', cand_s, torch.float32, (R, C)),
                               ('cand_i', cand_i, torch.int32, (R, C))):
        if t.dtype != dt or tuple(t.shape) != shape:
            raise ValueError(f'beam_candidates: {name} must be {shape} {dt}, got {tuple(t.shape)} {t.dtype}')
    if not logits.is_cuda:
        raise RuntimeError('beam_candidates runs on a CUDA device only (there is no CPU fallback)')
    _check_cuda('beam_candidates', (scores, cand_s, cand_i), logits.device)
    ld = logits.stride(0) if R > 1 else V
    with torch.cuda.device(logits.device):
        _lib.check(_lib.load().quip_beam_candidates(logits.data_ptr(), ld, scores.data_ptr(), cand_s.data_ptr(),
                                                    cand_i.data_ptr(), R, V, K, C,
                                                    torch.cuda.current_stream(logits.device).cuda_stream))
    return cand_s, cand_i


ES_MODES = {False: 0, True: 1, 'never': 2}


def beam_select(cand_s, cand_i, eos, budget, step, pen, st, K, V, early_stopping, never_long):
    """quip_beam_select: merge each prompt's K candidate lists (cand_s / cand_i (B * K, C), beam_candidates) and apply
    HF's running-beam, finished-slot, early-stop and done rules (include/quip_b200.h) at step step (1,) int64, with
    eos (n_eos <= 3,) int64, budget (B,) int64 and pen (max_new + 1,) fp32 = n ** length_penalty.  st: the state
    tensors by name -- score (B * K,) fp32; hist, hist_tmp, fin_tok, fin_tmp (B, K, max_new) int64; fin_score (B, K)
    fp32; fin_len (B, K) int64; fin_filled (B, K), heur (B,), done (B,) uint8; tokens, parents, adv (B * K,) int64 --
    updated in place.  early_stopping: False, True or 'never'.  CUDA, one device, contiguous; checked before the
    launch, which runs on the current stream."""
    if early_stopping not in ES_MODES:
        raise ValueError(f"beam_select: early_stopping must be False, True or 'never', got {early_stopping!r}")
    if cand_s.dim() != 2 or cand_s.dtype != torch.float32 or cand_i.dtype != torch.int32 or cand_i.shape != cand_s.shape:
        raise ValueError(f'beam_select: cand_s (R, C) fp32 and cand_i (R, C) int32, got {tuple(cand_s.shape)} '
                         f'{cand_s.dtype} / {tuple(cand_i.shape)} {cand_i.dtype}')
    R, C = cand_s.shape
    if not (1 <= K <= BEAM_MAX_K and K <= C <= BEAM_MAX_C) or R % K or K * V > 2 ** 31 - 1 or V < 1:
        raise ValueError(f'beam_select: need 1 <= K <= {BEAM_MAX_K}, K <= C <= {BEAM_MAX_C}, K | R, got R {R}, K {K}, '
                         f'C {C}, V {V}')
    B = R // K
    max_new = st['hist'].shape[-1] if st['hist'].dim() == 3 else -1
    if max_new < 1 or eos.dim() != 1 or eos.numel() > BEAM_MAX_EOS:
        raise ValueError(f'beam_select: hist must be (B, K, max_new >= 1) and eos at most {BEAM_MAX_EOS} ids')
    want = dict(score=((R,), torch.float32), hist=((B, K, max_new), torch.int64),
                hist_tmp=((B, K, max_new), torch.int64), fin_score=((B, K), torch.float32),
                fin_len=((B, K), torch.int64), fin_tok=((B, K, max_new), torch.int64),
                fin_tmp=((B, K, max_new), torch.int64), fin_filled=((B, K), torch.uint8), heur=((B,), torch.uint8),
                done=((B,), torch.uint8), tokens=((R,), torch.int64), parents=((R,), torch.int64),
                adv=((R,), torch.int64))
    args = [('eos', eos, eos.shape, torch.int64), ('budget', budget, (B,), torch.int64),
            ('step', step, (1,), torch.int64), ('pen', pen, (max_new + 1,), torch.float32)]
    args += [(n, st[n], shape, dt) for n, (shape, dt) in want.items()]
    for name, t, shape, dt in args:
        if t.dtype != dt or tuple(t.shape) != tuple(shape):
            raise ValueError(f'beam_select: {name} must be {tuple(shape)} {dt}, got {tuple(t.shape)} {t.dtype}')
    _check_cuda('beam_select', [cand_s, cand_i] + [t for _, t, _, _ in args], cand_s.device)
    with torch.cuda.device(cand_s.device):
        _lib.check(_lib.load().quip_beam_select(
            cand_s.data_ptr(), cand_i.data_ptr(), eos.data_ptr() if eos.numel() else None, eos.numel(),
            budget.data_ptr(), step.data_ptr(), pen.data_ptr(), *[st[n].data_ptr() for n in want if n != 'adv'],
            st['adv'].data_ptr(), B, K, C, V, max_new, ES_MODES[early_stopping], int(bool(never_long)),
            torch.cuda.current_stream(cand_s.device).cuda_stream))


def kv_beam_fork(k_pool, v_pool, table, table_tmp, parents, lens, scratch0, k_scale=None, v_scale=None):
    """quip_kv_beam_fork: after a beam select, row r with parents[r] != r takes its parent's table entries for the
    spans before its current one and a copy of its parent's slots 64 * cur .. lens[r] - 1 of the current span, in every
    layer of the pools k_pool / v_pool (L, n_pages, nkv, 64, hd) (fp16, or float8_e4m3fn with fp32 k_scale / v_scale
    (L, n_pages, nkv, 64)), through scratch pages scratch0 .. scratch0 + R - 1 (include/quip_b200.h).  table /
    table_tmp (R, max_pages) int32, parents / lens (R,) int64.  CUDA, one device, contiguous; checked before the
    launches (two, on the current stream)."""
    fp8 = _kv_format('kv_beam_fork', k_pool, v_pool, k_scale, v_scale)
    if k_pool.dim() != 5 or k_pool.shape[0] < 1 or k_pool.shape[3] != KV_PAGE or v_pool.shape != k_pool.shape:
        raise ValueError(f'kv_beam_fork: pools must be (L, n_pages, nkv, {KV_PAGE}, hd), got {tuple(k_pool.shape)} / '
                         f'{tuple(v_pool.shape)}')
    L, n_pages, nkv, _, hd = k_pool.shape
    if (hd * k_pool.element_size()) % 16:
        raise ValueError(f'kv_beam_fork: a head vector must be a multiple of 16 bytes, got hd {hd}')
    if fp8 and (tuple(k_scale.shape) != (L, n_pages, nkv, KV_PAGE) or v_scale.shape != k_scale.shape):
        raise ValueError(f'kv_beam_fork: scales must be {(L, n_pages, nkv, KV_PAGE)} fp32')
    if table.dtype != torch.int32 or table.dim() != 2 or table_tmp.shape != table.shape or table_tmp.dtype != torch.int32:
        raise ValueError(f'kv_beam_fork: table and table_tmp must be (R, max_pages) int32, got {tuple(table.shape)} / '
                         f'{tuple(table_tmp.shape)}')
    R = table.shape[0]
    _check_i64('kv_beam_fork', parents=(parents, (R,)), lens=(lens, (R,)))
    if isinstance(scratch0, bool) or int(scratch0) != scratch0 or not 0 <= scratch0 <= n_pages - R:
        raise ValueError(f'kv_beam_fork: scratch pages {scratch0} .. {scratch0} + {R} - 1 lie outside the pool of '
                         f'{n_pages}')
    _check_cuda('kv_beam_fork', (k_pool, v_pool, k_scale, v_scale, table, table_tmp, parents, lens), k_pool.device)
    kv = _kv_cache('kv_beam_fork', k_pool[0], v_pool[0], k_scale[0] if fp8 else None, v_scale[0] if fp8 else None,
                   table, R)                                         # layer 0; the kernels step n_pages per layer
    with torch.cuda.device(k_pool.device):
        _lib.check(_lib.load().quip_kv_beam_fork(C.byref(kv), L, table_tmp.data_ptr(), parents.data_ptr(),
                                                 lens.data_ptr(), R, int(scratch0),
                                                 torch.cuda.current_stream(k_pool.device).cuda_stream))


PROC_MAX_V, PROC_MAX_EOS, PROC_MAX_BAD, PROC_BAD_LEN = 2 ** 18, 8, 256, 16


def logits_process(logits, T, hist, last, prompt_len, penalty, ngram, min_new, eos, bad, bad_len, tokens=None,
                   rows=None):
    """quip_logits_process: the repetition penalty, no-repeat n-gram, bad-word and min_new_tokens rule of
    include/quip_b200.h, in place on logits (R, V) fp16 (stride(1) == 1, any stride(0) >= V).  Row r is offset r % T of
    decoder row rows[r // T] (rows (R // T,) int64; default r // T), whose history is hist[b, :last[b] + 1] (hist
    (B, max_len) int64, last (B,) int64) and the drafts tokens[b, 1 .. r % T] (tokens (B, T) int64, needed when T > 1).
    prompt_len (B,) int64, penalty (B,) fp32, ngram and min_new (B,) int32; eos (n_eos <= 8,) int64; bad (n_bad <= 256,
    16) int64 with bad_len (n_bad,) int32 in [1, 16].  CUDA, one device; everything is checked before the launch, which
    runs on the current stream.  Returns logits."""
    if logits.dim() != 2 or logits.dtype != torch.float16:
        raise ValueError(f'logits_process: logits must be (R, V) fp16, got {tuple(logits.shape)} {logits.dtype}')
    R, V = logits.shape
    if not 1 <= V <= PROC_MAX_V or (R > 1 and logits.stride(0) < V) or (V > 1 and logits.stride(1) != 1):
        raise ValueError(f'logits_process: logits rows must be unit-stride, not overlap and hold 1 .. {PROC_MAX_V} '
                         f'values, got shape {tuple(logits.shape)} strides {tuple(logits.stride())}')
    if isinstance(T, bool) or int(T) != T or T < 1 or R % T:
        raise ValueError(f'logits_process: T must be an integer >= 1 dividing R = {R}, got {T!r}')
    if hist.dim() != 2:
        raise ValueError(f'logits_process: hist must be (B, max_len), got {tuple(hist.shape)}')
    B, max_len = hist.shape
    n_eos, n_bad = eos.numel(), bad.shape[0] if bad.dim() == 2 else -1
    if not 0 <= n_eos <= PROC_MAX_EOS or not 0 <= n_bad <= PROC_MAX_BAD:
        raise ValueError(f'logits_process: at most {PROC_MAX_EOS} eos ids and {PROC_MAX_BAD} bad words, got {n_eos} '
                         f'and {n_bad}')
    if T > 1 and tokens is None:
        raise ValueError('logits_process: T > 1 needs the drafts (tokens)')
    if rows is None and R // T != B:
        raise ValueError(f'logits_process: {R // T} logits rows of T = {T} for {B} history rows: pass rows')
    checks = [('hist', hist, torch.int64, (B, max_len)), ('last', last, torch.int64, (B,)),
              ('prompt_len', prompt_len, torch.int64, (B,)), ('penalty', penalty, torch.float32, (B,)),
              ('ngram', ngram, torch.int32, (B,)), ('min_new', min_new, torch.int32, (B,)),
              ('eos', eos, torch.int64, (n_eos,)), ('bad', bad, torch.int64, (n_bad, PROC_BAD_LEN)),
              ('bad_len', bad_len, torch.int32, (n_bad,))]
    if tokens is not None:
        checks.append(('tokens', tokens, torch.int64, (B, T)))
    if rows is not None:
        checks.append(('rows', rows, torch.int64, (R // T,)))
    for name, t, dt, shape in checks:
        if t.dtype != dt or tuple(t.shape) != shape:
            raise ValueError(f'logits_process: {name} must be {shape} {dt}, got {tuple(t.shape)} {t.dtype}')
    if not logits.is_cuda:
        raise RuntimeError('logits_process runs on a CUDA device only (there is no CPU fallback)')
    _check_cuda('logits_process', [t for _, t, _, _ in checks], logits.device)
    ld = logits.stride(0) if R > 1 else V
    p = lambda t: None if t is None or t.numel() == 0 else t.data_ptr()
    with torch.cuda.device(logits.device):
        _lib.check(_lib.load().quip_logits_process(logits.data_ptr(), ld, R, int(T), V, p(rows), hist.data_ptr(),
                                                   last.data_ptr(), p(tokens), prompt_len.data_ptr(),
                                                   penalty.data_ptr(), ngram.data_ptr(), min_new.data_ptr(), p(eos),
                                                   n_eos, p(bad), p(bad_len), n_bad, B, max_len,
                                                   torch.cuda.current_stream(logits.device).cuda_stream))
    return logits


CONSTRAIN_MAX_V, CONSTRAIN_MAX_T = 2 ** 18, 8


def _constraint_table(fn, offsets, ids, next):
    """(S, nnz) of a packed token-automaton table after checking its shapes and dtypes (its contents are checked where
    it is packed: constrain.pack_automata)."""
    if offsets.dtype != torch.int32 or offsets.dim() != 1 or offsets.numel() < 1:
        raise ValueError(f'{fn}: offsets must be (S + 1,) int32, got {tuple(offsets.shape)} {offsets.dtype}')
    nnz = ids.numel()
    for name, t in (('ids', ids), ('next', next)):
        if t.dtype != torch.int32 or tuple(t.shape) != (nnz,):
            raise ValueError(f'{fn}: {name} must be (nnz = {nnz},) int32, got {tuple(t.shape)} {t.dtype}')
    return offsets.numel() - 1, nnz


def constrain_mask(logits, T, state, offsets, ids, next, tokens=None, rows=None):
    """quip_constrain_mask: the token-automaton mask rule of include/quip_b200.h, in place on logits (R, V) fp16
    (stride(1) == 1, any stride(0) >= V).  Row r is offset r % T of decoder row rows[r // T] (rows (R // T,) int64;
    default r // T), whose state state[b] (state (B,) int32, -1: unconstrained) is walked over the drafts
    tokens[b, 1 .. r % T] (tokens (B, T) int64, needed when T > 1) through the table offsets (S + 1,), ids and next
    (nnz,) int32.  CUDA, one device; everything is checked before the launch, which runs on the current stream.
    Returns logits."""
    if logits.dim() != 2 or logits.dtype != torch.float16:
        raise ValueError(f'constrain_mask: logits must be (R, V) fp16, got {tuple(logits.shape)} {logits.dtype}')
    R, V = logits.shape
    if not 1 <= V <= CONSTRAIN_MAX_V or (R > 1 and logits.stride(0) < V) or (V > 1 and logits.stride(1) != 1):
        raise ValueError(f'constrain_mask: logits rows must be unit-stride, not overlap and hold 1 .. '
                         f'{CONSTRAIN_MAX_V} values, got shape {tuple(logits.shape)} strides {tuple(logits.stride())}')
    if isinstance(T, bool) or int(T) != T or not 1 <= T <= CONSTRAIN_MAX_T or R % T:
        raise ValueError(f'constrain_mask: T must be an integer in [1, {CONSTRAIN_MAX_T}] dividing R = {R}, got {T!r}')
    if state.dtype != torch.int32 or state.dim() != 1 or state.numel() < 1:
        raise ValueError(f'constrain_mask: state must be (B,) int32, got {tuple(state.shape)} {state.dtype}')
    B = state.numel()
    S, nnz = _constraint_table('constrain_mask', offsets, ids, next)
    if T > 1 and tokens is None:
        raise ValueError('constrain_mask: T > 1 needs the drafts (tokens)')
    if rows is None and R // T != B:
        raise ValueError(f'constrain_mask: {R // T} logits rows of T = {T} for {B} states: pass rows')
    if tokens is not None and (tokens.dtype != torch.int64 or tuple(tokens.shape) != (B, T)):
        raise ValueError(f'constrain_mask: tokens must be {(B, T)} int64, got {tuple(tokens.shape)} {tokens.dtype}')
    if rows is not None and (rows.dtype != torch.int64 or tuple(rows.shape) != (R // T,)):
        raise ValueError(f'constrain_mask: rows must be {(R // T,)} int64, got {tuple(rows.shape)} {rows.dtype}')
    if not logits.is_cuda:
        raise RuntimeError('constrain_mask runs on a CUDA device only (there is no CPU fallback)')
    _check_cuda('constrain_mask', (state, offsets, ids, next, tokens, rows), logits.device)
    ld = logits.stride(0) if R > 1 else V
    p = lambda t: None if t is None or t.numel() == 0 else t.data_ptr()
    with torch.cuda.device(logits.device):
        _lib.check(_lib.load().quip_constrain_mask(logits.data_ptr(), ld, R, int(T), V, p(rows), p(tokens),
                                                   state.data_ptr(), B, offsets.data_ptr(), p(ids), p(next), S, nnz,
                                                   torch.cuda.current_stream(logits.device).cuda_stream))
    return logits


def constrain_advance(state, tokens, offsets, ids, next, counts=None, rows=None):
    """quip_constrain_advance: state[b] (state (B,) int32) walked over the first counts[n] (counts (N,) int64; default
    T) of the committed tokens (N, T) int64 of entry n, b = rows[n] (rows (N,) int64, distinct; default n), through the
    table offsets (S + 1,), ids and next (nnz,) int32 (include/quip_b200.h).  CUDA, one device; checked before the
    launch, which runs on the current stream.  Returns state."""
    if state.dtype != torch.int32 or state.dim() != 1 or state.numel() < 1:
        raise ValueError(f'constrain_advance: state must be (B,) int32, got {tuple(state.shape)} {state.dtype}')
    if tokens.dtype != torch.int64 or tokens.dim() != 2 or not 1 <= tokens.shape[1] <= CONSTRAIN_MAX_T:
        raise ValueError(f'constrain_advance: tokens must be (N, T <= {CONSTRAIN_MAX_T}) int64, got '
                         f'{tuple(tokens.shape)} {tokens.dtype}')
    B, (N, T) = state.numel(), tokens.shape
    S, nnz = _constraint_table('constrain_advance', offsets, ids, next)
    if rows is None and N != B:
        raise ValueError(f'constrain_advance: {N} token rows for {B} states: pass rows')
    for name, t in (('counts', counts), ('rows', rows)):
        if t is not None and (t.dtype != torch.int64 or tuple(t.shape) != (N,)):
            raise ValueError(f'constrain_advance: {name} must be ({N},) int64, got {tuple(t.shape)} {t.dtype}')
    if not state.is_cuda:
        raise RuntimeError('constrain_advance runs on a CUDA device only (there is no CPU fallback)')
    _check_cuda('constrain_advance', (tokens, offsets, ids, next, counts, rows), state.device)
    p = lambda t: None if t is None or t.numel() == 0 else t.data_ptr()
    with torch.cuda.device(state.device):
        _lib.check(_lib.load().quip_constrain_advance(state.data_ptr(), B, tokens.data_ptr(), T, N, T, p(rows),
                                                      p(counts), offsets.data_ptr(), p(ids), p(next), S, nnz,
                                                      torch.cuda.current_stream(state.device).cuda_stream))
    return state
