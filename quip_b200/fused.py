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


def _kv_layout(fn, k_cache, B, page_table):
    """(rows, slots, max_len) of one layer's cache k_cache (rows, nkv, slots, hd): the contiguous cache (B, nkv, max_len,
    hd) without a page table; with page_table (B, max_pages) int32, pools (n_pages, nkv, 64, hd) and max_len =
    max_pages * 64 (include/quip_b200.h has the rule).  Checks the table's dtype, shape, device and alignment and the
    pools' alignment; the callers check the rest of the shapes against these."""
    if page_table is None:
        return B, k_cache.shape[2], k_cache.shape[2]
    if page_table.dtype != torch.int32 or page_table.dim() != 2 or page_table.shape[0] != B or page_table.shape[1] < 1:
        raise ValueError(f'{fn}: page_table must be (B={B}, max_pages >= 1) int32, got {tuple(page_table.shape)} '
                         f'{page_table.dtype}')
    if k_cache.dim() != 4 or k_cache.shape[2] != KV_PAGE or k_cache.shape[0] < 1:
        raise ValueError(f'{fn}: with a page table the caches are pools (n_pages, nkv, {KV_PAGE}, hd), got '
                         f'{tuple(k_cache.shape)}')
    if page_table.shape[1] > (2 ** 31 - 1) // KV_PAGE:
        raise ValueError(f'{fn}: {page_table.shape[1]} pages per row: max_pages * {KV_PAGE} must fit int32')
    if not page_table.is_cuda or page_table.device != k_cache.device or not page_table.is_contiguous():
        raise ValueError(f'{fn}: page_table must be a contiguous CUDA tensor on the caches\' device')
    if page_table.data_ptr() % 4 or k_cache.data_ptr() % 16:
        raise ValueError(f'{fn}: page_table must be 4-byte aligned and the pools 16-byte aligned')
    return k_cache.shape[0], KV_PAGE, page_table.shape[1] * KV_PAGE


def _paged_args(page_table, n_pages):
    return (page_table.data_ptr(), page_table.shape[1], n_pages)


def decode_attention(q, k_new, v_new, k_cache, v_cache, positions, scale, k_scale=None, v_scale=None, page_table=None):
    """quip_decode_attention on torch tensors: append k_new / v_new (B, nkv, hd) at slot positions[b] of one layer's
    k_cache / v_cache (B, nkv, max_len, hd) and attend q (B, nh, hd) over slots 0 .. positions[b].  fp16, CUDA,
    contiguous; positions (B,) int64 on the same device.  Returns (B, nh, hd) fp16, on the current stream.

    Caches of dtype torch.float8_e4m3fn take quip_decode_attention_fp8 and need their per-slot fp32 scales k_scale /
    v_scale (B, nkv, max_len): k_new / v_new are quantized on append (include/quip_b200.h has the format).

    page_table (B, max_pages) int32: the caches are page pools (n_pages, nkv, 64, hd), scales (n_pages, nkv, 64), and
    slot j of row b lives at slot j % 64 of page page_table[b, j // 64] (quip_decode_attention_paged(_fp8)); a row that
    would touch a page id outside [0, n_pages) writes nothing there and gets NaN."""
    if k_cache.dtype == torch.float8_e4m3fn:
        return _decode_attention_fp8(q, k_new, v_new, k_cache, v_cache, k_scale, v_scale, positions, scale, page_table)
    if k_scale is not None or v_scale is not None:
        raise ValueError('decode_attention: k_scale / v_scale go with float8_e4m3fn caches only')
    ts = (q, k_new, v_new, k_cache, v_cache)
    for t in ts + (positions,):
        if not t.is_cuda:
            raise RuntimeError('decode_attention runs on a CUDA device only (there is no CPU fallback)')
        if t.device != q.device:
            raise ValueError('decode_attention: all tensors must be on one device')
        if not t.is_contiguous():
            raise ValueError('decode_attention takes contiguous tensors')
    if any(t.dtype != torch.float16 for t in ts) or positions.dtype != torch.int64:
        raise ValueError('decode_attention takes fp16 q / k / v / caches and int64 positions')
    if q.dim() != 3 or k_cache.dim() != 4:
        raise ValueError(f'decode_attention: q must be (B, nh, hd) and the caches (B, nkv, max_len, hd), got '
                         f'{tuple(q.shape)} and {tuple(k_cache.shape)}')
    B, nh, hd = q.shape
    nkv = k_cache.shape[1]
    rows, slots, max_len = _kv_layout('decode_attention', k_cache, B, page_table)
    if (tuple(k_cache.shape) != (rows, nkv, slots, hd) or v_cache.shape != k_cache.shape or
            tuple(k_new.shape) != (B, nkv, hd) or v_new.shape != k_new.shape or tuple(positions.shape) != (B,)):
        raise ValueError(f'decode_attention: shapes q {tuple(q.shape)}, k_new {tuple(k_new.shape)}, v_new '
                         f'{tuple(v_new.shape)}, caches {tuple(k_cache.shape)} / {tuple(v_cache.shape)}, positions '
                         f'{tuple(positions.shape)} do not agree')
    lib = _lib.load()
    need = C.c_size_t(0)
    _lib.check(lib.quip_decode_attention_workspace_bytes(B, nh, hd, max_len, C.byref(need)))
    ws = torch.empty(max(int(need.value), 16), dtype=torch.uint8, device=q.device)
    out = torch.empty_like(q)
    st = torch.cuda.current_stream(q.device).cuda_stream
    with torch.cuda.device(q.device):
        if page_table is not None:
            _lib.check(lib.quip_decode_attention_paged(q.data_ptr(), k_new.data_ptr(), v_new.data_ptr(),
                                                       k_cache.data_ptr(), v_cache.data_ptr(), positions.data_ptr(),
                                                       out.data_ptr(), B, nh, nkv, hd, C.c_float(scale), ws.data_ptr(),
                                                       ws.numel(), *_paged_args(page_table, rows), st))
        else:
            _lib.check(lib.quip_decode_attention(q.data_ptr(), k_new.data_ptr(), v_new.data_ptr(), k_cache.data_ptr(),
                                                 v_cache.data_ptr(), positions.data_ptr(), out.data_ptr(), B, nh, nkv,
                                                 hd, max_len, C.c_float(scale), ws.data_ptr(), ws.numel(), st))
    return out


def _check_cuda(fn, ts, dev):
    for t in ts:
        if not t.is_cuda:
            raise RuntimeError(f'{fn} runs on a CUDA device only (there is no CPU fallback)')
        if t.device != dev:
            raise ValueError(f'{fn}: all tensors must be on one device')
        if not t.is_contiguous():
            raise ValueError(f'{fn} takes contiguous tensors')


def _decode_attention_fp8(q, k_new, v_new, k_cache, v_cache, k_scale, v_scale, positions, scale, page_table):
    if k_scale is None or v_scale is None:
        raise ValueError('decode_attention: float8_e4m3fn caches need k_scale and v_scale')
    if (any(t.dtype != torch.float16 for t in (q, k_new, v_new)) or v_cache.dtype != torch.float8_e4m3fn or
            k_scale.dtype != torch.float32 or v_scale.dtype != torch.float32 or positions.dtype != torch.int64):
        raise ValueError('decode_attention: an e4m3 step takes fp16 q / k / v, float8_e4m3fn caches, fp32 scales and '
                         'int64 positions')
    if q.dim() != 3 or k_cache.dim() != 4:
        raise ValueError(f'decode_attention: q must be (B, nh, hd) and the caches (B, nkv, max_len, hd), got '
                         f'{tuple(q.shape)} and {tuple(k_cache.shape)}')
    B, nh, hd = q.shape
    nkv = k_cache.shape[1]
    rows, slots, max_len = _kv_layout('decode_attention', k_cache, B, page_table)
    if (tuple(k_cache.shape) != (rows, nkv, slots, hd) or v_cache.shape != k_cache.shape or
            tuple(k_new.shape) != (B, nkv, hd) or v_new.shape != k_new.shape or tuple(positions.shape) != (B,) or
            tuple(k_scale.shape) != (rows, nkv, slots) or v_scale.shape != k_scale.shape):
        raise ValueError(f'decode_attention: shapes q {tuple(q.shape)}, k_new {tuple(k_new.shape)}, v_new '
                         f'{tuple(v_new.shape)}, caches {tuple(k_cache.shape)} / {tuple(v_cache.shape)}, scales '
                         f'{tuple(k_scale.shape)} / {tuple(v_scale.shape)}, positions {tuple(positions.shape)} do not agree')
    _check_cuda('decode_attention', (q, k_new, v_new, k_cache, v_cache, k_scale, v_scale, positions), q.device)
    lib = _lib.load()
    need = C.c_size_t(0)
    _lib.check(lib.quip_decode_attention_workspace_bytes(B, nh, hd, max_len, C.byref(need)))
    ws = torch.empty(max(int(need.value), 16), dtype=torch.uint8, device=q.device)
    out = torch.empty_like(q)
    st = torch.cuda.current_stream(q.device).cuda_stream
    with torch.cuda.device(q.device):
        if page_table is not None:
            _lib.check(lib.quip_decode_attention_paged_fp8(q.data_ptr(), k_new.data_ptr(), v_new.data_ptr(),
                                                           k_cache.data_ptr(), v_cache.data_ptr(), k_scale.data_ptr(),
                                                           v_scale.data_ptr(), positions.data_ptr(), out.data_ptr(), B,
                                                           nh, nkv, hd, C.c_float(scale), ws.data_ptr(), ws.numel(),
                                                           *_paged_args(page_table, rows), st))
        else:
            _lib.check(lib.quip_decode_attention_fp8(q.data_ptr(), k_new.data_ptr(), v_new.data_ptr(),
                                                     k_cache.data_ptr(), v_cache.data_ptr(), k_scale.data_ptr(),
                                                     v_scale.data_ptr(), positions.data_ptr(), out.data_ptr(), B, nh,
                                                     nkv, hd, max_len, C.c_float(scale), ws.data_ptr(), ws.numel(), st))
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


def extend_attention(q, k_new, v_new, k_cache, v_cache, positions, scale, k_scale=None, v_scale=None, page_table=None):
    """quip_extend_attention(_fp8) on torch tensors: append token i of k_new / v_new (B, T, nkv, hd) at slot
    positions[b] + i of one layer's caches (B, nkv, max_len, hd) and attend q (B, T, nh, hd) causally over slots
    0 .. positions[b] + i.  fp16 q / k / v; fp16 caches, or float8_e4m3fn caches with fp32 k_scale / v_scale
    (B, nkv, max_len).  CUDA, one device, contiguous; positions (B,) int64.  Returns (B, T, nh, hd) fp16.
    page_table: page pools as in decode_attention (quip_extend_attention_paged(_fp8))."""
    fp8 = k_cache.dtype == torch.float8_e4m3fn
    if not fp8 and (k_scale is not None or v_scale is not None):
        raise ValueError('extend_attention: k_scale / v_scale go with float8_e4m3fn caches only')
    if fp8 and (k_scale is None or v_scale is None):
        raise ValueError('extend_attention: float8_e4m3fn caches need k_scale and v_scale')
    cdt = torch.float8_e4m3fn if fp8 else torch.float16
    if (any(t.dtype != torch.float16 for t in (q, k_new, v_new)) or k_cache.dtype != cdt or v_cache.dtype != cdt or
            positions.dtype != torch.int64 or (fp8 and (k_scale.dtype != torch.float32 or v_scale.dtype != torch.float32))):
        raise ValueError('extend_attention takes fp16 q / k / v, fp16 or float8_e4m3fn caches (fp32 scales) and int64 '
                         'positions')
    if q.dim() != 4 or k_cache.dim() != 4:
        raise ValueError(f'extend_attention: q must be (B, T, nh, hd) and the caches (B, nkv, max_len, hd), got '
                         f'{tuple(q.shape)} and {tuple(k_cache.shape)}')
    B, T, nh, hd = q.shape
    nkv = k_cache.shape[1]
    rows, slots, max_len = _kv_layout('extend_attention', k_cache, B, page_table)
    if (tuple(k_cache.shape) != (rows, nkv, slots, hd) or v_cache.shape != k_cache.shape or
            tuple(k_new.shape) != (B, T, nkv, hd) or v_new.shape != k_new.shape or tuple(positions.shape) != (B,) or
            (fp8 and (tuple(k_scale.shape) != (rows, nkv, slots) or v_scale.shape != k_scale.shape))):
        raise ValueError(f'extend_attention: shapes q {tuple(q.shape)}, k_new {tuple(k_new.shape)}, v_new '
                         f'{tuple(v_new.shape)}, caches {tuple(k_cache.shape)} / {tuple(v_cache.shape)}, positions '
                         f'{tuple(positions.shape)} do not agree')
    ts = (q, k_new, v_new, k_cache, v_cache, positions) + ((k_scale, v_scale) if fp8 else ())
    _check_cuda('extend_attention', ts, q.device)
    lib = _lib.load()
    need = C.c_size_t(0)
    _lib.check(lib.quip_extend_attention_workspace_bytes(B, T, nh, hd, max_len, C.byref(need)))
    ws = torch.empty(max(int(need.value), 16), dtype=torch.uint8, device=q.device)
    out = torch.empty_like(q)
    st = torch.cuda.current_stream(q.device).cuda_stream
    with torch.cuda.device(q.device):
        if page_table is not None and fp8:
            _lib.check(lib.quip_extend_attention_paged_fp8(q.data_ptr(), k_new.data_ptr(), v_new.data_ptr(),
                                                           k_cache.data_ptr(), v_cache.data_ptr(), k_scale.data_ptr(),
                                                           v_scale.data_ptr(), positions.data_ptr(), out.data_ptr(), B, T,
                                                           nh, nkv, hd, C.c_float(scale), ws.data_ptr(), ws.numel(),
                                                           *_paged_args(page_table, rows), st))
        elif page_table is not None:
            _lib.check(lib.quip_extend_attention_paged(q.data_ptr(), k_new.data_ptr(), v_new.data_ptr(),
                                                       k_cache.data_ptr(), v_cache.data_ptr(), positions.data_ptr(),
                                                       out.data_ptr(), B, T, nh, nkv, hd, C.c_float(scale),
                                                       ws.data_ptr(), ws.numel(), *_paged_args(page_table, rows), st))
        elif fp8:
            _lib.check(lib.quip_extend_attention_fp8(q.data_ptr(), k_new.data_ptr(), v_new.data_ptr(), k_cache.data_ptr(),
                                                     v_cache.data_ptr(), k_scale.data_ptr(), v_scale.data_ptr(),
                                                     positions.data_ptr(), out.data_ptr(), B, T, nh, nkv, hd, max_len,
                                                     C.c_float(scale), ws.data_ptr(), ws.numel(), st))
        else:
            _lib.check(lib.quip_extend_attention(q.data_ptr(), k_new.data_ptr(), v_new.data_ptr(), k_cache.data_ptr(),
                                                 v_cache.data_ptr(), positions.data_ptr(), out.data_ptr(), B, T, nh, nkv,
                                                 hd, max_len, C.c_float(scale), ws.data_ptr(), ws.numel(), st))
    return out


def _check_chunk(fn, k_cache, v_cache, positions, counts, k_scale, v_scale, page_table=None):
    """The checks kv_append and prefill_attention share: cache and scale dtypes, positions / counts (B,) int64, and the
    page table with its pools.  Returns (whether the caches are e4m3, B, rows, max_len) (_kv_layout)."""
    fp8 = k_cache.dtype == torch.float8_e4m3fn
    if not fp8 and (k_scale is not None or v_scale is not None):
        raise ValueError(f'{fn}: k_scale / v_scale go with float8_e4m3fn caches only')
    if fp8 and (k_scale is None or v_scale is None):
        raise ValueError(f'{fn}: float8_e4m3fn caches need k_scale and v_scale')
    cdt = torch.float8_e4m3fn if fp8 else torch.float16
    if (k_cache.dtype != cdt or v_cache.dtype != cdt or positions.dtype != torch.int64 or counts.dtype != torch.int64 or
            (fp8 and (k_scale.dtype != torch.float32 or v_scale.dtype != torch.float32))):
        raise ValueError(f'{fn} takes fp16 or float8_e4m3fn caches (fp32 scales) and int64 positions and counts')
    if k_cache.dim() != 4:
        raise ValueError(f'{fn}: the caches must be (B, nkv, max_len, hd), got {tuple(k_cache.shape)}')
    B = k_cache.shape[0] if page_table is None else (positions.shape[0] if positions.dim() == 1 else -1)
    nkv = k_cache.shape[1]
    rows, slots, max_len = _kv_layout(fn, k_cache, B, page_table)
    if (v_cache.shape != k_cache.shape or tuple(positions.shape) != (B,) or tuple(counts.shape) != (B,) or
            (fp8 and (tuple(k_scale.shape) != (rows, nkv, slots) or v_scale.shape != k_scale.shape))):
        raise ValueError(f'{fn}: shapes caches {tuple(k_cache.shape)} / {tuple(v_cache.shape)}, positions '
                         f'{tuple(positions.shape)}, counts {tuple(counts.shape)} do not agree')
    return fp8, B, rows, max_len


def kv_append(k_new, v_new, k_cache, v_cache, positions, counts, k_scale=None, v_scale=None, page_table=None):
    """quip_kv_append(_fp8) on torch tensors: token i of k_new / v_new (B, T, nkv, hd) fp16 to slot positions[b] + i of
    one layer's caches (B, nkv, max_len, hd) for i < counts[b]; nothing else is written.  fp16 caches, or
    float8_e4m3fn caches with fp32 k_scale / v_scale (B, nkv, max_len), quantized on the way.  CUDA, one device,
    contiguous; positions / counts (B,) int64.  On the current stream.  page_table: page pools as in decode_attention
    (quip_kv_append_paged(_fp8)); a slot whose page id lies outside the pool is not written."""
    fp8, B, rows, max_len = _check_chunk('kv_append', k_cache, v_cache, positions, counts, k_scale, v_scale, page_table)
    if k_new.dtype != torch.float16 or v_new.dtype != torch.float16:
        raise ValueError('kv_append takes fp16 k_new / v_new')
    nkv, hd = k_cache.shape[1], k_cache.shape[3]
    if k_new.dim() != 4 or k_new.shape[0] != B or tuple(k_new.shape[2:]) != (nkv, hd) or v_new.shape != k_new.shape:
        raise ValueError(f'kv_append: k_new {tuple(k_new.shape)} / v_new {tuple(v_new.shape)} must be (B, T, nkv, hd) '
                         f'for caches {tuple(k_cache.shape)}')
    T = k_new.shape[1]
    ts = (k_new, v_new, k_cache, v_cache, positions, counts) + ((k_scale, v_scale) if fp8 else ())
    _check_cuda('kv_append', ts, k_new.device)
    lib, st = _lib.load(), torch.cuda.current_stream(k_new.device).cuda_stream
    with torch.cuda.device(k_new.device):
        if page_table is not None and fp8:
            _lib.check(lib.quip_kv_append_paged_fp8(k_new.data_ptr(), v_new.data_ptr(), k_cache.data_ptr(),
                                                    v_cache.data_ptr(), k_scale.data_ptr(), v_scale.data_ptr(),
                                                    positions.data_ptr(), counts.data_ptr(), B, T, nkv, hd,
                                                    *_paged_args(page_table, rows), st))
        elif page_table is not None:
            _lib.check(lib.quip_kv_append_paged(k_new.data_ptr(), v_new.data_ptr(), k_cache.data_ptr(),
                                                v_cache.data_ptr(), positions.data_ptr(), counts.data_ptr(), B, T, nkv,
                                                hd, *_paged_args(page_table, rows), st))
        elif fp8:
            _lib.check(lib.quip_kv_append_fp8(k_new.data_ptr(), v_new.data_ptr(), k_cache.data_ptr(), v_cache.data_ptr(),
                                              k_scale.data_ptr(), v_scale.data_ptr(), positions.data_ptr(),
                                              counts.data_ptr(), B, T, nkv, hd, max_len, st))
        else:
            _lib.check(lib.quip_kv_append(k_new.data_ptr(), v_new.data_ptr(), k_cache.data_ptr(), v_cache.data_ptr(),
                                          positions.data_ptr(), counts.data_ptr(), B, T, nkv, hd, max_len, st))


def prefill_attention(q, k_cache, v_cache, positions, counts, scale, k_scale=None, v_scale=None, page_table=None):
    """quip_prefill_attention(_fp8) on torch tensors: q (B, T, nh, hd) fp16 attends causally over one layer's caches
    (B, nkv, max_len, hd), which already hold the chunk (kv_append): token i of row b over slots 0 .. positions[b] + i
    for i < counts[b]; rows i >= counts[b] are zero.  fp16 caches, or float8_e4m3fn caches with fp32 k_scale / v_scale.
    CUDA, one device, contiguous; positions / counts (B,) int64.  Returns (B, T, nh, hd) fp16, on the current stream.
    page_table: page pools as in decode_attention (quip_prefill_attention_paged(_fp8))."""
    fp8, B, rows, max_len = _check_chunk('prefill_attention', k_cache, v_cache, positions, counts, k_scale, v_scale,
                                         page_table)
    if q.dtype != torch.float16 or q.dim() != 4:
        raise ValueError(f'prefill_attention: q must be (B, T, nh, hd) fp16, got {tuple(q.shape)} {q.dtype}')
    T, nh, hd = q.shape[1:]
    nkv = k_cache.shape[1]
    if q.shape[0] != B or k_cache.shape[3] != hd:
        raise ValueError(f'prefill_attention: q {tuple(q.shape)} and caches {tuple(k_cache.shape)} do not agree')
    ts = (q, k_cache, v_cache, positions, counts) + ((k_scale, v_scale) if fp8 else ())
    _check_cuda('prefill_attention', ts, q.device)
    out = torch.empty_like(q)
    lib, st = _lib.load(), torch.cuda.current_stream(q.device).cuda_stream
    with torch.cuda.device(q.device):
        if page_table is not None and fp8:
            _lib.check(lib.quip_prefill_attention_paged_fp8(q.data_ptr(), k_cache.data_ptr(), v_cache.data_ptr(),
                                                            k_scale.data_ptr(), v_scale.data_ptr(), positions.data_ptr(),
                                                            counts.data_ptr(), out.data_ptr(), B, T, nh, nkv, hd,
                                                            C.c_float(scale), *_paged_args(page_table, rows), st))
        elif page_table is not None:
            _lib.check(lib.quip_prefill_attention_paged(q.data_ptr(), k_cache.data_ptr(), v_cache.data_ptr(),
                                                        positions.data_ptr(), counts.data_ptr(), out.data_ptr(), B, T,
                                                        nh, nkv, hd, C.c_float(scale), *_paged_args(page_table, rows),
                                                        st))
        elif fp8:
            _lib.check(lib.quip_prefill_attention_fp8(q.data_ptr(), k_cache.data_ptr(), v_cache.data_ptr(),
                                                      k_scale.data_ptr(), v_scale.data_ptr(), positions.data_ptr(),
                                                      counts.data_ptr(), out.data_ptr(), B, T, nh, nkv, hd, max_len,
                                                      C.c_float(scale), st))
        else:
            _lib.check(lib.quip_prefill_attention(q.data_ptr(), k_cache.data_ptr(), v_cache.data_ptr(),
                                                  positions.data_ptr(), counts.data_ptr(), out.data_ptr(), B, T, nh, nkv,
                                                  hd, max_len, C.c_float(scale), st))
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
