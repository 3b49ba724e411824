"""Torch (CPU or CUDA) restatement of the e4m3 KV-cache format of csrc/attn_decode.cu and include/quip_b200.h.

A cached head vector x (the hd values of one layer, row, kv head and slot, taken in fp32) is stored as

    amax = max_i |x_i|;   s = amax / 448 (fp32), s = 1 when amax == 0;   q_i = e4m3fn(x_i / s)   (round to nearest even)

and read back as float(q_i) * s.  |x_i / s| < 464, so torch's non-saturating conversion gives the bytes the kernels'
saturating cvt gives.  `attention` is float64 attention over a cache read back that way, with the appended slot
quantized like every other slot.
"""
import torch

E4M3_MAX = 448.0


def quantize(x):
    """x (..., hd) -> (q (..., hd) float8_e4m3fn, s (...) fp32)."""
    x = x.float()
    amax = x.abs().amax(-1)
    # a tensor divisor: torch's CUDA division by a Python scalar multiplies by its reciprocal, which is not IEEE division
    s = torch.where(amax == 0, torch.ones_like(amax), amax / torch.full_like(amax, E4M3_MAX))
    return (x / s[..., None]).to(torch.float8_e4m3fn), s


def dequantize(q, s, dtype=torch.float32):
    return (q.to(torch.float32) * s[..., None].float()).to(dtype)


def attention(q, k_new, v_new, k_cache, v_cache, k_scale, v_scale, positions, scale):
    """float64 o (B, nh, hd) of one step: k_new / v_new (B, nkv, hd) quantized into slot positions[b], attention of
    q (B, nh, hd) over slots 0 .. positions[b] of the dequantized e4m3 cache (B, nkv, max_len, hd) / scales
    (B, nkv, max_len).  Slots past positions[b] are not looked at."""
    B, nh, hd = q.shape
    G = nh // k_new.shape[1]
    kq, ks = quantize(k_new)
    vq, vs = quantize(v_new)
    out = torch.empty(B, nh, hd, dtype=torch.float64, device=q.device)
    for b in range(B):
        p = int(positions[b])
        K = k_cache[b, :, :p + 1].to(torch.float64) * k_scale[b, :, :p + 1, None].double()
        V = v_cache[b, :, :p + 1].to(torch.float64) * v_scale[b, :, :p + 1, None].double()
        K[:, p] = kq[b].to(torch.float64) * ks[b, :, None].double()
        V[:, p] = vq[b].to(torch.float64) * vs[b, :, None].double()
        K, V = K.repeat_interleave(G, 0), V.repeat_interleave(G, 0)
        sc = torch.einsum('hd,hjd->hj', q[b].double(), K) * scale
        out[b] = torch.einsum('hj,hjd->hd', torch.softmax(sc, -1), V)
    return out
