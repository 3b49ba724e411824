"""Code <-> value maps and quantizer parameters (CPU oracle, numpy).

Restates, with the reference's own dtypes and rounding points:
  * Quantizer.find_params for the weight / per-channel / asymmetric case
    (reference quant.py:57-136 with perchannel=True, sym=False, weight=True,
    mse=False -- the only configuration opt.py:100-129 ever builds);
  * the qfn 'a' and qfn 'b' grid maps of quantize_weight_vecbal
    (reference vector_balance.py:514-530; quant.py:6-15);
  * the inverse map grid value -> integer code used for the bit-exact check;
  * the affine form  W = scales * code - zeros  that Quant3Linear stores
    (reference quant.py:186-191) and the packed kernels consume.

Test infrastructure only (see oracle/__init__.py).
"""
import numpy as np

f16, f32, f64 = np.float16, np.float32, np.float64


def maxq_of(bits):
    # quant.py:40
    return (1 << int(bits)) - 1


def find_params_qfna(w, bits):
    """Per-output-channel asymmetric (scale, zero), each float32 of shape (N,1).

    quant.py:62-64 flattens the weight to (N, K); :76-78 take the row min/max
    against a float32 zeros vector (which promotes fp16 weights to float32);
    :86-88 replace an all-zero row by [-1, 1]; :90 scale=(max-min)/maxq;
    :94 zero=round(-min/scale); :123-127 reshape to (N,1).
    """
    maxq = f32(maxq_of(bits))
    x = np.asarray(w).reshape(w.shape[0], -1)
    xmin = np.minimum(x.min(axis=1).astype(f32), f32(0))
    xmax = np.maximum(x.max(axis=1).astype(f32), f32(0))
    dead = (xmin == 0) & (xmax == 0)
    xmin[dead] = -1
    xmax[dead] = +1
    scale = ((xmax - xmin) / maxq).astype(f32)
    zero = np.round(-xmin / scale).astype(f32)       # half-to-even, like torch.round
    return scale.reshape(-1, 1), zero.reshape(-1, 1)


def qfnb_scale(w):
    """qfn 'b' scale: 2.4*rms(w) evaluated in the weight's own dtype.

    vector_balance.py:522 with an fp16 `w` (bal.py:22): every elementwise op
    rounds to fp16; the `+ 1e-16` is absorbed (SURVEY A7).  The mean's fp32
    accumulation order is torch-internal, so this helper is only used to
    sanity-check captured scales, never to derive codes.
    """
    w = np.asarray(w)
    if w.dtype == f16:
        sq = (w.astype(f32) * w.astype(f32)).astype(f16)
        mean = f16(sq.astype(f64).sum() / sq.size)
        return f16(f16(f32(2.4) * f32(f16(np.sqrt(f32(mean))))) + f16(1e-16))
    return w.dtype.type(2.4 * np.sqrt(np.mean(np.square(w.astype(f64)))) + 1e-16)


def grid_qfna(codes, scale, zero):
    """fp16 grid value of integer codes, qfn 'a': vector_balance.py:519-520.

    scale*(wr - zero) is evaluated in float32 (scale/zero are float32 even for
    fp16 weights, SURVEY a1) and then `.half()`.
    """
    c = np.asarray(codes).astype(f32)
    return (np.asarray(scale, f32) * (c - np.asarray(zero, f32))).astype(f16)


def grid_qfnb(codes, scale, bits):
    """fp16 grid value of integer codes, qfn 'b': vector_balance.py:528-530.

    `wr` is float32 (round_ldl is called on w.float(), :445), so
    ((wr / maxq) * 2 - 1) is float32; the product with the 0-dim fp16 `scale`
    stays float32; `.half()` rounds once.
    """
    maxq = f32(maxq_of(bits))
    c = np.asarray(codes).astype(f32)
    t = (c / maxq) * f32(2) - f32(1)
    return (t * f32(scale)).astype(f16)


def lut_qfnb(scale, bits):
    return grid_qfnb(np.arange(maxq_of(bits) + 1), scale, bits)


def codes_from_grid_qfna(q, scale, zero, bits):
    """Inverse of grid_qfna, the same rounding Quant3Linear.pack applies
    (quant.py:190-191: round((W + zero*scale) / scale))."""
    c = np.round(np.asarray(q, f64) / np.asarray(scale, f64) + np.asarray(zero, f64))
    assert c.min() >= 0 and c.max() <= maxq_of(bits)
    return c.astype(np.uint8)


def codes_from_grid_qfnb(q, scale, bits):
    maxq = maxq_of(bits)
    c = np.round((np.asarray(q, f64) / f64(scale) + 1.0) / 2.0 * maxq)
    assert c.min() >= 0 and c.max() <= maxq
    return c.astype(np.uint8)


def affine_qfna(scale, zero):
    """(scales, zeros) with W = scales*code - zeros; zeros is stored
    pre-multiplied exactly as Quant3Linear.pack does (quant.py:186)."""
    scale = np.asarray(scale, f32).reshape(-1, 1)
    zero = np.asarray(zero, f32).reshape(-1, 1)
    return scale.copy(), (zero * scale).astype(f32)


def affine_qfnb(scale, bits, n_rows):
    """qfn 'b' written in the same affine form: ((c/maxq)*2-1)*s = (2s/maxq)*c - s."""
    s = f32(scale)
    scales = np.full((n_rows, 1), f32(2) * s / f32(maxq_of(bits)), f32)
    zeros = np.full((n_rows, 1), s, f32)
    return scales, zeros


def kernel_affine(scales, zeros, bits):
    """The two per-row coefficients the sm_90a kernels apply in their epilogue.

    The kernels contract x against d = (code - cbar) / 2^bits with
    cbar = (2^bits - 1)/2 (exactly representable in fp16 for bits in {2,3,4}),
    so   sum_k x_k (scales*c_k - zeros) = P * sum_k x_k d_k + R * sum_k x_k
    with P = scales * 2^bits and R = scales * cbar - zeros.
    """
    cbar = f32(maxq_of(bits)) / f32(2)
    P = (np.asarray(scales, f32).reshape(-1) * f32(1 << bits)).astype(f32)
    R = (np.asarray(scales, f32).reshape(-1) * cbar - np.asarray(zeros, f32).reshape(-1)).astype(f32)
    return P, R
