"""Quantizer / QuantLinear / make_quant -- the reference's quant.py surface, backed by sm_90a kernels.

Reference surface kept (Cornell-RelaxML/QuIP, quant.py):
  * `Quantizer` (quant.py:23-163): `configure / find_params / quantize / enabled / ready`, buffers
    `maxq / scale / zero`, value maps qfn 'a' | 'b' | 'c' (quant.py:6-21);
  * the packed-linear module contract of `Quant3Linear` (quant.py:172-233) and `Quant4Linear`
    (zeroShot/models/quant.py:183-212): buffers `qweight / scales / zeros / bias` with
    W = scales*code - zeros (zeros stored pre-multiplied, quant.py:186), `pack(linear, scales,
    zeros)`, `forward(x)`;
  * `make_quant*` tree surgery by dotted name (quant.py:236-246).

What is new: bits in {2,3,4}, any number of tokens, no-bias layers (Llama), K % 128 == 0 instead of
K % 1024 == 0, and the incoherence data the reference throws away (scaleWH, butterfly factors of
U and V) stored as buffers so the fused forward can un-project at run time.  `forward` calls the C
ABI (include/quip_b200.h); there is no CPU path.
"""
import ctypes as C
from typing import Optional

import torch
import torch.nn as nn

from . import _lib
from .capture import Butterfly, LayerParts, butterfly_factors
from .incoherence import fold_inv_scale, plan_side

# ----------------------------------------------------------------------------------------------
# value maps (quant.py:6-21)
# ----------------------------------------------------------------------------------------------


def quantize_qfna(x, scale, zero, maxq):
    q = (torch.round(x / scale) + zero).clamp(0, maxq)
    return scale * (q - zero)


def quantize_qfnb(x, scale, maxq):
    q = torch.round(((x / scale) + 1) / 2 * maxq).clamp(0, maxq)
    return ((q / maxq) * 2 - 1) * scale


def quantize_qfnc(x, scale, zero, maxq):
    q = torch.round(((x / scale) + zero).clamp(0, maxq))
    return scale * (q - zero)


class Quantizer(nn.Module):
    """Per-channel min/max quantizer parameters (reference quant.py:23-163)."""

    def __init__(self, shape=1):
        super().__init__()
        self.register_buffer('maxq', torch.tensor(0))
        self.register_buffer('scale', torch.zeros(shape))
        self.register_buffer('zero', torch.zeros(shape))

    def configure(self, bits, perchannel=False, sym=True, qfn='a', mse=False, norm=2.4, grid=100, maxshrink=.8):
        self.maxq = torch.tensor(2 ** bits - 1)
        self.perchannel, self.sym, self.qfn = perchannel, sym, qfn
        self.mse, self.norm, self.grid, self.maxshrink = mse, norm, grid, maxshrink

    # quant.py:50-55
    def find_params(self, x, weight=False):
        if self.qfn in ('a', 'c'):
            self._find_minmax(x, weight)
        elif self.qfn == 'b':
            self.maxq = self.maxq.to(x.device)
            self.scale = None          # 2.4*rms(w) is only known after preproc (quant.py:138-142)
            self.zero = None

    def _rows(self, x, weight):
        shape = x.shape
        if not self.perchannel:
            return x.flatten().unsqueeze(0)
        if weight:
            return x.flatten(1)
        if len(shape) == 4:
            return x.permute(1, 0, 2, 3).flatten(1)
        if len(shape) == 3:
            return x.reshape(-1, shape[-1]).t()
        return x.t()

    def _find_minmax(self, x, weight):
        dev = x.device
        self.maxq = self.maxq.to(dev)
        shape = x.shape
        rows = self._rows(x, weight)
        zero_f32 = torch.zeros(rows.shape[0], device=dev)             # float32: promotes fp16 rows (quant.py:76-78)
        lo = torch.minimum(rows.min(1)[0], zero_f32)
        hi = torch.maximum(rows.max(1)[0], zero_f32)
        if self.sym:
            hi = torch.maximum(lo.abs(), hi)
            neg = lo < 0
            lo = torch.where(neg, -hi, lo)
        dead = (lo == 0) & (hi == 0)
        lo = torch.where(dead, torch.full_like(lo, -1), lo)
        hi = torch.where(dead, torch.full_like(hi, 1), hi)

        def params(lo_, hi_):
            sc = (hi_ - lo_) / self.maxq
            ze = torch.full_like(sc, (self.maxq + 1) / 2) if self.sym else torch.round(-lo_ / sc)
            return sc, ze
        scale, zero = params(lo, hi)
        if self.mse:                                                   # quant.py:96-114 shrink search
            best = torch.full([rows.shape[0]], float('inf'), device=dev)
            for i in range(int(self.maxshrink * self.grid)):
                f = 1 - i / self.grid
                sc1, ze1 = params(f * lo, f * hi)
                if self.sym:
                    ze1 = zero
                err = (quantize_qfna(rows, sc1.unsqueeze(1), ze1.unsqueeze(1), self.maxq) - rows).abs().pow(self.norm).sum(1)
                better = err < best
                best = torch.where(better, err, best)
                scale = torch.where(better, sc1, scale)
                zero = torch.where(better, ze1, zero)
        if not self.perchannel:
            rep = shape[0] if weight else (shape[1] if len(shape) != 3 else shape[2])
            scale, zero = scale.repeat(rep), zero.repeat(rep)
        if weight:
            view = [-1] + [1] * (len(shape) - 1)
        elif len(shape) == 4:
            view = (1, -1, 1, 1)
        elif len(shape) == 3:
            view = (1, 1, -1)
        else:
            view = (1, -1)
        self.scale, self.zero = scale.reshape(view), zero.reshape(view)

    def quantize(self, x):
        if self.qfn == 'a':
            assert self.ready()
            return quantize_qfna(x, self.scale, self.zero, self.maxq)
        if self.qfn == 'b':
            assert torch.all(self.maxq != 0)
            self.scale = 2.4 * x.square().mean().sqrt() + 1e-16       # quant.py:150
            return quantize_qfnb(x, self.scale, self.maxq)
        if self.qfn == 'c':
            assert self.ready()
            return quantize_qfnc(x, self.scale, self.zero, self.maxq)
        return NotImplementedError()

    def enabled(self):
        return self.maxq > 0

    def ready(self):
        return self.scale is not None and torch.all(self.scale != 0)


# ----------------------------------------------------------------------------------------------
# packing helpers
# ----------------------------------------------------------------------------------------------
_SB_WORDS = {2: 128, 3: 192, 4: 256}


def packed_words(N, K, bits):
    if N % 16 or K % 128 or bits not in _SB_WORDS:
        raise ValueError(f'packed layout needs N % 16 == 0, K % 128 == 0, bits in (2,3,4); got N={N} K={K} bits={bits}')
    return (N // 16) * (K // 128) * _SB_WORDS[bits]


def _native_fields(N, K, bits, device):
    """(word index, bit shift, code shift, field bits) per plane -- same map as oracle/packing.py."""
    n = torch.arange(N, device=device)[:, None]
    k = torch.arange(K, device=device)[None, :]
    rb, r = n // 16, n % 16
    g, hi = r % 8, r // 8
    ks, kk = k // 128, k % 128
    ch, t, pos = kk // 32, (kk % 32) // 8, kk % 8
    lane, e = g * 4 + t, pos % 2
    base = (rb * (K // 128) + ks) * _SB_WORDS[bits]
    u = pos // 2
    j = 2 * ((u % 2) * 2 + u // 2) + hi
    if bits == 2:
        return [(base + lane * 4 + ch, 2 * j + 16 * e, 0, 2)]
    if bits == 4:
        jp = 2 * ((pos % 4) // 2) + hi
        return [(base + (ch // 2) * 128 + lane * 4 + (ch % 2) * 2 + pos // 4, 4 * jp + 16 * e, 0, 4)]
    return [(base + lane * 4 + ch, 2 * j + 16 * e, 1, 2),
            (base + 128 + lane * 2 + ch // 2, 8 * (ch % 2) + j + 16 * e, 0, 1)]


def fragment_order(f: torch.Tensor) -> torch.Tensor:
    """Block-diagonal factors (nblk, p, p) fp16, row-major  ->  mma.m16n8k16 B-fragment order (QuipPass.factors_frag):
    [blk][n-tile][k/32][lane = 4g+t][q][pair], element (i = 8nt+g, k = 32j + 16(q//2) + 8(q%2) + 2t + pair)."""
    nblk, p, _ = f.shape
    v = f.reshape(nblk, p // 8, 8, p // 32, 2, 2, 4, 2)          # blk, nt, g, j, q//2, q%2, t, pair
    return v.permute(0, 1, 3, 2, 6, 4, 5, 7).contiguous()        # blk, nt, j, g, t, q//2, q%2, pair


def pack_codes(codes: torch.Tensor, bits: int) -> torch.Tensor:
    """codes (N, K) uint8 -> native packed int32 words.  On CUDA tensors this is quip_pack_codes (the GPU
    packer the reference leaves as a TODO, opt.py:302); on CPU tensors the same bit layout is built with
    torch index ops (host-side formatting, like the reference's numpy packer quant.py:185-220)."""
    N, K = codes.shape
    words = packed_words(N, K, bits)
    codes = codes.to(torch.uint8).contiguous()
    if codes.is_cuda:
        out = torch.empty(words, dtype=torch.int32, device=codes.device)
        lib = _lib.load()
        with torch.cuda.device(codes.device):
            _lib.check(lib.quip_pack_codes(_lib.ptr(codes), N, K, bits, _lib.ptr(out),
                                           C.c_void_p(torch.cuda.current_stream().cuda_stream)))
        return out
    c = codes.to(torch.int64)
    out = torch.zeros(words, dtype=torch.int64)
    for word, shift, cshift, nb in _native_fields(N, K, bits, codes.device):
        field = (c >> cshift) & ((1 << nb) - 1)
        out.index_add_(0, word.expand(N, K).reshape(-1), (field << shift.expand(N, K)).reshape(-1))
    out = torch.where(out >= 2 ** 31, out - 2 ** 32, out)
    return out.to(torch.int32)


def unpack_codes(qweight: torch.Tensor, N: int, K: int, bits: int) -> torch.Tensor:
    """Inverse of pack_codes -> (N, K) uint8; used for the bit-exact code check."""
    packed_words(N, K, bits)
    if qweight.is_cuda:
        out = torch.empty((N, K), dtype=torch.uint8, device=qweight.device)
        lib = _lib.load()
        with torch.cuda.device(qweight.device):
            _lib.check(lib.quip_unpack_codes(_lib.ptr(qweight.contiguous()), N, K, bits, _lib.ptr(out),
                                             C.c_void_p(torch.cuda.current_stream().cuda_stream)))
        return out
    q = qweight.to(torch.int64) & 0xFFFFFFFF
    c = torch.zeros((N, K), dtype=torch.int64)
    for word, shift, cshift, nb in _native_fields(N, K, bits, qweight.device):
        c |= ((q[word.expand(N, K)] >> shift.expand(N, K)) & ((1 << nb) - 1)) << cshift
    return c.to(torch.uint8)


def convert_ref_qweight(ref_qweight: torch.Tensor, K: int, N: int, bits: int) -> torch.Tensor:
    """Reference packed layouts (quant.py:192-220 3-bit, zeroShot/models/quant.py:193-199 4-bit, natural
    2-bit) -> codes (N, K) uint8, on the GPU."""
    if not ref_qweight.is_cuda:
        raise RuntimeError('convert_ref_qweight runs on the GPU; move the tensor to a CUDA device')
    assert tuple(ref_qweight.shape) == (K * bits // 32, N)
    out = torch.empty((N, K), dtype=torch.uint8, device=ref_qweight.device)
    lib = _lib.load()
    with torch.cuda.device(ref_qweight.device):
        _lib.check(lib.quip_convert_ref(_lib.ptr(ref_qweight.contiguous()), K, N, bits, _lib.ptr(out),
                                        C.c_void_p(torch.cuda.current_stream().cuda_stream)))
    return out


# ----------------------------------------------------------------------------------------------
# workspace (one per device, grown on demand; the 16 KiB header stays zero between calls)
# ----------------------------------------------------------------------------------------------
_workspaces = {}
_retired = []          # outgrown workspaces: a captured CUDA graph may still address them, so they are never freed


def _workspace(device, nbytes, stream_ptr=None):
    """One workspace per (device, stream): kernels of different streams may run concurrently.

    A workspace that is outgrown is kept alive (`_retired`) instead of freed: its address may be baked into a captured
    CUDA graph (GraphDecoder, GraphedSampleNLL), and torch hands out stream handles from a small pool, so a later,
    larger request can arrive under the same (device, stream) key.  Growth at least doubles, which bounds the retired
    bytes by the size of the live workspace."""
    if stream_ptr is None:
        stream_ptr = torch.cuda.current_stream(device).cuda_stream
    key = (device, stream_ptr)
    ws = _workspaces.get(key)
    if ws is None or ws.numel() < nbytes:
        if ws is not None:
            _retired.append(ws)
            nbytes = max(nbytes, 2 * ws.numel())
        ws = torch.zeros(max(nbytes, 1 << 20), dtype=torch.uint8, device=device)
        _workspaces[key] = ws
    return ws


class SiblingGroup:
    """Sibling QuantLinears that consume the SAME input (q/k/v; gate/up) run concurrently on side streams.

    Each packed forward is a chain of ~7 dependent kernels, several of them latency- rather than
    bandwidth-bound, and the contraction's tile count rarely fills a whole number of waves; three independent
    chains interleave on the SMs instead of queueing.  The first sibling called with a new input launches all
    of them (itself on the caller's stream, the others on their own streams after an event on the input);
    the later siblings return the already-launched result after making the caller's stream wait for it.
    Results are bit-identical to the serial order (same kernels, per-stream workspaces)."""

    def __init__(self, members):
        self.members = list(members)
        self.streams = None
        self._key = None
        self._x = None
        self._outs = [None] * len(self.members)
        self._events = [None] * len(self.members)
        for i, m in enumerate(self.members):
            m._group, m._group_index = self, i

    def dissolve(self):
        for m in self.members:
            m._group, m._group_index = None, 0
        self._x, self._key = None, None
        self._outs = [None] * len(self.members)

    def get(self, index, x, variant=None):
        # the pending input is held by a strong reference and compared by identity: its id / address cannot be reused by a
        # different tensor while sibling outputs are pending
        key = (x.data_ptr(), tuple(x.shape), x._version, variant)
        if x is not self._x or key != self._key or self._outs[index] is None:
            self._outs = [None] * len(self.members)         # outputs of an abandoned input are dropped
            self._x = x
            dev = x.device
            if self.streams is None or self.streams[0].device != dev:
                self.streams = [torch.cuda.Stream(device=dev) for _ in self.members[1:]]
            cur = torch.cuda.current_stream(dev)
            # inside a CUDA-graph capture the allocator's blocks are reused in stream order within the graph, and every
            # side stream starts behind `ready`: no record_stream there (it is an eager-mode allocator hint)
            capturing = torch.cuda.is_current_stream_capturing()
            ready = torch.cuda.Event()
            ready.record(cur)
            order = [index] + [j for j in range(len(self.members)) if j != index]
            for slot, j in enumerate(order):
                if slot == 0:
                    self._outs[j] = self.members[j]._forward_impl(x, variant=variant)
                    self._events[j] = None
                    continue
                st = self.streams[slot - 1]
                st.wait_event(ready)
                with torch.cuda.stream(st):
                    y = self.members[j]._forward_impl(x, variant=variant)
                    ev = torch.cuda.Event()
                    ev.record(st)
                if not capturing:
                    x.record_stream(st)
                self._outs[j], self._events[j] = y, ev
            self._key = key
        y, ev = self._outs[index], self._events[index]
        self._outs[index] = None
        if all(o is None for o in self._outs):
            self._x = None                                  # every sibling consumed: release the input
        if ev is not None:
            cur = torch.cuda.current_stream(x.device)
            cur.wait_event(ev)
            if not torch.cuda.is_current_stream_capturing():
                y.record_stream(cur)
        return y


def group_siblings(model):
    """Group q/k/v and gate/up (Llama) or q/k/v (OPT) QuantLinears of every decoder layer.  Returns the groups."""
    groups = []
    for mod in model.modules():
        for names in (('q_proj', 'k_proj', 'v_proj'), ('gate_proj', 'up_proj')):
            members = [getattr(mod, n, None) for n in names]
            if all(isinstance(m, QuantLinear) for m in members):
                groups.append(SiblingGroup(members))
    return groups


# ----------------------------------------------------------------------------------------------
# QuantLinear
# ----------------------------------------------------------------------------------------------
_INCOH_MODES = {None: None, 0: 'blocked', 1: 'kron', 2: 'noperm', 'blocked': 'blocked', 'kron': 'kron', 'noperm': 'noperm'}


class QuantLinear(nn.Module):
    """Packed 2/3/4-bit linear with fused dequant and incoherence un-projection.

    y = ((x / scaleWH) V^T) Q^T U + bias,   Q = scales*code - zeros      (SURVEY a6)

    `incoh` mirrors --pre_proj / --pre_proj_extra (method.py:125-180): None (no projection), 'blocked'
    (extra=0, what --incoh_processing actually runs, SURVEY A1), 'kron' (extra=1), 'noperm' (extra=2).
    `rescale` mirrors --pre_rescale.
    """

    def __init__(self, bits, infeatures, outfeatures, bias=True, incoh=None, rescale=False):
        super().__init__()
        if bits not in (2, 3, 4):
            raise NotImplementedError('Only 2, 3 and 4 bits are supported.')
        self.bits, self.infeatures, self.outfeatures = bits, infeatures, outfeatures
        self.in_features, self.out_features = infeatures, outfeatures
        self.incoh = _INCOH_MODES[incoh]
        self.rescale = bool(rescale)
        K, N = infeatures, outfeatures
        self.register_buffer('qweight', torch.zeros(packed_words(N, K, bits), dtype=torch.int32))
        self.register_buffer('scales', torch.zeros((N, 1)))
        self.register_buffer('zeros', torch.zeros((N, 1)))
        self.register_buffer('bias', torch.zeros(N, dtype=torch.float16) if bias else None)
        self.register_buffer('inv_scale', torch.ones(K) if rescale else None)
        # meta: [format version, symmetric grid, inv_scale folded into V factors, V idx identity, U idx identity]
        self.register_buffer('meta', torch.tensor([1, 0, 0, 0, 0], dtype=torch.int32))
        if self.incoh:
            for side, n in (('v', K), ('u', N)):
                p1, p2 = butterfly_factors(n)
                first, second = (p1, p2) if side == 'v' else (p2, p1)       # V: COL then ROW; U: ROW^T then COL^T
                nb0 = 1 if self.incoh == 'kron' else n // first
                nb1 = 1 if self.incoh == 'kron' else n // second
                self.register_buffer(f'{side}_idx', torch.arange(n, dtype=torch.int32))
                self.register_buffer(f'{side}_f0', torch.zeros((nb0, first, first), dtype=torch.float16))
                self.register_buffer(f'{side}_f1', torch.zeros((nb1, second, second), dtype=torch.float16))
        self._desc = None
        self._group, self._group_index = None, 0

    # -- construction ------------------------------------------------------------------------
    def pack(self, linear, scales, zeros):
        """Reference contract (quant.py:185-220): `linear.weight` holds grid values of a per-channel
        asymmetric quantizer (qfn 'a', no incoherence); `scales`/`zeros` are the Quantizer's.  Codes are
        recovered as round((W + zero*scale)/scale) exactly like quant.py:186-191."""
        if self.incoh or self.rescale:
            raise ValueError('pack(linear, scales, zeros) cannot recover U/V/scaleWH from a dense weight; '
                             'use pack_parts() with a capture of the quantization run')
        scales = scales.float().reshape(-1, 1)
        zeros_mul = zeros.float().reshape(-1, 1) * scales
        W = linear.weight.data.float()
        codes = torch.round((W + zeros_mul) / scales)
        if codes.min() < 0 or codes.max() > 2 ** self.bits - 1:
            raise ValueError('weights are not on the quantizer grid')
        bias = linear.bias.data if linear.bias is not None else None
        self._install(codes.to(torch.uint8), scales, zeros_mul, bias)

    def pack_parts(self, parts: LayerParts):
        """Build the packed module from a capture of the reference's quantization (quip_b200/capture.py)."""
        N, K = parts.codes.shape
        assert (K, N, parts.bits) == (self.infeatures, self.outfeatures, self.bits)
        codes, scales, zeros = parts.codes, parts.scales.float().reshape(-1, 1), parts.zeros.float().reshape(-1, 1)
        folded = 0
        if (parts.V is not None) != bool(self.incoh) or (parts.scaleWH is not None) != self.rescale:
            raise ValueError('layer parts do not match the module configuration (incoh / rescale)')
        inv_scale = None if parts.scaleWH is None else (1.0 / parts.scaleWH.float())
        if self.incoh:
            vp, up = plan_side(parts.V, 'V'), plan_side(parts.U, 'U')
            if inv_scale is not None and fold_inv_scale(vp, inv_scale):
                folded = 1
            codes = codes[:, vp.order.to(codes.device)]
            o = up.order.to(codes.device)
            codes, scales, zeros = codes[o], scales[o], zeros[o]
            for side, plan in (('v', vp), ('u', up)):
                n = plan.n
                idx = plan.idx if plan.idx is not None else torch.arange(n)
                getattr(self, f'{side}_idx').copy_(idx.to(torch.int32))
                self.meta[3 if side == 'v' else 4] = int(plan.idx is None)
                for i, ps in enumerate(plan.passes):
                    buf = getattr(self, f'{side}_f{i}')
                    assert tuple(buf.shape) == tuple(ps.factors.shape), (buf.shape, ps.factors.shape)
                    buf.copy_(ps.factors.to(torch.float16))
        if inv_scale is not None:
            self.inv_scale.copy_(inv_scale)
        self.meta[2] = folded
        self._install(codes, scales, zeros, parts.bias)

    def _install(self, codes, scales, zeros, bias):
        dev = self.qweight.device
        self.qweight.copy_(pack_codes(codes.to(dev), self.bits))
        self.scales.copy_(scales)
        self.zeros.copy_(zeros)
        cbar = (2 ** self.bits - 1) / 2.0
        sym = bool(torch.all((self.scales * cbar - self.zeros).abs() <= 1e-6 * self.zeros.abs().clamp_min(1e-30)))
        self.meta[1] = int(sym)
        if bias is not None:
            if self.bias is None:
                raise ValueError('module was built without a bias')
            self.bias.copy_(bias.to(torch.float16))
        self._desc = None

    def codes(self):
        """Integer codes (N, K) uint8 in packed (layout) order -- for the bit-exact check."""
        return unpack_codes(self.qweight, self.outfeatures, self.infeatures, self.bits)

    # -- C ABI descriptor ----------------------------------------------------------------------
    # dtypes the C ABI reads the buffers as (include/quip_b200.h): a blanket model.half() / .float() / .to(dtype) must not
    # change them -- the kernels would reinterpret the bytes
    _BUFFER_DTYPES = dict(qweight=torch.int32, meta=torch.int32, v_idx=torch.int32, u_idx=torch.int32, scales=torch.float32,
                          zeros=torch.float32, inv_scale=torch.float32, bias=torch.float16, v_f0=torch.float16,
                          v_f1=torch.float16, u_f0=torch.float16, u_f1=torch.float16)

    def _apply(self, fn, *a, **kw):
        self._desc = None
        out = super()._apply(fn, *a, **kw)
        for name, dt in self._BUFFER_DTYPES.items():
            buf = self._buffers.get(name)
            if buf is not None and buf.dtype != dt:
                self._buffers[name] = buf.to(dt)
        return out

    # the cached descriptor holds ctypes pointers into this module's buffers: copies and pickles rebuild it lazily
    _TRANSIENT = ('_desc', '_desc_ref', '_frag_keep', '_u_inv', '_ws_need', 'meta_host', '_variants')

    def __getstate__(self):
        st = dict(self.__dict__)
        for k in self._TRANSIENT:
            st.pop(k, None)
        st['_desc'] = None
        st['_group'], st['_group_index'] = None, 0
        return st

    def __deepcopy__(self, memo):
        import copy
        new = self.__class__.__new__(self.__class__)
        memo[id(self)] = new
        for k, v in self.__getstate__().items():
            new.__dict__[k] = copy.deepcopy(v, memo)
        return new

    def _load_from_state_dict(self, *a, **kw):
        self._desc = None                       # cached host copies (meta, fragment-order factors, inverse index) are stale
        return super()._load_from_state_dict(*a, **kw)

    def _side(self, side, n):
        s = _lib.QuipSide()
        if not self.incoh:
            s.n, s.npass = 0, 0
            return s
        p1, p2 = butterfly_factors(n)
        layout_a = p2 >= p1
        col = dict(p=p1, nblk=p2, strided=int(layout_a))
        row = dict(p=p2, nblk=p1, strided=int(not layout_a))
        order = (col, row) if side == 'v' else (row, col)
        s.n, s.npass = n, 2
        for i, d in enumerate(order):
            f = getattr(self, f'{side}_f{i}')
            s.passes[i].p, s.passes[i].nblk, s.passes[i].strided = d['p'], d['nblk'], d['strided']
            s.passes[i].shared = int(f.shape[0] == 1 and d['nblk'] > 1)
            s.passes[i].factors = f.data_ptr()
            s.passes[i].factors_frag = None
            if d['p'] in (32, 64) and n <= 4096:
                # tensor-core fragment order for the one-kernel sides (include/quip_b200.h): derived, not a checkpoint buffer
                frag = fragment_order(f)
                self._frag_keep[f'{side}{i}'] = frag
                s.passes[i].factors_frag = frag.data_ptr()
        identity = bool(self.meta_host[3 if side == 'v' else 4])
        s.idx = None if identity else getattr(self, f'{side}_idx').data_ptr()
        s.inv_idx = None
        if side == 'u' and not identity:
            # inverse of the output gather, derived once (not a checkpoint buffer): lets the few-token forward
            # scatter the last U pass straight into y
            idx = self.u_idx
            inv = torch.empty_like(idx)
            inv[idx.long()] = torch.arange(idx.numel(), dtype=idx.dtype, device=idx.device)
            self._u_inv = inv
            s.inv_idx = inv.data_ptr()
        return s

    def _descriptor(self):
        if self._desc is None:
            self.meta_host = self.meta.tolist()
            self._frag_keep = {}
            for name, dt in self._BUFFER_DTYPES.items():
                buf = self._buffers.get(name)
                if buf is not None and buf.dtype != dt:
                    raise TypeError(f'QuantLinear buffer {name!r} is {buf.dtype}, the packed kernels read it as {dt}')
            d = _lib.QuipLinearDesc()
            d.K, d.N, d.bits = self.infeatures, self.outfeatures, self.bits
            d.flags = _lib.QUIP_FLAG_SYMMETRIC if self.meta_host[1] else 0
            d.qweight, d.scales, d.zeros = self.qweight.data_ptr(), self.scales.data_ptr(), self.zeros.data_ptr()
            d.bias = None if self.bias is None else self.bias.data_ptr()
            use_scale = self.rescale and not self.meta_host[2]
            d.inv_scale = self.inv_scale.data_ptr() if use_scale else None
            d.V, d.U = self._side('v', self.infeatures), self._side('u', self.outfeatures)
            self._desc = d
            self._desc_ref = C.byref(d)
            self._ws_need = {}
            self._variants = {}
        return self._desc

    # -- layout-order variants (the glue of the fused Llama stack moves the permutations into its own kernels) -------
    def gather_index(self, side):
        """The index vector of the K-side ('v': layout[l] = x[idx[l]]) or N-side ('u': y[j] = layout[idx[j]]) gather as an
        int64 tensor, or None when it is the identity / the layer has no incoherence sides."""
        self._descriptor()
        if not self.incoh or self.meta_host[3 if side == 'v' else 4]:
            return None
        return getattr(self, f'{side}_idx').long()

    def layout_variant_ok(self, skip_in=False, skip_out=False):
        """Can forward_layout() skip the input gather (x already in V layout order) / the output gather (return y in U layout
        order)?  Needs the 1/scaleWH folded into the V factors (no per-feature scale left at the gather) and no bias."""
        self._descriptor()
        if not self.incoh:
            return False
        if skip_in and self.rescale and not self.meta_host[2]:
            return False
        if skip_out and self.bias is not None:
            return False
        return True

    def _variant(self, skip_in, skip_out):
        self._descriptor()
        key = (bool(skip_in), bool(skip_out))
        v = self._variants.get(key)
        if v is None:
            if not self.layout_variant_ok(skip_in, skip_out):
                raise ValueError('this layer cannot skip the requested gather (per-feature scale or bias at the gather)')
            d = _lib.QuipLinearDesc()
            C.memmove(C.byref(d), C.byref(self._desc), C.sizeof(d))
            if skip_in:
                d.V.idx = None
            if skip_out:
                d.U.idx, d.U.inv_idx = None, None
            v = self._variants[key] = (d, C.byref(d), {})
        return v

    def forward_layout(self, x, skip_in=False, skip_out=False):
        """forward() with the input taken in V layout order (skip_in: x[..., l] is already x_plain[..., v_idx[l]]) and / or the
        output returned in U layout order (skip_out: y_plain[..., j] = y[..., u_idx[j]]).  The permutations are pure data
        movement; callers that own the neighbouring elementwise kernels fold them there (quip_b200/fused.py)."""
        if not (skip_in or skip_out):
            return self.forward(x)
        variant = (bool(skip_in), bool(skip_out))
        if self._group is not None and x.is_cuda:          # siblings (gate / up) take the same variant, on their side streams
            return self._group.get(self._group_index, x, variant=variant)
        return self._forward_impl(x, variant=variant)

    # -- forward -------------------------------------------------------------------------------
    def forward(self, x):
        if self._group is not None and x.is_cuda:
            return self._group.get(self._group_index, x)
        return self._forward_impl(x)

    def _forward_impl(self, x, variant=None):
        if x.shape[-1] != self.infeatures:
            raise ValueError(f'expected last dimension {self.infeatures}, got {tuple(x.shape)}')
        if not (x.is_cuda and self.qweight.is_cuda):
            raise RuntimeError('QuantLinear.forward runs on a CUDA device only (there is no CPU fallback)')
        dtype = x.dtype
        xh = x.reshape(-1, self.infeatures)
        if xh.dtype != torch.float16:
            xh = xh.to(torch.float16)
        xh = xh.contiguous()
        M = xh.shape[0]
        y = torch.empty((M, self.outfeatures), dtype=torch.float16, device=x.device)
        if M:
            lib = _lib.load()
            d = self._descriptor()
            dref, ws_need = self._desc_ref, self._ws_need
            if variant is not None:
                d, dref, ws_need = self._variant(*variant)
            need = ws_need.get(M)                       # per token count: one C call the first time, a dict hit after
            if need is None:
                nb = C.c_size_t()
                _lib.check(lib.quip_qlinear_workspace_bytes(C.byref(d), M, C.byref(nb)))
                need = ws_need[M] = nb.value
            stream = torch.cuda.current_stream(x.device)
            ws = _workspace(x.device, need, stream.cuda_stream)
            if x.device.index == torch.cuda.current_device():
                _lib.check(lib.quip_qlinear_forward(dref, xh.data_ptr(), y.data_ptr(), M, ws.data_ptr(), ws.numel(),
                                                    stream.cuda_stream))
            else:
                with torch.cuda.device(x.device):
                    _lib.check(lib.quip_qlinear_forward(dref, xh.data_ptr(), y.data_ptr(), M, ws.data_ptr(),
                                                        ws.numel(), stream.cuda_stream))
        y = y.reshape(*x.shape[:-1], self.outfeatures)
        return y if dtype == torch.float16 else y.to(dtype)

    def extra_repr(self):
        return (f'in={self.infeatures}, out={self.outfeatures}, bits={self.bits}, bias={self.bias is not None}, '
                f'incoh={self.incoh}, rescale={self.rescale}')



# ----------------------------------------------------------------------------------------------
# the reference's own packed modules, running on the replacement of its absent quant_cuda extension
# ----------------------------------------------------------------------------------------------
def _vecquant(vec, mat, mul, scales, zeros, bits):
    if not (vec.is_cuda and mat.is_cuda and mul.is_cuda):
        raise RuntimeError('vecquant matmul runs on a CUDA device only (there is no CPU fallback)')
    K = vec.numel()
    N = mul.numel()
    if mat.dtype != torch.int32 or tuple(mat.shape) != (K * bits // 32, N):
        raise ValueError(f'packed matrix must be int32 ({K * bits // 32}, {N}), got {mat.dtype} {tuple(mat.shape)}')
    if vec.dtype != torch.float32 or mul.dtype != torch.float32 or not mul.is_contiguous():
        raise ValueError('vec and mul must be fp32 (mul contiguous: it is accumulated in place)')
    sc, ze = scales.reshape(-1).float().contiguous(), zeros.reshape(-1).float().contiguous()
    lib = _lib.load()
    with torch.cuda.device(vec.device):
        _lib.check(lib.quip_vecquant_matmul(_lib.ptr(vec.contiguous()), _lib.ptr(mat.contiguous()), _lib.ptr(mul), _lib.ptr(sc),
                                            _lib.ptr(ze), K, N, bits, C.c_void_p(torch.cuda.current_stream().cuda_stream)))


def vecquant3matmul(vec, mat, mul, scales, zeros):
    """quant_cuda.vecquant3matmul (quant.py:229-230): mul += (scales*code - zeros) . vec on the reference's 3-bit layout."""
    _vecquant(vec, mat, mul, scales, zeros, 3)


def vecquant4matmul(vec, mat, mul, scales, zeros):
    """quant_cuda.vecquant4matmul (zeroShot/models/quant.py:207-208), the 4-bit layout of Quant4Linear."""
    _vecquant(vec, mat, mul, scales, zeros, 4)


class Quant3Linear(nn.Module):
    """The reference's Quant3Linear (quant.py:173-233) with the same buffers, layout and single-token contract -- a
    state_dict written from the reference's module loads unchanged -- on quip_vecquant_matmul instead of quant_cuda.
    `to_native()` converts it into the QuantLinear of this package (any token count, tensor cores)."""
    BITS = 3

    def __init__(self, infeatures, outfeatures):
        super().__init__()
        self.infeatures, self.outfeatures = infeatures, outfeatures
        self.register_buffer('zeros', torch.zeros((outfeatures, 1)))
        self.register_buffer('scales', torch.zeros((outfeatures, 1)))
        self.register_buffer('bias', torch.zeros(outfeatures))
        self.register_buffer('qweight', torch.zeros((infeatures * self.BITS // 32, outfeatures), dtype=torch.int32))

    def forward(self, x):
        if x.shape[-1] == x.numel():                                  # quant.py:223: one token only
            outshape = list(x.shape)
            y = self.bias.float().clone()
            outshape[-1] = self.bias.numel()
            _vecquant(x.reshape(-1).float(), self.qweight, y, self.scales, self.zeros, self.BITS)
            return y.to(x.dtype).reshape(outshape)
        raise ValueError('Only supports a single token currently.')

    def to_native(self):
        q = QuantLinear(self.BITS, self.infeatures, self.outfeatures, bias=True).to(self.qweight.device)
        codes = convert_ref_qweight(self.qweight, self.infeatures, self.outfeatures, self.BITS)
        q._install(codes, self.scales.float().reshape(-1, 1), self.zeros.float().reshape(-1, 1), self.bias)
        return q


class Quant4Linear(Quant3Linear):
    """zeroShot/models/quant.py:185-212 (buffers and forward; construct empty and load_state_dict, or pack with
    quip_b200.quant.make_quant4 for the native module)."""
    BITS = 4

def spec_from_parts(parts: LayerParts):
    """Constructor keyword arguments of the QuantLinear that can hold `parts`."""
    incoh = None
    if parts.V is not None:
        kron = parts.V.B0.shape[0] == 1 and parts.V.n // parts.V.p1 > 1
        ident = torch.equal(parts.V.p_in, torch.arange(parts.V.n)) and torch.equal(parts.V.p_out, torch.arange(parts.V.n))
        incoh = 'kron' if kron else ('noperm' if ident else 'blocked')
    return dict(bits=parts.bits, bias=parts.bias is not None, incoh=incoh, rescale=parts.scaleWH is not None)


def make_quant(module, names, bits=None, name='', **kw):
    """Replace, in place, every attribute of `module` whose dotted name is in `names` by a QuantLinear of
    the same in/out features (reference make_quant3, quant.py:236-246).  `names` may be an iterable of
    names (all layers share `bits` / **kw) or a dict name -> LayerParts | dict of constructor kwargs."""
    if isinstance(module, QuantLinear):
        return
    for attr in dir(module):
        tmp = getattr(module, attr)
        name1 = name + '.' + attr if name != '' else attr
        if name1 in names and isinstance(tmp, nn.Module) and hasattr(tmp, 'in_features'):
            spec = dict(bits=bits, bias=getattr(tmp, 'bias', None) is not None, **kw)
            if isinstance(names, dict):
                v = names[name1]
                spec.update(spec_from_parts(v) if isinstance(v, LayerParts) else (v or {}))
            b = spec.pop('bits')
            setattr(module, attr, QuantLinear(b, tmp.in_features, tmp.out_features, **spec))
    for name1, child in module.named_children():
        make_quant(child, names, bits=bits, name=name + '.' + name1 if name != '' else name1, **kw)


def make_quant3(module, names, name=''):
    """Drop-in for the reference's 3-bit entry point (quant.py:236-246)."""
    make_quant(module, names, bits=3, name=name)


def make_quant4(module, quantizers, name=''):
    """Drop-in for zeroShot/models/quant.py:215-228 (constructs and packs from the quantizers)."""
    layers = {n: m for n, m in module.named_modules() if (name + '.' + n if name else n) in quantizers}
    make_quant(module, list(quantizers.keys()), bits=4, name=name)
    for n, lin in layers.items():
        full = name + '.' + n if name else n
        q = dict(module.named_modules())[n]
        q.pack(lin, quantizers[full].scale, quantizers[full].zero)
