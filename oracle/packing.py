"""Packed-integer layouts (CPU oracle, numpy, bit-exact).

Reference layouts (what a reference-quantized checkpoint would hold):
  * 3-bit: Quant3Linear.pack, reference quant.py:185-220 -- codes transposed to
    (K, N), 32 consecutive k packed into 3 int32 rows; codes 10 and 21 of every
    32 straddle a word boundary.  Requires K % 1024 == 0 there (quant.py:182);
    the restatement only needs K % 32 == 0.
  * 4-bit: Quant4Linear.__init__, reference zeroShot/models/quant.py:193-199 --
    8 codes per word, code i at bits 4*(i%8) of row i//8.
  * 2-bit: not defined by the reference; the natural extension (16 codes per
    word, code i at bits 2*(i%16) of row i//16) is provided for completeness.

Native layout (what the sm_90a kernels read; documented in DESIGN.md):
  The (N, K) code matrix is cut into super-blocks of 16 rows x 128 k, stored
  [row_block][k_superblock].  Inside a super-block the data are laid out per
  *lane* l = 4*g + t of a warp, lane l owning rows {g, g+8} and, in each of the
  4 chunks of 32 k, the 8 consecutive k = 32*ch + 8*t + [0,8).  Those 16 codes
  per (lane, chunk) are stored as 8 "pairs" (two consecutive k of one row), the
  first element of a pair in the low half-word and the second in the high one,
  so that one shift + one LOP3 drops both into the mantissa of an fp16 pair.
  Pair u = pos//2 of row half r = (row >= 8) sits in slot j = 2*perm(u) + r,
  perm = [0,2,1,3]: then byte b of the word holds k offsets {0,2,1,3}[b] (low
  nibble) and 4+{0,2,1,3}[b] (high nibble), each nibble = (row g, row g+8), which
  is what the int8 tensor-core path masks out with four ANDs (csrc/common.cuh):
      bits=2: 1 word / (lane,chunk): pair j at bits 2j and 16+2j;
              lane's 4 chunk words are contiguous (one 128-bit load).
      bits=4: 2 words / (lane,chunk) (pos 0-3, pos 4-7): slot j' = 2*((pos%4)//2) + (row >= 8)
              at bits 4j', 16+4j';
              two 128-bit segments per super-block (chunks 0-1, chunks 2-3).
      bits=3: the upper two bits use the bits=2 layout ("hi plane"), followed by a
              "lo plane" of the lowest bit: 2 words / lane, word ch//2, pair
              8*(ch%2)+j at bits jj and 16+jj.
  This is exactly the A-fragment ownership of mma.sync.m16n8k16 (rows g/g+8,
  k-pairs) with k re-labelled so a lane's 8 k's are contiguous, which also makes
  them one 16-byte chunk of a 128B-swizzled K-major wgmma operand row.

Test infrastructure only (see oracle/__init__.py).
"""
import numpy as np

SB_ROWS, SB_K = 16, 128
SB_WORDS = {2: 128, 3: 192, 4: 256}


# --------------------------------------------------------------------------
# reference layouts
# --------------------------------------------------------------------------
def ref_pack3(codes_nk):
    """quant.py:192-220.  codes (N, K) uint8 < 8  ->  qweight int32 (K*3/32, N)."""
    c = np.ascontiguousarray(np.asarray(codes_nk).T).astype(np.uint32)      # (K, N) quant.py:192
    K, N = c.shape
    assert K % 32 == 0
    g = c.reshape(K // 32, 32, N)
    q = np.zeros((K // 32, 3, N), np.uint32)
    for j in range(10):                                                      # :200-201
        q[:, 0] |= g[:, j] << np.uint32(3 * j)
    q[:, 0] |= g[:, 10] << np.uint32(30)                                     # :203 (upper bit falls off)
    q[:, 1] |= (g[:, 10] >> np.uint32(2)) & np.uint32(1)                     # :205
    for j in range(10):                                                      # :207-208
        q[:, 1] |= g[:, 11 + j] << np.uint32(3 * j + 1)
    q[:, 1] |= g[:, 21] << np.uint32(31)                                     # :210
    q[:, 2] |= (g[:, 21] >> np.uint32(1)) & np.uint32(3)                     # :212
    for j in range(10):                                                      # :214-215
        q[:, 2] |= g[:, 22 + j] << np.uint32(3 * j + 2)
    return q.reshape(K // 32 * 3, N).view(np.int32)


def ref_unpack3(qweight, K):
    q = np.asarray(qweight).view(np.uint32)
    N = q.shape[1]
    q = q.reshape(K // 32, 3, N)
    g = np.zeros((K // 32, 32, N), np.uint32)
    for j in range(10):
        g[:, j] = (q[:, 0] >> np.uint32(3 * j)) & np.uint32(7)
        g[:, 11 + j] = (q[:, 1] >> np.uint32(3 * j + 1)) & np.uint32(7)
        g[:, 22 + j] = (q[:, 2] >> np.uint32(3 * j + 2)) & np.uint32(7)
    g[:, 10] = (q[:, 0] >> np.uint32(30)) | ((q[:, 1] & np.uint32(1)) << np.uint32(2))
    g[:, 21] = (q[:, 1] >> np.uint32(31)) | ((q[:, 2] & np.uint32(3)) << np.uint32(1))
    return np.ascontiguousarray(g.reshape(K, N).T).astype(np.uint8)


def ref_pack4(codes_nk):
    """zeroShot/models/quant.py:193-199: qweight[i//8] |= code[i] << 4*(i%8)."""
    c = np.ascontiguousarray(np.asarray(codes_nk).T).astype(np.uint32)
    K, N = c.shape
    assert K % 8 == 0
    g = c.reshape(K // 8, 8, N)
    q = np.zeros((K // 8, N), np.uint32)
    for i in range(8):
        q |= g[:, i] << np.uint32(4 * i)
    return q.view(np.int32)


def ref_unpack4(qweight, K):
    q = np.asarray(qweight).view(np.uint32)
    N = q.shape[1]
    g = np.stack([(q >> np.uint32(4 * i)) & np.uint32(15) for i in range(8)], axis=1)
    return np.ascontiguousarray(g.reshape(K, N).T).astype(np.uint8)


def ref_pack2(codes_nk):
    """Natural 2-bit extension of the reference scheme (SURVEY a3)."""
    c = np.ascontiguousarray(np.asarray(codes_nk).T).astype(np.uint32)
    K, N = c.shape
    assert K % 16 == 0
    g = c.reshape(K // 16, 16, N)
    q = np.zeros((K // 16, N), np.uint32)
    for i in range(16):
        q |= g[:, i] << np.uint32(2 * i)
    return q.view(np.int32)


def ref_unpack2(qweight, K):
    q = np.asarray(qweight).view(np.uint32)
    N = q.shape[1]
    g = np.stack([(q >> np.uint32(2 * i)) & np.uint32(3) for i in range(16)], axis=1)
    return np.ascontiguousarray(g.reshape(K, N).T).astype(np.uint8)


# --------------------------------------------------------------------------
# native fragment-major layout
# --------------------------------------------------------------------------
def native_words(N, K, bits):
    assert N % SB_ROWS == 0 and K % SB_K == 0 and bits in (2, 3, 4)
    return (N // SB_ROWS) * (K // SB_K) * SB_WORDS[bits]


def _coords(N, K):
    n = np.arange(N, dtype=np.int64)[:, None]
    k = np.arange(K, dtype=np.int64)[None, :]
    rb, r = n // 16, n % 16
    g, hi_row = r % 8, r // 8
    ks, kk = k // 128, k % 128
    ch, t, pos = kk // 32, (kk % 32) // 8, kk % 8
    lane = g * 4 + t
    e = pos % 2
    sb = rb * (K // 128) + ks
    return sb, lane, ch, pos, hi_row, e


def native_index(N, K, bits):
    """For every (n, k): list of (word index, bit shift, code-bit shift, nbits) planes."""
    sb, lane, ch, pos, hi_row, e = _coords(N, K)
    base = sb * SB_WORDS[bits]
    u = pos // 2
    j = 2 * ((u % 2) * 2 + u // 2) + hi_row           # pair slot 0..7 inside a (lane, chunk), see below
    if bits == 2:
        return [(base + lane * 4 + ch, 2 * j + 16 * e, 0, 2)]
    if bits == 4:
        w = pos // 4
        jp = 2 * ((pos % 4) // 2) + hi_row
        word = base + (ch // 2) * 128 + lane * 4 + (ch % 2) * 2 + w
        return [(word, 4 * jp + 16 * e, 0, 4)]
    hi = (base + lane * 4 + ch, 2 * j + 16 * e, 1, 2)
    jj = 8 * (ch % 2) + j
    lo = (base + 128 + lane * 2 + ch // 2, jj + 16 * e, 0, 1)
    return [hi, lo]


def native_pack(codes_nk, bits):
    c = np.asarray(codes_nk).astype(np.uint32)
    N, K = c.shape
    out = np.zeros(native_words(N, K, bits), np.uint32)
    for word, shift, cshift, nb in native_index(N, K, bits):
        field = (c >> np.uint32(cshift)) & np.uint32((1 << nb) - 1)
        np.add.at(out, np.broadcast_to(word, c.shape).ravel(),
                  (field << shift.astype(np.uint32)).ravel())
    return out.view(np.int32)


def native_unpack(qweight, N, K, bits):
    q = np.asarray(qweight).view(np.uint32).ravel()
    c = np.zeros((N, K), np.uint32)
    for word, shift, cshift, nb in native_index(N, K, bits):
        w = q[np.broadcast_to(word, c.shape)]
        c |= ((w >> shift.astype(np.uint32)) & np.uint32((1 << nb) - 1)) << np.uint32(cshift)
    return c.astype(np.uint8)
