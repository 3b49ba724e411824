"""Prompt-lookup drafting and acceptance of speculative generation (include/quip_b200.h: quip_ngram_draft,
quip_spec_accept) as plain numpy loops: the reference the torch restatements in quip_b200/decode.py and the kernels of
csrc/spec.cu are checked against."""
import numpy as np


def ngram_draft(hist, positions, k, n_min, n_max):
    """tokens (B, 1 + k): the current token hist[b, c], c = positions[b], and k drafts.  The match is the end e < c whose
    common suffix with hist[b, ..c] is longest (capped at n_max, at least n_min), the latest e on ties; the drafts copy
    what followed it, u[e + 1 ..], where u is the history up to c followed by the drafts themselves.  No match: the
    current token repeated.  c outside [0, max_len): zeros."""
    hist = np.asarray(hist, dtype=np.int64)
    B, max_len = hist.shape
    out = np.zeros((B, k + 1), dtype=np.int64)
    for b in range(B):
        c = int(positions[b])
        if not 0 <= c < max_len:
            continue
        h = hist[b]
        best_l, best_e = 0, -1
        for e in range(c):
            length = 0
            while length < n_max and length <= e and h[e - length] == h[c - length]:
                length += 1
            if length >= n_min and (length > best_l or (length == best_l and e > best_e)):
                best_l, best_e = length, e
        u = list(h[:c + 1])
        for i in range(1, k + 1):
            u.append(u[c] if best_e < 0 else u[best_e + i])
        out[b] = u[c:]
    return out


def spec_accept(tokens, targets, generated, hist, positions, n_gen, accepted, max_new):
    """In place on numpy int64 arrays: for each row with n_gen < max_new, a = the longest prefix of drafts with
    tokens[b][i] == targets[b][i - 1], e = min(a + 1, max_new - n_gen); targets[b][:e] go to generated[b, n_gen ..] and
    hist[b, positions + 1 ..] (below max_len); positions and n_gen advance by e, accepted by e - 1."""
    B, T = tokens.shape
    for b in range(B):
        g = int(n_gen[b])
        if not 0 <= g < max_new:
            continue
        a = 0
        while a < T - 1 and tokens[b, a + 1] == targets[b, a]:
            a += 1
        e = min(a + 1, max_new - g)
        c = int(positions[b])
        for j in range(e):
            generated[b, g + j] = targets[b, j]
            if 0 <= c + 1 + j < hist.shape[1]:
                hist[b, c + 1 + j] = targets[b, j]
        positions[b] = c + e
        n_gen[b] = g + e
        accepted[b] += e - 1
