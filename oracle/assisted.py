"""Assisted generation (quip_b200/decode.py: AssistedDecoder) as a cache-free loop: each model is re-run on the whole
sequence for every token it scores.  Because nothing is cached, a decoder that matches it keeps its assistant's cache
right across rounds (the T = 2 catch-up step over the current token and the one before it)."""
import numpy as np


def assisted_generate(target_fn, assistant_fn, prompt, max_new, k, select):
    """target_fn / assistant_fn: a sequence of ids -> its logits (len, vocab), row j predicting token j + 1.
    select(z, t): the token chosen from logits z (vocab,) as generated token t (argmax, or a seeded draw at step t).

    The first token is select(target(prompt)[-1], 0).  A round with g tokens generated and the sequence seq (prompt and
    tokens) drafts d_1 .. d_k, d_i = select(assistant(seq + d_1 .. d_(i-1))[-1], g + i - 1); scores y_i =
    select(target(seq + d_1 .. d_k)[len(seq) - 1 + i], g + i) for i = 0 .. k; and takes y_0 .. y_a, a the longest prefix
    with d_(i+1) == y_i, cut to max_new tokens in all.  Returns (the max_new tokens, the drafts accepted in each round:
    the tokens it took minus one)."""
    seq = [int(x) for x in prompt]
    out = [int(select(np.asarray(target_fn(seq))[-1], 0))]
    seq.append(out[0])
    rounds = []
    while len(out) < max_new:
        g = len(out)
        drafts = []
        for i in range(k):
            drafts.append(int(select(np.asarray(assistant_fn(seq + drafts))[-1], g + i)))
        z = np.asarray(target_fn(seq + drafts))
        targets = [int(select(z[len(seq) - 1 + i], g + i)) for i in range(k + 1)]
        a = 0
        while a < k and drafts[a] == targets[a]:
            a += 1
        e = min(a + 1, max_new - g)
        out += targets[:e]
        seq += targets[:e]
        rounds.append(e - 1)
    return out, rounds
