"""Continuation scoring (quip_b200.decode.score, PromptDecoder.prefill_scores, quip_b200.zeroshot.PackedLM) on tiny fp32
HF models on the CPU, where csrc/logprob.cu's rule runs as its torch restatement.

tests/golden/loglik.npz holds the reference harness's own answers (oracle/gen_golden_loglik.py) on a GQA Llama and a
post-LN OPT with project_in / project_out, for string requests under the tokenizer [ord(c) % V for c in s]."""
import json
import os

import numpy as np
import pytest
import torch

from oracle import loglik
from quip_b200 import decode
from quip_b200.decode import PromptDecoder, score
from quip_b200.zeroshot import PackedLM

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'loglik.npz')


def _fixture():
    z = np.load(GOLDEN)
    meta = json.loads(str(z['meta']))
    return z, meta


def _fixture_model(z, meta, kind):
    from transformers import LlamaConfig, LlamaForCausalLM, OPTConfig, OPTForCausalLM
    cfg = meta['configs'][kind]
    m = (OPTForCausalLM(OPTConfig(**cfg)) if kind == 'opt' else LlamaForCausalLM(LlamaConfig(**cfg))).float().eval()
    sd = {k[len(kind) + 1:]: torch.from_numpy(z[k]) for k in z.files if k.startswith(kind + '/')}
    m.load_state_dict(sd)
    return m


class _Tok:
    def __init__(self, V, eot):
        self.V, self.eos_token_id = V, eot

    def encode(self, s, add_special_tokens=True):
        assert add_special_tokens is False
        return [ord(c) % self.V for c in s]


def _requests(z):
    return list(zip(z['contexts'].tolist(), z['continuations'].tolist()))


@pytest.mark.parametrize('kind', ['llama', 'opt'])
@pytest.mark.parametrize('kw', [dict(), dict(share_prompt_prefixes=False), dict(prefill_chunk_size=7)])
def test_packed_lm_reproduces_the_reference_harness(kind, kw):
    z, meta = _fixture()
    m = _fixture_model(z, meta, kind)
    lm = PackedLM(m, _Tok(meta['V'], meta['eot']), batch_size=meta['batch_size'], max_length=meta['max_length'], **kw)
    got = lm.loglikelihood(_requests(z))
    want_lp, want_g = z[f'{kind}_logprob'], z[f'{kind}_greedy']
    assert len(got) == len(want_lp)
    for i, ((lp, g), wl, wg) in enumerate(zip(got, want_lp, want_g)):
        assert abs(lp - wl) <= 1e-5, (i, lp, wl)
        assert g == bool(wg), i


def test_the_fixture_shares_pages_and_truncates():
    z, meta = _fixture()
    tok = _Tok(meta['V'], meta['eot'])
    reqs = _requests(z)
    ctxs = [[meta['eot']] if c == '' else tok.encode(c, False) for c, _ in reqs]
    conts = [tok.encode(x, False) for _, x in reqs]
    wins = decode.score_windows(ctxs, conts, meta['max_length'])
    assert any(len(c) + len(x) > meta['max_length'] + 1 for c, x in zip(ctxs, conts))
    assert len(wins) < len(reqs)                                       # repeated requests are computed once
    B, shared = meta['batch_size'], 0
    for s in range(0, len(wins), B):                                   # the batches score() plans
        part = wins[s:s + B]
        heads = [torch.tensor(w[0][:len(w[0]) - len(w[1]) + 1]) for w in part]
        shared += sum(1 for x in decode.plan_prefix_pages(heads, [len(w[0]) for w in part])[2] if x)
    assert shared >= 3


def test_window_arithmetic_equals_the_reference_inputs():
    z, meta = _fixture()
    tok = _Tok(meta['V'], meta['eot'])
    reqs = _requests(z)
    ctxs = [[meta['eot']] if c == '' else tok.encode(c, False) for c, _ in reqs]
    conts = [tok.encode(x, False) for _, x in reqs]
    want = loglik.windows(ctxs, conts, meta['max_length'])
    got = decode.score_windows(ctxs, conts, meta['max_length'])
    assert [(list(a), list(b), list(c)) for a, b, c in got] == [(list(a), list(b), list(c)) for a, b, c in want]
    for kind in ('llama', 'opt'):
        rows = z[f'{kind}_inps']
        assert rows.shape[0] == len(want)
        for row, (inp, _, _) in zip(rows, want):
            assert np.trim_zeros(row, 'b').tolist() == inp                 # no token of the fixture is 0


def test_cpu_rule_equals_the_float64_oracle():
    g = torch.Generator().manual_seed(0)
    x = (torch.randn(9, 37, generator=g) * 4).half()
    x[1, 5] = x[1, 20] = x[1].max() + 1                                 # a tie: the lower index wins
    x[2, 3] = float('nan')
    t = torch.randint(0, 37, (9,), generator=g)
    t[1], t[4], t[5] = 5, -1, 37
    lp, gr = decode._token_logprobs_torch(x, t)
    want_lp, want_g = loglik.token_logprobs(x.float().numpy(), t.numpy())
    np.testing.assert_allclose(lp.double().numpy(), want_lp, rtol=0, atol=1e-5)
    assert np.isnan(lp.numpy()).tolist() == np.isnan(want_lp).tolist()
    assert gr.numpy().tolist() == want_g.tolist()
    assert int(gr[1]) == 1


# ---- invariances on the four tiny models of test_generate.py

KINDS = ['llama_mha', 'llama_gqa', 'opt_pre_ln', 'opt_post_ln']


def _model(kind):
    torch.manual_seed(0)
    if kind.startswith('opt'):
        from transformers import OPTConfig, OPTForCausalLM
        pre = kind == 'opt_pre_ln'
        cfg = OPTConfig(hidden_size=64, ffn_dim=128, num_hidden_layers=2, num_attention_heads=4, vocab_size=199,
                        max_position_embeddings=40, word_embed_proj_dim=64 if pre else 48, do_layer_norm_before=pre)
        return OPTForCausalLM(cfg).float().eval()
    from transformers import LlamaConfig, LlamaForCausalLM
    cfg = LlamaConfig(hidden_size=128, intermediate_size=352, num_hidden_layers=2, num_attention_heads=4,
                      num_key_value_heads=4 if kind == 'llama_mha' else 2, vocab_size=199, max_position_embeddings=64)
    return LlamaForCausalLM(cfg).float().eval()


def _docs(kind, seed=0):
    """Multiple-choice documents: a shared context and 2-4 continuations each, sized to the model's positions."""
    g = torch.Generator().manual_seed(seed)
    short = kind.startswith('opt')                                    # 40 learned positions
    ctxs, conts = [], []
    for d in range(5):
        n = int(torch.randint(3, 25 if short else 150, (1,), generator=g))
        ctx = torch.randint(3, 199, (n,), generator=g).tolist()
        for _ in range(int(torch.randint(2, 5, (1,), generator=g))):
            ctxs.append(ctx)
            conts.append(torch.randint(3, 199, (int(torch.randint(1, 8, (1,), generator=g)),), generator=g).tolist())
    return ctxs, conts, (39 if short else 200)


def _close(a, b, tol=1e-6):
    assert len(a) == len(b)
    for i, ((la, ga), (lb, gb)) in enumerate(zip(a, b)):
        assert abs(la - lb) <= tol * max(1.0, abs(lb)), (i, la, lb)
        assert ga == gb, i


@pytest.mark.parametrize('kind', KINDS)
def test_shared_batch_size_and_chunk_size_do_not_change_the_scores(kind):
    m = _model(kind)
    ctxs, conts, L = _docs(kind)
    base = score(m, ctxs, conts, batch_size=4, max_length=L, share_prompt_prefixes=False, prefill_chunk_size=64)
    _close(score(m, ctxs, conts, batch_size=4, max_length=L, prefill_chunk_size=64), base)
    for bs in (1, 3, 100):
        _close(score(m, ctxs, conts, batch_size=bs, max_length=L, prefill_chunk_size=64), base)
    for c in (1, 7):
        _close(score(m, ctxs, conts, batch_size=4, max_length=L, prefill_chunk_size=c), base)


@pytest.mark.parametrize('kind', ['llama_gqa', 'opt_post_ln'])
def test_e4m3_scores_equal_teacher_forced_prefill_over_the_quantized_cache(kind):
    m = _model(kind)
    ctxs, conts, L = _docs(kind, seed=1)
    ctxs, conts = ctxs[:5], conts[:5]
    got = score(m, ctxs, conts, batch_size=2, max_length=L, kv_dtype=torch.float8_e4m3fn, prefill_chunk_size=16)
    for (lp, gr), c, x in zip(got, ctxs, conts):
        inp = (c + x)[-(L + 1):][:-1]
        tot, greedy = 0.0, True
        for k, t in enumerate(x):
            j = len(inp) - len(x) + k                                   # position j predicts x[k]
            dec = PromptDecoder(m, max_len=len(inp), batch=1, kv_dtype=torch.float8_e4m3fn)
            logits = dec.prefill([torch.tensor(inp[:j + 1])], chunk=16)[0].float()
            tot += float(torch.log_softmax(logits, -1)[t])
            greedy &= int(logits.argmax()) == t
        assert abs(lp - tot) <= 1e-5, (lp, tot)
        assert gr == greedy


def test_prefill_scores_positions_and_scored_count():
    m = _model('llama_gqa')
    dec = PromptDecoder(m, max_len=20, batch=2)
    p = [torch.arange(3, 15), torch.arange(5, 10)]
    lp, gr = dec.prefill_scores(p, [torch.tensor([7, 8, 9]), torch.tensor([], dtype=torch.long)], chunk=4)
    assert lp.shape == (3,) and gr.dtype == torch.bool
    assert dec.positions.tolist() == [12, 5]
    with torch.no_grad():
        full = torch.log_softmax(m(p[0][None]).logits[0].float(), -1)
    want = full[torch.arange(9, 12), torch.tensor([7, 8, 9])]
    torch.testing.assert_close(lp, want, rtol=0, atol=1e-5)


def test_argument_errors_are_raised_before_any_work(monkeypatch):
    m = _model('llama_mha')

    def boom(*a, **k):
        raise AssertionError('work started')
    monkeypatch.setattr(PromptDecoder, '__init__', boom)
    ok_c, ok_x = [[3, 4]], [[5]]
    cases = [
        (dict(contexts=[[3]], continuations=[]), 'contexts'),
        (dict(contexts=[], continuations=[]), 'no requests'),
        (dict(contexts=[[]], continuations=ok_x), 'empty context'),
        (dict(contexts=ok_c, continuations=[[]]), 'empty continuation'),
        (dict(contexts=[[3, 199]], continuations=ok_x), 'token ids'),
        (dict(contexts=ok_c, continuations=[[-1]]), 'token ids'),
        (dict(contexts=ok_c, continuations=ok_x, batch_size=0), 'batch_size'),
        (dict(contexts=ok_c, continuations=ok_x, batch_size=2.5), 'batch_size'),
        (dict(contexts=ok_c, continuations=ok_x, prefill_chunk_size=None), 'prefill_chunk_size'),
        (dict(contexts=ok_c, continuations=ok_x, prefill_chunk_size=0), 'chunk size'),
        (dict(contexts=ok_c, continuations=ok_x, max_length=0), 'max_length'),
        (dict(contexts=ok_c, continuations=[[5, 6, 7]], max_length=2), 'longer than max_length'),
        (dict(contexts=ok_c, continuations=ok_x, kv_dtype=torch.bfloat16), 'kv_dtype'),
    ]
    for kw, msg in cases:
        with pytest.raises(ValueError, match=msg):
            score(m, **kw)
    o = _model('opt_pre_ln')
    with pytest.raises(ValueError, match='learned positions'):
        score(o, ok_c, ok_x, max_length=41)
    monkeypatch.undo()
    lm = PackedLM(m, _Tok(199, 1), batch_size=2, max_length=32)
    with pytest.raises(NotImplementedError):
        lm.loglikelihood_rolling([('a',)])
    with pytest.raises(NotImplementedError):
        lm.greedy_until([('a', ['.'])])
    dec = PromptDecoder(m, max_len=16, batch=1)
    with pytest.raises(ValueError, match='targets must lie'):
        dec.prefill_scores([torch.arange(3, 9)], [torch.tensor([199])], chunk=4)
    with pytest.raises(ValueError, match='at most its prompt length'):
        dec.prefill_scores([torch.arange(3, 6)], [torch.arange(3, 7)], chunk=4)
    with pytest.raises(ValueError, match='page_table needs a paged'):
        dec.prefill_scores([torch.arange(3, 6)], [torch.arange(3, 4)], chunk=4, page_table=[[0]])
    paged = PromptDecoder(m, max_len=16, batch=1, n_pages=2)
    with pytest.raises(ValueError, match='page ids'):
        paged.prefill([torch.arange(3, 6)], chunk=4, page_table=[[2]])
