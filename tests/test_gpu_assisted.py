"""Assisted generation on the GPU (quip_b200/decode.py: AssistedDecoder, generate(assistant_model=...)) on the synthetic
packed models of test_gpu_speculative.py, each with a shallower packed assistant of the same vocabulary: graph replay
against the eager round, the target as its own assistant (rejections only at near ties), assisted against plain
generation, the verify step's logits against eager HF, and sampled runs from run to run."""
import pytest
import torch

pytestmark = pytest.mark.gpu

KINDS = [(4, 64), (2, 64), (2, 128), 'opt']


def _tiny(kind):
    from test_gpu_speculative import _tiny as tiny
    return tiny(kind)


def _assistant(kind):
    """One decoder layer of the target's shape with other weights: same vocabulary, drafts that are often wrong."""
    from transformers import LlamaConfig, OPTConfig
    from quip_b200.synth import build_synthetic_model
    if kind == 'opt':
        cfg = OPTConfig(hidden_size=256, ffn_dim=1024, num_hidden_layers=1, num_attention_heads=4, vocab_size=320,
                        max_position_embeddings=128, word_embed_proj_dim=256)
    else:
        nkv, hd = kind
        cfg = LlamaConfig(hidden_size=4 * hd, intermediate_size=512, num_hidden_layers=1, num_attention_heads=4,
                          num_key_value_heads=nkv, vocab_size=320, max_position_embeddings=128)
    return build_synthetic_model(cfg, torch.device('cuda:0'), bits=2, incoh='blocked', rescale=True, seed=6, seqlen=64)


def _prompts(shared=False):
    from test_gpu_speculative import _prompts as prompts
    if not shared:
        return prompts()
    g = torch.Generator().manual_seed(8)
    base = torch.randint(0, 320, (70,), generator=g)
    return [base, torch.cat((base[:66], torch.tensor([3, 4]))), torch.randint(0, 320, (9,), generator=g)]


def _run(model, assistant, prompts, n, k, capture, kv_dtype=None, shared=False, record=False):
    """An AssistedDecoder's run: (decoder, [(n_gen before, n_gen after, the verify logits (B, T, vocab), the
    assistant's k logits (B, vocab) when record)] per round).  shared: a paged cache planned by plan_prefix_pages,
    prefilled in chunks of 32."""
    from quip_b200.decode import AssistedDecoder, plan_prefix_pages
    max_len = max(p.numel() for p in prompts) + n + k
    kw, pre = {}, {}
    if shared:
        table, n_pages, starts = plan_prefix_pages(prompts, [p.numel() + n + k for p in prompts],
                                                   max_pages=-(-max_len // 64))
        kw, pre = dict(page_table=table, n_pages=n_pages), dict(chunk=32, starts=starts)
    dec = AssistedDecoder(model, assistant, max_len=max_len, batch=len(prompts), max_new=n, draft_tokens=k,
                          kv_dtype=kv_dtype, **kw)
    if capture:
        dec.capture()
    drafts = []
    if record:                                        # eager only: the assistant's logits of every draft
        assist = dec._assist

        def logged(tokens):
            z = assist(tokens)
            drafts[-1].append(z.float().clone())
            return z
        dec._assist = logged
    log = []
    with torch.no_grad():
        dec.prefill(prompts, **pre)
        for _ in range(n - 1):
            drafts.append([])
            g0 = dec.n_gen.clone()
            logits = dec.step().float().clone()
            log.append((g0, dec.n_gen.clone(), logits, drafts[-1]))
    return dec, log


def _plain(model, prompts, n, kv_dtype=None, shared=False):
    """The captured PromptDecoder's tokens and logits per generated token (index j predicts generated[j])."""
    from quip_b200.decode import PromptDecoder, plan_prefix_pages
    max_len = max(p.numel() for p in prompts) + n
    kw, pre = {}, {}
    if shared:
        table, n_pages, starts = plan_prefix_pages(prompts, [p.numel() + n for p in prompts],
                                                   max_pages=-(-max_len // 64))
        kw, pre = dict(page_table=table, n_pages=n_pages), dict(chunk=32, starts=starts)
    dec = PromptDecoder(model, max_len=max_len, batch=len(prompts), max_new=n, kv_dtype=kv_dtype, **kw).capture()
    with torch.no_grad():
        logits = [dec.prefill(prompts, **pre).float().clone()]
        logits += [dec.step().float().clone() for _ in range(n - 1)]
    return dec.generated.cpu(), logits


@pytest.mark.parametrize('kind', KINDS)
def test_assisted_graph_replay_equals_the_eager_round(kind):
    model, assistant = _tiny(kind), _assistant(kind)
    for k in (1, 4):
        e, elog = _run(model, assistant, _prompts(), 16, k, capture=False)
        g, glog = _run(model, assistant, _prompts(), 16, k, capture=True)
        assert torch.equal(e.generated, g.generated) and torch.equal(e.accepted, g.accepted)
        for (a0, a1, la, _), (b0, b1, lb, _) in zip(elog, glog):
            assert torch.equal(a0, b0) and torch.equal(a1, b1) and torch.equal(la, lb)


@pytest.mark.parametrize('kind', KINDS)
def test_self_assisted_rounds_reject_a_draft_only_at_a_near_tie(kind):
    """With the target as its own assistant a draft and the target's token come from the same model on the same
    prefix by two routes (the assistant's T = 2 and T = 1 steps, the verify step at T = k + 1), so they differ only
    where the target's top-2 gap is within twice the largest logit difference of the two routes."""
    model = _tiny(kind)
    n, k = 24, 4
    dec, log = _run(model, model, _prompts(), n, k, capture=False, record=True)
    full = rejected = 0
    for g0, g1, logits, drafts in log:
        for b in range(logits.shape[0]):
            s, e = int(g0[b]), int(g1[b])
            if s >= n:
                continue
            a = e - s - 1                                            # drafts accepted
            if a == k:
                full += 1
            elif e < n:                                              # a rejection, not the budget's cut
                rejected += 1
                zt, za = logits[b, a], drafts[a][b]
                top2 = zt.topk(2).values
                assert float(top2[0] - top2[1]) <= 2 * float((zt - za).abs().max()), (b, s, a)
    assert full > rejected and full >= 5, (full, rejected)


@pytest.mark.parametrize('shared', [False, True])
@pytest.mark.parametrize('kv_dtype', [None, torch.float8_e4m3fn])
@pytest.mark.parametrize('kind', KINDS)
def test_assisted_equals_plain_generation_away_from_near_ties(kind, kv_dtype, shared):
    """As for prompt lookup: a token can differ only where the plain run's top-2 gap is at most twice the largest
    logit difference of the two runs at that position; up to the first such position the tokens must agree."""
    model, assistant = _tiny(kind), _assistant(kind)
    prompts, n, k = _prompts(shared), 20, 3
    dec, log = _run(model, assistant, prompts, n, k, capture=True, kv_dtype=kv_dtype, shared=shared)
    plain_gen, plogits = _plain(model, prompts, n, kv_dtype=kv_dtype, shared=shared)
    gen = dec.generated.cpu()
    checked = 0
    for b in range(len(prompts)):
        slog = {}
        for g0, g1, logits, _ in log:
            for i in range(int(g1[b]) - int(g0[b])):
                slog[int(g0[b]) + i] = logits[b, i]
        assert int(gen[b, 0]) == int(plain_gen[b, 0])
        for j in range(1, n):
            top2 = plogits[j][b].topk(2).values
            if float(top2[0] - top2[1]) <= 2 * float((slog[j] - plogits[j][b]).abs().max()):
                break
            assert int(gen[b, j]) == int(plain_gen[b, j]), (b, j)
            checked += 1
    assert checked >= n, checked


def _norms(model):
    from test_gpu_speculative import _norms as norms
    return norms(model)


@pytest.mark.parametrize('kv_dtype', [None, torch.float8_e4m3fn])
@pytest.mark.parametrize('kind', KINDS)
def test_assisted_verify_logits_match_eager_hf(kind, kv_dtype):
    import bench
    model, assistant = _tiny(kind), _assistant(kind)
    prompts, n = _prompts(), 20
    dec, log = _run(model, assistant, prompts, n, 4, capture=True, kv_dtype=kv_dtype)
    gen = dec.generated.cpu()
    assert dec.n_gen.tolist() == [n] * len(prompts)
    worst = control = 0.0
    for b, p in enumerate(prompts):
        fed = torch.cat((p, gen[b, :n - 1])).cuda()[None]
        runs = []
        for flip in (False, True):
            hooks = bench._ulp_flip_hooks(_norms(model), 3e-5, seed=b) if flip else []
            try:
                with torch.no_grad():
                    runs.append(model(fed).logits[0].float())
            finally:
                for hk in hooks:
                    hk.remove()
        want, ctrl = runs
        P = p.numel()
        for g0, g1, logits, _ in log:
            s, e = int(g0[b]), int(g1[b])
            for i in range(e - s):
                assert int(logits[b, i].argmax()) == int(gen[b, s + i]), (b, s, i)
                w = want[P + s - 1 + i]
                worst = max(worst, float((logits[b, i] - w).norm() / w.norm()))
                control = max(control, float((ctrl[P + s - 1 + i] - w).norm() / w.norm()))
    if kv_dtype is None:
        assert worst < max(2e-3, 3.0 * control), (worst, control)
    else:                                                             # one e4m3 rounding of every cached key and value
        assert worst < 0.1, (worst, control)


def test_sampled_assisted_generation_is_reproducible():
    from quip_b200.decode import generate
    model = _tiny((2, 64))
    prompts = _prompts()
    kw = dict(do_sample=True, seed=[1, 2, 3], top_k=20, temperature=0.8)
    for assistant in (model, _assistant((2, 64))):
        runs = []
        for _ in range(2):
            stats = {}
            runs.append(generate(model, prompts, 24, assistant_model=assistant, num_assistant_tokens=4,
                                 spec_stats=stats, **kw))
            assert [o.numel() for o in runs[-1]] == [24] * 3
        assert all(torch.equal(x, y) for x, y in zip(*runs))
        if assistant is model:
            assert sum(stats['accepted']) > 0
