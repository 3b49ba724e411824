"""quip_token_logprobs (csrc/logprob.cu) against the float64 oracle (oracle/loglik.py), and decode.score on a 7B-shaped
packed model against the reference harness's recipe (padded batch through model(ids), fp32 log_softmax, gather)."""
import numpy as np
import pytest
import torch

from oracle import loglik
from quip_b200 import fused

pytestmark = pytest.mark.gpu


def _run(x, t):
    lp = torch.full(t.shape, 7.0, dtype=torch.float32, device='cuda')
    gr = torch.full(t.shape, 9, dtype=torch.uint8, device='cuda')
    fused.token_logprobs(x, t, lp, gr)
    torch.cuda.synchronize()
    return lp, gr


def _check(x, t, lp, gr, rows):
    want_lp, want_g = loglik.token_logprobs(x[rows].float().cpu().numpy(), t[rows].cpu().numpy())
    got = lp[rows].double().cpu().numpy()
    m = np.abs(np.nan_to_num(x[rows].float().cpu().numpy(), nan=0.0)).max(1)
    ok = np.isnan(want_lp)
    assert (np.isnan(got) == ok).all()
    err = np.abs(got - want_lp)[~ok]
    assert (err <= 1e-5 + 1e-6 * m[~ok]).all(), err.max()
    assert gr[rows].cpu().numpy().tolist() == want_g.tolist()


@pytest.mark.parametrize('V', [1, 7, 199, 32000, 50272, 128256])
@pytest.mark.parametrize('R', [1, 3, 300, 4096])
def test_kernel_matches_the_float64_oracle_on_strided_unaligned_rows(R, V):
    g = torch.Generator(device='cuda').manual_seed(R * 7 + V)
    pad, off = 3 + V % 5, 1 + R % 7                                  # unaligned ld and row start
    buf = (torch.randn(R * (V + pad) + off + 8, generator=g, device='cuda') * 3).half()
    x = buf[off:off + R * (V + pad)].view(R, V + pad)[:, :V]
    t = torch.randint(0, V, (R,), generator=g, device='cuda')
    if R >= 3 and V > 4:                                               # planted ties at and around the target
        for r in range(min(R, 64)):
            top = x[r].max() + 1
            j = int(t[r])
            if r % 4 == 0:
                x[r, j] = top
                x[r, (j + 1) % V] = top                               # tie above: target wins only if lower
            elif r % 4 == 1:
                x[r, j] = top
                x[r, (j - 1) % V] = top                               # tie below: the lower index wins
            elif r % 4 == 2:
                x[r, j] = top
    lp, gr = _run(x, t)
    rows = np.arange(R) if R * V <= 2 ** 22 else np.unique(np.r_[np.arange(64), np.linspace(0, R - 1, 64).astype(int)])
    _check(x, t, lp, gr, rows)
    lp2, gr2 = _run(x, t)                                              # a second launch: the same bits
    assert torch.equal(lp.view(torch.int32), lp2.view(torch.int32)) and torch.equal(gr, gr2)


def test_nan_rows_and_out_of_range_targets_give_nan_and_zero_and_touch_nothing_else():
    R, V = 6, 1000
    g = torch.Generator(device='cuda').manual_seed(3)
    x = torch.randn(R, V, generator=g, device='cuda').half()
    x[1, 999] = float('nan')
    x[2, 0] = float('nan')
    t = torch.tensor([5, 5, 5, -1, V, 2 ** 40], dtype=torch.long, device='cuda')
    lp = torch.full((R + 2,), 7.0, device='cuda')
    gr = torch.full((R + 2,), 9, dtype=torch.uint8, device='cuda')
    fused.token_logprobs(x, t, lp[1:R + 1], gr[1:R + 1])
    torch.cuda.synchronize()
    assert float(lp[0]) == 7.0 and float(lp[-1]) == 7.0 and int(gr[0]) == 9 and int(gr[-1]) == 9
    assert not torch.isnan(lp[1]) and torch.isnan(lp[2:R + 1]).all()
    assert gr[2:R + 1].eq(0).all()
    _check(x, t.clamp(-1, V), lp[1:R + 1], gr[1:R + 1], np.arange(R))


def test_wrapper_checks_arguments_before_any_launch():
    x = torch.zeros(4, 10, dtype=torch.float16, device='cuda')
    t = torch.zeros(4, dtype=torch.long, device='cuda')
    lp = torch.zeros(4, device='cuda')
    gr = torch.zeros(4, dtype=torch.uint8, device='cuda')
    with pytest.raises(ValueError, match='fp16'):
        fused.token_logprobs(x.float(), t, lp, gr)
    with pytest.raises(ValueError, match='unit-stride'):
        fused.token_logprobs(x.t(), t, lp, gr)
    with pytest.raises(ValueError, match='targets'):
        fused.token_logprobs(x, t.int(), lp, gr)
    with pytest.raises(ValueError, match='greedy_out'):
        fused.token_logprobs(x, t, lp, gr.bool())
    with pytest.raises(RuntimeError, match='CUDA'):
        fused.token_logprobs(x, t.cpu(), lp, gr)


# ---- end to end on a 7B-shaped packed model (4 of its 32 layers)

@pytest.fixture(scope='module')
def model7b():
    from quip_b200.synth import build_synthetic_model, model_config
    cfg = model_config('llama7b', num_hidden_layers=4)
    return build_synthetic_model(cfg, torch.device('cuda:0'), bits=2, seed=3, seqlen=1024)


def _workload(V, docs=12, seed=0):
    g = torch.Generator().manual_seed(seed)
    ctxs, conts = [], []
    for _ in range(docs):
        ctx = torch.randint(0, V, (int(torch.randint(64, 300, (1,), generator=g)),), generator=g).tolist()
        for _ in range(4):
            ctxs.append(ctx)
            conts.append(torch.randint(0, V, (int(torch.randint(1, 17, (1,), generator=g)),), generator=g).tolist())
    return ctxs, conts


def reference_recipe(model, ctxs, conts, batch_size, max_length):
    """The harness's _loglikelihood_tokens on the packed model: right-padded batches through model(ids), fp32
    log_softmax of every position, gather; per-token log-probs and the margin of the argmax over the runner-up."""
    from quip_b200.decode import score_windows
    reqs = score_windows(ctxs, conts, max_length)
    res = [None] * len(ctxs)
    for s in range(0, len(reqs), batch_size):
        part = reqs[s:s + batch_size]
        P = len(part[0][0])
        ids = torch.zeros(len(part), P, dtype=torch.long)
        for b, (inp, _, _) in enumerate(part):
            ids[b, :len(inp)] = torch.tensor(inp)
        with torch.no_grad():
            logits = model(ids.cuda()).logits
        for b, (inp, cont, idx) in enumerate(part):
            n = len(cont)
            x = logits[b, len(inp) - n:len(inp)].float()
            lp = torch.log_softmax(x, -1).gather(-1, torch.tensor(cont, device='cuda')[:, None])[:, 0]
            top2 = x.topk(2, -1).values
            for i in idx:
                res[i] = (lp.double().cpu(), (x.argmax(-1).cpu() == torch.tensor(cont)),
                          (top2[:, 0] - top2[:, 1]).cpu())
    return res


def test_score_against_the_reference_recipe_within_three_times_the_control(model7b):
    import bench
    from quip_b200.decode import score
    from test_gpu_generate import _norms
    V = model7b.config.vocab_size
    ctxs, conts = _workload(V)
    L = 1024
    ref = reference_recipe(model7b, ctxs, conts, 8, L)
    other = reference_recipe(model7b, ctxs, conts, 3, L)               # the recipe at another batch composition
    batch_control = max(float((a[0] - b[0]).abs().max()) for a, b in zip(ref, other))
    # the packed GEMMs give every token the same bits at any batch composition (batch_control is 0), so the control is
    # the project's rounding-level one: the recipe against itself with one-ulp flips in 3e-5 of its norm outputs
    hooks = bench._ulp_flip_hooks(_norms(model7b), 3e-5, seed=1)
    try:
        ctl = reference_recipe(model7b, ctxs, conts, 8, L)
    finally:
        for hk in hooks:
            hk.remove()
    control = max(float((a[0] - b[0]).abs().max()) for a, b in zip(ref, ctl))
    runs = {share: score(model7b, ctxs, conts, batch_size=8, max_length=L, share_prompt_prefixes=share)
            for share in (False, True)}
    bound = 3 * control
    print(f'per-token control: batch composition {batch_control:.2e}, ulp flips {control:.2e}')
    for share, got in runs.items():
        worst = 0.0
        for (lp, g), (rlp, rg, margin), x in zip(got, ref, conts):
            worst = max(worst, abs(lp - float(rlp.sum())) / len(x))
            if g != bool(rg.all()):
                assert float(margin.min()) < 0.05, (share, margin)      # a near-tie decides the flag
        print(f'share={share}: worst per-request |diff| / tokens against the recipe {worst:.2e}')
        assert worst <= bound, (share, worst, control)
    for (a, ga), (b, gb), x in zip(runs[False], runs[True], conts):
        assert abs(a - b) / len(x) <= bound
    e4 = score(model7b, ctxs, conts, batch_size=8, max_length=L, kv_dtype=torch.float8_e4m3fn)
    diff = max(abs(a - b) for (a, _), (b, _) in zip(e4, runs[False]))
    agree = np.mean([ga == gb for (_, ga), (_, gb) in zip(e4, runs[False])])
    print(f'control {control:.2e}; e4m3 vs fp16: largest logprob difference {diff:.3e}, is_greedy agreement {agree:.3f}')
    assert np.isfinite(diff)
