"""The sampling kernel (csrc/sample.cu, quip_sample) against oracle/sampling.py, its distribution, determinism and row
independence, and sampled generation (PromptDecoder(sampling=True), generate(do_sample=True)) on synthetic packed models."""
import numpy as np
import pytest
import torch

from oracle import sampling as S

pytestmark = pytest.mark.gpu

# (temperature, top_k, top_p); top_k None: V + 3.  Tie-heavy and all-equal rows take settings that keep few tokens: the
# oracle's margin is relative to S, so a flat row with every token kept lies near a boundary by that measure.
RANDOM = [(0.7, 50, 0.9), (0.6, 0, 0.9), (0.6, 0, 1.0), (1.3, 20, 1.0), (0.0, 0, 1.0), (0.8, 1, 1.0), (1.0, 5, 0.5),
          (0.5, None, 0.95), (1.0, 0, 1e-6), (1.0, 3, 0.01), (2.0, 40, 0.8)]
FLAT = [(0.7, 5, 1.0), (1.0, 1, 1.0), (0.0, 0, 1.0), (1.0, 3, 0.9), (1.0, 0, 1e-6), (2.0, 10, 1.0), (0.9, 12, 0.45)]


def _rows(V, B, seed):
    """Logits (B, V) fp16 on the CPU -- random (scale 4 or 8), tie-heavy (6 distinct values) and all-equal rows in turn --
    with mixed per-row settings and seeds (bits >= 2^63 included)."""
    g = torch.Generator().manual_seed(seed)
    x = torch.empty(B, V)
    T, k, p, sd = [], [], [], []
    for b in range(B):
        kind = b % 3
        if kind == 0:
            x[b] = torch.randn(V, generator=g) * (4.0 if b % 2 else 8.0)
            t, kk, pp = RANDOM[(b // 3) % len(RANDOM)]
        else:
            x[b] = torch.randint(0, 6, (V,), generator=g).float() * 1.5 if kind == 1 else 0.25
            t, kk, pp = FLAT[(b // 3 + kind) % len(FLAT)]
        T.append(t)
        k.append(V + 3 if kk is None else kk)
        p.append(pp)
        sd.append(int(torch.randint(0, 2 ** 62, (1,), generator=g)) * 4 + b % 4)
    return x.half(), T, k, p, sd


def _bits(seeds):
    return torch.tensor([s - 2 ** 64 if s >= 2 ** 63 else s for s in seeds], dtype=torch.int64)


def _launch(x, T, k, p, seeds, t):
    from quip_b200 import fused
    dev = 'cuda'
    out = torch.full((x.shape[0],), -1, dtype=torch.int64, device=dev)
    fused.sample(x.to(dev).contiguous(), torch.tensor(T, dtype=torch.float32, device=dev),
                 torch.tensor(k, dtype=torch.int32, device=dev), torch.tensor(p, dtype=torch.float32, device=dev),
                 _bits(seeds).to(dev), torch.tensor([t], dtype=torch.int64, device=dev), out)
    return out.cpu()


VS = [1, 7, 320, 32000, 32001, 50272, 128256]
BS = [1, 5, 64]


def _oracle(x, T, k, p, sd, t):
    return [S.sample_row(x[b].float().numpy(), T[b], k[b], p[b], sd[b], t) for b in range(x.shape[0])]


def test_kernel_picks_the_oracle_token():
    total = amb = 0
    bad = []
    for V in VS:
        for B in BS:
            t = V % 997 + B
            x, T, k, p, sd = _rows(V, B, seed=V + B)
            got = _launch(x, T, k, p, sd, t)
            want = _oracle(x, T, k, p, sd, t)
            for b in range(B):
                g = int(got[b])
                assert 0 <= g < V, (V, B, b, g)
                total += 1
                if want[b]['ambiguous']:
                    amb += 1
                    continue
                if g != want[b]['token']:
                    bad.append((V, B, b, T[b], k[b], p[b], g, want[b]['token']))
    assert not bad, (len(bad), bad[:5])
    assert amb < 0.01 * total, (amb, total)


def test_greedy_rows_equal_argmax_bit_for_bit():
    for V in (7, 320, 32001, 128256):
        g = torch.Generator().manual_seed(V)
        B = 48
        x = torch.randn(B, V, generator=g).half()
        x[1::2] = (torch.randint(0, 4, (B // 2, V), generator=g).float() * 0.5).half()      # tie-heavy rows
        x[2] = 0.0
        x[4, ::2] = -0.0                                              # -0 and +0 are equal: the first index wins
        T = [0.0 if b % 2 else 0.9 for b in range(B)]
        k = [0 if b % 2 else 1 for b in range(B)]
        got = _launch(x, T, k, [0.5] * B, list(range(B)), 3)
        assert torch.equal(got, x.cuda().argmax(-1).cpu()), V


def test_draws_follow_the_oracle_distribution():
    """One peaked row (V = 1000) with T = 0.8, top-k 200, drawn with seeds 0 .. 65535 in one launch: a chi-square test
    against the oracle's float64 probabilities, bins pooled to expected counts >= 5, passes at p-value 1e-6; no draw lies
    outside the top-k set."""
    from scipy.stats import chisquare
    V, N = 1000, 65536
    g = torch.Generator().manual_seed(42)
    row = (torch.randn(V, generator=g) * 2.5).half()
    T, k = 0.8, 200
    got = _launch(row[None].expand(N, V).contiguous(), [T] * N, [k] * N, [1.0] * N, list(range(N)), 5)
    want = S.sample_row(row.float().numpy(), T, k, 1.0, 0, 5)
    kept, probs = want['kept'], want['probs']
    assert np.isin(got.numpy(), kept).all()
    counts = np.bincount(got.numpy(), minlength=V)[kept].astype(np.float64)
    exp = probs * N
    order = np.argsort(exp)
    obs_b, exp_b, po, pe = [], [], 0.0, 0.0
    for i in order:                                                   # pool the smallest bins until each holds >= 5
        po, pe = po + counts[i], pe + exp[i]
        if pe >= 5:
            obs_b.append(po)
            exp_b.append(pe)
            po = pe = 0.0
    if pe:
        obs_b[-1] += po
        exp_b[-1] += pe
    assert chisquare(obs_b, exp_b).pvalue > 1e-6


def test_deterministic_and_independent_of_the_other_rows():
    V, B = 50272, 64
    x, T, k, p, sd = _rows(V, B, seed=9)
    a = _launch(x, T, k, p, sd, 17)
    assert torch.equal(a, _launch(x, T, k, p, sd, 17))
    y, T2, k2, p2, sd2 = _rows(V, B, seed=10)
    for b in (0, 1, 2, 30):
        y[b], T2[b], k2[b], p2[b], sd2[b] = x[b], T[b], k[b], p[b], sd[b]
    c = _launch(y, T2, k2, p2, sd2, 17)
    for b in (0, 1, 2, 30):
        assert int(c[b]) == int(a[b]), b
    one = _launch(x[30:31], T[30:31], k[30:31], p[30:31], sd[30:31], 17)
    assert int(one[0]) == int(a[30])


@pytest.mark.parametrize('kv', [None, torch.float8_e4m3fn])
@pytest.mark.parametrize('kind', [(2, 64), (2, 128), 'opt'])
def test_sampling_decoder_graph_equals_eager_and_the_oracle(kind, kv):
    from test_gpu_generate import _prompts, _tiny
    from quip_b200.decode import PromptDecoder
    model = _tiny(kind)
    prompts, n = _prompts(), 10
    settings = dict(temperature=[0.9, 1.2, 0.7], top_k=[0, 40, 5], top_p=[0.95, 1.0, 0.8], seed=[3, 2 ** 64 - 5, 11])
    runs = []
    for graph in (False, True):
        with torch.no_grad():
            dec = PromptDecoder(model, max_len=40, batch=3, max_new=n, kv_dtype=kv, sampling=True)
            dec.set_sampling(**settings)
            if graph:
                dec.capture()
            logits = [dec.prefill(prompts).float().cpu()]
            logits += [dec.step().float().cpu() for _ in range(n - 1)]
            runs.append((dec.generated.cpu(), logits))
    (ge, le), (gg, lg) = runs
    assert torch.equal(ge, gg)
    for a, b in zip(le, lg):
        assert torch.equal(a, b)
    checked = 0
    for t in range(n):
        for b in range(3):
            w = S.sample_row(lg[t][b].numpy(), settings['temperature'][b], settings['top_k'][b], settings['top_p'][b],
                             settings['seed'][b], t)
            if not w['ambiguous']:
                assert int(gg[b, t]) == w['token'], (t, b)
                checked += 1
    assert checked >= 0.7 * 3 * n


@pytest.mark.parametrize('kind', [(2, 64), 'opt'])
def test_generate_top_k_one_equals_greedy(kind):
    from test_gpu_generate import _prompts, _tiny
    from quip_b200.decode import generate
    model = _tiny(kind)
    prompts = _prompts()
    want = generate(model, prompts, 16)
    got = generate(model, prompts, 16, do_sample=True, top_k=1, temperature=0.8, seed=[1, 2, 3])
    assert all(torch.equal(a, b) for a, b in zip(got, want))
    sampled = generate(model, prompts, 16, do_sample=True, temperature=1.0, seed=[1, 2, 3])
    again = generate(model, prompts, 16, do_sample=True, temperature=1.0, seed=[1, 2, 3])
    assert all(torch.equal(a, b) for a, b in zip(sampled, again))
