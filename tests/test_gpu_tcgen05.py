"""Tensor-core (wgmma + TMA) GEMM vs the CPU oracle (kept in its own file: see tests/test_gpu_kernels.py)."""
import numpy as np
import pytest

from oracle import forward as ofw
from test_gpu_kernels import _qgemm_case

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize('bits', [2, 3, 4])
@pytest.mark.parametrize('M', [33, 128, 129, 300, 2048])
@pytest.mark.parametrize('symmetric', [True, False])
def test_qgemm_tc_vs_oracle(bits, M, symmetric):
    from gpu_util import run_qgemm
    shapes = [(128, 128), (256, 1024), (384, 640)] if M < 2048 else [(512, 1024)]
    for (N, K) in shapes:
        codes, scales, zeros, X, bias, want = _qgemm_case(bits, N, K, M, symmetric, bits * 10 + M)
        z, _ = run_qgemm(codes, scales, zeros, bits, X, path=2, bias=bias, symmetric=symmetric)
        assert not np.isnan(z.astype(np.float32)).any()
        err = ofw.rel_err(z, want)
        assert err < 3e-4, (bits, M, symmetric, N, K, err)


def test_qgemm_tc_small_M_and_ragged_N():
    from gpu_util import run_qgemm
    for (N, K, M) in [(48, 256, 5), (144, 384, 40), (4096, 4096, 64)]:
        codes, scales, zeros, X, bias, want = _qgemm_case(2, N, K, M, False, N + M)
        z, _ = run_qgemm(codes, scales, zeros, 2, X, path=2, bias=bias, symmetric=False)
        assert ofw.rel_err(z, want) < 3e-4, (N, K, M)


def test_tc_and_skinny_agree():
    from gpu_util import run_qgemm
    codes, scales, zeros, X, bias, want = _qgemm_case(2, 512, 1024, 24, True, 99)
    a, _ = run_qgemm(codes, scales, zeros, 2, X, path=1, bias=bias, symmetric=True)
    b, _ = run_qgemm(codes, scales, zeros, 2, X, path=2, bias=bias, symmetric=True)
    assert ofw.rel_err(a, b) < 2e-4


def test_big_block_pass_on_tensor_cores():
    """Block-diagonal pass with 688 x 688 blocks (the 11008 side of Llama-2-7B) through the TMA-fed wgmma kernel."""
    from gpu_util import run_pass
    from oracle import butterfly as obf
    for (p, nblk, M, shared) in [(688, 16, 2048, False), (224, 32, 300, False), (128, 8, 129, True), (96, 4, 64, False)]:
        rng = np.random.default_rng(p + M)
        n = p * nblk
        X = rng.standard_normal((M, n)).astype(np.float16)
        F = (rng.standard_normal((1 if shared else nblk, p, p)) / np.sqrt(p)).astype(np.float16)
        want = obf.apply_pass(X.astype(np.float64), F.astype(np.float64), p, nblk, False)
        got = run_pass(X, F, p, nblk, False, impl=0)
        assert ofw.rel_err(got, want) < 4e-4, (p, nblk, M)
        legacy = run_pass(X, F, p, nblk, False, impl=3)        # mma.sync tiled kernel
        assert ofw.rel_err(legacy, want) < 4e-4
