"""CPU oracle for the QuIP packed-linear hot path.  TEST INFRASTRUCTURE ONLY.

This package restates, in numpy / CPU torch, the algorithm of the reference's
(Cornell-RelaxML/QuIP) hot path so the CUDA kernels can be checked against it:

  qmath.py      code <-> value maps and quantizer parameters
                (reference quant.py:6-21, 57-163; vector_balance.py:499-532)
  packing.py    reference 3-/4-bit packed layouts (quant.py:185-220,
                zeroShot/models/quant.py:185-199), the natural 2-bit extension,
                and the native fragment-major layout the sm_90a kernels read
  butterfly.py  structured orthogonal multiply (method.py:16-78)
  forward.py    W_ref reconstruction (method.py:195-214) and the factored
                forward  y = ((x / s) V^T) Q^T U + b
  evalloop.py   port of the per-layer eval loop (opt.py:193-299,
                llama.py:174-253) used as the CPU baseline

Only `tests/`, `__graft_entry__.smoke()` and `bench.py`'s cpu_baseline /
`--impl reference` legs may import this package, and only as the checker.
Nothing under `quip_b200/` imports it; the product path fails loudly when the
CUDA extension is missing.

Parity pinning: the reference ships NO golden vectors or tests for this path
(SURVEY.md section 4).  The oracle is therefore pinned against outputs of the
reference itself, generated in the build container by `oracle/gen_golden.py`
(which imports /root/reference with a `primefac` stand-in) and committed under
`tests/golden/`.  `tests/test_oracle_golden.py` re-checks every restatement
here against those files.  The one boundary that stays unpinned is the absent
third-party `quant_cuda.vecquant{3,4}matmul` extension (IST-DASLab/gptq, no
version pinned anywhere in the reference): its semantics are inferred from the
reference's `pack()` routines and call signature only.
"""
