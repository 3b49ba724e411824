"""quip_b200: H100-native packed QuantLinear path for QuIP-quantized OPT / Llama models.

Host code is Python/PyTorch mirroring the reference's quant.py / opt.py / llama.py surface; the
compute runs in hand-written sm_90a kernels behind a C ABI (include/quip_b200.h,
quip_b200/libquip_b200.so).  Importing the package does not load the library; the first packed
forward (or `quip_b200._lib.load()`) does, and fails loudly if it is missing.
"""
from .quant import QuantLinear, Quantizer, make_quant, make_quant3, make_quant4  # noqa: F401
from .modelutils import find_layers  # noqa: F401

__all__ = ['QuantLinear', 'Quantizer', 'make_quant', 'make_quant3', 'make_quant4', 'find_layers']
