"""supir_b200 — H100 (sm_90a) backend for SUPIR's EDM sampling hot path.

Hand-written CUDA kernels behind a C ABI (include/supir_b200.h, supir_b200/csrc/), driven by host classes that mirror
the reference's sgm / SUPIR plugin surface (same class names, constructor parameters, state_dict keys and call
signatures). See DESIGN.md and INTEGRATION.md. There is no CPU or PyTorch fallback for the compute path.
"""
__version__ = "0.1.0"
