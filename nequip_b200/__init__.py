"""nequip_b200 -- H100-native (sm_90a) implementation of NequIP's per-edge equivariant
convolution hot path, behind the reference's ``TensorProductScatter`` operator interface.

Layout:
  csrc/        CUDA: libnqb.so runtime (C ABI in include/nqb.h) + device vocabulary of the
               generated tensor-product kernels
  codegen.py   per-signature kernel generator;  cg.py / irreps.py: host-side tables
  build.py     in-tree nvcc builds (sm_90a)
  ops.py       torch autograd glue over the C ABI (no CPU fallback)
  nn/          host-side mirrors of the reference's operator interface
"""
from .irreps import Irrep, Irreps, build_tp_instructions  # noqa: F401

__version__ = "0.1.0"
