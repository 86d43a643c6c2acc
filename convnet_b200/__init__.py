"""convnet_b200 — H100-native (sm_90a) conv / pool / response-norm / gradient-sync hot path of
TorontoDeepLearning/convnet behind the reference's own C ABI.

The product is the C-ABI shared library convnet_b200/lib/libconvnet_b200.so
(include/*.h).  This package is the thin host side used by tests and bench:
  abi       ctypes mirror of cudamat / Shape4D / ConvDesc (cudamat/cudamat.py:127-185)
  lib       loads the library and declares every entry point (fails loudly if it is missing)
  matrix    CUDAMatrix: a column-major device matrix + Shape4D (mirror of cudamat.CUDAMatrix)
  conv_gemm the reference's python binding surface (cudamat/cudamat_conv_gemm.py:61-157)
"""
from .abi import ConvDesc, GetConvDesc, Shape4D, cudamat, num_modules  # noqa: F401

__version__ = "0.1.0"
