"""ctypes door onto oracle/_ref/libcudamat_conv_gemm_ref.so (TEST INFRASTRUCTURE).

That file is the reference's own CUDA implementation of the path — cudamat/cudamat_conv_gemm.cu and
cudamat_conv3d_gemm.cu compiled UNMODIFIED for sm_90 by oracle/Makefile — so on the GPU it is
"the reference on the same inputs" at BASELINE sizes, where the CPU oracle would take hours (tests record its outputs
into tests/golden/ref_cuda_samples.npz, see tests/test_gpu_vs_reference_cuda.py).
It exports the same ABI-1 symbols as the product, so the product's python surface
(convnet_b200.conv_gemm.Binding) is simply bound to it.  Only tests/ may import this module.
"""
import ctypes as ct
import os

from convnet_b200.conv_gemm import Binding
from convnet_b200.lib import SIGNATURES

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PATH = os.path.join(ROOT, "oracle", "_ref", "libcudamat_conv_gemm_ref.so")

# what cudamat_conv_gemm.cuh:36-138 declares and the tests call
_NAMES = ["convUpGemm", "convDownGemm", "convOutpGemm", "localUpGemm", "localDownGemm", "localOutpGemm",
          "MaxPoolGemm", "AvgPoolGemm", "MaxPoolUndoGemm", "AvgPoolUndoGemm", "UpSampleGemm", "DownSampleGemm",
          "ResponseNormCrossMapGemm", "ResponseNormCrossMapUndoGemm", "convUp3DGemm", "convDown3DGemm",
          "convOutp3DGemm", "ResponseNormCrossMap3DGemm", "ResponseNormCrossMap3DUndoGemm"]

_lib = None


def available():
    return os.path.exists(PATH)


def load():
    global _lib
    if _lib is None:
        lib = ct.CDLL(PATH, mode=ct.RTLD_LOCAL)      # same symbol names as the product: keep them out of the global scope
        for n in _NAMES:
            fn = getattr(lib, n)
            fn.argtypes = SIGNATURES[n]
            fn.restype = None
        # the reference uses the legacy cuBLAS API, which its host (src/matrix.cc:510 -> cudamat.cu:57) initialises
        # with cublasInit(); the symbol is reachable through the library's own dependency on libcublas
        init = lib.cublasInit
        init.restype = ct.c_int
        status = init()
        assert status == 0, "cublasInit failed: %d" % status
        _lib = lib
    return _lib


def binding():
    """the ABI-1 python surface bound to the reference's CUDA library"""
    return Binding(load, "gemm")
