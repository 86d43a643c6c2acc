"""GPU parity tests (run with -m gpu on an H100): every C-ABI entry point of
libconvnet_b200.so against the CPU oracle and the committed golden vectors.

Metric: the reference's own Diff = max|a-b| / mean|a+b| (py/test_conv.py:382-385).
Tolerances (stated once, used everywhere):
  FP32 mode (CUDA-core fp32)            : 1e-4  — the reference's own bar (py/test_conv.py:387)
  TF32 mode (mma.sync tf32)             : 5e-3  — the tensor core reads the fp32 operands' top 19 bits
                                                   (10-bit mantissa, truncated), fp32 accumulate
  BF16 mode (wgmma, bf16 operands)      : 2.5e-2 — operands rounded to bf16 (8-bit mantissa, nearest even) by the
                                                   staging pass, fp32 accumulate
  max-pool values                       : bit-exact
  avg-pool / pool-undo / response-norm  : 1e-4  (rnorm uses __powf like the reference GPU build)
"""
import numpy as np
import pytest

from cases import F, GOLDEN_2D, GOLDEN_3D, Z, geo2d, geo3d, load_golden
from convnet_b200.abi import GetConvDesc, num_modules
from oracle_lib import Diff

pytestmark = pytest.mark.gpu

TOL = {"fp32": 1e-4, "tf32": 5e-3, "bf16": 2.5e-2}
TOL_MEM = 1e-4


@pytest.fixture(scope="module")
def gpu():
    import torch
    assert torch.cuda.is_available(), "these tests need a CUDA device"
    from convnet_b200 import conv_gemm as cg
    from convnet_b200 import lib
    from convnet_b200.matrix import CUDAMatrix
    lib.load()

    class G:
        pass
    g = G()
    g.cg, g.lib, g.M, g.torch = cg, lib, CUDAMatrix, torch
    g.up = lambda a, s4=None: CUDAMatrix.from_numpy(a, s4)
    g.new = lambda r, c, s4=None: CUDAMatrix(r, c, s4)

    def nan_like(r, c, s4=None):
        m = CUDAMatrix(r, c, s4)
        m.fill_(float("nan"))
        return m
    g.nan = nan_like
    yield g
    lib.set_precision("tf32")


# ------------------------------------------------------------------------------------------
# 1. golden vectors produced by the reference's py/conv_cpu.py
# ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", ["fp32", "tf32", "bf16"])
@pytest.mark.parametrize("name", GOLDEN_2D)
def test_golden_conv2d(gpu, name, mode):
    gpu.lib.set_precision(mode)
    g = load_golden(name)
    d, pd, ish, fsh, tsh, psh = geo2d(g)
    N = g["N"]
    images, filters, derivs = gpu.up(g["images"], ish), gpu.up(g["filters"], fsh), gpu.up(g["derivs"], tsh)
    out = gpu.nan(N, g["convUp"].shape[1], tsh); gpu.cg.convUp(images, filters, out, d)
    assert Diff(out.asarray(), g["convUp"]) < TOL[mode]
    out = gpu.nan(N, g["convDown"].shape[1], ish); gpu.cg.convDown(derivs, filters, out, d)
    assert Diff(out.asarray(), g["convDown"]) < TOL[mode]
    out = gpu.nan(*g["convOutp"].shape, fsh); gpu.cg.convOutp(images, derivs, out, d)
    assert Diff(out.asarray(), g["convOutp"]) < TOL[mode]
    # ABI-2 partial sums
    chunks = g["convOutpPartial"].shape[1] // g["convOutp"].shape[1]
    out = gpu.nan(*g["convOutpPartial"].shape, (g["Cout"], g["kx"], g["ky"], g["Cin"] * chunks))
    gpu.cg.convOutpPartial(images, derivs, out, d, g["psy"], g["psx"])
    assert Diff(out.asarray(), g["convOutpPartial"]) < TOL[mode]


@pytest.mark.parametrize("name", GOLDEN_2D)
def test_golden_pool_rnorm2d(gpu, name):
    g = load_golden(name)
    d, pd, ish, fsh, tsh, psh = geo2d(g)
    N = g["N"]
    pim, pdv = gpu.up(g["pool_images"], ish), gpu.up(g["pool_derivs"], psh)
    mx = gpu.nan(N, g["maxPool"].shape[1], psh); gpu.cg.MaxPool(pim, mx, pd)
    assert np.array_equal(mx.asarray(), g["maxPool"])
    av = gpu.nan(N, g["avgPool"].shape[1], psh); gpu.cg.AvgPool(pim, av, pd)
    assert Diff(av.asarray(), g["avgPool"]) < TOL_MEM
    out = gpu.nan(N, g["maxPoolUndo"].shape[1], ish); gpu.cg.MaxPoolUndo(pim, pdv, mx, out, pd)
    assert Diff(out.asarray(), g["maxPoolUndo"]) < TOL_MEM
    out = gpu.nan(N, g["avgPoolUndo"].shape[1], ish); gpu.cg.AvgPoolUndo(pdv, out, pd)
    assert Diff(out.asarray(), g["avgPoolUndo"]) < TOL_MEM
    images, rdv = gpu.up(g["images"], ish), gpu.up(g["rnorm_derivs"], ish)
    for blocked in (False, True):
        tag = "_blocked" if blocked else ""
        out = gpu.nan(*g["images"].shape, ish)
        gpu.cg.ResponseNormCrossMap(images, out, g["sizeF"], g["add_scale"], g["pow_scale"], blocked)
        assert Diff(out.asarray(), g["rnorm" + tag]) < TOL_MEM
        out = gpu.nan(*g["images"].shape, ish)
        gpu.cg.ResponseNormCrossMapUndo(rdv, images, out, g["sizeF"], g["add_scale"], g["pow_scale"], blocked)
        assert Diff(out.asarray(), g["rnormUndo" + tag]) < TOL_MEM


@pytest.mark.parametrize("mode", ["fp32", "tf32", "bf16"])
@pytest.mark.parametrize("name", GOLDEN_3D)
def test_golden_3d(gpu, name, mode):
    gpu.lib.set_precision(mode)
    g = load_golden(name)
    d, pd, ish, fsh, tsh, psh = geo3d(g)
    N = g["N"]
    images, filters, derivs = gpu.up(g["images"], ish), gpu.up(g["filters"], fsh), gpu.up(g["derivs"], tsh)
    out = gpu.nan(N, g["convUp3D"].shape[1], tsh); gpu.cg.convUp3D(images, filters, out, d)
    assert Diff(out.asarray(), g["convUp3D"]) < TOL[mode]
    out = gpu.nan(N, g["convDown3D"].shape[1], ish); gpu.cg.convDown3D(derivs, filters, out, d)
    assert Diff(out.asarray(), g["convDown3D"]) < TOL[mode]
    out = gpu.nan(*g["convOutp3D"].shape, fsh); gpu.cg.convOutp3D(images, derivs, out, d)
    assert Diff(out.asarray(), g["convOutp3D"]) < TOL[mode]
    pim, pdv = gpu.up(g["pool_images"], ish), gpu.up(g["pool_derivs"], psh)
    mx = gpu.nan(N, g["maxPool3D"].shape[1], psh); gpu.cg.MaxPool3D(pim, mx, pd)
    assert np.array_equal(mx.asarray(), g["maxPool3D"])
    av = gpu.nan(N, g["avgPool3D"].shape[1], psh); gpu.cg.AvgPool3D(pim, av, pd)
    assert Diff(av.asarray(), g["avgPool3D"]) < TOL_MEM
    out = gpu.nan(N, g["maxPool3DUndo"].shape[1], ish); gpu.cg.MaxPool3DUndo(pim, pdv, mx, out, pd)
    assert Diff(out.asarray(), g["maxPool3DUndo"]) < TOL_MEM
    out = gpu.nan(N, g["avgPool3DUndo"].shape[1], ish); gpu.cg.AvgPool3DUndo(pdv, out, pd)
    assert Diff(out.asarray(), g["avgPool3DUndo"]) < TOL_MEM


# ------------------------------------------------------------------------------------------
# 2. seeded shapes against the oracle (sizes the oracle finishes in seconds)
# ------------------------------------------------------------------------------------------
CONV_CASES = {
    # name: N, W, H, Cin, Cout, ky, kx, sy, sx, py, px
    "testconv_full": (128, 12, 12, 32, 64, 3, 3, 2, 2, 1, 1),     # py/test_conv.py:394-441
    "alex_conv1": (32, 57, 57, 3, 96, 7, 7, 2, 2, 1, 1),          # conv1 geometry, image cut to 57
    "alex_conv2": (32, 27, 27, 96, 256, 5, 5, 2, 2, 1, 1),        # conv2 geometry, image cut to 27
    "alex_conv3": (32, 14, 14, 256, 384, 3, 3, 1, 1, 1, 1),       # conv3 exact (batch 32)
    "alex_conv5": (32, 14, 14, 384, 512, 3, 3, 1, 1, 0, 0),       # conv5 exact, p0
    "one_by_one": (64, 14, 14, 384, 768, 1, 1, 1, 1, 0, 0),       # nin3_1 (ConvOneToOne as 1x1 conv)
    "fc_like": (128, 1, 1, 1152, 10, 1, 1, 1, 1, 0, 0),           # mnist FC as a conv on a 1x1 image
    "mnist_conv1": (100, 28, 28, 1, 48, 4, 4, 1, 1, 0, 0),        # examples/mnist-conv batch 100
    "mnist_conv2": (100, 11, 11, 48, 128, 4, 4, 1, 1, 0, 0),
    "ragged_batch": (37, 9, 8, 12, 20, 3, 2, 2, 1, 1, 0),         # N % 4 != 0, rectangular everything
    "single_image": (1, 6, 6, 4, 8, 3, 3, 1, 1, 1, 1),
    "batch_260": (260, 7, 7, 32, 64, 3, 3, 1, 1, 1, 1),           # N % 128 != 0, N % 4 == 0
    "cin8_cout16": (32, 12, 12, 8, 16, 3, 3, 1, 1, 1, 1),         # one K block, mostly zero-filled
    "cin24_s2": (32, 6, 6, 24, 16, 3, 3, 2, 2, 1, 1),
    "cin16_1x1": (32, 6, 6, 16, 24, 1, 1, 1, 1, 0, 0),
    "fc_splitk": (128, 1, 1, 2048, 512, 1, 1, 1, 1, 0, 0),        # FC: 2 output tiles, 64 K blocks -> split-K + reduce
    "fc_splitk_b32": (32, 1, 1, 1024, 256, 1, 1, 1, 1, 0, 0),     # partial m-tile with split-K
}


def _conv_case(shape, seed=5):
    N, W, H, Cin, Cout, ky, kx, sy, sx, py, px = shape
    modY, modX = num_modules(H, ky, sy, py), num_modules(W, kx, sx, px)
    d = GetConvDesc(Cin, Cout, ky, kx, sy, sx, py, px)
    ish, fsh, tsh = (N, W, H, Cin), (Cout, kx, ky, Cin), (N, modX, modY, Cout)
    r = np.random.RandomState(seed)
    images = F(r.randn(N, W * H * Cin))
    filters = F(r.randn(Cout, kx * ky * Cin) / np.sqrt(kx * ky * Cin))
    derivs = F(r.randn(N, modX * modY * Cout))
    return d, ish, fsh, tsh, images, filters, derivs


_ORACLE_CACHE = {}


def _oracle_conv(oracle, case):
    """oracle results for a CONV_CASES entry, computed once and shared by both precision modes."""
    if case not in _ORACLE_CACHE:
        d, ish, fsh, tsh, images, filters, derivs = _conv_case(CONV_CASES[case])
        N = ish[0]
        up = Z(*derivs.shape); oracle.convUp(images, filters, up, ish, fsh, tsh, d)
        init = F(np.random.RandomState(9).randn(*images.shape))
        dn = init.copy(order="F"); oracle.convDown(derivs, filters, dn, tsh, fsh, ish, d, 1.0)
        dw = Z(*filters.shape); oracle.convOutp(images, derivs, dw, ish, tsh, fsh, d, 0.0, 1.0 / N)
        _ORACLE_CACHE[case] = (up, init, dn, dw)
    return _ORACLE_CACHE[case]


@pytest.mark.parametrize("mode", ["fp32", "tf32", "bf16"])
@pytest.mark.parametrize("case", sorted(CONV_CASES))
def test_conv_vs_oracle(gpu, oracle, case, mode):
    gpu.lib.set_precision(mode)
    d, ish, fsh, tsh, images, filters, derivs = _conv_case(CONV_CASES[case])
    r_up, init, r_dn, r_dw = _oracle_conv(oracle, case)
    N = ish[0]
    gi, gf, gd = gpu.up(images, ish), gpu.up(filters, fsh), gpu.up(derivs, tsh)
    # fprop, overwrite into NaN-poisoned memory (scaleTargets == 0 must not read the target)
    out = gpu.nan(N, derivs.shape[1], tsh); gpu.cg.convUp(gi, gf, out, d, 0)
    assert Diff(out.asarray(), r_up) < TOL[mode], gpu.lib.last_conv_path()
    # dgrad, accumulate (scaleTargets = 1)
    out = gpu.up(init, ish); gpu.cg.convDown(gd, gf, out, d, 1)
    assert Diff(out.asarray(), r_dn) < TOL[mode], gpu.lib.last_conv_path()
    # wgrad with the Edge layer's scaleOutput = scale_gradients / batch (conv_edge.cc:206-208)
    out = gpu.nan(*filters.shape, fsh); gpu.cg.convOutp(gi, gd, out, d, 0, 1.0 / N)
    assert Diff(out.asarray(), r_dw) < TOL[mode], gpu.lib.last_conv_path()


def test_tensor_core_path_is_taken(gpu):
    """In TF32 mode the AlexNet 3x3 layers must run on the tensor cores, not fall through."""
    gpu.lib.set_precision("tf32")
    d, ish, fsh, tsh, images, filters, derivs = _conv_case(CONV_CASES["alex_conv3"])
    gi, gf, gd = gpu.up(images, ish), gpu.up(filters, fsh), gpu.up(derivs, tsh)
    out = gpu.new(ish[0], derivs.shape[1], tsh); gpu.cg.convUp(gi, gf, out, d)
    assert gpu.lib.last_conv_path() == "tc-tf32"
    out = gpu.new(*images.shape, ish); gpu.cg.convDown(gd, gf, out, d)
    assert gpu.lib.last_conv_path() == "tc-tf32"
    out = gpu.new(*filters.shape, fsh); gpu.cg.convOutp(gi, gd, out, d)
    assert gpu.lib.last_conv_path() == "tc-tf32"
    gpu.lib.set_precision("bf16")
    out = gpu.new(ish[0], derivs.shape[1], tsh); gpu.cg.convUp(gi, gf, out, d)
    assert gpu.lib.last_conv_path() == "tc-bf16"
    out = gpu.new(*images.shape, ish); gpu.cg.convDown(gd, gf, out, d)
    assert gpu.lib.last_conv_path() == "tc-bf16"
    out = gpu.new(*filters.shape, fsh); gpu.cg.convOutp(gi, gd, out, d)
    assert gpu.lib.last_conv_path() == "tc-bf16"


@pytest.mark.parametrize("mode", ["fp32", "tf32", "bf16"])
def test_conv_scale_targets_semantics(gpu, oracle, mode):
    gpu.lib.set_precision(mode)
    d, ish, fsh, tsh, images, filters, derivs = _conv_case((32, 10, 10, 16, 32, 3, 3, 1, 1, 1, 1))
    gi, gf, gd = gpu.up(images, ish), gpu.up(filters, fsh), gpu.up(derivs, tsh)
    r = np.random.RandomState(2)
    for st in (1.0, 0.5):
        init = F(r.randn(*derivs.shape)); out = gpu.up(init, tsh); gpu.cg.convUp(gi, gf, out, d, st)
        ref = init.copy(order="F"); oracle.convUp(images, filters, ref, ish, fsh, tsh, d, st)
        assert Diff(out.asarray(), ref) < TOL[mode]
        init = F(r.randn(*filters.shape)); out = gpu.up(init, fsh); gpu.cg.convOutp(gi, gd, out, d, st, 0.25)
        ref = init.copy(order="F"); oracle.convOutp(images, derivs, ref, ish, tsh, fsh, d, st, 0.25)
        assert Diff(out.asarray(), ref) < TOL[mode]
    out = gpu.nan(*images.shape, ish); gpu.cg.convDown(gd, gf, out, d, 0)
    ref = Z(*images.shape); oracle.convDown(derivs, filters, ref, tsh, fsh, ish, d, 0.0)
    assert Diff(out.asarray(), ref) < TOL[mode]


@pytest.mark.parametrize("mode", ["fp32", "tf32", "bf16"])
def test_conv_channel_subranges(gpu, oracle, mode):
    """input/output channel slices (cudamat_conv_gemm.cu:607-613)."""
    gpu.lib.set_precision(mode)
    N, W, H, Cin, Cout = 16, 8, 8, 24, 32
    d = GetConvDesc(Cin, Cout, 3, 3, 1, 1, 1, 1, input_channel_begin=8, input_channel_end=24,
                    output_channel_begin=16, output_channel_end=32)
    ish, fsh, tsh = (N, W, H, Cin), (16, 3, 3, 16), (N, 8, 8, Cout)
    r = np.random.RandomState(3)
    images, filters, derivs = F(r.randn(N, W * H * Cin)), F(r.randn(16, 9 * 16)), F(r.randn(N, 64 * Cout))
    gi, gf, gd = gpu.up(images, ish), gpu.up(filters, fsh), gpu.up(derivs, tsh)
    init = F(r.randn(N, 64 * Cout)); out = gpu.up(init, tsh); gpu.cg.convUp(gi, gf, out, d, 1)
    ref = init.copy(order="F"); oracle.convUp(images, filters, ref, ish, fsh, tsh, d, 1.0)
    assert Diff(out.asarray(), ref) < TOL[mode]
    init = F(r.randn(N, 64 * Cin)); out = gpu.up(init, ish); gpu.cg.convDown(gd, gf, out, d, 0.5)
    ref = init.copy(order="F"); oracle.convDown(derivs, filters, ref, tsh, fsh, ish, d, 0.5)
    assert Diff(out.asarray(), ref) < TOL[mode]
    out = gpu.nan(16, 144, fsh); gpu.cg.convOutp(gi, gd, out, d, 0, 1.0)
    ref = Z(16, 144); oracle.convOutp(images, derivs, ref, ish, tsh, fsh, d)
    assert Diff(out.asarray(), ref) < TOL[mode]


def test_local_untied_filters(gpu, oracle):
    """localUp/Down/Outp (cudamat_conv_gemm.cu:1448-1467), module i uses filter block i."""
    N, W, H, Cin, Cout = 8, 6, 6, 4, 8
    d = GetConvDesc(Cin, Cout, 3, 3, 1, 1, 1, 1)
    mods = 36
    ish, fsh, tsh = (N, W, H, Cin), (Cout, 3, 3, Cin * mods), (N, 6, 6, Cout)
    r = np.random.RandomState(4)
    images, filters, derivs = F(r.randn(N, W * H * Cin)), F(r.randn(Cout, 9 * Cin * mods)), F(r.randn(N, mods * Cout))
    gi, gf, gd = gpu.up(images, ish), gpu.up(filters, fsh), gpu.up(derivs, tsh)
    out = gpu.nan(N, mods * Cout, tsh); gpu.cg.localUp(gi, gf, out, d)
    ref = Z(N, mods * Cout); oracle.convUp(images, filters, ref, ish, fsh, tsh, d, conv=False)
    assert Diff(out.asarray(), ref) < 1e-4
    out = gpu.nan(*images.shape, ish); gpu.cg.localDown(gd, gf, out, d)
    ref = Z(*images.shape); oracle.convDown(derivs, filters, ref, tsh, fsh, ish, d, conv=False)
    assert Diff(out.asarray(), ref) < 1e-4
    out = gpu.nan(*filters.shape, fsh); gpu.cg.localOutp(gi, gd, out, d)
    ref = Z(*filters.shape); oracle.convOutp(images, derivs, ref, ish, tsh, fsh, d, conv=False)
    assert Diff(out.asarray(), ref) < 1e-4


# ------------------------------------------------------------------------------------------
# 3. pooling / response norm against the oracle, incl. the edge cases the domain has
# ------------------------------------------------------------------------------------------
POOL_CASES = {
    # N, W, H, C, k, s, p
    "alex_pool1": (32, 110, 110, 8, 3, 2, 1),
    "alex_pool5": (64, 12, 12, 64, 3, 2, 1),
    "mnist_pool": (100, 25, 25, 6, 4, 2, 0),
    "global": (16, 6, 6, 10, 6, 1, 0),                # kernel = image (maxpool_edge.cc:20-22)
    "ragged": (7, 9, 9, 5, 3, 2, 1),
    "stride_gt_k": (8, 10, 10, 4, 2, 3, 0),
}


@pytest.mark.parametrize("case", sorted(POOL_CASES))
def test_pool_vs_oracle(gpu, oracle, case):
    N, W, H, C, k, s, p = POOL_CASES[case]
    mod = num_modules(W, k, s, p)
    d = GetConvDesc(C, C, k, k, s, s, p, p)
    ish, psh = (N, W, H, C), (N, mod, mod, C)
    r = np.random.RandomState(8)
    # quantised inputs force ties: every equal element must receive the gradient (gemm.cu:291)
    images = F(np.round(r.rand(N, W * H * C) * 8) / 8)
    grads = F(r.randn(N, mod * mod * C))
    gi, gg = gpu.up(images, ish), gpu.up(grads, psh)
    mx = gpu.nan(N, mod * mod * C, psh); gpu.cg.MaxPool(gi, mx, d)
    rmx = Z(N, mod * mod * C); oracle.pool(True, images, rmx, ish, psh, d)
    assert np.array_equal(mx.asarray(), rmx)
    av = gpu.nan(N, mod * mod * C, psh); gpu.cg.AvgPool(gi, av, d)
    rav = Z(N, mod * mod * C); oracle.pool(False, images, rav, ish, psh, d)
    assert Diff(av.asarray(), rav) < TOL_MEM
    for st in (0.0, 1.0):
        init = F(r.randn(*images.shape))
        out = gpu.up(init, ish) if st else gpu.nan(*images.shape, ish)
        gpu.cg.MaxPoolUndo(gi, gg, mx, out, d, st)
        ref = init.copy(order="F"); oracle.maxPoolUndo(images, grads, rmx, ref, ish, psh, d, st)
        assert Diff(out.asarray(), ref) < TOL_MEM
        out = gpu.up(init, ish) if st else gpu.nan(*images.shape, ish)
        gpu.cg.AvgPoolUndo(gg, out, d, st)
        ref = init.copy(order="F"); oracle.avgPoolUndo(grads, ref, psh, ish, d, st)
        assert Diff(out.asarray(), ref) < TOL_MEM


def test_up_down_sample(gpu, oracle):
    N, W, C, f = 12, 5, 6, 3
    small, big = (N, W, W, C), (N, W * f, W * f, C)
    d = GetConvDesc(C, C, f, f, f, f, 0, 0)
    r = np.random.RandomState(1)
    a = F(r.randn(N, W * W * C)); ga = gpu.up(a, small)
    out = gpu.nan(N, W * f * W * f * C, big); gpu.cg.UpSample(ga, out, f)
    ref = Z(N, W * f * W * f * C); oracle.avgPoolUndo(a, ref, small, big, d, 0.0, float(f * f))
    assert Diff(out.asarray(), ref) < TOL_MEM
    b = F(r.randn(N, W * f * W * f * C)); gb = gpu.up(b, big)
    out = gpu.nan(N, W * W * C, small); gpu.cg.DownSample(gb, out, f)
    ref = Z(N, W * W * C); oracle.pool(False, b, ref, big, small, d)
    assert Diff(out.asarray(), ref) < TOL_MEM


RNORM_CASES = {
    # N, W, H, F, sizeF, alpha, beta
    "alex_rnorm1": (16, 55, 55, 96, 24, 5e-4, 0.75),
    "alex_rnorm2": (32, 14, 14, 256, 64, 5e-4, 0.75),
    "testconv": (128, 12, 12, 32, 8, 0.005, 0.75),
    "window_gt_channels": (8, 4, 4, 6, 9, 0.01, 0.5),
    "size1": (8, 4, 4, 6, 1, 0.01, 0.5),
    "even_window": (5, 3, 3, 10, 4, 0.1, 1.0),
    "huge_window": (4, 2, 2, 700, 500, 1e-3, 0.75),   # ring spills to workspace
}


@pytest.mark.parametrize("blocked", [False, True])
@pytest.mark.parametrize("case", sorted(RNORM_CASES))
def test_rnorm_vs_oracle(gpu, oracle, case, blocked):
    N, W, H, nf, sizeF, alpha, beta = RNORM_CASES[case]
    ish = (N, W, H, nf)
    r = np.random.RandomState(6)
    x, dy = F(r.randn(N, W * H * nf)), F(r.randn(N, W * H * nf))
    gx, gdy = gpu.up(x, ish), gpu.up(dy, ish)
    out = gpu.nan(*x.shape, ish); gpu.cg.ResponseNormCrossMap(gx, out, sizeF, alpha, beta, blocked)
    ref = Z(*x.shape); oracle.rnorm(x, ref, nf, sizeF, alpha, beta, blocked)
    assert Diff(out.asarray(), ref) < TOL_MEM
    out = gpu.nan(*x.shape, ish); gpu.cg.ResponseNormCrossMapUndo(gdy, gx, out, sizeF, alpha, beta, blocked)
    ref = Z(*x.shape); oracle.rnormUndo(dy, x, ref, nf, sizeF, alpha, beta, blocked)
    assert Diff(out.asarray(), ref) < 2 * TOL_MEM


def test_rnorm3d_frames(gpu, oracle):
    N, W, H, nf, T = 8, 5, 5, 12, 3
    ish = (N, W, H, nf * T)
    r = np.random.RandomState(6)
    x, dy = F(r.randn(N, W * H * nf * T)), F(r.randn(N, W * H * nf * T))
    gx, gdy = gpu.up(x, ish), gpu.up(dy, ish)
    out = gpu.nan(*x.shape, ish); gpu.cg.ResponseNormCrossMap3D(gx, out, 5, 0.01, 0.75, False, T)
    ref = Z(*x.shape)
    fr = W * H * nf
    for t in range(T):     # cudamat_conv3d_gemm.cu:167-189: each frame normalised on its own
        a, b = F(x[:, t * fr:(t + 1) * fr]), Z(N, fr)
        oracle.rnorm(a, b, nf, 5, 0.01, 0.75, False); ref[:, t * fr:(t + 1) * fr] = b
    assert Diff(out.asarray(), ref) < TOL_MEM
    out = gpu.nan(*x.shape, ish); gpu.cg.ResponseNormCrossMap3DUndo(gdy, gx, out, 5, 0.01, 0.75, False, T)
    for t in range(T):
        a, g_, b = F(x[:, t * fr:(t + 1) * fr]), F(dy[:, t * fr:(t + 1) * fr]), Z(N, fr)
        oracle.rnormUndo(g_, a, b, nf, 5, 0.01, 0.75, False); ref[:, t * fr:(t + 1) * fr] = b
    assert Diff(out.asarray(), ref) < 2 * TOL_MEM


# ------------------------------------------------------------------------------------------
# 4. BASELINE-size property tests (no oracle: size-independent identities)
# ------------------------------------------------------------------------------------------
FULL = {
    "conv2_b128": (128, 55, 55, 96, 256, 5, 5, 2, 2, 1, 1),
    "conv3_b256": (256, 14, 14, 256, 384, 3, 3, 1, 1, 1, 1),
    "conv4_b256": (256, 14, 14, 768, 384, 3, 3, 1, 1, 1, 1),
    "conv1_b128": (128, 224, 224, 3, 96, 7, 7, 2, 2, 1, 1),
}


@pytest.mark.parametrize("mode", ["fp32", "tf32", "bf16"])
@pytest.mark.parametrize("case", sorted(FULL))
def test_full_size_adjoint_identity(gpu, case, mode):
    """<convUp(x,w), d> == <x, convDown(d,w)> == <w, convOutp(x,d)> at the BASELINE layer sizes:
    fprop, dgrad and wgrad are the three faces of one trilinear form, so any indexing or
    accumulation error in one of them breaks the equality."""
    torch = gpu.torch
    gpu.lib.set_precision(mode)
    N, W, H, Cin, Cout, ky, kx, sy, sx, py, px = FULL[case]
    modY, modX = num_modules(H, ky, sy, py), num_modules(W, kx, sx, px)
    d = GetConvDesc(Cin, Cout, ky, kx, sy, sx, py, px)
    ish, fsh, tsh = (N, W, H, Cin), (Cout, kx, ky, Cin), (N, modX, modY, Cout)
    g = torch.Generator(device="cuda").manual_seed(1)
    x = gpu.new(N, W * H * Cin, ish); x.storage.normal_(generator=g)
    w = gpu.new(Cout, kx * ky * Cin, fsh); w.storage.normal_(generator=g).mul_(1.0 / np.sqrt(kx * ky * Cin))
    dv = gpu.new(N, modX * modY * Cout, tsh); dv.storage.normal_(generator=g)
    up = gpu.nan(N, modX * modY * Cout, tsh); gpu.cg.convUp(x, w, up, d)
    dn = gpu.nan(N, W * H * Cin, ish); gpu.cg.convDown(dv, w, dn, d)
    dw = gpu.nan(Cout, kx * ky * Cin, fsh); gpu.cg.convOutp(x, dv, dw, d)
    a = torch.dot(up.storage.double(), dv.storage.double()).item()
    b = torch.dot(dn.storage.double(), x.storage.double()).item()
    c = torch.dot(dw.storage.double(), w.storage.double()).item()
    scale = np.sqrt(float(up.storage.numel()))          # |<u,d>| ~ sqrt(n) * sigma_u * sigma_d
    tol = {"fp32": 5e-3, "tf32": 5e-2, "bf16": 1.5e-1}[mode]
    assert torch.isfinite(up.storage).all() and torch.isfinite(dn.storage).all() and torch.isfinite(dw.storage).all()
    assert abs(a - b) / scale < tol and abs(a - c) / scale < tol, (a, b, c, scale)


def test_full_size_pool_rnorm_properties(gpu):
    """pool1 / rnorm1 at batch 128 (BASELINE config 2 sizes)."""
    torch = gpu.torch
    N, W, C = 128, 110, 96
    mod = num_modules(W, 3, 2, 1)
    d = GetConvDesc(C, C, 3, 3, 2, 2, 1, 1)
    ish, psh = (N, W, W, C), (N, mod, mod, C)
    g = torch.Generator(device="cuda").manual_seed(2)
    x = gpu.new(N, W * W * C, ish); x.storage.normal_(generator=g)
    gr = gpu.new(N, mod * mod * C, psh); gr.storage.normal_(generator=g)
    mx = gpu.nan(N, mod * mod * C, psh); gpu.cg.MaxPool(x, mx, d)
    # max-pool == torch max_pool2d on the [C*, W, W, N] view (values are exact)
    xt = x.storage.view(C, W, W, N).permute(3, 0, 1, 2)
    ref = torch.nn.functional.max_pool2d(xt, 3, 2, 1).permute(1, 2, 3, 0).contiguous().view(-1)
    assert torch.equal(mx.storage, ref)
    # avg-pool undo conserves mass: sum(undo(g)) == sum(g) (every window divides by its own clipped size)
    und = gpu.nan(N, W * W * C, ish); gpu.cg.AvgPoolUndo(gr, und, d)
    s1, s2 = und.storage.double().sum().item(), gr.storage.double().sum().item()
    assert abs(s1 - s2) < 1e-3 * np.sqrt(gr.storage.numel())
    # max-pool undo routes exactly the incoming gradient when there are no ties (continuous inputs)
    und = gpu.nan(N, W * W * C, ish); gpu.cg.MaxPoolUndo(x, gr, mx, und, d)
    s1 = und.storage.double().sum().item()
    assert abs(s1 - s2) < 1e-3 * np.sqrt(gr.storage.numel())
    # response norm: directional finite difference of the forward equals <undo(dy), v>
    Wn, Cn, k = 55, 96, 24
    rsh = (N, Wn, Wn, Cn)
    xs = gpu.new(N, Wn * Wn * Cn, rsh); xs.storage.normal_(generator=g)
    v = torch.randn(xs.storage.numel(), device="cuda", generator=g)
    dy = gpu.new(N, Wn * Wn * Cn, rsh); dy.storage.normal_(generator=g)
    eps = 1e-2
    xp = gpu.new(N, Wn * Wn * Cn, rsh); xp.storage.copy_(xs.storage + eps * v)
    xm = gpu.new(N, Wn * Wn * Cn, rsh); xm.storage.copy_(xs.storage - eps * v)
    yp, ym = gpu.nan(N, Wn * Wn * Cn, rsh), gpu.nan(N, Wn * Wn * Cn, rsh)
    gpu.cg.ResponseNormCrossMap(xp, yp, k, 5e-4, 0.75, False)
    gpu.cg.ResponseNormCrossMap(xm, ym, k, 5e-4, 0.75, False)
    dx = gpu.nan(N, Wn * Wn * Cn, rsh); gpu.cg.ResponseNormCrossMapUndo(dy, xs, dx, k, 5e-4, 0.75, False)
    fd = torch.dot(dy.storage.double(), (yp.storage.double() - ym.storage.double()) / (2 * eps)).item()
    an = torch.dot(dx.storage.double(), v.double()).item()
    assert abs(fd - an) < 2e-3 * np.sqrt(v.numel()), (fd, an)


@pytest.mark.parametrize("mode", ["fp32", "tf32", "bf16"])
def test_fused_epilogues(gpu, oracle, mode):
    """convnet_b200_fuse_next: bias + ReLU in the fprop epilogue, ReLU' mask in dgrad / pool-undo epilogues must equal the
    unfused sequence (conv -> AddRowVec -> LowerBound(0); conv -> ApplyDerivativeOfActivation)."""
    torch = gpu.torch
    gpu.lib.set_precision(mode)
    L = gpu.lib.load()
    d, ish, fsh, tsh, images, filters, derivs = _conv_case((128, 10, 10, 32, 64, 3, 3, 1, 1, 1, 1))
    N = ish[0]
    gi, gf, gd = gpu.up(images, ish), gpu.up(filters, fsh), gpu.up(derivs, tsh)
    r = np.random.RandomState(4)
    bias = torch.from_numpy(r.randn(64).astype(np.float32)).cuda()
    # fprop: bias + relu
    ref = Z(*derivs.shape); oracle.convUp(images, filters, ref, ish, fsh, tsh, d)
    ref = np.maximum(ref.reshape(N, 64, 100) + bias.cpu().numpy()[None, :, None], 0).reshape(N, -1)   # cols = mod + 100*o
    out = gpu.nan(N, derivs.shape[1], tsh)
    L.convnet_b200_fuse_next(bias.data_ptr(), 1, None); gpu.cg.convUp(gi, gf, out, d)
    assert Diff(out.asarray(), ref) < 2 * TOL[mode]          # half the entries are clamped to 0: the Diff denominator halves
    out2 = gpu.nan(N, derivs.shape[1], tsh); gpu.cg.convUp(gi, gf, out2, d)      # the request was one-shot
    assert (out2.asarray() < 0).any()
    # dgrad: mask
    state = F(r.randn(*images.shape)); gs = gpu.up(state, ish)
    ref = Z(*images.shape); oracle.convDown(derivs, filters, ref, tsh, fsh, ish, d)
    ref = np.where(state > 0, ref, 0).astype(np.float32)
    out = gpu.nan(*images.shape, ish)
    L.convnet_b200_fuse_next(None, 0, gs.ptr); gpu.cg.convDown(gd, gf, out, d)
    assert Diff(out.asarray(), ref) < 2 * TOL[mode]
    # max-pool undo: mask
    pd = GetConvDesc(32, 32, 3, 3, 2, 2, 1, 1)
    psh = (N, 5, 5, 32)
    pim = F(r.rand(*images.shape)); gpim = gpu.up(pim, ish)
    grads = F(r.randn(N, 25 * 32)); gg = gpu.up(grads, psh)
    mx = gpu.nan(N, 25 * 32, psh); gpu.cg.MaxPool(gpim, mx, pd)
    ref = Z(*images.shape); oracle.maxPoolUndo(pim, grads, mx.asarray(), ref, ish, psh, pd)
    ref = np.where(state > 0, ref, 0).astype(np.float32)
    out = gpu.nan(*images.shape, ish)
    L.convnet_b200_fuse_next(None, 0, gs.ptr); gpu.cg.MaxPoolUndo(gpim, gg, mx, out, pd)
    assert Diff(out.asarray(), ref) < TOL_MEM


@pytest.mark.parametrize("mode", ["tf32", "bf16"])
def test_split_k_fused_epilogues(gpu, oracle, mode):
    """FC-shaped calls leave most SMs idle, so their K loop is split across CTAs and a second kernel reduces the partial
    sums; bias + ReLU (fprop), the ReLU' mask (dgrad) and scaleTargets then ride in that reduction kernel."""
    torch = gpu.torch
    gpu.lib.set_precision(mode)
    L = gpu.lib.load()
    d, ish, fsh, tsh, images, filters, derivs = _conv_case((128, 1, 1, 2048, 512, 1, 1, 1, 1, 0, 0))
    N, Cout = ish[0], 512
    gi, gf, gd = gpu.up(images, ish), gpu.up(filters, fsh), gpu.up(derivs, tsh)
    r = np.random.RandomState(4)
    bias = torch.from_numpy(r.randn(Cout).astype(np.float32)).cuda()
    ref = Z(*derivs.shape); oracle.convUp(images, filters, ref, ish, fsh, tsh, d)
    ref = np.maximum(ref + bias.cpu().numpy()[None, :], 0)
    out = gpu.nan(N, derivs.shape[1], tsh)
    L.convnet_b200_fuse_next(bias.data_ptr(), 1, None); gpu.cg.convUp(gi, gf, out, d)
    assert Diff(out.asarray(), ref) < 2 * TOL[mode]
    state = F(r.randn(*images.shape)); gs = gpu.up(state, ish)
    init = F(r.randn(*images.shape))
    ref = init.copy(order="F"); oracle.convDown(derivs, filters, ref, tsh, fsh, ish, d, 1.0)     # scaleTargets = 1
    ref = np.where(state > 0, ref, 0).astype(np.float32)
    out = gpu.up(init, ish)
    L.convnet_b200_fuse_next(None, 0, gs.ptr); gpu.cg.convDown(gd, gf, out, d, 1)
    assert Diff(out.asarray(), ref) < 2 * TOL[mode]
