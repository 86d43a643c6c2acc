"""The R-operators, within-map normalisation, RGB -> YUV and convInnerpGemm on the GPU: element by element against the
float64 restatements of tests/abi_rest_exact.py at every dispatch branch, and against the reference's own CUDA kernels
(oracle/_ref/libcudamat_conv_gemm_ref.so and libcudamat_conv_ref.so) at py/test_conv.py's shapes and AlexNet's
hidden1 shapes at batch 128.  Every call writes into a NaN-sentinel buffer with guard zones and counts its launches."""
import ctypes as ct
import os

import numpy as np
import pytest
import torch

import abi_rest_exact as ax
import pool_exact as px
from gpu_buffers import guards_ok, launched, matrix
from pool_exact import PG

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_GEMM = os.path.join(ROOT, "oracle", "_ref", "libcudamat_conv_gemm_ref.so")
REF_CONV = os.path.join(ROOT, "oracle", "_ref", "libcudamat_conv_ref.so")
GEMM_NAMES = ["MaxPoolRpropGemm", "ResponseNormCrossMapRpropGemm", "convInnerpGemm"]
CONV_NAMES = ["ResponseNorm", "ResponseNormUndo", "ContrastNorm", "ContrastNormUndo", "RGBToYUV"]


class Env:
    pass


@pytest.fixture(scope="module")
def env():
    from convnet_b200 import conv_gemm as cg
    from convnet_b200 import lib
    e = Env()
    e.L = lib.load()
    e.cg, e.lib = cg, lib
    lib.set_precision("fp32")
    return e


def _rand(n, seed, dyadic=False):
    g = torch.Generator(device="cpu").manual_seed(seed)
    if dyadic:
        return (torch.randint(-64, 65, (n,), generator=g).float() / 16).cuda()
    return torch.randn(n, generator=g).cuda()


def _mat(rows, cols, s4, data=None, offset=0):
    m, buf = matrix(rows, cols, s4, offset)
    if data is not None:
        m.storage.copy_(data)
    return m, buf


def _ok(y, e, what):
    v = px.check(y, e)
    assert v.ok, "%s: %s" % (what, v)


def _one_launch(env, fn, n=1):
    a = launched(env, fn)
    b = launched(env, fn)
    assert a == n and b == n, (a, b)


# ---------------------------------------------------------------------------------------------------------------------
# element by element, every branch
# ---------------------------------------------------------------------------------------------------------------------
MAX_CASES = [PG(8, 12, 12, 8, 3, 3, 2, 2, 1, 1), PG(6, 9, 7, 5, 3, 2, 2, 1, 0, 1), PG(4, 10, 10, 3, 4, 4, 3, 3, 0, 0)]


@pytest.mark.parametrize("ci", range(len(MAX_CASES)))
@pytest.mark.parametrize("st", [0.0, 1.0, 0.5])
def test_max_pool_rprop(env, ci, st):
    g = MAX_CASES[ci]
    n_in, n_out = g.N * g.W * g.H * g.C, g.N * g.modX * g.modY * g.C
    x, R = _rand(n_in, 1 + ci, True), _rand(n_in, 11 + ci, True)
    im, _ = _mat(*g.in_dims(), g.in_shape(), x)
    rm, _ = _mat(*g.in_dims(), g.in_shape(), R)
    mx, _ = _mat(*g.out_dims(), g.out_shape())
    env.cg.MaxPool(im, mx, g.desc())
    t0 = _rand(n_out, 21 + ci, True)
    out, buf = _mat(*g.out_dims(), g.out_shape(), t0 if st else None)
    _one_launch(env, lambda: (out.storage.copy_(t0) if st else None,
                              env.cg.MaxPoolRprop(im, rm, mx, out, g.desc(), st)) and None)
    assert guards_ok(buf, 0, n_out)
    _ok(out.storage, ax.max_rprop(g, x, R, mx.storage, st, t0, exact_arm=True), ax.max_rprop_branch(g.N))


RN_CASES = [  # (N, S, F, k, blocked): tile vec / tile scalar (L % 4 != 0) / ring (no tile for 512 channels)
    (8, 6, 32, 5, False), (8, 6, 32, 5, True), (5, 3, 24, 4, False), (5, 3, 24, 4, True),
    (4, 3, 512, 9, False), (4, 3, 512, 9, True), (3, 3, 96, 96, False)]


@pytest.mark.parametrize("case", RN_CASES, ids=lambda c: "N%d_S%d_F%d_k%d_%s" % (c[0], c[1], c[2], c[3], "bl" if c[4] else "un"))
def test_rnorm_rprop(env, case):
    N, S, F, k, blocked = case
    n = N * S * S * F
    x, R = _rand(n, 31), _rand(n, 32)
    s4 = (N, S, S, F)
    im, _ = _mat(N, S * S * F, s4, x)
    rm, _ = _mat(N, S * S * F, s4, R)
    out, buf = _mat(N, S * S * F, s4)
    _one_launch(env, lambda: env.cg.ResponseNormCrossMapRprop(im, rm, out, k, 0.01, 0.75, blocked))
    assert guards_ok(buf, 0, n)
    _ok(out.storage, ax.rnorm_rprop(x, R, F, k, 0.01, 0.75, blocked), ax.rnorm_rprop_branch(N * S * S, F, blocked))


MAP_CASES = [  # (N, S, F, sizeX): vector / scalar images, small and large windows, windows wider than the map
    (8, 12, 4, 3), (8, 12, 4, 9), (6, 7, 3, 4), (6, 7, 3, 10), (20, 5, 2, 5), (4, 13, 2, 2)]


@pytest.mark.parametrize("case", MAP_CASES, ids=lambda c: "N%d_S%d_F%d_X%d" % c)
@pytest.mark.parametrize("contrast", [False, True])
def test_mapnorm(env, case, contrast):
    N, S, F, sizeX = case
    n = N * S * S * F
    alpha, beta = 0.02, 0.75
    s4 = (N, S, S, F)
    x = _rand(n, 41)
    md_t = _rand(n, 42) if contrast else x
    im, _ = _mat(N, S * S * F, s4, x)
    md, _ = _mat(N, S * S * F, s4, md_t)
    dn, bd = _mat(N, S * S * F, s4)
    tg, bt = _mat(N, S * S * F, s4)
    if contrast:
        _one_launch(env, lambda: env.cg.ContrastNorm(im, md, dn, tg, F, sizeX, alpha, beta))
    else:
        _one_launch(env, lambda: env.cg.ResponseNorm(im, dn, tg, F, sizeX, alpha, beta))
    assert guards_ok(bd, 0, n) and guards_ok(bt, 0, n)
    branch = ax.mapnorm_branch(N, False)
    _ok(dn.storage, ax.mapnorm_denoms(md_t, N, S, F, sizeX, alpha), branch + " denoms")
    _ok(tg.storage, ax.mapnorm_targets(x, dn.storage, beta), branch + " targets")
    # the undo on the forward pass's own outputs
    og_t = _rand(n, 43)
    og, _ = _mat(N, S * S * F, s4, og_t)
    acts_before = tg.storage.clone()
    du, bu = _mat(N, S * S * F, s4)
    if contrast:
        _one_launch(env, lambda: env.cg.ContrastNormUndo(og, dn, md, tg, du, F, sizeX, alpha, beta))
    else:
        _one_launch(env, lambda: env.cg.ResponseNormUndo(og, dn, im, tg, du, F, sizeX, alpha, beta))
    assert guards_ok(bu, 0, n)
    assert torch.equal(tg.storage, acts_before), "the undo must not overwrite acts"
    _ok(du.storage, ax.mapnorm_undo(og_t, dn.storage, md_t, tg.storage, N, S, F, sizeX, alpha, beta),
        ax.mapnorm_branch(N, True))


@pytest.mark.parametrize("N,S", [(8, 12), (5, 7)])
def test_rgb_to_yuv(env, N, S):
    n = N * S * S * 3
    x = _rand(n, 51)
    im, _ = _mat(N, S * S * 3, (N, S, S, 3), x)
    out, buf = _mat(N, S * S * 3, (N, S, S, 3))
    _one_launch(env, lambda: env.cg.RGBToYUV(im, out))
    assert guards_ok(buf, 0, n)
    _ok(out.storage, ax.rgb_to_yuv(x), ax.yuv_branch(N * S * S))


INNERP_CASES = [  # (PG, splits > 1?)
    PG(8, 12, 12, 4, 3, 3, 2, 2, 1, 1), PG(6, 9, 8, 3, 2, 3, 1, 2, 0, 1), PG(64, 30, 30, 16, 5, 5, 1, 1, 2, 2)]


@pytest.mark.parametrize("ci", range(len(INNERP_CASES)))
@pytest.mark.parametrize("st,so", [(0.0, 1.0), (1.0, 1.0), (0.5, 0.25)])
def test_innerp(env, ci, st, so):
    g = INNERP_CASES[ci]
    x = _rand(g.N * g.W * g.H * g.C, 61 + ci)
    dv = _rand(g.N * g.modX * g.modY * g.C, 71 + ci)
    im, _ = _mat(*g.in_dims(), g.in_shape(), x)
    de, _ = _mat(*g.out_dims(), g.out_shape(), dv)
    t0 = _rand(g.kx * g.ky, 81)
    out, buf = _mat(1, g.kx * g.ky, (1, g.kx, g.ky, 1), t0 if st else None)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    launches = ax.innerp_launches(g.N, g.C * g.modX * g.modY, sms)
    _one_launch(env, lambda: (out.storage.copy_(t0) if st else None, env.cg.convInnerp(im, de, out, g.desc(), st, so))
                and None, launches)
    assert guards_ok(buf, 0, g.kx * g.ky)
    _ok(out.storage, ax.innerp(g, x, dv, st, t0, so, sms), "innerp launches=%d" % launches)


def test_splits_cover_both_branches():
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    got = {ax.innerp_launches(g.N, g.C * g.modX * g.modY, sms) for g in INNERP_CASES}
    assert got == {1, 2}


def test_branches_are_all_reached():
    assert {ax.max_rprop_branch(g.N) for g in MAX_CASES} == {"pool_rprop_kernel<4>", "pool_rprop_kernel<1>"}
    rn = {ax.rnorm_rprop_branch(N * S * S, F, bl) for N, S, F, k, bl in RN_CASES}
    assert {b[1] for b in rn} == {"vec", "scalar", "ring"}
    assert {b[0] for b in rn} >= {"rnorm_rprop_kernel<true>", "rnorm_rprop_kernel<false>"}
    assert {ax.mapnorm_branch(c[0], False) for c in MAP_CASES} == {"mapnorm_kernel<false, 4>", "mapnorm_kernel<false, 1>"}


# ---------------------------------------------------------------------------------------------------------------------
# the writer protocol, and no symbol aborts
# ---------------------------------------------------------------------------------------------------------------------
def test_staged_copies_of_written_tensors_are_dropped(env):
    L = env.L
    N, S, F = 4, 6, 8
    n = N * S * S * F
    s4 = (N, S, S, F)
    ms = {k: _mat(N, S * S * F, s4, _rand(n, i))[0] for i, k in enumerate("abcdef")}
    a, b, c, d, e, f = (ms[k] for k in "abcdef")

    def check(fn, written):
        for m in written:
            L.convnet_b200_bf16_stage(m.ptr, n)
            assert L.convnet_b200_bf16_is_staged(m.ptr, n) == 1
        fn()
        torch.cuda.synchronize()
        for m in written:
            assert L.convnet_b200_bf16_is_staged(m.ptr, n) == 0, "a stale bf16 copy survived the write"

    env.lib.set_precision("bf16")                   # staged copies exist in bf16 mode only
    try:
        check(lambda: env.cg.ResponseNormCrossMapRprop(a, b, c, 5, 1e-3, 0.75, False), [c])
        check(lambda: env.cg.ResponseNorm(a, d, e, F, 3, 1e-3, 0.75), [d, e])
        check(lambda: env.cg.ContrastNorm(a, b, d, e, F, 3, 1e-3, 0.75), [d, e])
        check(lambda: env.cg.ResponseNormUndo(b, d, a, e, f, F, 3, 1e-3, 0.75), [f])
        check(lambda: env.cg.ContrastNormUndo(b, d, a, e, f, F, 3, 1e-3, 0.75), [f])
        y = _mat(N, S * S * 3, (N, S, S, 3))[0]
        check(lambda: env.cg.RGBToYUV(_mat(N, S * S * 3, (N, S, S, 3), _rand(N * S * S * 3, 9))[0], y), [])
        g = PG(N, S, S, F, 2, 2, 2, 2)
        mx = _mat(*g.out_dims(), g.out_shape())[0]
        env.cg.MaxPool(a, mx, g.desc())
        t = _mat(*g.out_dims(), g.out_shape())[0]
        L.convnet_b200_bf16_stage(t.ptr, g.N * 9 * F)
        env.cg.MaxPoolRprop(a, b, mx, t, g.desc())
        torch.cuda.synchronize()
        assert L.convnet_b200_bf16_is_staged(t.ptr, g.N * 9 * F) == 0
        # a requested copy is produced after the write
        L.convnet_b200_emit_bf16_next()
        env.cg.ResponseNorm(a, d, e, F, 3, 1e-3, 0.75)
        torch.cuda.synchronize()
        assert L.convnet_b200_bf16_is_staged(e.ptr, n) == 1
    finally:
        for m in (c, d, e, f):
            L.convnet_b200_bf16_invalidate(m.ptr)
        env.lib.set_precision("fp32")


def test_every_symbol_runs_at_a_tiny_shape(env):
    g = PG(4, 4, 4, 2, 2, 2, 2, 2)
    n_in, n_out = g.N * 16 * 2, g.N * 4 * 2
    im, _ = _mat(*g.in_dims(), g.in_shape(), _rand(n_in, 1))
    rm, _ = _mat(*g.in_dims(), g.in_shape(), _rand(n_in, 2))
    mx, _ = _mat(*g.out_dims(), g.out_shape())
    env.cg.MaxPool(im, mx, g.desc())
    t, _ = _mat(*g.out_dims(), g.out_shape())
    env.cg.MaxPoolRprop(im, rm, mx, t, g.desc())
    r2, _ = _mat(*g.in_dims(), g.in_shape())
    env.cg.ResponseNormCrossMapRprop(im, rm, r2, 2, 1e-3, 0.75, False)
    ip, _ = _mat(1, 4, (1, 2, 2, 1))
    env.cg.convInnerp(im, mx, ip, g.desc())
    dn, _ = _mat(*g.in_dims(), g.in_shape())
    tg, _ = _mat(*g.in_dims(), g.in_shape())
    env.cg.ResponseNorm(im, dn, tg, 2, 3, 1e-3, 0.75)
    env.cg.ResponseNormUndo(rm, dn, im, tg, r2, 2, 3, 1e-3, 0.75)
    env.cg.ContrastNorm(im, rm, dn, tg, 2, 3, 1e-3, 0.75)
    env.cg.ContrastNormUndo(rm, dn, rm, tg, r2, 2, 3, 1e-3, 0.75)
    c3, _ = _mat(4, 12, (4, 2, 2, 3), _rand(48, 3))
    y3, _ = _mat(4, 12, (4, 2, 2, 3))
    env.cg.RGBToYUV(c3, y3)
    torch.cuda.synchronize()
    for m in (t, r2, ip, dn, tg, y3):
        assert torch.isfinite(m.storage).all()


# ---------------------------------------------------------------------------------------------------------------------
# against the reference's own CUDA kernels
# ---------------------------------------------------------------------------------------------------------------------
_ref = {}


def _reflib(path, names):
    if path not in _ref:
        if not os.path.exists(path):
            pytest.skip("%s was not built (the reference tree was absent at build time)" % os.path.basename(path))
        import ref_cuda_lib
        ref_cuda_lib.load()                          # cublasInit for the legacy cuBLAS calls of the reference
        lib = ct.CDLL(path, mode=ct.RTLD_LOCAL)
        from convnet_b200.lib import SIGNATURES
        for nm in names:
            getattr(lib, nm).argtypes = SIGNATURES[nm]
            getattr(lib, nm).restype = None
        _ref[path] = lib
    from convnet_b200.conv_gemm import Binding
    return Binding(lambda: _ref[path], "gemm")


def _rel(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / b.norm().clamp_min(1e-300))


TEST_CONV_POOL = PG(128, 12, 12, 32, 3, 3, 2, 2, 1, 1)


@pytest.mark.parametrize("g", [TEST_CONV_POOL, ax.alexnet_shapes(128)[0]], ids=["test_conv", "alexnet_hidden1"])
@pytest.mark.parametrize("st", [0.0, 1.0])
def test_max_pool_rprop_vs_reference_cuda(env, g, st):
    ref = _reflib(REF_GEMM, GEMM_NAMES)
    n_in, n_out = g.N * g.W * g.H * g.C, g.N * g.modX * g.modY * g.C
    x, R, t0 = _rand(n_in, 91), _rand(n_in, 92), _rand(n_out, 93)
    im, _ = _mat(*g.in_dims(), g.in_shape(), x)
    rm, _ = _mat(*g.in_dims(), g.in_shape(), R)
    mx, _ = _mat(*g.out_dims(), g.out_shape())
    env.cg.MaxPool(im, mx, g.desc())
    ours, _ = _mat(*g.out_dims(), g.out_shape(), t0)
    theirs, _ = _mat(*g.out_dims(), g.out_shape(), t0)
    env.cg.MaxPoolRprop(im, rm, mx, ours, g.desc(), st)
    ref.MaxPoolRprop(im, rm, mx, theirs, g.desc(), st)
    torch.cuda.synchronize()
    assert torch.equal(ours.storage.view(torch.int32), theirs.storage.view(torch.int32)), "max-pool R-op is not bit-exact"


@pytest.mark.parametrize("shape,k,alpha", [((128, 12, 12, 32), 8, 0.005), ((128, 55, 55, 96), 5, 1e-4)],
                         ids=["test_conv", "alexnet_hidden1"])
@pytest.mark.parametrize("blocked", [False, True])
def test_rnorm_rprop_vs_reference_cuda(env, shape, k, alpha, blocked):
    ref = _reflib(REF_GEMM, GEMM_NAMES)
    N, S, _, F = shape
    n = N * S * S * F
    x, R = _rand(n, 94), _rand(n, 95)
    im, _ = _mat(N, S * S * F, shape, x)
    rm, _ = _mat(N, S * S * F, shape, R)
    ours, _ = _mat(N, S * S * F, shape)
    theirs, _ = _mat(N, S * S * F, shape)
    env.cg.ResponseNormCrossMapRprop(im, rm, ours, k, alpha, 0.75, blocked)
    ref.ResponseNormCrossMapRprop(im, rm, theirs, k, alpha, 0.75, blocked)
    torch.cuda.synchronize()
    assert _rel(ours.storage, theirs.storage) < 1e-4


@pytest.mark.parametrize("g", [TEST_CONV_POOL, ax.alexnet_shapes(128)[0]], ids=["test_conv", "alexnet_hidden1"])
@pytest.mark.parametrize("st,so", [(0.0, 1.0), (0.5, 2.0)])
def test_innerp_vs_reference_cuda(env, g, st, so):
    ref = _reflib(REF_GEMM, GEMM_NAMES)
    x, dv, t0 = _rand(g.N * g.W * g.H * g.C, 96), _rand(g.N * g.modX * g.modY * g.C, 97), _rand(g.kx * g.ky, 98)
    im, _ = _mat(*g.in_dims(), g.in_shape(), x)
    de, _ = _mat(*g.out_dims(), g.out_shape(), dv)
    ours, _ = _mat(1, g.kx * g.ky, (1, g.kx, g.ky, 1), t0)
    theirs, _ = _mat(1, g.kx * g.ky, (1, g.kx, g.ky, 1), t0)
    env.cg.convInnerp(im, de, ours, g.desc(), st, so)
    ref.convInnerp(im, de, theirs, g.desc(), st, so)
    torch.cuda.synchronize()
    assert _rel(ours.storage, theirs.storage) < 1e-4


@pytest.mark.parametrize("shape", [(128, 12, 12, 32), (128, 55, 55, 96)], ids=["test_conv", "alexnet_hidden1"])
@pytest.mark.parametrize("sizeX", [5, 9])
@pytest.mark.parametrize("contrast", [False, True])
def test_mapnorm_vs_reference_cuda(env, shape, sizeX, contrast):
    ref = _reflib(REF_CONV, CONV_NAMES)
    N, S, _, F = shape
    n = N * S * S * F
    alpha, beta = 1e-3, 0.75
    x = _rand(n, 101)
    md_t = _rand(n, 102) if contrast else x
    og_t = _rand(n, 103)
    mats = {k: _mat(N, S * S * F, shape)[0] for k in ("dn", "tg", "dn_r", "tg_r", "du", "du_r", "acts_r")}
    im, _ = _mat(N, S * S * F, shape, x)
    md, _ = _mat(N, S * S * F, shape, md_t)
    og, _ = _mat(N, S * S * F, shape, og_t)
    m = mats
    if contrast:
        env.cg.ContrastNorm(im, md, m["dn"], m["tg"], F, sizeX, alpha, beta)
        ref.ContrastNorm(im, md, m["dn_r"], m["tg_r"], F, sizeX, alpha, beta)
    else:
        env.cg.ResponseNorm(im, m["dn"], m["tg"], F, sizeX, alpha, beta)
        ref.ResponseNorm(im, m["dn_r"], m["tg_r"], F, sizeX, alpha, beta)
    torch.cuda.synchronize()
    assert _rel(m["dn"].storage, m["dn_r"].storage) < 1e-4
    assert _rel(m["tg"].storage, m["tg_r"].storage) < 1e-4
    m["acts_r"].storage.copy_(m["tg"].storage)        # the reference overwrites its acts argument
    # for sizeX >= 6 the reference's undo (kRNormUndo2 with add = true at scaleTargets 0) computes 0 * target + result,
    # so it reads its target: give it zeros rather than the NaN sentinel (the product never reads the target)
    m["du_r"].storage.zero_()
    inputs = md if contrast else im
    if contrast:
        env.cg.ContrastNormUndo(og, m["dn"], inputs, m["tg"], m["du"], F, sizeX, alpha, beta)
        ref.ContrastNormUndo(og, m["dn"], inputs, m["acts_r"], m["du_r"], F, sizeX, alpha, beta)
    else:
        env.cg.ResponseNormUndo(og, m["dn"], inputs, m["tg"], m["du"], F, sizeX, alpha, beta)
        ref.ResponseNormUndo(og, m["dn"], inputs, m["acts_r"], m["du_r"], F, sizeX, alpha, beta)
    torch.cuda.synchronize()
    assert _rel(m["du"].storage, m["du_r"].storage) < 1e-4


@pytest.mark.parametrize("N,S", [(128, 12), (128, 224)], ids=["test_conv", "alexnet_input"])
def test_rgb_to_yuv_vs_reference_cuda(env, N, S):
    ref = _reflib(REF_CONV, CONV_NAMES)
    n = N * S * S * 3
    im, _ = _mat(N, S * S * 3, (N, S, S, 3), _rand(n, 104))
    ours, _ = _mat(N, S * S * 3, (N, S, S, 3))
    theirs, _ = _mat(N, S * S * 3, (N, S, S, 3))
    env.cg.RGBToYUV(im, ours)
    ref.RGBToYUV(im, theirs)
    torch.cuda.synchronize()
    assert _rel(ours.storage, theirs.storage) < 1e-4
