"""The float64 restatements of tests/abi_rest_exact.py, without a GPU: the two R-operators against the reference's own
CPU code (py/conv_cpu.py, where the reference tree exists), the within-map norms and RGB -> YUV on cases small enough to
check by hand, and the python surface against the C signatures."""
import ast
import ctypes as ct
import os

import numpy as np
import pytest
import torch

import abi_rest_exact as ax
import pool_exact as px
from convnet_b200 import conv_gemm
from convnet_b200.lib import SIGNATURES
from pool_exact import PG

REF_CPU = "/root/reference/py/conv_cpu.py"
reflib = pytest.mark.skipif(not os.path.exists(REF_CPU), reason="the reference tree is not present")


def _conv_cpu(*names):
    """the named functions of the reference's py/conv_cpu.py (python 2: xrange, integer '/'), compiled for python 3"""
    lines = open(REF_CPU).read().split("\n")
    want = set(names) | {"ComputeDenoms", "GetBounds", "GetBoundsInv"}
    src, keep = [], False
    for ln in lines:                               # the file is python 2 as a whole: take the wanted functions only
        if ln and not ln[0].isspace():
            keep = ln.startswith("def ") and ln[4:].split("(")[0] in want
        if keep:
            src.append(ln)
    tree = ast.parse("\n".join(src))

    class FloorDiv(ast.NodeTransformer):          # every '/' in these functions is between ints (shapes and strides)
        def visit_BinOp(self, node):
            self.generic_visit(node)
            if isinstance(node.op, ast.Div):
                node.op = ast.FloorDiv()
            return node

    body = [FloorDiv().visit(n) for n in tree.body if isinstance(n, ast.FunctionDef) and n.name in want]
    ns = {"np": np, "xrange": range}
    exec(compile(ast.fix_missing_locations(ast.Module(body=body, type_ignores=[])), REF_CPU, "exec"), ns)
    return ns


def _fm(a):
    """(rows, cols) numpy -> the flat column-major fp32 tensor the kernels see"""
    return torch.from_numpy(np.ascontiguousarray(np.asarray(a, dtype=np.float32).T).reshape(-1))


def _ok(y, e):
    v = px.check(y, e)
    assert v.ok, v


# ---------------------------------------------------------------------------------------------------------------------
# the R-operators against py/conv_cpu.py, at py/test_conv.py's shapes
# ---------------------------------------------------------------------------------------------------------------------
@reflib
def test_max_pool_rprop_matches_conv_cpu():
    cpu = _conv_cpu("MaxPool", "MaxPoolRprop")
    r = np.random.RandomState(1)
    N, S, C = 128, 12, 32
    g = PG(N, S, S, C, 3, 3, 2, 2, 1, 1)
    images = r.randn(N, S * S * C).astype(np.float32)
    R = r.randn(N, S * S * C).astype(np.float32)
    x = _fm(images)
    maxes_flat = px.pool_fwd(g, x, True).ref.to(torch.float32)
    maxes = maxes_flat.numpy().reshape(-1, N).T
    spec = (C, 3, 3, 2, 2, 1, 1)
    out = cpu["MaxPoolRprop"](images, R, maxes, (N, S, S, C), spec)
    e = ax.max_rprop(g, x, _fm(R), maxes_flat)
    _ok(_fm(out), e)


@reflib
@pytest.mark.parametrize("blocked", [False, True])
def test_rnorm_rprop_matches_conv_cpu(blocked):
    cpu = _conv_cpu("ResponseNormCrossMapRprop")
    r = np.random.RandomState(2 + blocked)
    N, S, C, k, alpha, beta = 128, 12, 32, 8, 0.005, 0.75
    images = r.randn(N, S * S * C).astype(np.float32)
    R = r.randn(N, S * S * C).astype(np.float32)
    out = cpu["ResponseNormCrossMapRprop"](images, R, (N, S, S, C), k, alpha, beta, blocked)
    e = ax.rnorm_rprop(_fm(images), _fm(R), C, k, alpha, beta, blocked)
    _ok(_fm(out), e)


def test_rnorm_rprop_is_the_directional_derivative():
    """t = d/de rnorm(x + e R) at e = 0, by a central difference in float64"""
    r = np.random.RandomState(5)
    F, L, k, alpha, beta = 12, 7, 5, 0.05, 0.75
    x = torch.from_numpy(r.randn(F * L).astype(np.float32))
    R = torch.from_numpy(r.randn(F * L).astype(np.float32))
    for blocked in (False, True):
        e = ax.rnorm_rprop(x, R, F, k, alpha, beta, blocked)
        h = 1e-6
        f = lambda t: px.rnorm_fwd(t, F, k, alpha, beta, blocked).ref
        num = (f(x.double() + h * R.double()) - f(x.double() - h * R.double())) / (2 * h)
        assert torch.allclose(e.ref, num, rtol=1e-6, atol=1e-8)


# ---------------------------------------------------------------------------------------------------------------------
# within-map normalisation and the colour transform by hand
# ---------------------------------------------------------------------------------------------------------------------
def _window_count(S, sizeX, p, inverse=False):
    off = sizeX // 2 - sizeX + 1 if inverse else -(sizeX // 2)
    return min(S, p + off + sizeX) - max(0, p + off)


@pytest.mark.parametrize("sizeX", [3, 4, 5, 8])
def test_mapnorm_constant_image(sizeX):
    N, S, F, alpha, beta, c = 2, 6, 2, 0.1, 0.75, 0.5
    md = torch.full((N * S * S * F,), c, dtype=torch.float32)
    d = ax.mapnorm_denoms(md, N, S, F, sizeX, alpha).ref.view(F, S, S, N)
    for y in range(S):
        for x in range(S):
            want = 1 + alpha * c * c * _window_count(S, sizeX, x) * _window_count(S, sizeX, y)
            assert abs(float(d[1, y, x, 0]) - want) < 1e-12, (y, x)
    t = ax.mapnorm_targets(md, d.reshape(-1).float(), beta).ref.view(F, S, S, N)
    assert abs(float(t[0, 0, 0, 1]) - c * float(d[0, 0, 0, 1].float()) ** -beta) < 1e-12


@pytest.mark.parametrize("sizeX", [2, 3])
def test_mapnorm_hot_pixel_at_a_border(sizeX):
    """one hot pixel at (x, y) = (0, 2): the denominators it raises are exactly the pixels whose window holds it"""
    N, S, F, alpha = 1, 5, 1, 1.0
    md = torch.zeros(S * S)
    md[0 + S * 2] = 3.0
    d = ax.mapnorm_denoms(md, N, S, F, sizeX, alpha).ref.view(S, S)
    lo = -(sizeX // 2)
    for y in range(S):
        for x in range(S):
            inside = y + lo <= 2 < y + lo + sizeX and x + lo <= 0 < x + lo + sizeX
            assert float(d[y, x]) == (10.0 if inside else 1.0), (y, x)
    # the undo gathers over the inverse window: the pixels q whose window holds p
    og = torch.zeros(S * S); og[0 + S * 2] = 1.0
    ones = torch.ones(S * S)
    u = ax.mapnorm_undo(og, ones, ones, ones, N, S, F, sizeX, 0.5, 1.0).ref.view(S, S)
    for y in range(S):
        for x in range(S):
            inside = 2 + lo <= y < 2 + lo + sizeX and 0 + lo <= x < 0 + lo + sizeX     # p in window(q = (0, 2))
            want = -1.0 * inside + (1.0 if (y, x) == (2, 0) else 0.0)
            assert abs(float(u[y, x]) - want) < 1e-12, (y, x, float(u[y, x]))


def test_yuv_of_primaries():
    px_n = 4
    img = torch.zeros(3 * px_n)
    img[0] = 1.0                  # pixel 0 red
    img[px_n + 1] = 1.0           # pixel 1 green
    img[2 * px_n + 2] = 1.0       # pixel 2 blue
    y = ax.rgb_to_yuv(img).ref.view(3, px_n)
    f = lambda v: float(np.float32(v))
    assert [float(y[i, 0]) for i in range(3)] == [f(0.2126), f(-0.09991), f(0.615)]
    assert [float(y[i, 1]) for i in range(3)] == [f(0.7152), f(-0.33609), f(-0.55861)]
    assert [float(y[i, 2]) for i in range(3)] == [f(0.0722), f(0.436), f(-0.05639)]
    assert float(y[:, 3].abs().sum()) == 0.0


def test_innerp_restatement_is_a_correlation():
    """innerp = the correlation of each image channel with the derivative of the same channel, summed"""
    r = np.random.RandomState(3)
    g = PG(3, 7, 6, 2, 3, 2, 2, 1, 1, 0)
    x = torch.from_numpy(r.randn(g.N * g.W * g.H * g.C).astype(np.float32))
    dv = torch.from_numpy(r.randn(g.N * g.modX * g.modY * g.C).astype(np.float32))
    e = ax.innerp(g, x, dv).ref.view(g.ky, g.kx)
    X = x.double().view(g.C, g.H, g.W, g.N)
    D = dv.double().view(g.C, g.modY, g.modX, g.N)
    for ty in range(g.ky):
        for tx in range(g.kx):
            s = 0.0
            for my in range(g.modY):
                for mx in range(g.modX):
                    Y, Xp = my * g.sy - g.py + ty, mx * g.sx - g.px + tx
                    if 0 <= Y < g.H and 0 <= Xp < g.W:
                        s += float((X[:, Y, Xp, :] * D[:, my, mx, :]).sum())
            assert abs(float(e[ty, tx]) - s) < 1e-10


# ---------------------------------------------------------------------------------------------------------------------
# the python surface
# ---------------------------------------------------------------------------------------------------------------------
class _Recorder:
    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        return lambda *args: self.calls.append((name, args))


class _M:
    p_mat = ct.pointer(ct.c_int(0))
    p_shape4d = ct.pointer(ct.c_int(0))
    shape4d = (4, 3, 3, 8)


NEW_CALLS = {
    "convInnerp": (lambda b, m: b.convInnerp(m, m, m, None), "convInnerpGemm"),
    "MaxPoolRprop": (lambda b, m: b.MaxPoolRprop(m, m, m, m, None), "MaxPoolRpropGemm"),
    "ResponseNormCrossMapRprop": (lambda b, m: b.ResponseNormCrossMapRprop(m, m, m, 5, 1e-4, 0.75, False),
                                  "ResponseNormCrossMapRpropGemm"),
    "ResponseNorm": (lambda b, m: b.ResponseNorm(m, m, m, 8, 5, 1e-4, 0.75), "ResponseNorm"),
    "ResponseNormUndo": (lambda b, m: b.ResponseNormUndo(m, m, m, m, m, 8, 5, 1e-4, 0.75), "ResponseNormUndo"),
    "ContrastNorm": (lambda b, m: b.ContrastNorm(m, m, m, m, 8, 5, 1e-4, 0.75), "ContrastNorm"),
    "ContrastNormUndo": (lambda b, m: b.ContrastNormUndo(m, m, m, m, m, 8, 5, 1e-4, 0.75), "ContrastNormUndo"),
    "RGBToYUV": (lambda b, m: b.RGBToYUV(m, m), "RGBToYUV"),
}


@pytest.mark.parametrize("method", sorted(NEW_CALLS))
@pytest.mark.parametrize("abi", ["gemm", "cc2"])
def test_binding_calls_the_c_symbol_with_its_signature(method, abi):
    rec = _Recorder()
    b = conv_gemm.Binding(lambda: rec, abi)
    call, symbol = NEW_CALLS[method]
    call(b, _M())
    assert len(rec.calls) == 1
    name, args = rec.calls[0]
    assert name == symbol
    sig = SIGNATURES[symbol]
    assert len(args) == len(sig), (symbol, len(args), len(sig))
    for a, t in zip(args, sig):
        if t in (ct.c_int, ct.c_float, ct.c_bool):
            assert isinstance(a, (int, float, bool)), (symbol, a, t)
        elif a is not None:
            assert isinstance(a, ct._Pointer), (symbol, a, t)


def test_module_level_names():
    for name in NEW_CALLS:
        assert callable(getattr(conv_gemm, name))


def test_dispatch_mirror():
    assert ax.innerp_splits(8, 12 * 5)[0] == 1
    assert ax.innerp_splits(128, 96 * 27 * 27)[0] > 1
    assert ax.rnorm_rprop_branch(1000, 32, False)[0] == "rnorm_tile_kernel<64, (cnb::RnPass)2>"
    assert ax.rnorm_rprop_branch(1000, 512, True) == ("rnorm_rprop_kernel<true>", "ring")
    assert ax.mapnorm_width(55, 5, True) == 16
