"""Pooling, response normalisation and their fused epilogues element by element against float64 (tests/pool_exact.py),
at every dispatch branch of pool.cu and rnorm.cu, and on whole BASELINE-size outputs.

Every call writes into a NaN-sentinel buffer with guard zones: a call with scaleTargets 0 must not read its target and
no call may touch the guards.  Every call asserts its launch count (the fused epilogues against their trailing passes:
colsum_finish against the two-kernel column sum, the in-kernel bf16 twin against a conversion pass, the fused ReLU
against cnb_relu), and runs twice with bit-identical results (no atomics, DESIGN.md).  Each case names the branch the
dispatch mirror of pool_exact.py gives it; test_kernel_names checks those names against the kernels CUPTI records.
Max-pool cases use dyadic inputs, so their undo and bias sums must equal float64 exactly.  A bf16 twin is read back
exactly through a bf16 1x1 conv with identity filters on the staged copy (no conversion launch).
"""
import dataclasses
import zlib

import pytest
import torch

import pool_exact as px
from gpu_buffers import check_twin as _check_twin, guards_ok as _guards_ok, launched as _launched, matrix as _matrix
from pool_exact import PG

pytestmark = pytest.mark.gpu

WORST = {}                 # (op, branch) -> largest |err|/bar


# ---------------------------------------------------------------------------------------------------------------------
# the case tables (importable without a GPU: tests/test_pool_exact_cpu.py checks them against the mirror)
# ---------------------------------------------------------------------------------------------------------------------
@dataclasses.dataclass
class Undo:
    st: float = 0.0
    mask: str = None          # None, "input" (the pool input) or "other"
    bias: bool = True
    bias_st: float = 0.0


@dataclasses.dataclass
class PoolCase:
    name: str
    g: PG
    is_max: bool
    fwd: str                  # branch the forward pass claims
    undo: str                 # branch every undo of the case claims (cache / mask / st given below)
    undos: tuple = (Undo(),)
    cache: bool = False
    so: float = 1.0
    offset: int = 0           # floats: 1 makes every operand 4 bytes off 16-byte alignment
    emit: bool = False
    abi: str = "gemm"
    undo_overrides: dict = None   # index in undos -> branch (the compare path after a tie-mask forward)

    @property
    def aligned(self):
        return self.offset % 4 == 0

    def undo_branch(self, i):
        return (self.undo_overrides or {}).get(i, self.undo)


@dataclasses.dataclass
class RnCase:
    name: str
    N: int
    W: int
    H: int
    F: int
    k: int
    fwd: str
    undo: str
    blocked: bool = False
    frames: int = 1
    alpha: float = 5e-4
    beta: float = 0.75
    relu: bool = False
    emit: bool = False
    offset: int = 0
    hot: float = 0.0          # > 0: post-ReLU input with the first eighth of the channels scaled by `hot`
    abi: str = "gemm"

    @property
    def L(self):
        return self.N * self.W * self.H


UNDOS_FULL = (Undo(0.0), Undo(1.0, bias_st=1.0), Undo(0.0, "input"), Undo(0.0, "other"), Undo(1.0, "input"))

# 2-D geometries of the pool kernels: (tag, ky, kx, sy, sx, py, px, W, H)
GEOMS = [
    ("k2s1", 2, 2, 1, 1, 0, 0, 9, 8),
    ("k1s1", 1, 1, 1, 1, 0, 0, 6, 5),
    ("k2s2", 2, 2, 2, 2, 0, 0, 11, 10),
    ("k3s2p1", 3, 3, 2, 2, 1, 1, 13, 11),
    ("k3s1p1", 3, 3, 1, 1, 1, 1, 7, 8),
    ("k2s3", 2, 2, 3, 3, 0, 0, 11, 11),            # stride > kernel: pixels no window covers
    ("k3s3", 3, 3, 3, 3, 1, 1, 10, 12),
    ("rect", 2, 3, 1, 2, 0, 1, 11, 9),             # kx != ky, sx != sy, px != py
    ("k4s2p1", 4, 4, 2, 2, 1, 1, 12, 10),
    ("k5s3p2", 5, 5, 3, 3, 2, 2, 13, 14),
    ("global", 6, 7, 1, 1, 0, 0, 7, 6),            # global pooling: one window per channel
    ("k2s1p2", 2, 2, 1, 1, 2, 2, 6, 5),            # padding == kernel: empty windows (NaN average)
    ("k2s1p3", 2, 3, 1, 1, 3, 3, 6, 5),            # padding > kernel: empty windows (signed zero average)
]


def _pool_cases():
    out = []
    for tag, ky, kx, sy, sx, py, pxx, W, H in GEOMS:
        for is_max in (True, False):
            for vtag, N, off in (("v4", 32, 0), ("v1n", 7, 0), ("v1mis", 32, 1)):
                if vtag == "v1mis" and tag not in ("k3s2p1", "k2s1", "k4s2p1", "k3s1p1", "k2s3", "rect", "k2s2", "k1s1"):
                    continue
                g = PG(N, W, H, 16, ky, kx, sy, sx, py, pxx)
                a = off % 4 == 0
                f = px.pool_fwd_branch(g, is_max, a).name
                u = px.pool_undo_branch(g, is_max, a).name
                undos = (Undo(0.0, "other"), Undo(1.0, bias_st=1.0))
                out.append(PoolCase("%s_%s_%s" % (tag, "max" if is_max else "avg", vtag), g, is_max, f, u, undos,
                                    offset=off,
                                    # (a NaN average of an empty window would poison the twin's 1x1 consumer)
                                    emit=vtag == "v4" and g.modX * g.modY > 1 and pxx < kx and py < ky))
    # 3-D: frames stacked as channel blocks
    for is_max in (True, False):
        g = PG(8, 6, 7, 4, 2, 2, 1, 1, 0, 0, T=5, kt=2, st_t=2)
        out.append(PoolCase("3d_%s" % ("max" if is_max else "avg"), g, is_max, px.pool_fwd_branch(g, is_max).name,
                            px.pool_undo_branch(g, is_max).name, (Undo(0.0, bias=False), Undo(0.5, "other", bias=False))))
    # the patch kernels: padding 0 / 1 / 2, with and without tie masks, scaleTargets 0 / 1, the ReLU' mask being the pool
    # input or a separate tensor (those two with st = 1 resp. a separate mask stay on the compare path)
    for p in (0, 1, 2):
        for cache in (False, True):
            for vtag, N, off in (("v4", 32, 0), ("v1", 6, 0)):
                if vtag == "v1" and p != 2:
                    continue
                g = PG(N, 13, 12, 16, 3, 3, 2, 2, p, p)
                v = 4 if N % 4 == 0 else 1
                base = "masked_patch<%d>" % v if cache else "patch<%d>" % v
                over = {3: "patch<%d>" % v, 4: "patch<%d>" % v} if cache else None
                out.append(PoolCase("patch_p%d_%s%s" % (p, "cache_" if cache else "", vtag), g, True,
                                    px.pool_fwd_branch(g, True).name, base, UNDOS_FULL, cache=cache, offset=off,
                                    emit=vtag == "v4", undo_overrides=over))
    g = PG(32, 12, 13, 16, 2, 3, 2, 2, 2, 1)            # rectangular patch window (3 wide, 2 high)
    out.append(PoolCase("patch_rect_cache", g, True, px.pool_fwd_branch(g, True).name, "masked_patch<4>", UNDOS_FULL,
                        cache=True, undo_overrides={3: "patch<4>", 4: "patch<4>"}))
    # scaleOutput of the forward pass (no tie masks then: they are recorded for unscaled outputs only)
    g = PG(32, 13, 13, 16, 3, 3, 2, 2, 1, 1)
    out.append(PoolCase("so_max", g, True, px.pool_fwd_branch(g, True).name, "patch<4>", (Undo(),), cache=True, so=0.5))
    out.append(PoolCase("so_avg", g, False, px.pool_fwd_branch(g, False).name,
                        px.pool_undo_branch(g, False).name, (Undo(0.0, "other"),), so=0.25))
    # ABI-2 entry points
    out.append(PoolCase("abi2_max", g, True, px.pool_fwd_branch(g, True).name, "patch<4>", (Undo(1.0),), abi="cc2"))
    out.append(PoolCase("abi2_avg", g, False, px.pool_fwd_branch(g, False).name, px.pool_undo_branch(g, False).name,
                        (Undo(1.0),), abi="cc2"))
    return out


POOL_CASES = _pool_cases()
POOL_BY_NAME = {c.name: c for c in POOL_CASES}
# the average cases once more under the sampling edges' requests (run_pool_epi); empty windows' NaN averages left out
EPI_CASES = [c for c in POOL_CASES if not c.is_max and c.g.px < c.g.kx and c.g.py < c.g.ky]


def _rn(name, N, W, H, F, k, **kw):
    c = RnCase(name, N, W, H, F, k, "", "", **kw)
    a = c.offset % 4 == 0
    c.fwd = px.rnorm_fwd_branch(c.L, F, k, c.blocked, a).name
    c.undo = px.rnorm_undo_branch(c.L, F, k, c.blocked, a).name
    return c


RN_CASES = [
    _rn("tile64", 32, 5, 4, 16, 5, emit=True),
    _rn("tile64_partial", 32, 3, 3, 24, 5),
    _rn("tile32", 32, 4, 4, 256, 9),
    _rn("tile_scalar_odd_L", 7, 5, 5, 20, 5),
    _rn("tile_scalar_misaligned", 32, 4, 4, 20, 5, offset=1),
    _rn("tile_relu_twin", 32, 6, 6, 32, 5, relu=True, emit=True),
    _rn("tile_blocked", 16, 5, 5, 20, 6, blocked=True),
    _rn("tile_3d", 16, 4, 4, 16, 5, frames=3, emit=True),
    _rn("tile_3d_blocked", 16, 4, 4, 12, 4, frames=2, blocked=True),
    _rn("size1", 16, 4, 4, 16, 1),
    _rn("even_k", 16, 4, 4, 32, 4),
    _rn("k_gt_F", 16, 4, 4, 8, 12),
    _rn("hot_x30", 32, 6, 6, 96, 24, hot=30.0),
    _rn("hot_x300", 32, 6, 6, 256, 64, hot=300.0),
    _rn("ring_seg", 8, 4, 4, 896, 5, relu=True, emit=True),
    _rn("ring_noseg", 32, 33, 33, 896, 5),
    _rn("ring_wide", 128, 46, 46, 896, 5),
    _rn("ring_gring_seg", 8, 4, 4, 896, 400),
    _rn("ring_blocked", 8, 4, 4, 900, 100, blocked=True),
    _rn("ring_blocked_gring", 8, 4, 4, 896, 400, blocked=True),
    _rn("ring_wide_gring", 128, 46, 46, 896, 96),
    _rn("ring_wide_blocked", 128, 46, 46, 896, 8, blocked=True),
    _rn("ring_wide_blocked_gring", 128, 46, 46, 896, 112, blocked=True),
    _rn("tile32_scalar", 7, 5, 5, 256, 9),
    _rn("undo_ring_seg", 8, 4, 4, 448, 5),
    _rn("undo_ring_noseg", 32, 33, 33, 448, 5),
    _rn("undo_ring_gring", 8, 4, 4, 448, 120),
    _rn("undo_ring_blocked", 8, 4, 4, 450, 50, blocked=True),
    _rn("abi2", 32, 5, 4, 16, 5, abi="cc2"),
]
RN_BY_NAME = {c.name: c for c in RN_CASES}


# ---------------------------------------------------------------------------------------------------------------------
# fixtures and buffers
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def env():
    assert torch.cuda.is_available(), "these tests need a CUDA device"
    from convnet_b200 import conv_gemm as cg
    from convnet_b200 import lib
    L = lib.load()

    class E:
        pass
    e = E()
    e.cg, e.lib, e.L = cg, lib, L
    e.sms = torch.cuda.get_device_properties(0).multi_processor_count
    yield e
    print("\nlargest |err|/bar per (op, branch):")
    for k in sorted(WORST):
        print("  %-10s %-34s %.3e" % (k[0], k[1], WORST[k]))


@pytest.fixture(autouse=True)
def hygiene(env):
    prec = env.L.convnet_b200_get_conv_precision()
    env.L.convnet_b200_set_conv_precision(2)            # bf16: the mode in which twins are emitted
    env.L.convnet_b200_bf16_invalidate(None)
    try:
        yield
    finally:
        env.L.convnet_b200_set_conv_precision(prec)
        env.L.convnet_b200_bf16_invalidate(None)
        env.L.cnb_relu_deriv(None, None, 0)           # consumes any fuse request a failed call left pending


def _fill(m, values):
    m.storage.copy_(values)
    return m


def _dyadic(n, gen, lo=-8, hi=9):
    return torch.randint(lo, hi, (n,), generator=gen, device="cuda").to(torch.float32) / 16


def _note(op, branch, v):
    WORST[(op, branch)] = max(WORST.get((op, branch), 0.0), v.worst)


# ---------------------------------------------------------------------------------------------------------------------
# pooling: one forward, then each undo of the case
# ---------------------------------------------------------------------------------------------------------------------
def _pool_fwd_call(env, c, x, out):
    L = env.L
    if c.cache:
        L.convnet_b200_pool_cache_next()
    if c.emit:
        L.convnet_b200_emit_bf16_next()
    d = c.g.desc()
    if c.abi == "cc2":
        (env.cg.cc2.MaxPool if c.is_max else env.cg.cc2.AvgPool)(x, out, d)
    else:
        (L.MaxPoolGemm if c.is_max else L.AvgPoolGemm)(x.p_mat, out.p_mat, x.p_shape4d, out.p_shape4d, d, 0.0, c.so)


def _pool_undo_call(env, c, u, x, gr, acts, tgt, mask, bias, bias_so):
    L = env.L
    if mask is not None:
        L.convnet_b200_fuse_next(None, 0, mask.data_ptr())
    if bias is not None:
        L.convnet_b200_fuse_next_bias_grad(bias.data_ptr(), u.bias_st, bias_so)
    if c.emit:
        L.convnet_b200_emit_bf16_next()
    b = env.cg.cc2 if c.abi == "cc2" else env.cg.gemm
    if c.is_max:
        b.MaxPoolUndo(x, gr, acts, tgt, c.g.desc(), u.st)
    else:
        b.AvgPoolUndo(gr, tgt, c.g.desc(), u.st)


def run_pool(env, c, inputs=None, check=True):
    """forward + undos of case c; returns the launched-branch bookkeeping for the kernel-name test"""
    g = c.g
    gen = torch.Generator(device="cuda").manual_seed(zlib.crc32(c.name.encode()))
    nin, nout = g.N * g.W * g.H * g.C * g.T, g.N * g.modX * g.modY * g.C * g.modT
    if inputs is not None:
        xv = inputs
    elif c.is_max:
        xv = _dyadic(nin, gen, -4, 5)                   # few distinct values: many ties
    else:
        xv = torch.randn(nin, generator=gen, device="cuda")
    x, _ = _matrix(*g.in_dims(), g.in_shape(), c.offset, guard=0)
    _fill(x, xv)
    out, obuf = _matrix(*g.out_dims(), g.out_shape(), c.offset)
    fb = px.pool_fwd_branch(g, c.is_max, c.aligned, c.cache, c.so)
    assert fb.name == c.fwd, (c.name, fb.name, c.fwd)
    tag = "%s fwd %s" % (c.name, c.fwd)
    launches = _launched(env, lambda: _pool_fwd_call(env, c, x, out))
    twin_pass = c.emit and not fb.in_kernel_twin
    assert launches == 1 + twin_pass, (tag, launches)
    assert _guards_ok(obuf, c.offset, nout), tag + ": wrote outside its target"
    first = out.storage.clone()
    if check:
        v = px.check(out.storage, px.pool_fwd(g, x.storage, c.is_max, c.so))
        _note("pool_fwd", c.fwd, v)
        print("%-50s %s" % (tag, v))
        assert v.ok, "%s: %s" % (tag, v)
        if c.emit:
            _check_twin(env, out, g.out_shape())
    # second forward into the same target (re-records the masks): bit-identical
    _launched(env, lambda: _pool_fwd_call(env, c, x, out))
    assert torch.equal(first.view(torch.int32), out.storage.view(torch.int32)), tag + ": not reproducible"
    exact_arm = c.is_max and c.so == 1.0
    grv = _dyadic(nout, gen) if exact_arm else torch.randn(nout, generator=gen, device="cuda")
    gr, _ = _matrix(*g.out_dims(), g.out_shape(), c.offset, guard=0)
    _fill(gr, grv)
    for i, u in enumerate(c.undos):
        want = c.undo_branch(i)
        ub = px.pool_undo_branch(g, c.is_max, c.aligned, u.mask, u.st, cached=c.cache and c.so == 1.0)
        assert ub.name == want, (c.name, i, ub.name, want)
        tag = "%s undo[st=%g mask=%s] %s" % (c.name, u.st, u.mask, want)
        tgt, tbuf = _matrix(*g.in_dims(), g.in_shape(), c.offset)
        if u.st != 0.0:                                 # else the NaN prefill: the call must not read it
            tgt.storage.copy_(_dyadic(nin, gen) if exact_arm else torch.randn(nin, generator=gen, device="cuda"))
        t0 = tgt.storage.clone()
        mask = None
        if u.mask == "input":
            mask = x.storage
        elif u.mask == "other":
            mbuf = torch.empty(nin + c.offset, device="cuda")
            mask = mbuf[c.offset:]
            mask.copy_(torch.randn(nin, generator=gen, device="cuda"))
        bias = b0 = None
        bias_so = 0.5 if exact_arm else 1.0 / 128
        if u.bias:
            b0 = _dyadic(g.C, gen) if exact_arm else torch.randn(g.C, generator=gen, device="cuda")
            bias = b0.clone()
        launches = _launched(env, lambda: _pool_undo_call(env, c, u, x, gr, out, tgt, mask, bias, bias_so))
        want_launches = 1 + (c.emit and not ub.in_kernel_twin) + ((1 if ub.slices else 2) if u.bias else 0)
        assert launches == want_launches, (tag, launches, want_launches)
        assert _guards_ok(tbuf, c.offset, nin), tag + ": wrote outside its target"
        y1 = tgt.storage.clone()
        bias1 = bias.clone() if bias is not None else None
        if check:
            if c.is_max:
                e = px.max_undo(g, x.storage, gr.storage, out.storage, u.st, t0, mask=mask, exact_arm=exact_arm)
            else:
                e = px.avg_undo(g, gr.storage, u.st, t0, mask=mask)
            v = px.check(tgt.storage, e)
            _note("pool_undo", want, v)
            print("%-50s %s" % (tag, v))
            assert v.ok, "%s: %s" % (tag, v)
            if bias is not None:
                per_thread, slices = px.bias_depth(ub, g)
                eb = px.bias_grad(tgt.storage, g.N * g.W * g.H, g.C, 1, b0, u.bias_st, bias_so, per_thread, slices,
                                  exact_arm=exact_arm)
                vb = px.check(bias, eb)
                _note("bias_grad", "%s/%d slices" % (ub.name.split("<")[0], slices), vb)
                assert vb.ok, "%s bias: %s" % (tag, vb)
            if c.emit:
                _check_twin(env, tgt, g.in_shape())
        # run it again from the same state: bit-identical target and bias gradient
        tgt.storage.copy_(t0)
        if bias is not None:
            bias.copy_(b0)
        _launched(env, lambda: _pool_undo_call(env, c, u, x, gr, out, tgt, mask, bias, bias_so))
        assert torch.equal(y1.view(torch.int32), tgt.storage.view(torch.int32)), tag + ": not reproducible"
        if bias is not None:
            assert torch.equal(bias1.view(torch.int32), bias.view(torch.int32)), tag + ": bias not reproducible"


@pytest.mark.parametrize("name", [c.name for c in POOL_CASES])
def test_pool_branch(env, name):
    run_pool(env, POOL_BY_NAME[name])


# ---------------------------------------------------------------------------------------------------------------------
# the fused epilogues of the average calls: the forward with ReLU, dropout, a scale, the bias gradient and the twin
# requested, the undo with a scale, the ReLU' mask, the bias gradient and the twin, each bit for bit against the unfused
# call followed by the stand-alone passes it replaces
# ---------------------------------------------------------------------------------------------------------------------
EPI_P, EPI_SCALE, EPI_SEED = 0.3, 1.0 / 0.7, 0x5EED1234


def _epi_call(env, c, fwd, src, tgt, mask, bias, st, request=True):
    L = env.L
    if request:
        if fwd:
            L.convnet_b200_fuse_next_act(None, 1, None)
            L.convnet_b200_fuse_next_dropout(EPI_P, EPI_SCALE, EPI_SEED)
        else:
            L.convnet_b200_fuse_next_act(None, 1, mask.data_ptr())
        L.convnet_b200_fuse_next_scale(EPI_SCALE)
        if bias is not None:
            L.convnet_b200_fuse_next_bias_grad(bias.data_ptr(), 0.5, 0.25)
        if c.emit:
            L.convnet_b200_emit_bf16_next()
    d = c.g.desc()
    if fwd:
        L.AvgPoolGemm(src.p_mat, tgt.p_mat, src.p_shape4d, tgt.p_shape4d, d, 0.0, c.so)
    else:
        env.cg.gemm.AvgPoolUndo(src, tgt, d, st)


def _epi_passes(env, fwd, y, mask):
    L, n = env.L, y.numel()
    scale = torch.full_like(y, EPI_SCALE)
    if fwd:
        L.cnb_relu(y.data_ptr(), n)
        L.cnb_dropout(y.data_ptr(), torch.empty_like(y).data_ptr(), n, EPI_P, EPI_SCALE, EPI_SEED)
    L.cnb_mult(y.data_ptr(), scale.data_ptr(), n)
    if not fwd:
        L.cnb_relu_deriv(y.data_ptr(), mask.data_ptr(), n)


def run_pool_epi(env, c, check=True):
    """forward then undo of case c, each unfused and then fused; returns the branches in launch order"""
    g = c.g
    gen = torch.Generator(device="cuda").manual_seed(zlib.crc32(("epi" + c.name).encode()))
    nin, nout = g.N * g.W * g.H * g.C * g.T, g.N * g.modX * g.modY * g.C * g.modT
    calls = ((True, g.in_dims(), g.in_shape(), g.out_dims(), g.out_shape(), nout, g.N * g.modX * g.modY),
             (False, g.out_dims(), g.out_shape(), g.in_dims(), g.in_shape(), nin, g.N * g.W * g.H))
    branches = []
    for fwd, sdims, sshape, tdims, tshape, n, rows in calls:
        st = 0.0 if fwd else 1.0
        src, _ = _matrix(*sdims, sshape, c.offset, guard=0)
        src.storage.normal_(generator=gen)
        t0 = torch.randn(n, generator=gen, device="cuda")
        mask = torch.randn(n, generator=gen, device="cuda")
        plain, _ = _matrix(*tdims, tshape, c.offset)
        plain.storage.copy_(t0)
        b0 = torch.randn(g.C, generator=gen, device="cuda")
        bias = b0.clone() if g.T == 1 else None          # (the edges ask a bias gradient of 2-D calls only)
        b = (px.pool_fwd_branch(g, False, c.aligned, so=c.so, epi=True) if fwd
             else px.pool_undo_branch(g, False, c.aligned, st=st, epi=True))
        branches += [(px.pool_fwd_branch(g, False, c.aligned, so=c.so) if fwd
                      else px.pool_undo_branch(g, False, c.aligned, st=st)), b]
        tag = "%s %s+epi %s" % (c.name, "fwd" if fwd else "undo", b.name)
        assert _launched(env, lambda: _epi_call(env, c, fwd, src, plain, mask, None, st, False)) == 1, tag
        _epi_passes(env, fwd, plain.storage, mask)
        tgt, tbuf = _matrix(*tdims, tshape, c.offset)
        tgt.storage.copy_(t0)
        launches = _launched(env, lambda: _epi_call(env, c, fwd, src, tgt, mask, bias, st))
        passes = 0 if b.fused else 3 if fwd else 2
        want = 1 + passes + (bias is not None and (1 if b.slices else 2)) + (c.emit and not b.in_kernel_twin)
        assert launches == want, (tag, launches, want)
        assert _guards_ok(tbuf, c.offset, n), tag + ": wrote outside its target"
        if not check:
            continue
        assert torch.equal(tgt.storage.view(torch.int32), plain.storage.view(torch.int32)), tag + ": not the passes' result"
        if bias is not None:
            per_thread, slices = px.bias_depth(b, g)
            vb = px.check(bias, px.bias_grad(tgt.storage, rows, g.C, 1, b0, 0.5, 0.25, per_thread, slices))
            _note("bias_grad", "%s/%d slices" % (b.name.split("<")[0], slices), vb)
            assert vb.ok, "%s bias: %s" % (tag, vb)
        if c.emit:
            _check_twin(env, tgt, tshape)
    return branches


@pytest.mark.parametrize("name", [c.name for c in EPI_CASES])
def test_pool_epilogue_branch(env, name):
    run_pool_epi(env, POOL_BY_NAME[name])


# ---------------------------------------------------------------------------------------------------------------------
# UpSample / DownSample
# ---------------------------------------------------------------------------------------------------------------------
def test_up_down_sample(env):
    f, N, w, h, C = 2, 32, 5, 6, 8
    big = PG(N, w * f, h * f, C, f, f, f, f)
    gen = torch.Generator(device="cuda").manual_seed(77)
    small, _ = _matrix(N, w * h * C, (N, w, h, C), guard=0)
    small.storage.normal_(generator=gen)
    tgt, tbuf = _matrix(N, w * h * C * f * f, big.in_shape())
    tgt.storage.normal_(generator=gen)
    t0 = tgt.storage.clone()
    assert _launched(env, lambda: env.cg.UpSample(small, tgt, f, 0.5)) == 1
    assert _guards_ok(tbuf, 0, tgt.storage.numel())
    v = px.check(tgt.storage, px.upsample(big, small.storage, 0.5, t0, f))
    _note("upsample", "undo_rows", v)
    assert v.ok, v
    down, dbuf = _matrix(N, w * h * C, (N, w, h, C))
    assert _launched(env, lambda: env.cg.DownSample(tgt, down, f)) == 1
    assert _guards_ok(dbuf, 0, down.storage.numel())
    v = px.check(down.storage, px.pool_fwd(big, tgt.storage, False))
    _note("downsample", "rows", v)
    assert v.ok, v


# ---------------------------------------------------------------------------------------------------------------------
# response normalisation
# ---------------------------------------------------------------------------------------------------------------------
def _rn_inputs(c, gen):
    n = c.L * c.F * c.frames
    if c.hot:
        x = torch.relu(torch.randn(n, generator=gen, device="cuda")).view(c.frames, c.F, c.L)
        x[:, : c.F // 8] *= c.hot
        x = x.reshape(-1)
    else:
        x = torch.randn(n, generator=gen, device="cuda")
    return x, torch.randn(n, generator=gen, device="cuda")


def _rn_fwd_call(env, c, x, out):
    if c.relu:
        env.L.convnet_b200_fuse_next(None, 1, None)
    if c.emit:
        env.L.convnet_b200_emit_bf16_next()
    if c.frames > 1:
        env.cg.ResponseNormCrossMap3D(x, out, c.k, c.alpha, c.beta, c.blocked, c.frames)
    elif c.abi == "cc2":
        env.cg.cc2.ResponseNormCrossMap(x, out, c.k, c.alpha, c.beta, c.blocked)
    else:
        env.cg.ResponseNormCrossMap(x, out, c.k, c.alpha, c.beta, c.blocked)


def _rn_undo_call(env, c, dy, x, acts, out):
    if c.emit:
        env.L.convnet_b200_emit_bf16_next()
    if c.frames > 1:
        env.cg.ResponseNormCrossMap3DUndo(dy, x, out, c.k, c.alpha, c.beta, c.blocked, c.frames)
    elif c.abi == "cc2":
        env.cg.cc2.ResponseNormCrossMapUndo(dy, x, out, c.k, c.alpha, c.beta, c.blocked, acts=acts)
    else:
        env.cg.ResponseNormCrossMapUndo(dy, x, out, c.k, c.alpha, c.beta, c.blocked)


def run_rnorm(env, c, inputs=None, check=True):
    gen = torch.Generator(device="cuda").manual_seed(zlib.crc32(c.name.encode()))
    shape = (c.N, c.W, c.H, c.F * c.frames)
    n = c.L * c.F * c.frames
    xv, dyv = inputs if inputs is not None else _rn_inputs(c, gen)
    a = c.offset % 4 == 0
    fb = px.rnorm_fwd_branch(c.L, c.F, c.k, c.blocked, a, env.sms)
    ub = px.rnorm_undo_branch(c.L, c.F, c.k, c.blocked, a, env.sms)
    assert (fb.name, ub.name) == (c.fwd, c.undo), (c.name, fb.name, ub.name)
    x, _ = _matrix(c.N, n // c.N, shape, c.offset, guard=0)
    _fill(x, xv)
    out, obuf = _matrix(c.N, n // c.N, shape, c.offset)
    tag = "%s fwd %s" % (c.name, c.fwd)
    launches = _launched(env, lambda: _rn_fwd_call(env, c, x, out))
    fused = px.rnorm_can_fuse(c.F)
    assert launches == c.frames + (c.relu and not fused) + (c.emit and not fused), (tag, launches)
    assert _guards_ok(obuf, c.offset, n), tag + ": wrote outside its target"
    y1 = out.storage.clone()
    if check:
        v = px.check(out.storage, px.rnorm_fwd(x.storage, c.F, c.k, c.alpha, c.beta, c.blocked, c.frames, c.relu))
        _note("rnorm_fwd", c.fwd, v)
        print("%-50s %s" % (tag, v))
        assert v.ok, "%s: %s" % (tag, v)
        if c.hot >= 300:
            # the kernel's error is of the prefix class: a bar charged on the window's own mass rejects it
            w = px.check(out.storage, px.rnorm_fwd(x.storage, c.F, c.k, c.alpha, c.beta, c.blocked, c.frames, c.relu,
                                                   local_bar=True))
            print("%-50s window-local bar: %s" % (tag, w))
            assert not w.ok, "hot channels: the window-local bar holds too, the case does not separate the bars"
        if c.emit:
            _check_twin(env, out, shape)
    _launched(env, lambda: _rn_fwd_call(env, c, x, out))
    assert torch.equal(y1.view(torch.int32), out.storage.view(torch.int32)), tag + ": not reproducible"
    dy, _ = _matrix(c.N, n // c.N, shape, c.offset, guard=0)
    _fill(dy, dyv)
    dx, dbuf = _matrix(c.N, n // c.N, shape, c.offset)
    tag = "%s undo %s" % (c.name, c.undo)
    launches = _launched(env, lambda: _rn_undo_call(env, c, dy, x, out, dx))
    assert launches == c.frames + c.emit, (tag, launches)
    assert _guards_ok(dbuf, c.offset, n), tag + ": wrote outside its target"
    d1 = dx.storage.clone()
    if check:
        v = px.check(dx.storage, px.rnorm_undo(dy.storage, x.storage, c.F, c.k, c.alpha, c.beta, c.blocked, c.frames))
        _note("rnorm_undo", c.undo, v)
        print("%-50s %s" % (tag, v))
        assert v.ok, "%s: %s" % (tag, v)
        if c.emit:
            _check_twin(env, dx, shape)
    _launched(env, lambda: _rn_undo_call(env, c, dy, x, out, dx))
    assert torch.equal(d1.view(torch.int32), dx.storage.view(torch.int32)), tag + ": not reproducible"


@pytest.mark.parametrize("name", [c.name for c in RN_CASES])
def test_rnorm_branch(env, name):
    c = RN_BY_NAME[name]
    if c.L * c.F * c.frames > (1 << 28):
        torch.cuda.empty_cache()
    run_rnorm(env, c)
    torch.cuda.empty_cache()


# ---------------------------------------------------------------------------------------------------------------------
# which kernel ran: the template names CUPTI records against the mirror
# ---------------------------------------------------------------------------------------------------------------------
def _hot_kernels(prof):
    from torch.autograd import DeviceType
    evs = [e for e in prof.events() if e.device_type == DeviceType.CUDA and
           ("pool_" in e.name or "rnorm_" in e.name) and "cnb::" in e.name]
    evs.sort(key=lambda e: e.time_range.start)
    return [e.name for e in evs]


def test_kernel_names(env):
    """every small branch case once more, unchecked, under torch.profiler: the pool / rnorm kernels CUPTI records must
    be, in order, the ones the mirror names (two launches per call: each call runs twice; the epilogue cases run each
    call unfused, then fused)"""
    from torch.profiler import ProfilerActivity, profile
    want = []
    small_rn = [c for c in RN_CASES if c.L * c.F < (1 << 22)]
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for c in POOL_CASES:
            env.L.convnet_b200_bf16_invalidate(None)
            run_pool(env, c, check=False)
            want += [px.pool_fwd_branch(c.g, c.is_max, c.aligned, c.cache, c.so).kernel] * 2
            for i, u in enumerate(c.undos):
                want += [px.pool_undo_branch(c.g, c.is_max, c.aligned, u.mask, u.st,
                                             cached=c.cache and c.so == 1.0).kernel] * 2
        for c in EPI_CASES:
            want += [b.kernel for b in run_pool_epi(env, c, check=False)]
        for c in small_rn:
            run_rnorm(env, c, check=False)
            a = c.offset % 4 == 0
            want += [px.rnorm_fwd_branch(c.L, c.F, c.k, c.blocked, a, env.sms).kernel] * (2 * c.frames)
            want += [px.rnorm_undo_branch(c.L, c.F, c.k, c.blocked, a, env.sms).kernel] * (2 * c.frames)
        torch.cuda.synchronize()
    got = _hot_kernels(prof)
    if not got:
        pytest.skip("torch.profiler recorded no kernels of the library in this process (CUPTI activity unavailable)")
    assert len(got) == len(want), (len(got), len(want))
    for i, (g_, w) in enumerate(zip(got, want)):
        assert w in g_, (i, w, g_)


# ---------------------------------------------------------------------------------------------------------------------
# whole outputs at BASELINE size: AlexNet's pools and response norms at batch 128, with the training step's options
# ---------------------------------------------------------------------------------------------------------------------
ALEX_POOL = {"pool1": (110, 96), "pool2": (27, 256), "pool5": (12, 512)}       # input side, channels; 3x3 / 2, pad 1
ALEX_RNORM = {"rnorm1": (55, 96, 24), "rnorm2": (14, 256, 64)}              # size, channels, sizeF (0.25 * channels)


@pytest.mark.parametrize("layer", list(ALEX_POOL))
def test_alexnet_pool(env, layer):
    """the training step's combination: tie masks recorded by the forward pass, the ReLU' mask being the pool input
    (a ReLU output), the bias gradient of the conv below fused, and bf16 twins of both outputs"""
    W, C = ALEX_POOL[layer]
    g = PG(128, W, W, C, 3, 3, 2, 2, 1, 1)
    gen = torch.Generator(device="cuda").manual_seed(zlib.crc32(layer.encode()))
    x = torch.relu(torch.randn(g.N * W * W * C, generator=gen, device="cuda"))
    c = PoolCase("alex_" + layer, g, True, px.pool_fwd_branch(g, True).name, "masked_patch<4>",
                 (Undo(0.0, "input", True),), cache=True, emit=True)
    run_pool(env, c, inputs=x)
    torch.cuda.empty_cache()


@pytest.mark.parametrize("layer", list(ALEX_RNORM))
def test_alexnet_rnorm(env, layer):
    W, F, k = ALEX_RNORM[layer]
    c = _rn("alex_" + layer, 128, W, W, F, k, relu=True, emit=True)
    gen = torch.Generator(device="cuda").manual_seed(zlib.crc32(layer.encode()))
    n = c.L * F
    x = torch.relu(torch.randn(n, generator=gen, device="cuda"))
    run_rnorm(env, c, inputs=(x, torch.randn(n, generator=gen, device="cuda") * 1e-3))
    torch.cuda.empty_cache()
