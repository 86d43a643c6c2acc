"""The elementwise kernels of csrc/elementwise.cu element by element against float64 (tests/elementwise_exact.py), at
every dispatch branch and on the `alexnet+bn` / AlexNet shapes at batch 128.

Every call writes into NaN-sentinel buffers with guard zones, 16-byte aligned or one float off: an output the call
does not read (dropout mask, batch-norm y / mu / sigma / gradients, a bias gradient with st = 0, the sum) keeps the NaN
prefill until the call writes it, and no call may touch the guards.  Every call asserts the branch the dispatch mirror
names and its launch count (a bf16 twin written in the kernel against a trailing conversion pass), and runs twice from
the same inputs with bit-identical results.  test_kernel_names checks the mirror's kernel names against the kernels
CUPTI records.  A bf16 twin is read back exactly through a bf16 1x1 conv with identity filters.
"""
import dataclasses
import os
import subprocess
import sys
import zlib

import numpy as np
import pytest
import torch

import conv_exact as cx
import elementwise_exact as ex
from gpu_buffers import check_twin, guards_ok, launched, matrix

pytestmark = pytest.mark.gpu

WORST = {}                 # (op, branch) -> largest |err|/bar
NEG_ZERO = {}              # op -> the signs fmaxf gave -0 inputs
RECORD = None              # list: the kernel names each call should launch (test_kernel_names)
SMS_H100 = ex.SMS
BIG = 2 ** 31 + 4099       # past the 32-bit index range, n % 4 == 3


# ---------------------------------------------------------------------------------------------------------------------
# the case tables (importable without a GPU: tests/test_elementwise_exact_cpu.py checks them against the mirror)
# ---------------------------------------------------------------------------------------------------------------------
@dataclasses.dataclass
class EwCase:
    name: str
    op: str                   # relu, relu_deriv, dropout, mult
    n: int
    off: int = 0              # the target's offset in floats
    off2: int = 0             # the second operand's (y, mask, b)
    emit: bool = False
    twin: tuple = None        # (N, W, H, C) view of the target for the twin read-back
    special: bool = False     # NaN, +-0, subnormals, infinities among the inputs
    p: float = 0.5
    scale: float = 2.0
    seed: int = 1234
    tie: tuple = ()           # dropout: p is set to u of this element (the >= threshold)
    branch: str = ""

    def mirror(self, sms=SMS_H100):
        return ex.n4_branch(self.op, self.n, self.off % 4 == 0, self.off2 % 4 == 0, sms)


GS_N = 16 * SMS_H100 * 256 * 4 + 6     # more float4 groups than 16 blocks per SM cover in one pass


def _ew(name, op, n, **kw):
    c = EwCase(name, op, n, **kw)
    c.branch = c.mirror().name
    return c


EW_CASES = []
for _op in ("relu", "relu_deriv", "dropout", "mult"):
    EW_CASES += [
        _ew("%s_n1" % _op, _op, 1),
        _ew("%s_n3" % _op, _op, 3, special=_op != "dropout"),
        _ew("%s_n4097" % _op, _op, 4097, special=_op != "dropout"),
        _ew("%s_n4098" % _op, _op, 4098),
        _ew("%s_n4099" % _op, _op, 4099),
        _ew("%s_vec_twin" % _op, _op, 8192, emit=True, twin=(32, 4, 4, 16)),
        _ew("%s_vec_special" % _op, _op, 8192, special=_op != "dropout"),
        _ew("%s_mis_target" % _op, _op, 8192, off=1, emit=True),
        _ew("%s_gs" % _op, _op, GS_N),
        _ew("%s_gs_vec" % _op, _op, GS_N + 394),
        _ew("%s_gs_scalar" % _op, _op, GS_N // 4 + 300, off=1),
    ]
    if _op != "relu":
        EW_CASES.append(_ew("%s_mis_second" % _op, _op, 8192, off2=1, emit=True))
EW_CASES += [
    _ew("dropout_p0", "dropout", 4099, p=0.0),
    _ew("dropout_tie_body", "dropout", 4103, tie=(1001,)),
    _ew("dropout_tie_tail", "dropout", 4103, tie=(4101,)),
    _ew("dropout_seed_wrap", "dropout", 4099, seed=2 ** 64 - 37),
    _ew("dropout_scale_1_over_0.7", "dropout", 4099, p=0.3, scale=float(np.float32(1 / 0.7))),
    _ew("dropout_fc_128x4096", "dropout", 128 * 4096, emit=True, twin=(128, 1, 1, 4096)),
    _ew("relu_conv1_128x55x55x96", "relu", 128 * 55 * 55 * 96, emit=True, twin=(128, 55, 55, 96)),
]
EW_BY_NAME = {c.name: c for c in EW_CASES}


@dataclasses.dataclass
class BiasCase:
    name: str
    rows: int
    cols: int
    relu: bool = False
    off: int = 0
    emit: bool = False
    twin: tuple = None
    special: bool = False
    branch: str = ""


def _bias(name, rows, cols, **kw):
    c = BiasCase(name, rows, cols, **kw)
    c.branch = ex.bias_branch(rows, cols, c.off % 4 == 0, c.relu).name
    return c


BIAS_CASES = []
for _r in (False, True):
    _t = "relu_" if _r else ""
    BIAS_CASES += [
        _bias(_t + "vec", 4000, 37, relu=_r, special=_r),
        _bias(_t + "rows_odd", 4001, 37, relu=_r, special=_r),
        _bias(_t + "rows_2", 4002, 5, relu=_r),
        _bias(_t + "misaligned", 4000, 37, relu=_r, off=1),
        _bias(_t + "tiny", 3, 5, relu=_r),
        _bias(_t + "twin", 512, 16, relu=_r, emit=True, twin=(32, 4, 4, 16)),
        _bias(_t + "gs_conv2", 128 * 27 * 27, 256, relu=_r),
        _bias(_t + "gs_scalar", 128 * 27 * 27 + 1, 256, relu=_r),
    ]
BIAS_BY_NAME = {c.name: c for c in BIAS_CASES}


@dataclasses.dataclass
class GradCase:
    name: str
    rows: int
    cols: int
    st: float = 0.0
    off: int = 0
    dyadic: bool = False
    branch: str = ""


def _grad(name, rows, cols, **kw):
    c = GradCase(name, rows, cols, **kw)
    c.branch = ex.bias_grad_branch(rows, cols, c.st).name
    return c


GRAD_CASES = []
for _st in (0.0, 1.0):
    _t = "st1_" if _st else ""
    GRAD_CASES += [
        _grad(_t + "c1_64slices", 65536 * 3 + 5, 1, st=_st, dyadic=True),
        _grad(_t + "c1_64slices_randn", 65536 * 3 + 5, 1, st=_st),
        _grad(_t + "c4096_1slice", 128, 4096, st=_st),
        _grad(_t + "rows_lt_1024", 1000, 3, st=_st, dyadic=True),
        _grad(_t + "c37_k_slices", 40000, 37, st=_st, off=1),
        _grad(_t + "c37_k_slices_dyadic", 40000, 37, st=_st, dyadic=True),
    ]
GRAD_BY_NAME = {c.name: c for c in GRAD_CASES}


@dataclasses.dataclass
class BnCase:
    name: str
    n: int
    C: int
    train: int = 1
    relu: int = 0
    run: bool = False
    off_x: int = 0
    off_y: int = 0            # y and the derivative (a layer's state and its derivative share the alignment)
    emit: bool = False
    twin: tuple = None
    kind: str = "randn"       # randn, offset (channel 0 at mean 1e3, sd 1e-2), dyadic (exact mean), pm1 (exact
                              # variance), grad_exact (caller's dyadic mu, sigma = 2: exact backward sums)
    eps: float = 1e-5
    f: float = 0.9
    stats: str = ""
    apply: str = ""
    backward: str = ""


def _bn(name, n, C, **kw):
    c = BnCase(name, n, C, **kw)
    ax, ay = c.off_x % 4 == 0, c.off_y % 4 == 0
    c.stats = ex.bn_stats_branch(n, C, ax, c.run).name
    c.apply = ex.bn_apply_branch(n, C, ax, ay, c.relu).name
    c.backward = ex.bn_backward_branch(n, C, ax, ay, c.train).name
    return c


BN_CASES = [
    _bn("n1", 1, 3, run=True),
    _bn("n1_test", 1, 2, train=0, relu=1),
    _bn("n4099_relu", 4099, 5, relu=1, run=True),
    _bn("n4098_test", 4098, 5, train=0, relu=1),
    _bn("x_aligned_y_misaligned", 4096, 5, off_y=1, run=True),
    _bn("x_misaligned", 4096, 3, off_x=1, relu=1),
    _bn("c1_1024_slices_pm1", 2 ** 21, 1, kind="pm1", run=True),
    _bn("c1_1024_slices_dyadic", 2 ** 21, 1, kind="dyadic", relu=1, train=0),
    _bn("c1_1024_slices_scalar", 2 ** 21, 1, off_x=1, relu=1),
    _bn("c1_1024_slices_scalar_test", 2 ** 21 + 2, 1, train=0, run=True),
    _bn("vec_k_slices_test", 4096, 5, train=0),
    _bn("c65535", 8, 65535, relu=1, run=True),
    _bn("train0_twin", 512, 16, train=0, emit=True, twin=(32, 4, 4, 16)),
    _bn("train1_relu_twin", 512, 16, relu=1, run=True, emit=True, twin=(32, 4, 4, 16)),
    _bn("offset_channel", 600000, 4, kind="offset", run=True),
    _bn("grad_exact", 2 ** 16, 3, kind="grad_exact"),
    _bn("grad_exact_scalar", 2 ** 16, 3, kind="grad_exact", off_x=1, off_y=1),
]
# the alexnet+bn layers at batch 128 (DESIGN.md §4.6), with the training step's options
ALEX_BN = {"hidden1_conv": (1548800, 96), "hidden2_conv": (93312, 256), "hidden3_conv_nin1": (25088, 768),
           "hidden4_conv": (25088, 384), "hidden5_conv_nin1": (18432, 1024), "hidden6": (128, 4096)}
BN_PROD = [_bn("alex_" + k, n, C, relu=1, run=True) for k, (n, C) in ALEX_BN.items()]
BN_BY_NAME = {c.name: c for c in BN_CASES + BN_PROD}


@dataclasses.dataclass
class SmCase:
    name: str
    rows: int
    cols: int
    kind: str = "randn"       # randn, scaled (x30, +1e4), tied, equal, onehot
    off: int = 0
    branch: str = ""


def _sm(name, rows, cols, **kw):
    c = SmCase(name, rows, cols, **kw)
    c.branch = ex.softmax_branch(rows, cols).name
    return c


SM_CASES = [_sm("r%d_c%d" % (r, c), r, c) for r in (1, 31, 32, 33, 129) for c in (1, 2, 7, 8, 9, 1000, 1001)]
SM_CASES += [
    _sm("scaled_r33_c1001", 33, 1001, kind="scaled"),
    _sm("scaled_r129_c9", 129, 9, kind="scaled"),
    _sm("scaled_r32_c7", 32, 7, kind="scaled"),
    _sm("tied_r32_c9", 32, 9, kind="tied"),
    _sm("tied_r31_c1000", 31, 1000, kind="tied"),
    _sm("equal_r33_c7", 33, 7, kind="equal"),
    _sm("equal_r129_c1000", 129, 1000, kind="equal"),
    _sm("equal_r1_c1", 1, 1, kind="equal"),
    _sm("onehot_r129_c1001", 129, 1001, kind="onehot"),
    _sm("onehot_r32_c9", 32, 9, kind="onehot"),
    _sm("misaligned_r31_c9", 31, 9, off=1),
    _sm("alex_128x1000", 128, 1000),
]
SM_BY_NAME = {c.name: c for c in SM_CASES}


@dataclasses.dataclass
class SumCase:
    name: str
    n: int
    dyadic: bool = False
    off: int = 0
    branch: str = ""


SUM_CASES = []
for _n in (1, 31, 256, 257, 10000):
    SUM_CASES.append(SumCase("n%d" % _n, _n, branch=ex.sum_branch(_n).name))
    SUM_CASES.append(SumCase("n%d_dyadic" % _n, _n, dyadic=True, off=1, branch=ex.sum_branch(_n).name))
SUM_BY_NAME = {c.name: c for c in SUM_CASES}


# ---------------------------------------------------------------------------------------------------------------------
# fixtures, buffers, bookkeeping
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
        print("  %-14s %-40s %.3e" % (k[0], k[1], WORST[k]))
    print("fmaxf(-0, 0) returned:", {k: sorted(v) for k, v in NEG_ZERO.items()})


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


def _flat(n, off, shape=None, guard=64):
    """(CUDAMatrix over n floats at `off`, its sentinel buffer)"""
    if shape is None:
        return matrix(1, n, (1, 1, 1, n), off, guard)
    return matrix(shape[0], n // shape[0], shape, off, guard)


def _gen(name):
    return torch.Generator(device="cuda").manual_seed(zlib.crc32(name.encode()))


def _dyadic(n, gen, lo=-8, hi=9):
    return torch.randint(lo, hi, (n,), generator=gen, device="cuda").to(torch.float32) / 16


SPECIALS = [float("nan"), -0.0, 0.0, 1e-45, -1e-45, 2.0 ** -130, -(2.0 ** -127), float("inf"), float("-inf")]


def _with_specials(v, gen):
    n = v.numel()
    k = min(n, len(SPECIALS) * 4)
    pos = torch.randperm(n, generator=gen, device="cuda")[:k]
    v[pos] = torch.tensor((SPECIALS * 4)[:k], device="cuda")
    return v


def _note(op, branch, v):
    WORST[(op, branch)] = max(WORST.get((op, branch), 0.0), v.worst)


def _ok(op, branch, tag, y, e):
    v = ex.check(y, e)
    _note(op, branch, v)
    print("%-60s %s" % (tag, v))
    assert v.ok, "%s: %s" % (tag, v)


def _call(env, br, fn, emit=False):
    """one library call: the launch count the mirror gives it, recorded for test_kernel_names"""
    if emit:
        env.L.convnet_b200_emit_bf16_next()
    n = launched(env, fn)
    assert n == br.launches(emit), (br.name, n, br.launches(emit))
    if RECORD is not None:
        RECORD.extend(br.kernels)


def _same(a, b):
    return torch.equal(a.view(torch.int32), b.view(torch.int32))


# ---------------------------------------------------------------------------------------------------------------------
# relu, relu', dropout, mult
# ---------------------------------------------------------------------------------------------------------------------
def _ew_fn(env, c, t, s, p):
    L = env.L
    if c.op == "relu":
        return lambda: L.cnb_relu(t.ptr, c.n)
    if c.op == "relu_deriv":
        return lambda: L.cnb_relu_deriv(t.ptr, s.ptr, c.n)
    if c.op == "dropout":
        return lambda: L.cnb_dropout(t.ptr, s.ptr, c.n, p, c.scale, c.seed)
    return lambda: L.cnb_mult(t.ptr, s.ptr, c.n)


def _dropout_p(c):
    if c.tie:
        return float(cx.dropout_u(c.seed, np.array(c.tie, dtype=np.uint64))[0])
    return c.p


def run_ew(env, c, check=True):
    gen = _gen(c.name)
    br = c.mirror(env.sms)
    assert br.name == c.branch, (c.name, br.name, c.branch)
    t, tbuf = _flat(c.n, c.off, c.twin)
    xv = torch.randn(c.n, generator=gen, device="cuda")
    if c.special:
        xv = _with_specials(xv, gen)
    t.storage.copy_(xv)
    s = sbuf = None
    if c.op != "relu":
        s, sbuf = _flat(c.n, c.off2)
        if c.op == "relu_deriv":
            yv = torch.relu(torch.randn(c.n, generator=gen, device="cuda")) * torch.sign(
                torch.randn(c.n, generator=gen, device="cuda"))
            s.storage.copy_(_with_specials(yv, gen) if c.special else yv)
        elif c.op == "mult":
            s.storage.copy_(torch.randn(c.n, generator=gen, device="cuda"))
    s0 = s.storage.clone() if s is not None else None
    p = _dropout_p(c)
    tag = "%s %s" % (c.name, c.branch)
    _call(env, br, _ew_fn(env, c, t, s, p), c.emit)
    assert guards_ok(tbuf, c.off, c.n), tag + ": wrote outside its target"
    if sbuf is not None:
        assert guards_ok(sbuf, c.off2, c.n), tag + ": wrote outside its second operand"
    y1, m1 = t.storage.clone(), s.storage.clone() if s is not None else None
    if check:
        if c.op == "relu":
            _ok("relu", c.branch, tag, t.storage, ex.relu(xv))
            nz = (xv == 0) & torch.signbit(xv)
            if bool(nz.any()):
                NEG_ZERO.setdefault("relu", set()).update(
                    "-0" if b else "+0" for b in torch.signbit(t.storage[nz]).tolist())
        elif c.op == "relu_deriv":
            _ok("relu_deriv", c.branch, tag, t.storage, ex.relu_deriv(xv, s0))
        elif c.op == "mult":
            _ok("mult", c.branch, tag, t.storage, ex.mult(xv, s0))
        else:
            ev, em = ex.dropout(xv, p, c.scale, c.seed)
            _ok("dropout", c.branch, tag, t.storage, ev)
            _ok("dropout_mask", c.branch, tag + " mask", s.storage, em)
            for k in c.tie:
                assert float(s.storage[k]) == c.scale, tag + ": the element at the threshold was dropped"
        if c.emit and c.twin:
            check_twin(env, t, c.twin)
    # the same call again from the same inputs: bit-identical
    t.storage.copy_(xv)
    if c.op == "dropout":
        s.storage.view(torch.int32).fill_(0x7FC0DEAD)
    _call(env, br, _ew_fn(env, c, t, s, p), c.emit)
    assert _same(y1, t.storage), tag + ": not reproducible"
    if s is not None:
        assert _same(m1, s.storage), tag + ": second operand not reproducible"


@pytest.mark.parametrize("name", [c.name for c in EW_CASES])
def test_elementwise_branch(env, name):
    c = EW_BY_NAME[name]
    run_ew(env, c)
    if c.n > (1 << 24):
        torch.cuda.empty_cache()


@pytest.mark.parametrize("op", ["relu", "dropout"])
def test_index_past_2_31(env, op):
    """n = 2^31 + 4099: windows around 2^31, the ends and a random sample of the in-place result"""
    n = BIG
    need = (2 if op == "dropout" else 1) * 4 * n + (2 << 30)
    if torch.cuda.mem_get_info()[0] < need:
        pytest.skip("needs %.1f GB of free device memory" % (need / 2 ** 30))
    br = ex.n4_branch(op, n, True, True, env.sms)
    assert br.name == "%s<vec+tail>|gs" % op, br.name
    gen = _gen("big_" + op)
    x = torch.empty(n + 64, dtype=torch.float32, device="cuda")
    x.view(torch.int32)[n:].fill_(0x7FC0DEAD)
    x[:n].normal_(generator=gen)
    mask = torch.empty(n + 64 if op == "dropout" else 0, dtype=torch.float32, device="cuda")
    mask.view(torch.int32).fill_(0x7FC0DEAD)
    # windows by slicing (torch's gather kernels do not take a source this long): both ends, 2^31 and 64 random ones
    w = 1 << 11                                         # < 4099: the window around 2^31 ends inside the target
    r = torch.Generator().manual_seed(31)
    starts = [0, 2 ** 31 - w, n - 2 * w] + torch.randint(0, n - 2 * w, (64,), generator=r).tolist()
    idx = torch.cat([torch.arange(s0, s0 + 2 * w) for s0 in starts])
    win = lambda t: torch.cat([t[s0:s0 + 2 * w] for s0 in starts])
    xv = win(x).clone()
    p, scale, seed = 0.5, 2.0, 2 ** 40 + 7
    if op == "relu":
        _call(env, br, lambda: env.L.cnb_relu(x.data_ptr(), n))
    else:
        _call(env, br, lambda: env.L.cnb_dropout(x.data_ptr(), mask.data_ptr(), n, p, scale, seed))
    assert bool((x.view(torch.int32)[n:] == 0x7FC0DEAD).all()), "wrote past the end"
    tag = "%s n=2^31+4099 %s" % (op, br.name)
    if op == "relu":
        _ok("relu", br.name, tag, win(x), ex.relu(xv))
    else:
        assert bool((mask.view(torch.int32)[n:] == 0x7FC0DEAD).all()), "mask: wrote past the end"
        ev, em = ex.dropout(xv, p, scale, seed, idx=idx.numpy())
        _ok("dropout", br.name, tag, win(x), ev)
        _ok("dropout_mask", br.name, tag + " mask", win(mask), em)
    del x, mask
    torch.cuda.empty_cache()


# ---------------------------------------------------------------------------------------------------------------------
# bias add, bias gradient
# ---------------------------------------------------------------------------------------------------------------------
def run_bias(env, c, check=True):
    gen = _gen(c.name)
    n = c.rows * c.cols
    br = ex.bias_branch(c.rows, c.cols, c.off % 4 == 0, c.relu, env.sms)
    assert br.name == c.branch, (c.name, br.name, c.branch)
    t, tbuf = _flat(n, c.off, c.twin)
    xv = torch.randn(n, generator=gen, device="cuda")
    if c.special:
        xv = _with_specials(xv, gen)
    t.storage.copy_(xv)
    b = torch.randn(c.cols, generator=gen, device="cuda")
    fn = env.L.cnb_add_channel_bias_relu if c.relu else env.L.cnb_add_channel_bias
    tag = "%s %s" % (c.name, c.branch)
    _call(env, br, lambda: fn(t.ptr, b.data_ptr(), c.rows, c.cols), c.emit)
    assert guards_ok(tbuf, c.off, n), tag + ": wrote outside its target"
    y1 = t.storage.clone()
    if check:
        _ok("bias_relu" if c.relu else "bias", c.branch, tag, t.storage, ex.bias_add(xv, b, c.rows, c.cols, c.relu))
        if c.emit and c.twin:
            check_twin(env, t, c.twin)
    t.storage.copy_(xv)
    _call(env, br, lambda: fn(t.ptr, b.data_ptr(), c.rows, c.cols), c.emit)
    assert _same(y1, t.storage), tag + ": not reproducible"


@pytest.mark.parametrize("name", [c.name for c in BIAS_CASES])
def test_bias_branch(env, name):
    run_bias(env, BIAS_BY_NAME[name])


def run_grad(env, c, check=True):
    gen = _gen(c.name)
    n = c.rows * c.cols
    br = ex.bias_grad_branch(c.rows, c.cols, c.st, env.sms)
    assert br.name == c.branch, (c.name, br.name, c.branch)
    d, _ = _flat(n, c.off, guard=0)
    d.storage.copy_(_dyadic(n, gen) if c.dyadic else torch.randn(n, generator=gen, device="cuda"))
    gb, gbuf = _flat(c.cols, c.off)
    if c.st != 0.0:                                     # else the NaN prefill: the call must not read it
        gb.storage.copy_(_dyadic(c.cols, gen) if c.dyadic else torch.randn(c.cols, generator=gen, device="cuda"))
    b0 = gb.storage.clone()
    so = 0.5 if c.dyadic else 1.0 / 128
    tag = "%s %s" % (c.name, c.branch)
    fn = lambda: env.L.cnb_channel_bias_grad(d.ptr, gb.ptr, c.rows, c.cols, c.st, so)
    _call(env, br, fn)
    assert guards_ok(gbuf, c.off, c.cols), tag + ": wrote outside its target"
    g1 = gb.storage.clone()
    if check:
        _ok("bias_grad", c.branch, tag, gb.storage,
            ex.bias_grad(d.storage, c.rows, c.cols, b0, c.st, so, env.sms, exact_arm=c.dyadic))
    gb.storage.copy_(b0)
    _call(env, br, fn)
    assert _same(g1, gb.storage), tag + ": not reproducible"


@pytest.mark.parametrize("name", [c.name for c in GRAD_CASES])
def test_bias_grad_branch(env, name):
    run_grad(env, GRAD_BY_NAME[name])


# ---------------------------------------------------------------------------------------------------------------------
# batch normalisation: statistics, apply, backward
# ---------------------------------------------------------------------------------------------------------------------
def _bn_inputs(c, gen):
    N = c.n * c.C
    if c.kind == "dyadic" or c.kind == "grad_exact":
        x = _dyadic(N, gen)
    elif c.kind == "pm1":
        x = torch.ones(c.C, c.n, device="cuda")
        x[:, : c.n // 2] = -1
        x = x[:, torch.randperm(c.n, generator=gen, device="cuda")].reshape(-1).contiguous()
    else:
        x = torch.randn(N, generator=gen, device="cuda")
        if c.kind == "offset":
            x[: c.n] = 1e3 + 1e-2 * torch.randn(c.n, generator=gen, device="cuda")
    d = _dyadic(N, gen) if c.kind == "grad_exact" else torch.randn(N, generator=gen, device="cuda")
    return x, d


def run_bn(env, c, check=True):
    gen = _gen(c.name)
    L, n, C = env.L, c.n, c.C
    N = n * C
    ax, ay = c.off_x % 4 == 0, c.off_y % 4 == 0
    bs = ex.bn_stats_branch(n, C, ax, c.run, env.sms)
    ba = ex.bn_apply_branch(n, C, ax, ay, c.relu, env.sms)
    bb = ex.bn_backward_branch(n, C, ax, ay, c.train, env.sms)
    assert (bs.name, ba.name, bb.name) == (c.stats, c.apply, c.backward), (c.name, bs.name, ba.name, bb.name)
    xv, dv = _bn_inputs(c, gen)
    x, _ = _flat(N, c.off_x, guard=0)
    x.storage.copy_(xv)
    gamma = torch.rand(C, generator=gen, device="cuda") + 0.5
    beta = torch.randn(C, generator=gen, device="cuda")
    slices, vec_s = ex.bn_slices(n, C, env.sms), n % 4 == 0 and ax
    # statistics
    mu, mubuf = _flat(C, 0)
    sg, sgbuf = _flat(C, 0)
    rm = rs = None
    if c.run:
        rm, rs = torch.randn(C, generator=gen, device="cuda"), torch.rand(C, generator=gen, device="cuda") + 0.5
    rm0, rs0 = (rm.clone(), rs.clone()) if c.run else (None, None)
    fn = lambda: L.cnb_bn_stats(x.ptr, n, C, c.eps, c.f, mu.ptr, sg.ptr, rm.data_ptr() if c.run else None,
                                rs.data_ptr() if c.run else None)
    tag = "%s stats %s" % (c.name, c.stats)
    _call(env, bs, fn)
    assert guards_ok(mubuf, 0, C) and guards_ok(sgbuf, 0, C), tag + ": wrote outside mu / sigma"
    got = [t.clone() for t in (mu.storage, sg.storage) + ((rm, rs) if c.run else ())]
    if check:
        exact_mean = c.kind in ("dyadic", "pm1")
        _ok("bn_mean", c.stats, tag + " mu", mu.storage, ex.bn_mean(x.storage, n, C, slices, vec_s, exact_mean))
        _ok("bn_sigma", c.stats, tag + " sigma", sg.storage,
            ex.bn_sigma(x.storage, n, C, mu.storage, c.eps, slices, vec_s, exact_arm=c.kind == "pm1"))
        if c.run:
            _ok("bn_running", c.stats, tag + " run_mu", rm, ex.bn_running(rm0, mu.storage, c.f))
            _ok("bn_running", c.stats, tag + " run_sigma", rs, ex.bn_running(rs0, sg.storage, c.f))
    if c.run:
        rm.copy_(rm0); rs.copy_(rs0)
    _call(env, bs, fn)
    again = (mu.storage, sg.storage) + ((rm, rs) if c.run else ())
    assert all(_same(a, b) for a, b in zip(got, again)), tag + ": not reproducible"
    # the mu / sigma the transform uses: the batch's, the test mode's constants, or the caller's exact ones
    if c.kind == "grad_exact":
        use_mu, use_sg = _dyadic(C, gen), torch.full((C,), 2.0, device="cuda")
    elif c.train:
        use_mu, use_sg = mu.storage.clone(), sg.storage.clone()
    else:
        use_mu, use_sg = torch.randn(C, generator=gen, device="cuda"), torch.rand(C, generator=gen, device="cuda") + 0.5
    # apply
    y, ybuf = _flat(N, c.off_y, (c.twin[0], c.twin[1], c.twin[2], C) if c.twin else None)
    fn = lambda: L.cnb_bn_apply(x.ptr, y.ptr, n, C, gamma.data_ptr(), beta.data_ptr(), use_mu.data_ptr(),
                                use_sg.data_ptr(), c.relu)
    tag = "%s apply %s" % (c.name, c.apply)
    _call(env, ba, fn, c.emit)
    assert guards_ok(ybuf, c.off_y, N), tag + ": wrote outside y"
    y1 = y.storage.clone()
    if check:
        _ok("bn_apply", c.apply, tag, y.storage, ex.bn_apply(x.storage, n, C, gamma, beta, use_mu, use_sg, c.relu))
        if c.emit and c.twin:
            check_twin(env, y, (c.twin[0], c.twin[1], c.twin[2], C))
    y.storage.view(torch.int32).fill_(0x7FC0DEAD)
    _call(env, ba, fn, c.emit)
    assert _same(y1, y.storage), tag + ": not reproducible"
    # backward, in place on the derivative
    dm, dbuf = _flat(N, c.off_y, (c.twin[0], c.twin[1], c.twin[2], C) if c.twin else None)
    dm.storage.copy_(dv)
    gg, ggbuf = _flat(C, 0)
    gbt, gbbuf = _flat(C, 0)
    fn = lambda: L.cnb_bn_backward(dm.ptr, x.ptr, n, C, gamma.data_ptr(), use_mu.data_ptr(), use_sg.data_ptr(),
                                   c.train, gg.ptr, gbt.ptr)
    tag = "%s backward %s" % (c.name, c.backward)
    _call(env, bb, fn, c.emit)
    assert guards_ok(dbuf, c.off_y, N) and guards_ok(ggbuf, 0, C) and guards_ok(gbbuf, 0, C), tag + ": wrote outside"
    got = [t.clone() for t in (dm.storage, gg.storage, gbt.storage)]
    if check:
        vec_b = n % 4 == 0 and ax and ay
        egg, egb = ex.bn_grads(dv, x.storage, n, C, use_mu, use_sg, slices, vec_b, exact_arm=c.kind == "grad_exact")
        _ok("bn_grad_gamma", c.backward, tag + " grad_gamma", gg.storage, egg)
        _ok("bn_grad_beta", c.backward, tag + " grad_beta", gbt.storage, egb)
        _ok("bn_backward", c.backward, tag, dm.storage,
            ex.bn_backward(dv, x.storage, n, C, gamma, use_mu, use_sg, gg.storage, gbt.storage, c.train))
        if c.emit and c.twin:
            check_twin(env, dm, (c.twin[0], c.twin[1], c.twin[2], C))
    dm.storage.copy_(dv)
    _call(env, bb, fn, c.emit)
    assert all(_same(a, b) for a, b in zip(got, (dm.storage, gg.storage, gbt.storage))), tag + ": not reproducible"


@pytest.mark.parametrize("name", [c.name for c in BN_CASES])
def test_bn_branch(env, name):
    run_bn(env, BN_BY_NAME[name])


@pytest.mark.parametrize("layer", list(ALEX_BN))
def test_alexnet_bn(env, layer):
    run_bn(env, BN_BY_NAME["alex_" + layer])
    torch.cuda.empty_cache()


# ---------------------------------------------------------------------------------------------------------------------
# softmax, sum
# ---------------------------------------------------------------------------------------------------------------------
def _sm_inputs(c, gen):
    n = c.rows * c.cols
    x = torch.randn(c.cols, c.rows, generator=gen, device="cuda") * 3
    if c.kind == "scaled":
        x = x * 10 + 1e4
    elif c.kind == "tied" and c.cols > 1:
        x[c.cols - 1] = x.max(0).values
        x[c.cols // 2] = x[c.cols - 1]
    elif c.kind == "equal":
        x = torch.full_like(x, 3.75)
    elif c.kind == "onehot":
        hot = torch.randint(0, c.cols, (c.rows,), generator=gen, device="cuda")
        x[hot, torch.arange(c.rows, device="cuda")] = x.max(0).values + 200
    return x.reshape(-1)[:n].contiguous()


def run_sm(env, c, check=True):
    gen = _gen(c.name)
    br = ex.softmax_branch(c.rows, c.cols)
    assert br.name == c.branch, (c.name, br.name, c.branch)
    n = c.rows * c.cols
    xv = _sm_inputs(c, gen)
    t, tbuf = _flat(n, c.off)
    t.storage.copy_(xv)
    fn = lambda: env.L.cnb_softmax(t.ptr, c.rows, c.cols)
    tag = "%s %s" % (c.name, c.branch)
    _call(env, br, fn)
    assert guards_ok(tbuf, c.off, n), tag + ": wrote outside its target"
    y1 = t.storage.clone()
    if check:
        exact = c.kind if c.kind in ("equal", "onehot") else None
        _ok("softmax", c.branch, tag, t.storage, ex.softmax(xv, c.rows, c.cols, exact))
    t.storage.copy_(xv)
    _call(env, br, fn)
    assert _same(y1, t.storage), tag + ": not reproducible"


@pytest.mark.parametrize("name", [c.name for c in SM_CASES])
def test_softmax_branch(env, name):
    run_sm(env, SM_BY_NAME[name])


def run_sum(env, c, check=True):
    gen = _gen(c.name)
    br = ex.sum_branch(c.n)
    a, _ = _flat(c.n, c.off, guard=0)
    a.storage.copy_(_dyadic(c.n, gen) if c.dyadic else torch.randn(c.n, generator=gen, device="cuda"))
    out, obuf = _flat(1, 0)
    fn = lambda: env.L.cnb_sum(a.ptr, out.ptr, c.n)
    tag = "sum %s %s" % (c.name, c.branch)
    _call(env, br, fn)
    assert guards_ok(obuf, 0, 1), tag + ": wrote outside its target"
    s1 = out.storage.clone()
    if check:
        _ok("sum", c.branch, tag, out.storage, ex.sum_ref(a.storage, exact_arm=c.dyadic))
    out.storage.view(torch.int32).fill_(0x7FC0DEAD)
    _call(env, br, fn)
    assert _same(s1, out.storage), tag + ": not reproducible"


@pytest.mark.parametrize("name", [c.name for c in SUM_CASES])
def test_sum_branch(env, name):
    run_sum(env, SUM_BY_NAME[name])


# ---------------------------------------------------------------------------------------------------------------------
# which kernel ran: the names CUPTI records against the mirror
# ---------------------------------------------------------------------------------------------------------------------
def _lib_kernels(prof):
    from torch.autograd import DeviceType
    evs = [e for e in prof.events() if e.device_type == DeviceType.CUDA and "cnb::" in e.name and
           any(k + "<" in e.name or k + "(" in e.name for k in ex.KERNEL_NAMES)]
    evs.sort(key=lambda e: e.time_range.start)
    return [e.name for e in evs]


def profile_kernel_names(env):
    """every small case once more, unchecked, under torch.profiler: (kernel names CUPTI recorded, the mirror's names for
    each call, in call order)"""
    from torch.profiler import ProfilerActivity, profile
    global RECORD
    RECORD = []
    try:
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for c in EW_CASES:
                if c.n < (1 << 22):
                    run_ew(env, c, check=False)
            for c in BIAS_CASES:
                if c.rows * c.cols < (1 << 22):
                    run_bias(env, c, check=False)
            for c in GRAD_CASES:
                run_grad(env, c, check=False)
            for c in BN_CASES:
                if c.n * c.C < (1 << 22):
                    run_bn(env, c, check=False)
            for c in SM_CASES:
                run_sm(env, c, check=False)
            for c in SUM_CASES:
                run_sum(env, c, check=False)
            torch.cuda.synchronize()
        want = RECORD
    finally:
        RECORD = None
    return _lib_kernels(prof), want


def test_kernel_names():
    """the elementwise kernels CUPTI records must be, in order, the ones the mirror names for each call.  The profiler
    session runs in a process of its own (tests/elementwise_names_worker.py): a second torch.profiler session in one
    process can miss a kernel record, and test_gpu_pool_exact.py's own session runs later in this one"""
    r = subprocess.run([sys.executable, os.path.join(os.path.dirname(os.path.abspath(__file__)),
                                                     "elementwise_names_worker.py")],
                       capture_output=True, text=True, timeout=900)
    out = r.stdout.strip().splitlines()
    if out and out[-1] == "NAMES-NONE":
        pytest.skip("torch.profiler recorded no kernels of the library (CUPTI activity unavailable)")
    assert r.returncode == 0 and out and out[-1].startswith("NAMES-OK"), (r.returncode, r.stdout[-2000:],
                                                                         r.stderr[-3000:])
