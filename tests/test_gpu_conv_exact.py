"""The conv kernels element by element against float64 on their own rounded operands (tests/conv_exact.py), at every
dispatch branch of conv_tc.cu, on whole BASELINE-size outputs, on persistent grids smaller than the GPU, and inside
NaN guard zones.

Each branch case names the branch it targets and asserts the path the call took and the kernels it launched, with the
operands pre-staged in bf16 mode so that no conversion pass is counted.  The launch count tells the branch apart:
split-K and wgrad reduction splits add a reduction launch, dgrad in fprop form launches once per stride phase plus once
for the first build of its filter banks, 3-D dgrad once per output frame (frame windows stride_t frames apart, which
overlap when kt > stride_t and leave frames unread when kt < stride_t).  Every tensor-core case is also a control: the same
output must FAIL the bar against the wrong operand models of its precision (conv_exact.CONTROLS), or the case is too weak
to see a rounding fault.
"""
import math
import zlib

import pytest
import torch

import conv_exact as cx
from conv_exact import Geo

pytestmark = pytest.mark.gpu

SENTINEL = 0x7FC0DEAD      # NaN bits of the guard zones and of targets the call must not read
GUARD = 64                 # floats of guard zone after each target
OFFSETS = (32, 36)         # target offsets in floats: 128-byte aligned, and 16-byte but not 128-byte aligned
WORST = {}                 # (op, path precision) -> largest |err|/S seen, printed at the end of the module


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
    print("\nlargest |err|/S per (op, precision):")
    for k in sorted(WORST):
        print("  %-6s %-5s %.3e" % (k[0], k[1], WORST[k]))


@pytest.fixture(autouse=True)
def hygiene(env):
    prec = env.L.convnet_b200_get_conv_precision()
    try:
        yield
    finally:
        env.L.convnet_b200_reserve_sms(0)
        env.L.convnet_b200_set_conv_precision(prec)
        env.L.convnet_b200_bf16_invalidate(None)
        env.L.cnb_relu_deriv(None, None, 0)          # consumes any fuse request a failed call left pending


# ---------------------------------------------------------------------------------------------------------------------
# buffers
# ---------------------------------------------------------------------------------------------------------------------
def _matrix(rows, cols, s4, offset=0, guard=0):
    """CUDAMatrix at `offset` floats into a sentinel-filled buffer with `guard` floats after it"""
    from convnet_b200.matrix import CUDAMatrix
    n = rows * cols
    buf = torch.empty(offset + n + guard, dtype=torch.float32, device="cuda")
    buf.view(torch.int32).fill_(SENTINEL)
    return CUDAMatrix(rows, cols, s4, storage=buf[offset:offset + n]), buf


def _randn(rows, cols, s4, gen, scale=1.0, offset=0):
    m, _ = _matrix(rows, cols, s4, offset)
    m.storage.normal_(generator=gen)
    if scale != 1.0:
        m.storage.mul_(scale)
    return m


def _sentinel_ok(t):
    return bool((t.view(torch.int32) == SENTINEL).all())


# ---------------------------------------------------------------------------------------------------------------------
# dispatch mirrors (conv_tc.cu) the cases use to state which side of a choice they are on
# ---------------------------------------------------------------------------------------------------------------------
def _pick_bn(cols, granule):
    tiles = -(-cols // 128)
    bn = -(-(-(-cols // tiles)) // granule) * granule
    return min(128, max(granule, bn))


def wgrad_splits(g, bf16, sms):
    """the reduction split count tc_conv_outp_impl picks (its cost model, restated)"""
    Cin, frames = g.Cin * g.kt, g.modT
    x_mode = Cin < 8
    nbc = -(-g.N // (64 if bf16 else 32))
    m_tiles = -(-g.Cout // 128)
    if x_mode:
        x_ct = min(Cin, 128 // (8 * g.ky))
        n_tiles = -(-Cin // x_ct)
    else:
        n_tiles = -(-Cin // _pick_bn(Cin, 16))
    units = g.modY * frames
    base = (1 if x_mode else g.kx * g.ky) * m_tiles * n_tiles
    row_us = 0.3 * g.modX * max(1, nbc // 2)
    dw_bytes = 4.0 * g.Cout * g.K
    cap = max(1, min(units, (4 * sms) // max(base, 1)))
    best, splits = 1e30, 1
    for sp in range(1, cap + 1):
        ups = -(-units // sp)
        real = -(-units // ups)
        waves = -(-(base * real) // sms)
        cost = waves * (ups * row_us + 1.5) + (dw_bytes * (real + 1) / 3e6 if real > 1 else 0.0)
        if cost < best - 1e-9:
            best, splits = cost, real
    while splits > 1 and g.Cout * g.K * splits * 4 > (1 << 30):
        splits -= 1
    ups = -(-units // splits)
    return -(-units // ups)


# ---------------------------------------------------------------------------------------------------------------------
# one call, checked
# ---------------------------------------------------------------------------------------------------------------------
class Case:
    def __init__(self, name, op, geo, branch, modes, path=None, launches=None, st=0.0, so=1.0, fuse=None,
                 stage=True, a_offset=0, split=None):
        self.name, self.op, self.g, self.branch, self.modes = name, op, geo, branch, modes
        self.path = path or {}          # mode -> expected path (default: the mode's tensor-core path)
        self.launches = launches or {}  # mode -> expected launch count (wgrad: from its split count)
        self.st, self.so, self.fuse, self.stage, self.a_offset, self.split = st, so, fuse, stage, a_offset, split

    def expected_path(self, mode):
        return self.path.get(mode, {"fp32": "cuda-core-fp32", "tf32": "tc-tf32", "bf16": "tc-bf16"}[mode])


def run(env, c, mode, offset=OFFSETS[0], reserve=0, controls=True):
    """run case `c` in `mode` and check it; returns (copy of the output, launches, path, target matrix)"""
    g, op = c.g, c.op
    env.lib.set_precision(mode)
    # fresh tensors may reuse a freed address: forget every staged copy and filter bank of the previous run
    env.L.convnet_b200_bf16_invalidate(None)
    gen = torch.Generator(device="cuda").manual_seed(zlib.crc32(c.name.encode()))
    img = _randn(*g.img_dims(), g.img_shape(), gen, offset=c.a_offset)
    flt = _randn(*g.flt_dims(), g.flt_shape(), gen, scale=1.0 / math.sqrt(g.K))
    der = _randn(*g.out_dims(), g.out_shape(), gen)
    a, b = {"fprop": (img, flt), "dgrad": (der, flt), "wgrad": (img, der)}[op]
    tdims, tshape = {"fprop": (g.out_dims(), g.out_shape()), "dgrad": (g.img_dims(), g.img_shape()),
                     "wgrad": (g.flt_dims(), g.flt_shape())}[op]
    out, buf = _matrix(*tdims, tshape, offset, GUARD)
    if c.st != 0.0:                 # else the target keeps its NaN prefill: the call must not read it
        out.storage.normal_(generator=gen)
    t0 = out.storage.clone()
    L = env.L
    fuse = c.fuse or {}
    bias = torch.randn(g.Cout, generator=gen, device="cuda") if "bias" in fuse else None
    mask = torch.randn(tdims[0] * tdims[1], generator=gen, device="cuda") if "mask" in fuse else None
    if mode == "bf16" and c.stage:
        for m in (a, b):
            L.convnet_b200_bf16_stage(m.ptr, m.rows * m.cols)
    L.convnet_b200_reserve_sms(reserve)
    L.convnet_b200_reset_launch_count()
    if bias is not None or "relu" in fuse or mask is not None:
        L.convnet_b200_fuse_next(bias.data_ptr() if bias is not None else None, int("relu" in fuse),
                                 mask.data_ptr() if mask is not None else None)
    if "drop" in fuse:
        L.convnet_b200_fuse_next_dropout(*fuse["drop"])
    if "emit" in fuse:
        L.convnet_b200_emit_bf16_next()
    d = g.desc()
    cg = env.cg
    three_d = g.T > 1 or g.kt > 1
    if op == "fprop":
        (cg.convUp3D if three_d else cg.convUp)(img, flt, out, d, c.st)
    elif op == "dgrad":
        (cg.convDown3D if three_d else cg.convDown)(der, flt, out, d, c.st)
    else:
        (cg.convOutp3D if three_d else cg.convOutp)(img, der, out, d, c.st, c.so)
    launches = int(L.convnet_b200_launch_count())
    path = env.lib.last_conv_path()
    L.convnet_b200_reserve_sms(0)
    torch.cuda.synchronize()
    n = tdims[0] * tdims[1]
    y = out.storage
    tag = "%s[%s] %s" % (c.name, mode, c.branch)
    assert _sentinel_ok(buf[:offset]) and _sentinel_ok(buf[offset + n:]), tag + ": wrote outside its target"
    kw = dict(t0=t0, st=c.st, so=c.so, bias=bias, relu="relu" in fuse, mask=mask, drop=fuse.get("drop"))
    kind = cx.PATH_MODEL[path]
    v = cx.check(op, g, y, cx.expect(op, g, a.storage, b.storage, kind, **kw), t0=t0)
    key = (op, kind)
    WORST[key] = max(WORST.get(key, 0.0), v.worst_ratio)
    print("%-40s path=%-14s launches=%-3d %s" % (tag, path, launches, v))
    assert v.ok, "%s path=%s: %s" % (tag, path, v)
    if controls:
        for wrong in cx.CONTROLS[kind]:
            w = cx.check(op, g, y, cx.expect(op, g, a.storage, b.storage, wrong, **kw), t0=t0)
            assert not w.ok, "%s: the output also passes against the wrong operand model %s (%s): case too weak" % (
                tag, wrong, w)
    return y.clone(), launches, path, out


# ---------------------------------------------------------------------------------------------------------------------
# the branch table
# ---------------------------------------------------------------------------------------------------------------------
TC = ("tf32", "bf16")
DROP = (0.25, 1.0 / 0.75, 987654321)


CASES = [
    # ---- fprop
    Case("fp_n128_cout64", "fprop", Geo(128, 8, 8, 64, 64, 3, 3, 1, 1, 1, 1),
         "N%128==0: merged A; Cout%chunk==0: merged B", TC, launches={"tf32": 1, "bf16": 1}),
    Case("fp_n64_cout72", "fprop", Geo(64, 7, 7, 32, 72, 3, 3, 1, 1, 1, 1),
         "N=64: unmerged A; Cout 72: unmerged B", TC, launches={"tf32": 1, "bf16": 1}),
    Case("fp_n96_cout40_cin72", "fprop", Geo(96, 6, 6, 72, 40, 3, 3, 1, 1, 1, 1),
         "ragged channel block (Cin 72), Cout 40, N 96", TC, launches={"tf32": 1, "bf16": 1}),
    Case("fp_rect", "fprop", Geo(32, 13, 9, 16, 24, 3, 5, 1, 2, 2, 1),
         "W!=H, kx!=ky, sx!=sy, px!=py", TC, launches={"tf32": 1, "bf16": 1}),
    Case("fp_pad_ge_kernel", "fprop", Geo(32, 6, 5, 16, 16, 2, 3, 1, 1, 3, 3),
         "padding >= kernel: windows wholly in padding", TC, launches={"tf32": 1, "bf16": 1}),
    Case("fp_fc_splitk", "fprop", Geo(128, 1, 1, 2048, 512, 1, 1),
         "FC: split-K + reduce_split", TC, launches={"tf32": 2, "bf16": 2}),
    Case("fp_fc_small_staged", "fprop", Geo(64, 1, 1, 512, 256, 1, 1),
         "FC, < 1024 rows, staged weights: bf16, split-K", TC, launches={"tf32": 2, "bf16": 2}),
    Case("fp_fc_small_unstaged", "fprop", Geo(64, 1, 1, 512, 256, 1, 1),
         "FC, < 1024 rows, weights not staged: tf32", ("bf16",), path={"bf16": "tc-tf32"}, launches={"bf16": 2},
         stage=False),
    Case("fp_x_cin3_k7_merged", "fprop", Geo(128, 29, 29, 3, 96, 7, 7, 2, 2, 1, 1),
         "x-mode Cin 3, ky 7 (two y-blocks), merged A and B", TC, path={"bf16": "tc-tf32"},
         launches={"tf32": 1, "bf16": 1}),
    Case("fp_x_cin1_k8x5", "fprop", Geo(64, 20, 20, 1, 40, 5, 8, 1, 1, 0, 0),
         "x-mode Cin 1, kx 8, ky 5 (two y-blocks), unmerged A and B", ("tf32",), launches={"tf32": 1}),
    Case("fp_x_cin7_k4x8", "fprop", Geo(96, 12, 14, 7, 64, 8, 4, 1, 2, 2, 1),
         "x-mode Cin 7, ky 8, unmerged A, merged B", ("tf32",), launches={"tf32": 1}),
    Case("fp_epilogue", "fprop", Geo(128, 8, 8, 32, 64, 3, 3, 1, 1, 1, 1),
         "bias + ReLU + dropout + bf16 twin in the epilogue", TC, launches={"tf32": 1, "bf16": 1},
         fuse={"bias": 1, "relu": 1, "drop": DROP, "emit": 1}),
    Case("fp_bf16_n36", "fprop", Geo(36, 8, 8, 16, 16, 3, 3, 1, 1, 1, 1),
         "N%8!=0 in bf16 mode: tf32", ("bf16",), path={"bf16": "tc-tf32"}, launches={"bf16": 1}),
    Case("fp_3d_cin9", "fprop", Geo(32, 10, 10, 3, 16, 3, 3, 1, 1, 1, 1, T=5, kt=3),
         "3-D: Cin 9 folded from 3 x kt 3, 3 frames", TC, launches={"tf32": 1, "bf16": 1}),
    Case("fp_3d_st2_kt3", "fprop", Geo(32, 8, 8, 4, 16, 3, 3, 1, 1, 1, 1, T=7, kt=3, st_t=2),
         "3-D, stride_t 2 < kt 3: 3 overlapping frame windows", TC, launches={"tf32": 1, "bf16": 1}),
    Case("fp_3d_st2_kt1", "fprop", Geo(32, 8, 8, 8, 16, 3, 3, 1, 1, 1, 1, T=7, kt=1, st_t=2),
         "3-D, kt 1 < stride_t 2: frames 1, 3, 5 read by no window", TC, launches={"tf32": 1, "bf16": 1}),
    Case("fp_subrange", "fprop", Geo(32, 8, 8, 32, 32, 3, 3, 1, 1, 1, 1, cin0=16, CinT=48, cout0=16, CoutT=64),
         "channel sub-ranges, scaleTargets 0.5", TC, launches={"tf32": 1, "bf16": 1}, st=0.5),
    Case("fp_unaligned_operand", "fprop", Geo(32, 8, 8, 16, 16, 3, 3, 1, 1, 1, 1),
         "images 4 bytes off 16-byte alignment: CUDA cores", TC, path={"tf32": "cuda-core-fp32",
                                                                        "bf16": "cuda-core-fp32"}, a_offset=1),
    # ---- dgrad
    Case("dg_fpform_s1", "dgrad", Geo(128, 8, 8, 32, 64, 3, 3, 1, 1, 1, 1),
         "fprop form, stride 1 (1 phase) / tf32 gather, merged", TC, launches={"tf32": 1, "bf16": 2}),
    Case("dg_fpform_s2_odd", "dgrad", Geo(128, 9, 9, 32, 32, 3, 3, 2, 2, 1, 1),
         "fprop form, stride 2 on odd size (phases of unequal size)", ("bf16",), launches={"bf16": 5}),
    Case("dg_fpform_s2_even_rect", "dgrad", Geo(128, 10, 8, 32, 16, 4, 3, 1, 2, 1, 0),
         "fprop form, sx 2 / sy 1 on even size", ("bf16",), launches={"bf16": 3}),
] + [
    Case("dg_fpform_s3_k5_p%d" % p, "dgrad", Geo(128, 11, 11, 32, 16, 5, 5, 3, 3, p, p),
         "fprop form, stride 3, kernel 5, padding %d" % p, ("bf16",), launches={"bf16": 10})
    for p in range(5)
] + [
    Case("dg_fpform_s3_k7_p%d" % p, "dgrad", Geo(128, 10, 10, 32, 16, 7, 7, 3, 3, p, p),
         "fprop form, stride 3, kernel 7, padding %d" % p, ("bf16",), launches={"bf16": 10})
    for p in (0, 3, 6)
] + [
    Case("dg_gather_st", "dgrad", Geo(128, 8, 8, 32, 64, 3, 3, 1, 1, 1, 1),
         "scaleTargets 0.5: gather form", TC, launches={"tf32": 1, "bf16": 1}, st=0.5),
    Case("dg_gather_k1_s2", "dgrad", Geo(128, 9, 9, 32, 32, 1, 1, 2, 2, 0, 0),
         "kernel 1 < stride 2: gather form, pixels no tap reaches", TC, launches={"tf32": 1, "bf16": 1}),
    Case("dg_n160", "dgrad", Geo(160, 7, 7, 16, 24, 3, 3, 1, 1, 1, 1),
         "N 160: the chunks of a tile on different pixels", TC, launches={"tf32": 1, "bf16": 1}),
    Case("dg_fc_splitk_mask", "dgrad", Geo(128, 1, 1, 1024, 2048, 1, 1),
         "FC: split-K with the ReLU' mask in reduce_split", TC, launches={"tf32": 2, "bf16": 2},
         fuse={"mask": 1}),
    Case("dg_mask", "dgrad", Geo(128, 8, 8, 32, 64, 3, 3, 1, 1, 1, 1),
         "ReLU' mask in the epilogue (fprop form / gather)", TC, launches={"tf32": 1, "bf16": 2},
         fuse={"mask": 1}),
] + [
    Case("dg_3d_st%s" % st, "dgrad", Geo(32, 8, 8, 4, 16, 3, 3, 1, 1, 1, 1, T=6, kt=3),
         "3-D, overlapping frame windows, scaleTargets %s: one launch per frame" % st, TC,
         launches={m: 4 + (st not in (0.0, 1.0)) for m in TC}, st=st)
    for st in (0.0, 0.5, 1.0)
] + [
    Case("dg_3d_st2_kt%d" % kt, "dgrad", Geo(32, 8, 8, cin, 16, 3, 3, 1, 1, 1, 1, T=T, kt=kt, st_t=2),
         "3-D, stride_t 2, kt %d (%s): one launch per output frame" % (kt, why), TC,
         launches={m: (T - kt) // 2 + 1 for m in TC})
    for kt, cin, T, why in ((3, 4, 7, "windows overlap on every second frame"), (2, 4, 8, "windows tile the frames"),
                            (1, 8, 7, "frames 1, 3, 5 read by no window: exactly 0"))
] + [
    Case("dg_subrange", "dgrad", Geo(32, 8, 8, 32, 32, 3, 3, 1, 1, 1, 1, cin0=16, CinT=48, cout0=8, CoutT=48),
         "channel sub-ranges, scaleTargets 1", TC, launches={"tf32": 1, "bf16": 1}, st=1.0),
    # ---- wgrad
    Case("wg_conv", "wgrad", Geo(32, 14, 14, 64, 64, 3, 3, 1, 1, 1, 1),
         "reduction splits > 1", TC, split=True),
    Case("wg_one_row", "wgrad", Geo(128, 16, 3, 64, 64, 3, 3, 1, 1, 0, 0),
         "one module row: reduction splits == 1", TC, split=False),
    Case("wg_dead_taps", "wgrad", Geo(256, 2, 2, 16, 16, 5, 5, 3, 3, 3, 3),
         "taps that land in no module: zero k-block group", TC),
    Case("wg_x_2tiles", "wgrad", Geo(32, 20, 20, 3, 32, 7, 7, 2, 2, 1, 1),
         "x-mode, ky 7: two channels per tile, two tiles", TC, path={"bf16": "tc-tf32"}),
    Case("wg_3d", "wgrad", Geo(32, 6, 6, 8, 16, 3, 3, 1, 1, 1, 1, T=5, kt=2),
         "3-D, 4 frames", TC),
    Case("wg_3d_st2_kt3", "wgrad", Geo(32, 8, 8, 4, 16, 3, 3, 1, 1, 1, 1, T=7, kt=3, st_t=2),
         "3-D, stride_t 2 < kt 3: 3 overlapping frame windows", TC),
    Case("wg_3d_st2_kt2", "wgrad", Geo(32, 8, 8, 8, 16, 3, 3, 1, 1, 1, 1, T=8, kt=2, st_t=2),
         "3-D, kt == stride_t 2: 4 frame windows that tile the frames", TC),
    Case("wg_st_so", "wgrad", Geo(32, 8, 8, 32, 32, 3, 3, 1, 1, 1, 1),
         "scaleTargets 0.5, scaleOutput 0.25", TC, st=0.5, so=0.25),
    Case("wg_fc_bf16", "wgrad", Geo(128, 1, 1, 512, 256, 1, 1),
         "FC, N%128==0 and Cin%32==0: bf16", TC, split=False),
    Case("wg_fc_declined", "wgrad", Geo(64, 1, 1, 512, 256, 1, 1),
         "FC with N 64 in bf16 mode: tf32", ("bf16",), path={"bf16": "tc-tf32"}, split=False),
    Case("wg_subrange", "wgrad", Geo(32, 8, 8, 32, 32, 3, 3, 1, 1, 1, 1, cin0=16, CinT=48, cout0=8, CoutT=48),
         "channel sub-ranges", TC),
]
BY_NAME = {c.name: c for c in CASES}
PARAMS = [(c.name, m) for c in CASES for m in c.modes + ("fp32",)]


@pytest.mark.parametrize("name,mode", PARAMS)
def test_branch(env, name, mode):
    c = BY_NAME[name]
    offset = OFFSETS[zlib.crc32(name.encode()) % 2]
    y, launches, path, out = run(env, c, mode, offset=offset, controls=True)
    assert path == c.expected_path(mode), (name, mode, path)
    if mode == "fp32":
        return
    want = c.launches.get(mode)
    if c.op == "wgrad":
        splits = wgrad_splits(c.g, path == "tc-bf16", env.sms)
        if c.split is not None:
            assert (splits > 1) == c.split, (name, mode, splits)
        want = 1 + (splits > 1)         # the tile kernel, + the partial-sum reduction
    if want is not None:
        assert launches == want, (name, mode, "launches", launches, want)
    if c.fuse and "emit" in c.fuse and mode == "bf16":
        _check_twin(env, c, out)


def _check_twin(env, c, out):
    """the bf16 twin the epilogue wrote is what a bf16 conv reading the output uses: it must be the round-to-nearest
    copy of the fp32 output (a consumer with a staged operand launches no conversion)"""
    L = env.L
    n = out.rows * out.cols
    assert L.convnet_b200_bf16_is_staged(out.ptr, n) == 1
    g = c.g
    g2 = Geo(g.N, g.modX, g.modY, g.Cout, 32, 3, 3, 1, 1, 1, 1)
    gen = torch.Generator(device="cuda").manual_seed(5)
    flt = _randn(*g2.flt_dims(), g2.flt_shape(), gen, scale=1.0 / math.sqrt(g2.K))
    L.convnet_b200_bf16_stage(flt.ptr, flt.rows * flt.cols)
    res, _ = _matrix(*g2.out_dims(), g2.out_shape())
    L.convnet_b200_reset_launch_count()
    env.cg.convUp(out, flt, res, g2.desc())
    assert int(L.convnet_b200_launch_count()) == 1 and env.lib.last_conv_path() == "tc-bf16"
    torch.cuda.synchronize()
    v = cx.check("fprop", g2, res.storage, cx.expect("fprop", g2, out.storage, flt.storage, "bf16"))
    assert v.ok, "consumer of the bf16 twin: %s" % v


# ---------------------------------------------------------------------------------------------------------------------
# persistent grids smaller than the GPU: the multi-tile walk and the ring-phase wrap
# ---------------------------------------------------------------------------------------------------------------------
SMALL_GRID = [("dg_gather_k1_s2", "bf16"), ("dg_gather_k1_s2", "tf32"), ("wg_dead_taps", "tf32"),
              ("wg_dead_taps", "bf16"), ("fp_x_cin3_k7_merged", "tf32"), ("dg_fpform_s2_odd", "bf16"),
              ("fp_3d_st2_kt3", "bf16"), ("dg_3d_st2_kt3", "tf32"), ("dg_3d_st2_kt1", "bf16"), ("wg_3d_st2_kt3", "bf16")]


@pytest.mark.parametrize("name,mode", SMALL_GRID)
def test_small_grid(env, name, mode):
    c = BY_NAME[name]
    full, l_full, p_full, _ = run(env, c, mode, controls=False)
    for reserve in (env.sms - 8, 16):
        y, launches, path, _ = run(env, c, mode, reserve=reserve, controls=False)
        assert path == p_full
        usable = env.sms - reserve
        same_split = (wgrad_splits(c.g, path == "tc-bf16", usable) == wgrad_splits(c.g, path == "tc-bf16", env.sms)
                      if c.op == "wgrad" else launches == l_full)
        if same_split:
            assert torch.equal(y.view(torch.int32), full.view(torch.int32)), (name, mode, reserve)


# ---------------------------------------------------------------------------------------------------------------------
# whole outputs at BASELINE size: every conv, 1x1 and FC layer of net A at batch 128, every element
# ---------------------------------------------------------------------------------------------------------------------
ALEX_CONV = {
    # name: W, H, Cin, Cout, ky, kx, sy, sx, py, px        (test_gpu_vs_reference_cuda.py)
    "conv1": (224, 224, 3, 96, 7, 7, 2, 2, 1, 1),
    "conv2": (55, 55, 96, 256, 5, 5, 2, 2, 1, 1),
    "nin2_1": (27, 27, 256, 256, 1, 1, 1, 1, 0, 0),
    "conv3": (14, 14, 256, 384, 3, 3, 1, 1, 1, 1),
    "nin3_1": (14, 14, 384, 768, 1, 1, 1, 1, 0, 0),
    "conv4": (14, 14, 768, 384, 3, 3, 1, 1, 1, 1),
    "nin4_1": (14, 14, 384, 768, 1, 1, 1, 1, 0, 0),
    "nin4_2": (14, 14, 768, 384, 1, 1, 1, 1, 0, 0),
    "conv5": (14, 14, 384, 512, 3, 3, 1, 1, 0, 0),
    "nin5_1": (12, 12, 512, 1024, 1, 1, 1, 1, 0, 0),
    "nin5_2": (12, 12, 1024, 512, 1, 1, 1, 1, 0, 0),
    "fc6": (1, 1, 18432, 4096, 1, 1, 1, 1, 0, 0),
    "fc7": (1, 1, 4096, 4096, 1, 1, 1, 1, 0, 0),
    "fc8": (1, 1, 4096, 1000, 1, 1, 1, 1, 0, 0),
}


@pytest.mark.parametrize("mode", ["fp32", "tf32", "bf16"])
@pytest.mark.parametrize("op", ["fprop", "dgrad", "wgrad"])
@pytest.mark.parametrize("layer", list(ALEX_CONV))
def test_alexnet_whole_output(env, layer, op, mode):
    W, H, Cin, Cout, ky, kx, sy, sx, py, px = ALEX_CONV[layer]
    c = Case("alex_%s_%s" % (layer, op), op, Geo(128, W, H, Cin, Cout, ky, kx, sy, sx, py, px), "BASELINE", (mode,),
             stage=False, so=1.0 / 128 if op == "wgrad" else 1.0)
    run(env, c, mode, controls=False)
