"""The float64 references and bars of tests/pool_exact.py, checked on the CPU: they agree with the C oracle (pinned to the
reference's CPU library) and with the golden vectors within the bars, the bars reject simulated kernel faults, the bar
of the response norm's window sums is charged on the right mass (an fp32 emulation of the tile kernel on hot channels),
and every branch of the dispatch mirror is targeted by a case of tests/test_gpu_pool_exact.py."""
import itertools

import numpy as np
import pytest
import torch

import pool_exact as px
from cases import F, GOLDEN_2D, GOLDEN_3D, load_golden
from pool_exact import PG


def _t(a):
    """Fortran numpy matrix -> flat torch buffer in the library's (column-major) order"""
    return torch.from_numpy(np.asarray(a, dtype=np.float32).reshape(-1, order="F").copy())


def _ok(y, e, what):
    v = px.check(_t(y) if isinstance(y, np.ndarray) else y, e)
    assert v.ok, (what, str(v))
    return v


def _fails(y, e, what):
    v = px.check(_t(y) if isinstance(y, np.ndarray) else y, e)
    assert not v.ok, (what, "the fault passes the bar", str(v))


# ---------------------------------------------------------------------------------------------------------------------
# 1. the references against the oracle and the golden vectors
# ---------------------------------------------------------------------------------------------------------------------
POOL_CASES = {
    "k3s2p1": PG(6, 11, 9, 5, 3, 3, 2, 2, 1, 1),
    "k3s2p2": PG(4, 10, 11, 3, 3, 3, 2, 2, 2, 2),
    "rect": PG(5, 11, 9, 4, 2, 3, 1, 2, 0, 1),
    "stride_gt_k": PG(4, 11, 11, 3, 2, 2, 3, 3, 0, 0),
    "k5s3p2": PG(3, 13, 14, 2, 5, 5, 3, 3, 2, 2),
    "global": PG(4, 7, 6, 3, 6, 7, 1, 1, 0, 0),
    "pad_eq_k": PG(3, 6, 5, 2, 2, 2, 1, 1, 2, 2),
    "pad_gt_k": PG(3, 6, 5, 2, 2, 3, 1, 1, 3, 3),
    "3d": PG(3, 6, 7, 2, 2, 2, 1, 1, 0, 0, T=5, kt=2, st_t=2),
}


def _pool_operands(g, seed, dyadic=False):
    r = np.random.RandomState(seed)
    nin, nout = g.in_dims()[1], g.out_dims()[1]
    if dyadic:
        x = F(r.randint(-4, 5, (g.N, nin)) / 16.0)
        gr = F(r.randint(-8, 9, (g.N, nout)) / 16.0)
        t0 = F(r.randint(-8, 9, (g.N, nin)) / 16.0)
    else:
        x = F(np.round(r.randn(g.N, nin) * 2) / 2 + 0.0)    # ties (no -0: fmaxf may return either zero)
        gr = F(r.randn(g.N, nout))
        t0 = F(r.randn(g.N, nin))
    return x, gr, t0


@pytest.mark.parametrize("case", sorted(POOL_CASES))
def test_pool_reference_matches_oracle(oracle, case):
    g = POOL_CASES[case]
    x, gr, t0 = _pool_operands(g, 3)
    d, ish, osh = g.desc(), g.in_shape(), g.out_shape()
    for is_max in (True, False):
        for so in (1.0, 0.5):
            y = np.zeros(g.out_dims(), np.float32, order="F")
            oracle.pool(int(is_max), x, y, ish, osh, d, so)
            _ok(y, px.pool_fwd(g, _t(x), is_max, so), (case, is_max, so))
    acts = np.zeros(g.out_dims(), np.float32, order="F")
    oracle.pool(1, x, acts, ish, osh, d, 1.0)
    for st in (0.0, 0.5):
        y = t0.copy(order="F")
        oracle.maxPoolUndo(x, gr, acts, y, ish, osh, d, st)
        _ok(y, px.max_undo(g, _t(x), _t(gr), _t(acts), st, _t(t0)), (case, "max undo", st))
        y = t0.copy(order="F")
        oracle.avgPoolUndo(gr, y, osh, ish, d, st, 1.0 if st == 0.0 else 0.25)
        _ok(y, px.avg_undo(g, _t(gr), st, _t(t0), 1.0 if st == 0.0 else 0.25), (case, "avg undo", st))


def test_empty_windows_are_pinned(oracle):
    """padding >= kernel: the reference's average of an empty window is 0 / (product of clipped extents): NaN where an
    extent is 0, a signed zero where it is negative; its maximum is the base value"""
    g = POOL_CASES["pad_gt_k"]
    x, _, _ = _pool_operands(g, 4)
    y = np.zeros(g.out_dims(), np.float32, order="F")
    oracle.pool(0, x, y, g.in_shape(), g.out_shape(), g.desc(), 1.0)
    e = px.pool_fwd(g, _t(x), False)
    ref = e.ref.to(torch.float32)
    assert bool(torch.isnan(ref).any()) and bool(((ref == 0) & torch.signbit(ref)).any())
    _ok(y, e, "pinned empty windows")
    oracle.pool(1, x, y, g.in_shape(), g.out_shape(), g.desc(), 1.0)
    assert (y == np.float32(-2e38)).any()
    _ok(y, px.pool_fwd(g, _t(x), True), "empty max windows")


def test_exact_arm_matches_oracle(oracle):
    """dyadic operands: the oracle's max undo (sequential atomics order) equals float64 bit for bit"""
    g = POOL_CASES["k3s2p2"]
    x, gr, t0 = _pool_operands(g, 5, dyadic=True)
    d, ish, osh = g.desc(), g.in_shape(), g.out_shape()
    acts = np.zeros(g.out_dims(), np.float32, order="F")
    oracle.pool(1, x, acts, ish, osh, d, 1.0)
    y = t0.copy(order="F")
    oracle.maxPoolUndo(x, gr, acts, y, ish, osh, d, 1.0)
    _ok(y, px.max_undo(g, _t(x), _t(gr), _t(acts), 1.0, _t(t0), exact_arm=True), "exact arm")


RN_CASES = [(20, 5, False), (20, 6, True), (32, 4, False), (8, 12, False), (16, 1, False), (21, 4, True)]


@pytest.mark.parametrize("F_,k,blocked", RN_CASES)
def test_rnorm_reference_matches_oracle(oracle, F_, k, blocked):
    r = np.random.RandomState(F_ * 100 + k)
    N, locs = 8, 12
    x = F(r.randn(N, locs * F_))
    dy = F(r.randn(N, locs * F_))
    for alpha, beta in ((5e-4, 0.75), (0.01, 0.5)):
        y = np.zeros_like(x)
        oracle.rnorm(x, y, F_, k, alpha, beta, blocked)
        _ok(y, px.rnorm_fwd(_t(x), F_, k, alpha, beta, blocked), ("rnorm", F_, k, blocked))
        y = np.zeros_like(x)
        oracle.rnormUndo(dy, x, y, F_, k, alpha, beta, blocked)
        _ok(y, px.rnorm_undo(_t(dy), _t(x), F_, k, alpha, beta, blocked), ("rnorm undo", F_, k, blocked))


@pytest.mark.parametrize("name", GOLDEN_2D + GOLDEN_3D)
def test_reference_matches_golden(name):
    g = load_golden(name)
    three = g["kind"] == "3d"
    pg = PG(g["N"], g["W"], g["H"], g["Cin"], g["ky"], g["kx"], g["sy"], g["sx"], g["py"], g["px"],
            **(dict(T=g["T"], kt=g["kt"], st_t=g["st"], pt=g["pt"]) if three else {}))
    sfx = "3D" if three else ""
    x, gr = _t(g["pool_images"]), _t(g["pool_derivs"])
    _ok(g["maxPool" + sfx], px.pool_fwd(pg, x, True), name)
    _ok(g["avgPool" + sfx], px.pool_fwd(pg, x, False), name)
    _ok(g["maxPool%sUndo" % sfx], px.max_undo(pg, x, gr, _t(g["maxPool" + sfx])), name)
    _ok(g["avgPool%sUndo" % sfx], px.avg_undo(pg, gr), name)
    if three:
        return
    imgs, dv = _t(g["images"]), _t(g["rnorm_derivs"])
    for blocked in (False, True):
        tag = "_blocked" if blocked else ""
        _ok(g["rnorm" + tag], px.rnorm_fwd(imgs, g["Cin"], g["sizeF"], g["add_scale"], g["pow_scale"], blocked), name)
        _ok(g["rnormUndo" + tag], px.rnorm_undo(dv, imgs, g["Cin"], g["sizeF"], g["add_scale"], g["pow_scale"], blocked),
            name)


# ---------------------------------------------------------------------------------------------------------------------
# 2. controls: simulated faults fail the bar on the case inputs
# ---------------------------------------------------------------------------------------------------------------------
def test_control_pool_window_and_region(oracle):
    g = POOL_CASES["k3s2p1"]
    x, gr, _ = _pool_operands(g, 6)
    d, ish, osh = g.desc(), g.in_shape(), g.out_shape()
    y = np.zeros(g.out_dims(), np.float32, order="F")
    oracle.pool(1, x, y, ish, osh, d, 1.0)
    _fails(y, px.pool_fwd(g, _t(x), True, fault="shift"), "max window shifted by one")
    oracle.pool(0, x, y, ish, osh, d, 1.0)
    _fails(y, px.pool_fwd(g, _t(x), False, fault="shift"), "avg window shifted by one")
    _fails(y, px.pool_fwd(g, _t(x), False, fault="unclipped"), "unclipped region count")
    u = np.zeros(g.in_dims(), np.float32, order="F")
    oracle.avgPoolUndo(gr, u, osh, ish, d, 0.0, 1.0)
    _fails(u, px.avg_undo(g, _t(gr), fault="unclipped"), "unclipped region count (undo)")


def test_control_ties_and_mask_bits(oracle):
    g = POOL_CASES["k3s2p2"]
    x, gr, t0 = _pool_operands(g, 7, dyadic=True)
    d, ish, osh = g.desc(), g.in_shape(), g.out_shape()
    acts = np.zeros(g.out_dims(), np.float32, order="F")
    oracle.pool(1, x, acts, ish, osh, d, 1.0)
    y = np.zeros(g.in_dims(), np.float32, order="F")
    oracle.maxPoolUndo(x, gr, acts, y, ish, osh, d, 0.0)
    args = (g, _t(x), _t(gr), _t(acts))
    _ok(y, px.max_undo(*args, exact_arm=True), "correct")
    _fails(y, px.max_undo(*args, exact_arm=True, fault="no_dup"), "ties not duplicated")
    _fails(y, px.max_undo(*args, exact_arm=True, fault="drop_bit"), "tie-mask bit (dx, dy) = (2, 2) dropped")
    # the random arm sees the missing duplicates too
    _fails(y, px.max_undo(*args, fault="no_dup"), "ties not duplicated (random arm)")


def test_control_relu_mask_order():
    """the ReLU' mask zeroes the OLD target too: applying it before adding st * old fails"""
    g = POOL_CASES["k3s2p1"]
    x, gr, t0 = _pool_operands(g, 8, dyadic=True)
    acts = px.pool_fwd(g, _t(x), True).ref.to(torch.float32)
    mask = torch.randn(g.in_dims()[0] * g.in_dims()[1], generator=torch.Generator().manual_seed(1))
    right = px.max_undo(g, _t(x), _t(gr), acts, 1.0, _t(t0), mask=mask, exact_arm=True)
    y = right.ref.to(torch.float32)
    _ok(y, right, "correct")
    _fails(y, px.max_undo(g, _t(x), _t(gr), acts, 1.0, _t(t0), mask=mask, exact_arm=True, fault="mask_first"),
           "mask applied before scaleTargets")


@pytest.mark.parametrize("blocked", [False, True])
def test_control_rnorm_windows(oracle, blocked):
    F_, k = 24, 6                                   # even k: the forward and inverse windows differ
    r = np.random.RandomState(9)
    x, dy = F(r.randn(8, 10 * F_)), F(r.randn(8, 10 * F_))
    a, b = 0.01, 0.75
    y = np.zeros_like(x)
    oracle.rnorm(x, y, F_, k, a, b, blocked)
    if not blocked:                                 # (blocked: both windows are the block)
        _fails(y, px.rnorm_fwd(_t(x), F_, k, a, b, blocked, fault="window_swap"), "forward and inverse windows swapped")
    _fails(y, px.rnorm_fwd(_t(x), F_, k, a, b, blocked, fault="blocked_swap"), "blocked / unblocked confused")
    y16 = px.round_mantissa(_t(y).to(torch.float64), 16).to(torch.float32)
    _fails(y16, px.rnorm_fwd(_t(x), F_, k, a, b, blocked), "result through 16 mantissa bits")
    u = np.zeros_like(x)
    oracle.rnormUndo(dy, x, u, F_, k, a, b, blocked)
    if not blocked:
        _fails(u, px.rnorm_undo(_t(dy), _t(x), F_, k, a, b, blocked, fault="window_swap"), "undo windows swapped")
    _fails(u, px.rnorm_undo(_t(dy), _t(x), F_, k, a, b, blocked, fault="blocked_swap"), "undo blocked confused")
    u16 = px.round_mantissa(_t(u).to(torch.float64), 16).to(torch.float32)
    _fails(u16, px.rnorm_undo(_t(dy), _t(x), F_, k, a, b, blocked), "undo through 16 mantissa bits")


def test_control_bias_sum():
    """one row missing from the bias sum fails the exact arm; an fp32 sum of the same rows passes the random arm"""
    C, rows = 8, 5000
    gen = torch.Generator().manual_seed(2)
    y = (torch.randint(-8, 9, (C * rows,), generator=gen) / 16.0).to(torch.float32)
    b0 = (torch.randint(-8, 9, (C,), generator=gen) / 16.0).to(torch.float32)
    s = y.view(C, rows).sum(1)                      # fp32, exact on these operands
    got = (1.0 * b0 + 0.5 * s).to(torch.float32)
    _ok(got, px.bias_grad(y, rows, C, 1, b0, 1.0, 0.5, 20, 4, exact_arm=True), "exact arm")
    _fails(got, px.bias_grad(y, rows, C, 1, b0, 1.0, 0.5, 20, 4, exact_arm=True, fault="drop_row"), "row missing")
    yr = torch.randn(C * rows, generator=gen)
    got = (yr.view(C, rows).sum(1) / 128).to(torch.float32)
    _ok(got, px.bias_grad(yr, rows, C, 1, torch.zeros(C), 0.0, 1.0 / 128, 20, 4), "random arm")


def test_control_twin_rounding():
    y = torch.randn(4096, generator=torch.Generator().manual_seed(3))
    rne, tr = px.bf16_rne(y), px.bf16_trunc(y)
    # the bit-level restatement of round-to-nearest-even at 16 dropped bits
    b = y.view(torch.int32).to(torch.int64) & 0xFFFFFFFF
    r = ((b + 0x7FFF + ((b >> 16) & 1)) & ~0xFFFF) & 0xFFFFFFFF
    r = torch.where(r >= 2 ** 31, r - 2 ** 32, r).to(torch.int32).view(torch.float32)
    assert torch.equal(rne.view(torch.int32), r.view(torch.int32))
    assert float((rne.view(torch.int32) != tr.view(torch.int32)).float().mean()) > 0.3, "truncation not told apart"


# ---------------------------------------------------------------------------------------------------------------------
# 3. the window-sum bar: an fp32 emulation of the tile kernel's prefix sums (rn_prefix, rnorm_fwd_tile_kernel)
# ---------------------------------------------------------------------------------------------------------------------
def _tile_fwd_emulated(x, F_, k, alpha, beta, TL):
    """x: (F, L) float32.  The kernel's exclusive fp32 prefix of x^2 in 128/TL channel segments (segment totals, then the
    running prefix offset by the earlier totals), S = Q[hi] - Q[lo] in fp32; the power in float64 (the emulation
    isolates the summation)"""
    nseg = 128 // TL
    sq = (x * x).astype(np.float32)
    fs = -(-F_ // nseg)
    Q = np.zeros((F_ + 1, x.shape[1]), np.float32)
    tots = []
    for s in range(nseg):
        t = np.zeros(x.shape[1], np.float32)
        for f in range(min(F_, s * fs), min(F_, s * fs + fs)):
            t = (t + sq[f]).astype(np.float32)
        tots.append(t)
    for s in range(nseg):
        run = np.zeros(x.shape[1], np.float32)
        for q in range(s):
            run = (run + tots[q]).astype(np.float32)
        for f in range(min(F_, s * fs), min(F_, s * fs + fs)):
            Q[f] = run
            run = (run + sq[f]).astype(np.float32)
        if min(F_, s * fs + fs) == F_ and min(F_, s * fs) < F_:
            Q[F_] = run
    a, b = k // 2, k - k // 2 - 1
    j = np.arange(F_)
    lo, hi = np.maximum(0, j - a), np.minimum(F_, j + b + 1)
    S = (Q[hi] - Q[lo]).astype(np.float32)
    base = (np.float32(1) + np.float32(alpha) * S).astype(np.float32)
    return (x * np.power(base.astype(np.float64), -beta)).astype(np.float32)


@pytest.mark.parametrize("F_,k,hot,TL", [(96, 24, 30.0, 64), (256, 64, 30.0, 32), (256, 64, 300.0, 32)])
def test_window_sum_bar_is_charged_on_the_prefix(F_, k, hot, TL):
    assert px.pick_tile(F_, 2) == TL
    r = np.random.RandomState(10)
    x = np.maximum(r.randn(F_, 2048), 0).astype(np.float32)
    x[: F_ // 8] *= np.float32(hot)
    y = _tile_fwd_emulated(x, F_, k, 5e-4, 0.75, TL)
    xt, yt = torch.from_numpy(x.reshape(-1)), torch.from_numpy(y.reshape(-1))
    v = _ok(yt, px.rnorm_fwd(xt, F_, k, 5e-4, 0.75, False), "prefix bar")
    rel = float(((yt.double() - px.rnorm_fwd(xt, F_, k, 5e-4, 0.75, False).ref).abs()
                 / px.rnorm_fwd(xt, F_, k, 5e-4, 0.75, False).ref.abs().clamp(min=1e-30)).max())
    print("F=%d k=%d hot x%g: max rel err %.2e, worst |err|/bar %.3f" % (F_, k, hot, rel, v.worst))
    if hot >= 300:
        assert rel > 1e-4          # above the README's fp32 figure: the error class the bar has to carry
        _fails(yt, px.rnorm_fwd(xt, F_, k, 5e-4, 0.75, False, local_bar=True), "window-local bar")
        assert v.worst > 1e-2, "the prefix bar is loose on the case that needs it"


# ---------------------------------------------------------------------------------------------------------------------
# 4. coverage: every branch of the mirror has a GPU case, and each case is on the branch it claims
# ---------------------------------------------------------------------------------------------------------------------
def _pool_universe():
    """every branch name the mirror returns over a grid of small geometries (planes of one channel below 2^31 floats:
    the K2 / K3 generic forward and the Q1 / Q2 generic undo are only reached by larger planes, 8 GiB per channel)"""
    fwd, undo = set(), set()
    for k, s, p in itertools.product((1, 2, 3, 4, 5), (1, 2, 3), (0, 1, 2, 3)):
        for kx, ky, sx, sy in ((k, k, s, s), (k, max(1, k - 1), s, max(1, s - 1))):
            for N, al in ((32, True), (7, True), (32, False)):
                g = PG(N, 12, 11, 4, ky, kx, sy, sx, min(p, ky - 1 + 1), min(p, kx - 1 + 1))
                if g.modX < 1 or g.modY < 1:
                    continue
                for is_max, epi in ((True, False), (False, False), (False, True)):
                    fwd.add(px.pool_fwd_branch(g, is_max, al, epi=epi).name)
                    for mask, st, cached in itertools.product((None, "input", "other"), (0.0, 1.0), (False, True)):
                        undo.add(px.pool_undo_branch(g, is_max, al, mask, st, cached, epi=epi).name)
    for is_max in (True, False):
        for N, al in ((32, True), (7, True)):
            g = PG(N, 6, 7, 2, 2, 2, 1, 1, 0, 0, T=5, kt=2, st_t=2)
            fwd.add(px.pool_fwd_branch(g, is_max, al).name)
            undo.add(px.pool_undo_branch(g, is_max, al).name)
    return fwd, undo


def _rn_universe():
    fwd, undo = set(), set()
    Ls = (128, 175, 288, 34848, 270848)
    for L, F_, k, blocked, al in itertools.product(Ls, (8, 20, 256, 448, 896), (1, 5, 8, 96, 120, 400), (False, True),
                                                   (True, False)):
        fwd.add(px.rnorm_fwd_branch(L, F_, k, blocked, al).name.split("|")[0])
        undo.add(px.rnorm_undo_branch(L, F_, k, blocked, al).name.split("|")[0])
    return fwd, undo


def test_every_mirror_branch_has_a_case():
    import test_gpu_pool_exact as T
    fwd, undo = set(), set()
    for c in T.POOL_CASES:
        assert px.pool_fwd_branch(c.g, c.is_max, c.aligned, c.cache, c.so).name == c.fwd, c.name
        fwd.add(c.fwd)
        for i, u in enumerate(c.undos):
            b = px.pool_undo_branch(c.g, c.is_max, c.aligned, u.mask, u.st, c.cache and c.so == 1.0).name
            assert b == c.undo_branch(i), (c.name, i, b)
            undo.add(b)
    for c in T.EPI_CASES:                            # the epilogue instances of the average row kernels
        fwd.add(px.pool_fwd_branch(c.g, False, c.aligned, so=c.so, epi=True).name)
        undo.add(px.pool_undo_branch(c.g, False, c.aligned, st=1.0, epi=True).name)
    want_f, want_u = _pool_universe()
    assert not want_f - fwd, ("pool forward branches without a case", sorted(want_f - fwd))
    assert not want_u - undo, ("pool undo branches without a case", sorted(want_u - undo))
    rf, ru = set(), set()
    for c in T.RN_CASES:
        a = c.offset % 4 == 0
        assert px.rnorm_fwd_branch(c.L, c.F, c.k, c.blocked, a).name == c.fwd, c.name
        assert px.rnorm_undo_branch(c.L, c.F, c.k, c.blocked, a).name == c.undo, c.name
        rf.add(c.fwd)
        ru.add(c.undo)
    want_f, want_u = _rn_universe()
    base = lambda s: {n.split("|")[0] for n in s}
    assert not want_f - base(rf), ("rnorm forward branches without a case", sorted(want_f - base(rf)))
    assert not want_u - base(ru), ("rnorm undo branches without a case", sorted(want_u - base(ru)))
    for attr in ("partial", "seg"):                  # the partial last tile and channel segments, both directions
        assert any(attr in n for n in rf) and any(attr in n for n in ru), attr
    # the combinations the issue of the fused epilogues names
    assert any(c.relu and c.emit and px.rnorm_can_fuse(c.F) for c in T.RN_CASES)
    assert any(c.relu and c.emit and not px.rnorm_can_fuse(c.F) for c in T.RN_CASES)
    assert any(c.hot >= 300 for c in T.RN_CASES) and any(c.frames > 1 for c in T.RN_CASES)
    assert {c.abi for c in T.POOL_CASES} == {"gemm", "cc2"} and {c.abi for c in T.RN_CASES} == {"gemm", "cc2"}
    for p in (0, 1, 2):
        for cache in (False, True):
            assert any(c.g.px == p and c.cache == cache and "patch" in c.undo for c in T.POOL_CASES), (p, cache)
