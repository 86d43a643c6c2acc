"""The references and bars of tests/elementwise_exact.py without a GPU: against the reference's CPU library (through
tests/golden/ref_elementwise.npz), against fp32 emulations of the kernels' summation orders (the bars must accept
them), against simulated faults (the bars must reject them), and the GPU case tables against the dispatch mirror."""
import itertools
import os

import numpy as np
import torch

import elementwise_exact as ex

U = ex.U
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_elementwise.npz")


def _ok(y, e, what):
    v = ex.check(y, e)
    assert v.ok, "%s: %s" % (what, v)
    return v


def _fails(y, e, what):
    v = ex.check(y, e)
    assert not v.ok, "%s: the fault passes (%s)" % (what, v)


def _t(a):
    return torch.from_numpy(np.ascontiguousarray(a))


def _colmajor(a):
    """a Fortran [rows x cols] array as the flat column-major fp32 tensor the kernels see"""
    return _t(np.asarray(a, np.float32).T.reshape(-1))


# ---------------------------------------------------------------------------------------------------------------------
# the reference's CPU library
# ---------------------------------------------------------------------------------------------------------------------
def test_kernels_against_the_reference_goldens():
    z = np.load(GOLDEN)
    # ReLU: lower_bound_scalar is the same fmax, bit for bit (zeros by value)
    _ok(_colmajor(z["relu_y"]), ex.relu(_colmajor(z["relu_x"])), "relu")
    # softmax: the reference sums the classes in order (depth cols), exp within 1 ulp; each side within its bar
    rows, cols = z["sm_x"].shape
    x = _colmajor(z["sm_x"])
    e = ex.softmax(x, rows, cols)
    X = x.to(torch.float64).view(cols, rows)
    dj = 2 * U + (X - X.max(0).values).abs() * U
    theirs = (1 + 2.0 ** -10) * (dj + dj.max(0).values + (cols + 2) * U) * e.ref.view(cols, rows) + 2.0 ** -146
    _ok(_colmajor(z["sm_p"]), ex.Expect(e.ref, e.bar + theirs.reshape(-1), e.exact), "softmax")
    # the equal-logit and one-hot images are exact on both sides
    p = z["sm_p"]
    assert (p[1] == np.float32(1) / np.float32(cols)).all() and (p[2] == (np.arange(cols) == 7)).all()
    # batch norm: ragged n, a channel at mean 1e3 / sd 1e-2.  The reference's sums run in order (depth n)
    n, C = z["bn_x"].shape
    bx, d = _colmajor(z["bn_x"]), _colmajor(z["bn_d"])
    gamma, beta, mu, sigma = (_t(z[k]) for k in ("bn_gamma", "bn_beta", "bn_mu", "bn_sigma"))
    eps = float(z["bn_eps"])
    slices = ex.bn_slices(n, C)
    em = ex.bn_mean(bx, n, C, slices, False)
    _ok(mu, ex.Expect(em.ref, em.bar + (n + 2) * U * bx.double().view(C, n).abs().sum(1) / n, em.exact), "bn mean")
    es = ex.bn_sigma(bx, n, C, mu, eps, slices, False)
    _ok(sigma, ex.Expect(es.ref, es.bar + ((n + 6) / 2 + 1) * U * es.ref, es.exact), "bn sigma")
    # y given the reference's own mu, sigma: ours is exact given them, theirs four roundings
    X = bx.double().view(C, n)
    xh = (X - mu.double().view(C, 1)) / sigma.double().view(C, 1)
    yref = xh * gamma.double().view(C, 1) + beta.double().view(C, 1)
    ybar = 4 * U * (xh * gamma.double().view(C, 1)).abs() + U * yref.abs()
    _ok(_colmajor(z["bn_y"]), ex.Expect(yref.reshape(-1), ybar.reshape(-1), torch.zeros(n * C, dtype=torch.bool)),
        "bn y")
    ours = ex.bn_apply(bx, n, C, gamma, beta, mu, sigma)
    _ok(_colmajor(z["bn_y"]), ex.Expect(ours.ref, ybar.reshape(-1) + 2 * U * yref.abs().reshape(-1),
                                        torch.zeros(n * C, dtype=torch.bool)), "bn y, our restatement")
    # the gradient means and dx
    egg, egb = ex.bn_grads(d, bx, n, C, mu, sigma, slices, False)
    D = d.double().view(C, n)
    _ok(_t(z["bn_grad_beta"]), ex.Expect(egb.ref, egb.bar + (n + 2) * U * D.abs().sum(1) / n, egb.exact), "grad beta")
    _ok(_t(z["bn_grad_gamma"]), ex.Expect(egg.ref, egg.bar + (n + 6) * U * (D * xh).abs().sum(1) / n, egg.exact),
        "grad gamma")
    gg, gb = egg.ref, egb.ref
    a = gamma.double().view(C, 1) / sigma.double().view(C, 1)
    dref = a * (D - gb.view(C, 1) - xh * gg.view(C, 1))
    # the reference subtracts mean(d - gg xhat) for gb, = gb - gg mean(xhat): charged with the whole mean of |xhat|
    dbar = a.abs() * (8 * U * (D.abs() + gb.abs().view(C, 1) + (xh * gg.view(C, 1)).abs())
                      + gg.abs().view(C, 1) * ((n + 8) * U * xh.abs().mean(1, keepdim=True) + xh.mean(1, keepdim=True).abs()))
    _ok(_colmajor(z["bn_dx"]), ex.Expect(dref.reshape(-1), dbar.reshape(-1), torch.zeros(n * C, dtype=torch.bool)),
        "bn dx")
    bk = ex.bn_backward(d, bx, n, C, gamma, mu, sigma, gg.float(), gb.float(), 1)
    _ok(bk.ref.float(), ex.Expect(dref.reshape(-1), dbar.reshape(-1), torch.zeros(n * C, dtype=torch.bool)),
        "bn dx, our restatement")


# ---------------------------------------------------------------------------------------------------------------------
# fp32 emulations of the correct kernels pass the bars
# ---------------------------------------------------------------------------------------------------------------------
def test_fma32_rounds_once():
    a = torch.tensor([1 + 2.0 ** -12, 3.0, 1.0], dtype=torch.float32)
    b = torch.tensor([1 + 2.0 ** -12, 1 / 3.0, 2.0 ** -30], dtype=torch.float32)
    c = torch.tensor([-1.0, -1.0, 1.0], dtype=torch.float32)
    got = ex.fma32(a, b, c)
    assert got[0] == 2.0 ** -11 + 2.0 ** -24                         # the product's low bits survive
    assert got[1] == float(np.float32(float(np.float32(3.0)) * float(np.float32(1 / 3.0)) - 1))
    assert got[2] == 1.0
    # a float64 midpoint between two fp32 numbers is rounded by the TwoSum error
    m = torch.tensor([1 + 2.0 ** -24], dtype=torch.float32)            # not representable: rounds to 1
    assert ex.fma32(torch.tensor([1.0]), torch.tensor([1.0]), torch.tensor([2.0 ** -24])) == 1.0
    t = ex.fma32(torch.tensor([1 + 2.0 ** -23]), torch.tensor([2.0 ** -24]), torch.tensor([1.0]))
    assert t == 1 + 2.0 ** -23, (t, m)                                # exact 1 + 2^-24 + 2^-47: just above the midpoint


def _sum_step(x2d, vec):
    def step(acc, r0, r1):
        if vec:
            v = x2d[:, 4 * r0:4 * r1].reshape(x2d.shape[0], -1, 4)
            return acc + ((v[..., 0] + v[..., 1]) + (v[..., 2] + v[..., 3]))
        return acc + x2d[:, r0:r1]
    return step


def _sqdev_step(x2d, mu, vec):
    def step(acc, r0, r1):
        if vec:
            v = x2d[:, 4 * r0:4 * r1].reshape(x2d.shape[0], -1, 4) - mu.view(-1, 1, 1)
            return acc + (ex.fma32(v[..., 0], v[..., 0], v[..., 1] * v[..., 1]) +
                          ex.fma32(v[..., 2], v[..., 2], v[..., 3] * v[..., 3]))
        dd = x2d[:, r0:r1] - mu.view(-1, 1)
        return ex.fma32(dd, dd, acc)
    return step


def test_bn_stats_emulation_passes_at_hidden1():
    """hidden1_conv's channel length (1,548,800 values) with the slice count 96 channels give it, float4 order"""
    n, Cfull = 1548800, 96
    slices = ex.bn_slices(n, Cfull)
    assert slices == 11
    g = torch.Generator().manual_seed(1)
    x = torch.randn(2, n, generator=g) * 2 + torch.tensor([[0.5], [1e3]])
    x[1] = 1e3 + 1e-2 * torch.randn(n, generator=g)
    flat = x.reshape(-1)
    s = ex.colsum_emulate(_sum_step(x, True), n, 2, slices, True)
    inv_n = torch.tensor(1.0 / n, dtype=torch.float32)
    mu = s * inv_n
    _ok(mu, ex.bn_mean(flat, n, 2, slices, True), "mean")
    q = ex.colsum_emulate(_sqdev_step(x, mu, True), n, 2, slices, True)
    sg = torch.sqrt(ex.fma32(q, inv_n.expand(2), torch.full((2,), 1e-5)))
    _ok(sg, ex.bn_sigma(flat, n, 2, mu, 1e-5, slices, True), "sigma")
    # the one-pass variance fails on the offset channel
    _fails(ex.bn_sigma_one_pass(flat, n, 2, 1e-5), ex.bn_sigma(flat, n, 2, mu, 1e-5, slices, True), "one-pass variance")


def test_bias_grad_and_bn_grad_emulations_pass():
    g = torch.Generator().manual_seed(2)
    rows, cols = 65536 * 3 + 5, 1                      # 64 slices, scalar
    d = torch.randn(cols, rows, generator=g)
    slices = ex.bias_grad_slices(rows, cols)
    assert slices == 64
    s = ex.colsum_emulate(_sum_step(d, False), rows, cols, slices, False)
    so = torch.tensor(1 / 128, dtype=torch.float32)
    b0 = torch.full((cols,), float("nan"))
    _ok(so * s, ex.bias_grad(d.reshape(-1), rows, cols, b0, 0.0, float(so)), "bias grad")
    # BnGradOp, float4 order
    n, C = 8192 * 3, 3
    x, dd = torch.randn(C, n, generator=g), torch.randn(C, n, generator=g)
    mu, sig = torch.randn(C, generator=g) * 0.1, torch.rand(C, generator=g) + 0.5
    inv = (1.0 / sig.double()).float()
    sl = ex.bn_slices(n, C)

    def gstep(acc, r0, r1):
        gv = dd[:, 4 * r0:4 * r1].reshape(C, -1, 4)
        v = (x[:, 4 * r0:4 * r1].reshape(C, -1, 4) - mu.view(-1, 1, 1)) * inv.view(-1, 1, 1)
        return acc + (ex.fma32(gv[..., 0], v[..., 0], gv[..., 1] * v[..., 1]) +
                      ex.fma32(gv[..., 2], v[..., 2], gv[..., 3] * v[..., 3]))
    s1 = ex.colsum_emulate(gstep, n, C, sl, True)
    s0 = ex.colsum_emulate(_sum_step(dd, True), n, C, sl, True)
    inv_n = torch.tensor(1.0 / n, dtype=torch.float32)
    egg, egb = ex.bn_grads(dd.reshape(-1), x.reshape(-1), n, C, mu, sig, sl, True)
    _ok(s1 * inv_n, egg, "grad gamma")
    _ok(s0 * inv_n, egb, "grad beta")


def test_softmax_and_sum_emulations_pass():
    g = torch.Generator().manual_seed(3)
    for rows, cols, scale, off in ((128, 1000, 3, 0), (33, 1001, 30, 1e4), (32, 9, 3, 0)):
        x = (torch.randn(cols * rows, generator=g) * scale + off).float()
        _ok(ex.softmax_emulate(x, rows, cols), ex.softmax(x, rows, cols), "softmax %dx%d" % (rows, cols))
    for n in (1, 31, 256, 257, 10000):
        a = torch.randn(n, generator=g)
        _ok(ex.sum_emulate(a).reshape(1), ex.sum_ref(a), "sum %d" % n)


# ---------------------------------------------------------------------------------------------------------------------
# simulated faults fail the bars
# ---------------------------------------------------------------------------------------------------------------------
def test_faults_bias_relu_dropout_mult():
    g = torch.Generator().manual_seed(4)
    rows, cols = 4001, 7
    x, b = torch.randn(rows * cols, generator=g), torch.randn(cols, generator=g)
    good = ex.bias_add(x, b, rows, cols, True)
    _fails(ex.bias_add(x, b, rows, cols, True, fault="mod_cols").ref.float(), good, "bias indexed by i % cols")
    _fails(ex.bias_add(x, b, rows, cols, True, fault="relu_first").ref.float(), good, "ReLU before the bias")
    # ReLU': >= on exact zeros, a flushed subnormal state
    y = torch.tensor([0.0, -0.0, 1e-45, 2.0 ** -130, float("nan"), 1.0, -1.0])
    d = torch.arange(1, 8, dtype=torch.float32)
    good = ex.relu_deriv(d, y)
    assert good.ref.tolist() == [0, 0, 3, 4, 0, 6, 0]
    _fails(ex.relu_deriv(d, y, "ge").ref.float(), good, "ReLU' with >=")
    _fails(ex.relu_deriv(d, y, "ftz").ref.float(), good, "ReLU' flushing subnormals")
    # ReLU of the special values
    r = ex.relu(torch.tensor([float("nan"), -0.0, 0.0, -1e-45, 1e-45, float("-inf")]))
    assert r.ref.tolist() == [0, 0, 0, 0, float(np.float32(1e-45)), 0] and not r.exact[1]
    # dropout: p at an element's u, the tail, the lanes, the mask
    n, seed, scale = 4103, 1234, 2.0
    n4 = n // 4
    kept, u = ex.cx.dropout_kept(n, 0.5, seed, return_u=True)
    xd = torch.randn(n, generator=g)
    for k in (1001, 4101):                               # one in the vector body, one in the tail
        p = float(u[k])
        gv, gm = ex.dropout(xd, p, scale, seed)
        fv, _ = ex.dropout(xd, p, scale, seed, fault="gt")
        assert gm.ref[k] == scale
        _fails(fv.ref.float(), gv, "dropout with > (p = u of element %d)" % k)
    gv, gm = ex.dropout(xd, 0.5, scale, seed)
    for f in ("tail0", "lanes"):
        fv, fm = ex.dropout(xd, 0.5, scale, seed, n4=n4, fault=f)
        _fails(fm.ref.float(), gm, "dropout " + f)
    _, fm = ex.dropout(xd, 0.5, scale, seed, fault="mask1")
    _fails(fm.ref.float(), gm, "a mask of 1")
    # u can be 1.0, and the seed wraps
    assert float(ex.cx.dropout_u(0, np.array([0], np.uint64))[0]) <= 1.0
    w = ex.cx.dropout_u(2 ** 64 - 2, np.arange(4, dtype=np.uint64))
    assert w[2] == ex.cx.dropout_u(0, np.array([0], np.uint64))[0]
    # mult
    a2, b2 = torch.randn(99, generator=g), torch.randn(99, generator=g)
    _ok((a2 * b2), ex.mult(a2, b2), "mult")
    _fails(ex.bf16_rne(a2 * b2), ex.mult(a2, b2), "a 16-bit product")


def test_faults_sums():
    g = torch.Generator().manual_seed(5)
    # bias grad reading its NaN target when st == 0; a dropped row (exact arm)
    rows, cols = 40000, 37
    d = (torch.randint(-8, 9, (rows * cols,), generator=g) / 16).float()
    b0 = torch.full((cols,), float("nan"))
    good = ex.bias_grad(d, rows, cols, b0, 0.0, 0.5, exact_arm=True)
    _ok(good.ref.float(), good, "bias grad, exact arm")
    _fails(ex.bias_grad(d, rows, cols, b0, 0.0, 0.5, fault="read_target").ref.float(), good, "st == 0 reads the target")
    _fails(ex.bias_grad(d, rows, cols, b0, 0.0, 0.5, fault="drop_row").ref.float(), good, "a dropped row")
    # a slice boundary that drops or doubles one element, at n = 2^21 (exact arms)
    n = 2 ** 21
    x = (torch.randint(-8, 9, (n,), generator=g) / 16).float()
    x[-1] = 0.5
    sl = ex.bn_slices(n, 1)
    em = ex.bn_mean(x, n, 1, sl, True, exact_arm=True)
    _fails(ex.bn_mean(x, n, 1, sl, True, fault="drop").ref.float(), em, "a dropped element")
    dup = x.clone()
    dup[: n // 2] = torch.cat([x[: n // 2 - 1], x[n // 2 - 2: n // 2 - 1]])
    _fails(ex.bn_mean(dup, n, 1, sl, True).ref.float(), em, "a doubled element")
    pm = torch.ones(n)
    pm[::2] = -1
    es = ex.bn_sigma(pm, n, 1, torch.zeros(1), 1e-5, sl, True, exact_arm=True)
    one_off = pm.clone()
    one_off[7] = 0.0                                   # one square left out of the sum
    _fails(ex.bn_sigma(one_off, n, 1, torch.zeros(1), 1e-5, sl, True).ref.float(), es, "variance, +-1 data")
    # the variance faults on a sd-1 channel: 1 / (n - 1), eps outside the root
    nb = 4096
    xb = torch.randn(nb, generator=g)
    mu = xb.double().mean().float().reshape(1)
    good = ex.bn_sigma(xb, nb, 1, mu, 1e-3, 1, True)
    for f in ("n_minus_1", "eps_outside"):
        _fails(ex.bn_sigma(xb, nb, 1, mu, 1e-3, 1, True, fault=f).ref.float(), good, f)
    # cnb_sum past 256 elements
    a = torch.randn(10000, generator=g)
    _fails(ex.sum_ref(a, fault="first256").ref.float(), ex.sum_ref(a), "sum stops at 256")


def test_faults_bn_elementwise():
    g = torch.Generator().manual_seed(6)
    n, C = 1000, 3
    x, d = torch.randn(n * C, generator=g), torch.randn(n * C, generator=g)
    gamma, beta = torch.rand(C, generator=g) + 0.5, torch.randn(C, generator=g)
    mu, sg = torch.randn(C, generator=g) * 0.1, torch.rand(C, generator=g) + 0.5
    good = ex.bn_apply(x, n, C, gamma, beta, mu, sg)
    _fails(ex.bn_apply(x, n, C, gamma, beta, mu, sg, fault="bf16_a").ref.float(), good, "gamma / sigma in bf16")
    # fma against a separately rounded product: a restatement that differs is caught bit for bit
    a = (gamma.double() / sg.double()).float()
    two = ((x.view(C, n) - mu.view(C, 1)) * a.view(C, 1) + beta.view(C, 1)).reshape(-1)
    assert not ex.check(two, good).ok
    gg, gb = torch.randn(C, generator=g) * 0.1, torch.randn(C, generator=g) * 0.1
    good = ex.bn_backward(d, x, n, C, gamma, mu, sg, gg, gb, 1)
    _fails(ex.bn_backward(d, x, n, C, gamma, mu, sg, gg, gb, 1, fault="no_xhat").ref.float(), good,
           "the xhat E[d xhat] term dropped")
    good0 = ex.bn_backward(d, x, n, C, gamma, mu, sg, gg, gb, 0)
    _fails(ex.bn_backward(d, x, n, C, gamma, mu, sg, gg, gb, 0, fault="train0_batch").ref.float(), good0,
           "train = 0 using batch terms")
    # the running averages are bit-exact: a separately rounded product differs somewhere on 4096 values
    run, val = torch.randn(4096, generator=g), torch.randn(4096, generator=g)
    f = torch.tensor(0.9, dtype=torch.float32)
    _fails((1 - f) * val + f * run, ex.bn_running(run, val, 0.9), "running average without the fma")


def test_faults_softmax():
    g = torch.Generator().manual_seed(7)
    rows, cols = 33, 1001
    x = torch.randn(cols, rows, generator=g) * 3
    hot = torch.randint(0, cols, (rows,), generator=g)
    hot[hot % 8 == 0] += 1                              # every maximum outside warp 0's columns
    x[hot, torch.arange(rows)] = x.max(0).values + 200
    x = x.reshape(-1)
    onehot = ex.softmax(x, rows, cols, exact="onehot")
    _ok(ex.softmax_emulate(x, rows, cols), onehot, "one-hot")
    _fails(ex.softmax_emulate(x, rows, cols, fault="one_warp"), onehot, "max over one warp")
    for c in (9, 1000):
        xs = torch.randn(c * 32, generator=g)
        _fails(ex.softmax_emulate(xs, 32, c, fault="drop_warp"), ex.softmax(xs, 32, c), "a warp's sum missing")
    eq = torch.full((7 * 33,), 2.5)
    _ok(ex.softmax_emulate(eq, 33, 7), ex.softmax(eq, 33, 7, exact="equal"), "equal logits")


# ---------------------------------------------------------------------------------------------------------------------
# every branch the mirror can return is claimed by a GPU case
# ---------------------------------------------------------------------------------------------------------------------
def test_every_mirror_branch_has_a_case():
    import test_gpu_elementwise_exact as T
    aligns = (True, False)
    claimed = {c.branch for c in T.EW_CASES}
    ns = (1, 2, 3, 4, 5, 4097, 4098, 4099, 8192, T.GS_N, T.GS_N + 2, T.GS_N + 394, 128 * 55 * 55 * 96)
    for op in ("relu", "relu_deriv", "dropout", "mult"):
        for n, a, b in itertools.product(ns, aligns, aligns):
            assert ex.n4_branch(op, n, a, b).name in claimed, (op, n, a, b)
    claimed = {c.branch for c in T.BIAS_CASES}
    for rows, cols, a, r in itertools.product((3, 4000, 4001, 4002, 93312, 93313), (5, 37, 256), aligns, (False, True)):
        assert ex.bias_branch(rows, cols, a, r).name in claimed, (rows, cols, a, r)
    claimed = {c.branch for c in T.GRAD_CASES}
    for rows, cols, st in itertools.product((100, 1000, 5000, 40000, 65536 * 3 + 5), (1, 3, 37, 600, 4096), (0.0, 1.0)):
        assert ex.bias_grad_branch(rows, cols, st).name in claimed, (rows, cols, st)
    cs = {c.stats for c in T.BN_CASES + T.BN_PROD}
    ca = {c.apply for c in T.BN_CASES + T.BN_PROD}
    cb = {c.backward for c in T.BN_CASES + T.BN_PROD}
    for n, C, ax, ay, flag in itertools.product((1, 8, 4096, 4099, 600000, 2 ** 21, 1548800), (1, 5, 96, 4096, 65535),
                                                aligns, aligns, (0, 1)):
        if n * C > 2 ** 31:
            continue
        assert ex.bn_stats_branch(n, C, ax, bool(flag)).name in cs, (n, C, ax, flag)
        assert ex.bn_apply_branch(n, C, ax, ay, flag).name in ca, (n, C, ax, ay, flag)
        assert ex.bn_backward_branch(n, C, ax, ay, flag).name in cb, (n, C, ax, ay, flag)
    claimed = {c.branch for c in T.SM_CASES}
    for r, c in itertools.product((1, 31, 32, 64, 129), (1, 7, 8, 9, 16, 1000, 1001)):
        assert ex.softmax_branch(r, c).name in claimed, (r, c)
    claimed = {c.branch for c in T.SUM_CASES}
    for n in (1, 255, 256, 257, 10 ** 6):
        assert ex.sum_branch(n).name in claimed, n
    # and every case table entry names the branch its own parameters give
    for c in T.EW_CASES:
        assert c.mirror().name == c.branch
