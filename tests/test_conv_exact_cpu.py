"""The float64 reference of tests/conv_exact.py, checked on the CPU: it agrees with the C oracle (itself pinned bit for
bit to the reference's CPU library) within the bar, its operand models match a bit-level restatement, and its bar rejects
simulated kernel faults that the Diff-based tolerances of the older tests let through."""
import numpy as np
import pytest
import torch

import conv_exact as cx
from cases import F, GOLDEN_2D, GOLDEN_3D, load_golden


def _t(a):
    """Fortran numpy matrix -> flat torch buffer in the library's (column-major) order"""
    return torch.from_numpy(np.asarray(a, dtype=np.float32).reshape(-1, order="F").copy())


def _agree(op, g, y, e, t0=None):
    v = cx.check(op, g, _t(y), e, t0=None if t0 is None else _t(t0))
    assert v.ok, (op, str(v))
    return v


# ---------------------------------------------------------------------------------------------------------------------
# 1. the validator against the oracle
# ---------------------------------------------------------------------------------------------------------------------
ORACLE_CASES = {
    # name: Geo(N, W, H, Cin, Cout, ky, kx, sy, sx, py, px, ...)
    "testconv_full": cx.Geo(128, 12, 12, 32, 64, 3, 3, 2, 2, 1, 1),
    "alex_conv1_cut": cx.Geo(8, 31, 31, 3, 96, 7, 7, 2, 2, 1, 1),
    "ragged_batch": cx.Geo(37, 9, 8, 12, 20, 3, 2, 2, 1, 1, 0),
    "single_image": cx.Geo(1, 6, 6, 4, 8, 3, 3, 1, 1, 1, 1),
    "fc_like": cx.Geo(64, 1, 1, 300, 10, 1, 1),
    "pad_ge_kernel": cx.Geo(8, 5, 6, 6, 8, 2, 3, 1, 2, 3, 3),
    "stride3_k5": cx.Geo(8, 11, 10, 8, 12, 5, 5, 3, 3, 2, 1),
    "subrange": cx.Geo(16, 8, 8, 16, 16, 3, 3, 1, 1, 1, 1, cin0=8, CinT=24, cout0=16, CoutT=32),
}


def _operands(g, seed):
    r = np.random.RandomState(seed)
    rows, cols = g.img_dims()
    images = F(r.randn(rows, cols))
    filters = F(r.randn(*g.flt_dims()) / np.sqrt(g.K))
    derivs = F(r.randn(*g.out_dims()))
    return r, images, filters, derivs


@pytest.mark.parametrize("case", sorted(ORACLE_CASES))
def test_reference_matches_oracle(oracle, case):
    g = ORACLE_CASES[case]
    r, images, filters, derivs = _operands(g, 11)
    ish, fsh, tsh, d = g.img_shape(), g.flt_shape(), g.out_shape(), g.desc()
    for st, so in ((0.0, 1.0), (0.5, 0.25)):
        t0 = F(r.randn(*g.out_dims()))
        up = t0.copy(order="F"); oracle.convUp(images, filters, up, ish, fsh, tsh, d, st, so)
        _agree("fprop", g, up, cx.expect("fprop", g, _t(images), _t(filters), "fp32", _t(t0), st, so), t0)
        t0 = F(r.randn(*g.img_dims()))
        dn = t0.copy(order="F"); oracle.convDown(derivs, filters, dn, tsh, fsh, ish, d, st, so)
        _agree("dgrad", g, dn, cx.expect("dgrad", g, _t(derivs), _t(filters), "fp32", _t(t0), st, so), t0)
        t0 = F(r.randn(*g.flt_dims()))
        dw = t0.copy(order="F"); oracle.convOutp(images, derivs, dw, ish, tsh, fsh, d, st, so)
        _agree("wgrad", g, dw, cx.expect("wgrad", g, _t(images), _t(derivs), "fp32", _t(t0), st, so), t0)


def test_reference_matches_oracle_3d(oracle):
    # frame windows 2 apart with kt = 3: dgrad windows overlap
    g = cx.Geo(8, 7, 6, 4, 12, 3, 3, 1, 1, 1, 1, T=7, kt=3, st_t=2)
    r, images, filters, derivs = _operands(g, 12)
    ish, fsh, tsh, d = g.img_shape(), g.flt_shape(), g.out_shape(), g.desc()
    for st in (0.0, 0.5):
        t0 = F(r.randn(*g.out_dims()))
        up = t0.copy(order="F"); oracle.convUp3D(images, filters, up, ish, fsh, tsh, d, st)
        _agree("fprop", g, up, cx.expect("fprop", g, _t(images), _t(filters), "fp32", _t(t0), st), t0)
        t0 = F(r.randn(*g.img_dims()))
        dn = t0.copy(order="F"); oracle.convDown3D(derivs, filters, dn, tsh, fsh, ish, d, st)
        _agree("dgrad", g, dn, cx.expect("dgrad", g, _t(derivs), _t(filters), "fp32", _t(t0), st), t0)
        t0 = F(r.randn(*g.flt_dims()))
        dw = t0.copy(order="F"); oracle.convOutp3D(images, derivs, dw, ish, tsh, fsh, d, st, 0.25)
        _agree("wgrad", g, dw, cx.expect("wgrad", g, _t(images), _t(derivs), "fp32", _t(t0), st, 0.25), t0)


@pytest.mark.parametrize("name", GOLDEN_2D + GOLDEN_3D)
def test_reference_matches_golden(name):
    """the committed outputs of the reference's own CPU conv (py/conv_cpu.py)"""
    z = load_golden(name)
    sfx = "3D" if name.startswith("ref3d") else ""
    kw = dict(T=z["T"], kt=z["kt"], st_t=z["st"]) if sfx else {}
    g = cx.Geo(z["N"], z["W"], z["H"], z["Cin"], z["Cout"], z["ky"], z["kx"], z["sy"], z["sx"], z["py"], z["px"], **kw)
    assert (g.modX, g.modY) == (z["modX"], z["modY"])
    im, fl, dv = _t(z["images"]), _t(z["filters"]), _t(z["derivs"])
    _agree("fprop", g, z["convUp" + sfx], cx.expect("fprop", g, im, fl, "fp32"))
    _agree("dgrad", g, z["convDown" + sfx], cx.expect("dgrad", g, dv, fl, "fp32"))
    _agree("wgrad", g, z["convOutp" + sfx], cx.expect("wgrad", g, im, dv, "fp32"))


def test_epilogue_reference():
    """bias + ReLU + dropout of fprop and the ReLU' mask of dgrad, against a direct float32 restatement"""
    g = cx.Geo(16, 6, 5, 8, 12, 3, 3, 1, 1, 1, 1)
    r, images, filters, derivs = _operands(g, 13)
    Nn, L = g.N, g.modX * g.modY
    im, fl = _t(images), _t(filters)
    bias = torch.from_numpy(r.randn(g.Cout).astype(np.float32))
    plain = cx.expect("fprop", g, im, fl, "fp32").ref
    y = torch.relu(plain.view(g.Cout, L, Nn) + bias.double().view(-1, 1, 1)).reshape(-1)
    kept = cx.dropout_kept(y.numel(), 0.3, 1234)
    y = torch.where(torch.from_numpy(kept), y * 2.0, torch.zeros_like(y)).float()
    e = cx.expect("fprop", g, im, fl, "fp32", bias=bias, relu=True, drop=(0.3, 2.0, 1234))
    assert cx.check("fprop", g, y, e).ok
    assert 0.2 < 1 - kept.mean() < 0.4 and bool(e.zero.any())
    mask = torch.from_numpy(r.randn(g.N * g.W * g.H * g.Cin).astype(np.float32))
    e = cx.expect("dgrad", g, _t(derivs), fl, "fp32", mask=mask)
    d = cx.expect("dgrad", g, _t(derivs), fl, "fp32").ref.float()
    assert cx.check("dgrad", g, torch.where(mask > 0, d, torch.zeros_like(d)), e).ok
    assert not cx.check("dgrad", g, d, e).ok          # an unmasked output fails


def test_dropout_hash_restatement():
    """hash_u32 (common.cuh) on known inputs: splitmix64's finaliser of seed + index, top 32 bits"""
    def splitmix(x):
        m = (1 << 64) - 1
        x = (x + 0x9E3779B97F4A7C15) & m
        x = ((x ^ (x >> 30)) * 0xBF58476D1CE4E5B9) & m
        x = ((x ^ (x >> 27)) * 0x94D049BB133111EB) & m
        return (x ^ (x >> 31)) >> 32
    xs = [0, 1, 2, 12345, (1 << 63) + 7, (1 << 64) - 1]
    assert [int(v) for v in cx.hash_u32(np.array(xs, dtype=np.uint64))] == [splitmix(x) for x in xs]


# ---------------------------------------------------------------------------------------------------------------------
# 2. operand models against a bit-level restatement
# ---------------------------------------------------------------------------------------------------------------------
def _edge_values():
    b = [0x00000000, 0x80000000, 0x00000001, 0x807FFFFF, 0x00400000, 0x007FFFFF,        # zeros, subnormals
         0x3F800000, 0x3F808000, 0x3F818000, 0x3F807FFF, 0x3F808001, 0xBF808000, 0xBF818000,  # bf16 ties / near ties
         0x3F801000, 0x3F803000, 0x3F800FFF, 0xBF801000, 0xBF803000,                     # tf32 ties
         0x7F7FFFFF, 0xFF7FFFFF, 0x7F7F8000, 0x7F7F7FFF, 0x7F800000, 0xFF800000]         # top of the range, inf
    r = np.random.RandomState(0).randint(0, 2 ** 32, 2000, dtype=np.uint64)
    bits = np.concatenate([np.array(b, dtype=np.uint64), r]).astype(np.uint32)
    bits = bits[~np.isnan(bits.view(np.float32))]
    return bits


def _rne(u, drop):
    u = u.astype(np.uint64)
    half = (1 << (drop - 1)) - 1
    r = (u + half + ((u >> drop) & 1)) >> drop << drop
    return (r & 0xFFFFFFFF).astype(np.uint32)


def _trunc(u, drop):
    return (u.astype(np.uint64) >> drop << drop).astype(np.uint32)


@pytest.mark.parametrize("kind", ["bf16", "tf32", "bf16_trunc", "tf32_rn"])
def test_operand_models_bitwise(kind):
    u = _edge_values()
    want = {"bf16": lambda v: _rne(v, 16), "tf32": lambda v: _trunc(v, 13),
            "bf16_trunc": lambda v: _trunc(v, 16), "tf32_rn": lambda v: _rne(v, 13)}[kind](u)
    x = torch.from_numpy(u.view(np.float32).copy())
    got = cx.MODELS[kind](x).numpy().view(np.uint32)
    finite = np.isfinite(u.view(np.float32))
    # rounding the largest finite values up gives +-inf, as __float2bfloat16_rn does
    assert np.array_equal(got[finite], want[finite]), [(hex(a), hex(b), hex(c)) for a, b, c in
                                                       zip(u[finite], got[finite], want[finite]) if b != c][:5]
    assert np.array_equal(got[~finite], u[~finite])
    assert cx.model(x, kind).dtype == torch.float64


def test_bf16_model_overflows_to_inf():
    # the largest finite floats lie above the largest bf16 + half an ulp: they round up to +-inf
    x = torch.from_numpy(np.array([0x7F7FFFFF, 0xFF7FFFFF, 0x7F7F8000], dtype=np.uint32).view(np.float32))
    assert torch.isinf(cx.MODELS["bf16"](x)).all()
    assert torch.isfinite(cx.MODELS["tf32"](x)).all()


# ---------------------------------------------------------------------------------------------------------------------
# 3. the bar has teeth: simulated kernels at conv3's GEMM shape (M 4096, K 2304, N 384) as an FC call
# ---------------------------------------------------------------------------------------------------------------------
SIM = cx.Geo(4096, 1, 1, 2304, 384, 1, 1)


@pytest.fixture(scope="module")
def sim():
    gen = torch.Generator().manual_seed(3)
    a = torch.randn(SIM.Cin * SIM.N, generator=gen)                       # images  [c][n]
    b = torch.randn(SIM.K * SIM.Cout, generator=gen) / np.sqrt(SIM.K)     # filters [k][o]
    exp = {kind: cx.expect("fprop", SIM, a, b, kind, so=SO) for kind in ("bf16", "tf32")}
    return a, b, exp


SO = 0.3          # an output scale bf16 cannot hold


def _gemm(a, b, kind, kblock_round=False, drop_k=None):
    """a simulated kernel: model-rounded operands, fp32 accumulate -> flat fprop output"""
    A = cx.MODELS[kind](a).view(SIM.Cin, SIM.N).t()          # (N, K)
    B = cx.MODELS[kind](b).view(SIM.K, SIM.Cout)             # (K, Cout)
    if kblock_round:
        acc = torch.zeros(SIM.N, SIM.Cout)
        for k0 in range(0, SIM.K, 64):
            acc += (A[:, k0:k0 + 64] @ B[k0:k0 + 64]).to(torch.bfloat16).float()
    else:
        acc = A @ B
    if drop_k is not None:
        acc[:128, :128] -= A[:128, drop_k:drop_k + 1] @ B[drop_k:drop_k + 1, :128]
    return acc.t().reshape(-1)                               # [o][n]


FAULTS = {
    # name: (operand model of the check, simulated output)
    "bf16_correct": ("bf16", lambda a, b: SO * _gemm(a, b, "bf16"), True),
    "tf32_correct": ("tf32", lambda a, b: SO * _gemm(a, b, "tf32"), True),
    "bf16_truncated_operands": ("bf16", lambda a, b: SO * _gemm(a, b, "bf16_trunc"), False),
    "bf16_kblock_partials_rounded": ("bf16", lambda a, b: SO * _gemm(a, b, "bf16", kblock_round=True), False),
    "bf16_output_scale_rounded": ("bf16", lambda a, b: float(torch.tensor(SO).to(torch.bfloat16)) * _gemm(a, b, "bf16"),
                                  False),
    "tf32_rounded_operands": ("tf32", lambda a, b: SO * _gemm(a, b, "tf32_rn"), False),
    "bf16_one_k_term_dropped_in_one_tile": ("bf16", lambda a, b: SO * _gemm(a, b, "bf16", drop_k=1000), False),
}


@pytest.mark.parametrize("fault", list(FAULTS))
def test_bar_rejects_simulated_faults(sim, fault):
    a, b, exp = sim
    kind, run, correct = FAULTS[fault]
    v = cx.check("fprop", SIM, run(a, b), exp[kind])
    assert v.ok == correct, (fault, str(v))
    if correct:
        assert v.worst_ratio < 2.0 ** -18, str(v)       # well inside the bar, not at its edge
    else:
        assert v.worst_ratio > 8 * cx.BAR, str(v)       # far outside it


def test_failure_report_names_the_element(sim):
    a, b, exp = sim
    y = SO * _gemm(a, b, "bf16")
    y[5 + SIM.N * 17] += 1.0                            # image 5, channel 17
    v = cx.check("fprop", SIM, y, exp["bf16"])
    assert not v.ok and "n=5 x=0 y=0 c=17" in v.where and v.share_over == 1.0 / y.numel()
