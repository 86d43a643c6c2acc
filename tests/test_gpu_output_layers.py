"""Logistic units and the output layers' loss functions and metrics on the GPU.

- The stand-alone passes (cnb_logistic, cnb_logistic_deriv), the loss and metric kernels (cnb_loss_deriv, cnb_metric)
  element by element against the float64 restatements and bars of tests/loss_ref.py, and against the reference's own CPU
  library (tests/golden/ref_loss.npz).
- The fused logistic epilogues (convnet_b200_fuse_next_act) bit for bit against the unfused call plus the pass, at the
  dispatch branches the fused ReLU reaches.
- Nets: back-propagation against a float64 autograd mirror sharing the native parameters, the grad check of logistic and
  non-softmax outputs, Net.metric(), training runs.
"""
import json
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import loss_ref as R
from conv_exact import Geo

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "ref_loss.npz")
NAN = 0x7FC0DEAD


@pytest.fixture(scope="module")
def env():
    assert torch.cuda.is_available()
    from convnet_b200 import conv_gemm as cg
    from convnet_b200 import lib, net
    L = lib.load()
    net.load_host()
    yield cg, lib, L, net
    lib.set_precision("tf32")


@pytest.fixture(autouse=True)
def hygiene(env):
    _, _, L, _ = env
    prec = L.convnet_b200_get_conv_precision()
    try:
        yield
    finally:
        L.convnet_b200_set_conv_precision(prec)
        L.convnet_b200_bf16_invalidate(None)
        L.cnb_relu_deriv(None, None, 0)                  # consumes any fuse request a failed call left pending


def _cm(a):
    """[images x cols] numpy -> column-major float32 device tensor (images fastest)"""
    return torch.tensor(np.asarray(a, np.float32).T.copy().ravel(), device="cuda")


def _rm(t, rows):
    """column-major device tensor -> [images x cols] float64 numpy"""
    return t.double().view(-1, rows).T.cpu().numpy()


def _ok(y, ref, bar):
    err = np.abs(np.asarray(y, np.float64) - ref)
    return bool(np.all(err <= bar)), float(np.max(err / np.where(bar > 0, bar, 1.0)))


# ---------------------------------------------------------------------------------------------------------------------
# the stand-alone passes
# ---------------------------------------------------------------------------------------------------------------------
def _read_twin(env, t, N, C):
    """the staged bf16 copy of the [N x 8*8*C] tensor t, read back exactly through a bf16 1x1 identity conv"""
    from convnet_b200.abi import GetConvDesc
    from convnet_b200.matrix import CUDAMatrix
    cg, lib, L, _ = env
    d = GetConvDesc(C, C, 1, 1, 1, 1, 0, 0)
    img = CUDAMatrix(N, 64 * C, (N, 8, 8, C), storage=t)
    eye = CUDAMatrix(C, C, (C, 1, 1, C), storage=torch.eye(C, device="cuda").reshape(-1).contiguous())
    out = CUDAMatrix(N, 64 * C, (N, 8, 8, C), storage=torch.empty(N * 64 * C, device="cuda"))
    assert L.convnet_b200_bf16_is_staged(t.data_ptr(), t.numel()) == 1
    cg.convUp(img, eye, out, d, 0)
    assert lib.last_conv_path() == "tc-bf16"
    torch.cuda.synchronize()
    return out.storage.clone()


@pytest.mark.parametrize("n,offset", [(1 << 20, 0), (1000003, 0), (4099, 1)], ids=["vec", "ragged", "misaligned"])
def test_logistic_passes_per_element(env, n, offset):
    _, lib, L, _ = env
    g = torch.Generator(device="cuda").manual_seed(n)
    buf = torch.randn(n + offset, device="cuda", generator=g) * 8
    buf[offset:offset + 8] = torch.tensor([0.0, -0.0, 30, -30, 88, -88, 95, -95])
    x = buf[offset:]
    x0 = x.double().cpu().numpy()
    L.cnb_logistic(x.data_ptr(), n)
    torch.cuda.synchronize()
    ok, worst = _ok(x.cpu().numpy(), R.sigmoid(x0), R.sigmoid_bar(x0))
    assert ok, worst
    d = torch.randn(n + offset, device="cuda", generator=g)[offset:]
    d0, s0 = d.double().cpu().numpy(), x.double().cpu().numpy()
    L.cnb_logistic_deriv(d.data_ptr(), x.data_ptr(), n)
    torch.cuda.synchronize()
    ok, worst = _ok(d.cpu().numpy(), R.logistic_deriv(d0, s0), R.logistic_deriv_bar(d0, s0))
    assert ok, worst
    # controls: the bars see a sign error and a missing (1 - s)
    assert not _ok(x.cpu().numpy(), R.sigmoid(-x0), R.sigmoid_bar(-x0))[0]
    assert not _ok(d.cpu().numpy(), d0 * s0, R.logistic_deriv_bar(d0, s0))[0]


def test_logistic_passes_bf16_twin(env):
    """convnet_b200_emit_bf16_next: both passes leave the round-to-nearest bf16 of what they store"""
    _, lib, L, _ = env
    lib.set_precision("bf16")
    N, C = 128, 16
    x = torch.randn(N * 64 * C, device="cuda") * 4
    L.convnet_b200_emit_bf16_next()
    L.cnb_logistic(x.data_ptr(), x.numel())
    assert torch.equal(_read_twin(env, x, N, C), x.to(torch.bfloat16).float())
    d = torch.randn_like(x)
    L.convnet_b200_emit_bf16_next()
    L.cnb_logistic_deriv(d.data_ptr(), x.data_ptr(), d.numel())
    assert torch.equal(_read_twin(env, d, N, C), d.to(torch.bfloat16).float())


# ---------------------------------------------------------------------------------------------------------------------
# loss functions and metrics
# ---------------------------------------------------------------------------------------------------------------------
def _inputs(loss, rows, cols, seed):
    rng = np.random.default_rng(seed)
    logits = rng.standard_normal((rows, cols)) * 3
    p = np.exp(logits - logits.max(1, keepdims=True)); p /= p.sum(1, keepdims=True)
    labels = rng.integers(0, cols, rows).astype(np.int32)
    if loss in (R.CE_MULTINOMIAL, R.CE_DISTRIBUTED, R.CLASS_MULTINOMIAL):
        y = p
        t = rng.uniform(0, 1, (rows, cols)); t /= t.sum(1, keepdims=True)
    elif loss in (R.CE_BINARY, R.CLASS_BINARY):
        y = rng.uniform(0, 1, (rows, cols))
        y[0, :3] = [0.0, 1.0, 0.5]
        t = (rng.uniform(0, 1, (rows, cols)) < 0.5).astype(np.float64)
        t[rng.uniform(0, 1, (rows, cols)) < 0.25] = -1                 # don't care
        t[:, 0] = rng.uniform(0, 1, rows)                              # soft targets
        t[min(2, rows - 1), :] = -1                                    # an image without a target
    else:
        y, t = rng.standard_normal((rows, cols)) * 2, rng.standard_normal((rows, cols))
    return np.float32(y), np.float32(t), labels


def _run_loss(env, loss, y, t, labels, weight):
    _, _, L, _ = env
    rows, cols = y.shape
    yd, td, ld = _cm(y), _cm(t), torch.tensor(labels, device="cuda")
    deriv = torch.empty(rows * cols, device="cuda"); deriv.view(torch.int32).fill_(NAN)
    value = torch.empty(rows, device="cuda"); value.view(torch.int32).fill_(NAN)
    L.cnb_loss_deriv(loss, yd.data_ptr(), td.data_ptr(), ld.data_ptr(), deriv.data_ptr(), value.data_ptr(), rows, cols, weight)
    metric = torch.empty(rows, device="cuda"); metric.view(torch.int32).fill_(NAN)
    L.cnb_metric(loss, yd.data_ptr(), td.data_ptr(), ld.data_ptr(), metric.data_ptr(), rows, cols)
    torch.cuda.synchronize()
    return _rm(deriv, rows), value.double().cpu().numpy(), metric


LOSSES = [R.SQUARED_ERROR, R.LINEAR_ERROR, R.CE_MULTINOMIAL, R.CE_BINARY, R.CE_DISTRIBUTED]
SHAPES = [(128, 10), (37, 21), (200, 1000), (1, 3), (130, 257)]


@pytest.mark.parametrize("weight", [1.0, 0.37])
@pytest.mark.parametrize("rows,cols", SHAPES)
@pytest.mark.parametrize("loss", LOSSES)
def test_loss_kernels_per_element(env, loss, rows, cols, weight):
    y, t, labels = _inputs(loss, rows, cols, rows * 1000 + cols)
    deriv, value, metric = _run_loss(env, loss, y, t, labels, weight)
    d, d_bar, v, v_bar = R.loss_ref(loss, y, t, labels, np.float32(weight))
    ok, worst = _ok(deriv, d, d_bar)
    assert ok, ("deriv", worst)
    ok, worst = _ok(value, v, v_bar)
    assert ok, ("value", worst)
    # a loss as the performance metric: the same per-image values, bit for bit
    assert np.array_equal(metric.double().cpu().numpy(), value)
    if loss == R.CE_BINARY:
        assert np.all(deriv[t < 0] == 0)
    if loss == R.CE_MULTINOMIAL and weight == 1.0:     # the kernel every softmax net has always run
        from convnet_b200 import lib
        L = lib.load()
        yd, ld = _cm(y), torch.tensor(labels, device="cuda")
        d2, v2 = torch.empty(rows * cols, device="cuda"), torch.empty(rows, device="cuda")
        L.cnb_softmax_ce_deriv(yd.data_ptr(), ld.data_ptr(), d2.data_ptr(), v2.data_ptr(), rows, cols)
        torch.cuda.synchronize()
        assert np.array_equal(_rm(d2, rows), deriv) and np.array_equal(v2.double().cpu().numpy(), value)


@pytest.mark.parametrize("rows,cols", SHAPES + [(64, 40)])
def test_metric_kernels(env, rows, cols):
    # CLASSIFICATION_MULTINOMIAL, with ties across and within lanes
    y, t, labels = _inputs(R.CLASS_MULTINOMIAL, rows, cols, cols)
    if cols >= 40:
        y[0, 5] = y[0, 37] = y[0].max() + 1                # lane 5 holds both: the first wins
        y[1, 33] = y[1, 2] = y[1].max() + 1                # lanes 1 and 2: lane 1 (column 33) wins
        labels[0], labels[1] = 5, 33
    _, _, m = _run_loss_metric(env, R.CLASS_MULTINOMIAL, y, t, labels)
    assert np.array_equal(m, R.classification_multinomial(y, labels))
    y, t, labels = _inputs(R.CLASS_BINARY, rows, cols, cols + 1)
    _, _, m = _run_loss_metric(env, R.CLASS_BINARY, y, t, labels)
    ref = R.classification_binary(y, t)
    assert np.allclose(m, ref, rtol=2 * R.U, atol=0), np.max(np.abs(m - ref))


def _run_loss_metric(env, metric, y, t, labels):
    _, _, L, _ = env
    rows, cols = y.shape
    yd, td, ld = _cm(y), _cm(t), torch.tensor(labels, device="cuda")
    out = torch.empty(rows, device="cuda"); out.view(torch.int32).fill_(NAN)
    L.cnb_metric(metric, yd.data_ptr(), td.data_ptr(), ld.data_ptr(), out.data_ptr(), rows, cols)
    torch.cuda.synchronize()
    return None, None, out.double().cpu().numpy()


def test_kernels_against_the_reference_goldens(env):
    """the kernels on the inputs of tests/golden/ref_loss.npz against what the reference's eigenmat functions returned
    for them.  Both sides carry their own rounding: each value must lie within the sum of the two bars of the exact one"""
    _, _, L, _ = env
    z = np.load(GOLDEN)
    rows, cols = z["x"].shape
    x = _cm(z["x"])
    L.cnb_logistic(x.data_ptr(), x.numel())
    d, s = _cm(z["d"]), _cm(z["s"])
    L.cnb_logistic_deriv(d.data_ptr(), s.data_ptr(), d.numel())
    torch.cuda.synchronize()
    assert np.all(np.abs(_rm(x, rows) - z["sigmoid"]) <= 2 * R.sigmoid_bar(z["x"]))
    assert np.all(np.abs(_rm(d, rows) - z["logistic_deriv"]) <= 2 * R.logistic_deriv_bar(z["d"], z["s"]))
    # apply_logistic_grad: CROSS_ENTROPY_BINARY's derivative, bit for bit (one rounded subtraction on both sides)
    deriv, value, _ = _run_loss(env, R.CE_BINARY, z["y"], z["t"], z["labels"].astype(np.int32), 1.0)
    assert np.array_equal(deriv, z["logistic_grad"].astype(np.float64))
    # the Bernoulli cross-entropy over the t >= 0 entries (the golden's don't-cares were given t = 0: left out here)
    ref = np.where(z["t"] >= 0, z["cross_entropy_bernoulli"], 0).astype(np.float64).sum(1)
    _, _, v, v_bar = R.loss_ref(R.CE_BINARY, z["y"], z["t"])
    assert np.all(np.abs(value - ref) <= 2 * v_bar)
    # CROSS_ENTROPY_MULTINOMIAL_DISTRIBUTED: compute_cross_entropy's terms summed per image
    _, value, _ = _run_loss(env, R.CE_DISTRIBUTED, z["p"], z["q"], z["labels"].astype(np.int32), 1.0)
    _, _, _, v_bar = R.loss_ref(R.CE_DISTRIBUTED, z["p"], z["q"])
    assert np.all(np.abs(value - z["cross_entropy"].astype(np.float64).sum(1)) <= 2 * v_bar)
    # the metrics: exactly the reference's decisions and shares
    _, _, m = _run_loss_metric(env, R.CLASS_MULTINOMIAL, z["p"], z["q"], z["labels"].astype(np.int32))
    assert np.array_equal(m, z["softmax_correct"])
    _, _, m = _run_loss_metric(env, R.CLASS_BINARY, z["y"], z["t"], z["labels"].astype(np.int32))
    assert np.array_equal(m, z["logistic_correct"].astype(np.float64))


# ---------------------------------------------------------------------------------------------------------------------
# fused epilogues
# ---------------------------------------------------------------------------------------------------------------------
def _m(rows, cols, s4, gen=None):
    from convnet_b200.matrix import CUDAMatrix
    t = torch.empty(rows * cols, dtype=torch.float32, device="cuda")
    if gen is not None:
        t.normal_(generator=gen)
    else:
        t.view(torch.int32).fill_(NAN)
    return CUDAMatrix(rows, cols, s4, storage=t)


# (name, geometry, conv or local, precisions): the branches the fused ReLU reaches
FUSE_CASES = [
    ("conv_merged", Geo(128, 8, 8, 64, 64, 3, 3, 1, 1, 1, 1), True, ("fp32", "tf32", "bf16")),
    ("conv_unmerged_ragged", Geo(96, 6, 6, 72, 40, 3, 3, 1, 1, 1, 1), True, ("fp32", "tf32", "bf16")),
    ("conv_stride2", Geo(128, 9, 9, 32, 32, 3, 3, 2, 2, 1, 1), True, ("tf32", "bf16")),
    ("fc_splitk", Geo(128, 1, 1, 2048, 512, 1, 1), True, ("fp32", "tf32", "bf16")),
    ("one_by_one", Geo(128, 13, 13, 96, 192, 1, 1), True, ("tf32", "bf16")),
    ("local_n128", Geo(128, 12, 12, 128, 128, 3, 3), False, ("fp32", "tf32", "bf16")),
]


@pytest.mark.parametrize("drop", [False, True], ids=["nodrop", "dropout"])
@pytest.mark.parametrize("name,g,conv,modes", FUSE_CASES, ids=[c[0] for c in FUSE_CASES])
def test_fused_logistic_is_bit_identical_to_the_passes(env, name, g, conv, modes, drop):
    """fprop: bias + sigma (+ dropout, + bf16 twin) in the epilogue == the call, the bias pass, cnb_logistic
    (, cnb_dropout); dgrad: sigma'(state) in the epilogue (or its trailing pass) == the call, cnb_logistic_deriv"""
    cg, lib, L, _ = env
    M = g.modX * g.modY
    per_feature = 1 if conv else M                     # bias per output channel, or per output feature (untied)
    gen = torch.Generator(device="cuda").manual_seed(sum(map(ord, name)))
    img = _m(g.N, g.W * g.H * g.Cin, (g.N, g.W, g.H, g.Cin), gen)
    banks = 1 if conv else M
    flt = _m(g.Cout, g.K * banks, (g.Cout, g.kx, g.ky, g.Cin * banks), gen)
    der = _m(g.N, M * g.Cout, (g.N, g.modX, g.modY, g.Cout), gen)
    bias = torch.randn(g.Cout * per_feature, device="cuda", generator=gen)
    d = g.desc()
    up, down = (cg.convUp, cg.convDown) if conv else (cg.localUp, cg.localDown)
    for mode in modes:
        lib.set_precision(mode)
        if mode == "bf16" and g.N * g.W * g.H < 1024:          # FC-shaped calls take bf16 with staged weights
            L.convnet_b200_bf16_stage(flt.ptr, flt.storage.numel())
        outs, paths = [], []
        for fused in (True, False):
            out = _m(g.N, M * g.Cout, (g.N, g.modX, g.modY, g.Cout))
            n_out = out.storage.numel()
            if fused:
                L.convnet_b200_fuse_next_act(bias.data_ptr(), 2, None)
                if drop:
                    L.convnet_b200_fuse_next_dropout(0.3, 1 / 0.7, 4242)
                up(img, flt, out, d, 0)
            else:
                up(img, flt, out, d, 0)
                L.cnb_add_channel_bias(out.ptr, bias.data_ptr(), n_out // (g.Cout * per_feature), g.Cout * per_feature)
                L.cnb_logistic(out.ptr, n_out)
                if drop:
                    L.cnb_dropout(out.ptr, torch.empty(n_out, device="cuda").data_ptr(), n_out, 0.3, 1 / 0.7, 4242)
            paths.append(lib.last_conv_path())
            torch.cuda.synchronize()
            outs.append(out.storage.clone())
        assert paths[0] == paths[1], paths
        assert torch.equal(outs[0].view(torch.int32), outs[1].view(torch.int32)), (name, mode, "fprop")
        if drop:
            continue
        state = torch.sigmoid(torch.randn(img.storage.numel(), device="cuda", generator=gen))
        res = []
        for fused in (True, False):
            t = _m(g.N, g.W * g.H * g.Cin, (g.N, g.W, g.H, g.Cin))
            if fused:
                L.convnet_b200_fuse_next_act(None, 2, state.data_ptr())
                down(der, flt, t, d, 0)
            else:
                down(der, flt, t, d, 0)
                L.cnb_logistic_deriv(t.ptr, state.data_ptr(), t.storage.numel())
            torch.cuda.synchronize()
            res.append(t.storage.clone())
        assert torch.equal(res[0].view(torch.int32), res[1].view(torch.int32)), (name, mode, "dgrad")


def test_fused_relu_through_the_new_entry_is_the_old_request(env):
    """convnet_b200_fuse_next_act(bias, 1, state) == convnet_b200_fuse_next(bias, 1, NULL) / (NULL, 0, state)"""
    cg, lib, L, _ = env
    g = Geo(128, 8, 8, 64, 64, 3, 3, 1, 1, 1, 1)
    gen = torch.Generator(device="cuda").manual_seed(5)
    img = _m(g.N, 64 * 64, (g.N, 8, 8, 64), gen)
    flt = _m(64, 9 * 64, (64, 3, 3, 64), gen)
    bias = torch.randn(64, device="cuda", generator=gen)
    state = torch.randn(img.storage.numel(), device="cuda", generator=gen)
    for mode in ("tf32", "bf16"):
        lib.set_precision(mode)
        a, b = _m(g.N, 64 * 64, (g.N, 8, 8, 64)), _m(g.N, 64 * 64, (g.N, 8, 8, 64))
        L.convnet_b200_fuse_next_act(bias.data_ptr(), 1, None); cg.convUp(img, flt, a, g.desc(), 0)
        L.convnet_b200_fuse_next(bias.data_ptr(), 1, None); cg.convUp(img, flt, b, g.desc(), 0)
        torch.cuda.synchronize()
        assert torch.equal(a.storage.view(torch.int32), b.storage.view(torch.int32))
        L.convnet_b200_fuse_next_act(None, 1, state.data_ptr()); cg.convDown(img, flt, a, g.desc(), 0)
        L.convnet_b200_fuse_next(None, 0, state.data_ptr()); cg.convDown(img, flt, b, g.desc(), 0)
        torch.cuda.synchronize()
        assert torch.equal(a.storage.view(torch.int32), b.storage.view(torch.int32))


# ---------------------------------------------------------------------------------------------------------------------
# nets
# ---------------------------------------------------------------------------------------------------------------------
# float64 autograd mirrors sharing the native parameters.  spec: ("conv", cout, k, stride, pad, act) |
# ("maxpool", k, s, p[, act]) | ("avgpool", k, s, p[, act]) | ("rnorm", k, alpha, beta, act) | ("fc", cout); act in {None, "relu",
# "logistic"}.  The output layer's activation and loss come from the model's suffix.
MIRRORS = {
    "tiny+logistic": dict(base="tiny", cin=8, size=12, spec=[
        ("conv", 16, 3, 1, 1, "logistic"), ("maxpool", 3, 2, 1), ("rnorm", 8, 0.01, 0.75, "logistic"),
        ("conv", 24, 1, 1, 0, "logistic"), ("conv", 16, 3, 2, 1, "logistic"), ("avgpool", 2, 2, 0), ("fc", 10)]),
    "tiny+soft-targets": dict(base="tiny", cin=8, size=12, spec=[
        ("conv", 16, 3, 1, 1, "relu"), ("maxpool", 3, 2, 1), ("rnorm", 8, 0.01, 0.75, "relu"),
        ("conv", 24, 1, 1, 0, "relu"), ("conv", 16, 3, 2, 1, "relu"), ("avgpool", 2, 2, 0), ("fc", 10)]),
    "logcheck": dict(base="gradcheck", cin=4, size=8, spec=[
        ("conv", 8, 3, 1, 1, "logistic"), ("avgpool", 3, 2, 1, "logistic"), ("rnorm", 4, 0.01, 0.75, "logistic"),
        ("conv", 12, 1, 1, 0, "logistic"), ("fc", 5)]),
    "lenet+binary-ce": dict(base="lenet", cin=1, size=28, spec=[
        ("conv", 48, 4, 1, 0, "relu"), ("maxpool", 4, 2, 0), ("conv", 128, 4, 1, 0, "relu"), ("maxpool", 4, 2, 0),
        ("fc", 10)]),
    "lenet+squared-error": dict(base="lenet", cin=1, size=28, spec=[
        ("conv", 48, 4, 1, 0, "relu"), ("maxpool", 4, 2, 0), ("conv", 128, 4, 1, 0, "relu"), ("maxpool", 4, 2, 0),
        ("fc", 10)]),
}


def _act(torch_, h, act):
    return torch_.relu(h) if act == "relu" else (torch_.sigmoid(h) if act == "logistic" else h)


def _targets(n, model, batch, gen):
    """fill the net's labels or targets; returns (labels, targets [batch x cols]) as float64 torch tensors"""
    out = n.model_output_layer(model)
    cols = n.num_classes
    if out["labels"]:
        lab = torch.randint(0, cols, (batch,), device="cuda", generator=gen, dtype=torch.int32)
        n.labels_tensor().copy_(lab)
        return lab.long(), None
    if out["loss_function"] == "CROSS_ENTROPY_BINARY":
        t = (torch.rand(batch, cols, device="cuda", generator=gen) < 0.5).float()
        t[torch.rand(batch, cols, device="cuda", generator=gen) < 0.2] = -1
    elif out["loss_function"] == "CROSS_ENTROPY_MULTINOMIAL_DISTRIBUTED":
        t = torch.softmax(3 * torch.randn(batch, cols, device="cuda", generator=gen), 1)
    else:
        t = torch.randn(batch, cols, device="cuda", generator=gen)
    n.targets_tensor().copy_(t.T.contiguous().view(-1))
    return None, t.double()


def _mirror(n, model, batch, labels, targets):
    import torch.nn.functional as Fn
    cfg = MIRRORS[model]
    P = n.params_tensor().double()
    edges = n.edges()
    params = {}
    C, S = cfg["cin"], cfg["size"]
    h = n.input_tensor().double().view(C, S, S, batch).permute(3, 0, 1, 2).contiguous()
    for i, e in enumerate(cfg["spec"]):
        off, size = edges[i][2], edges[i][3]
        if e[0] == "conv":
            _, cout, k, s, p, act = e
            cin = h.shape[1]
            K = cin * k * k
            flat = P[off:off + size].clone()
            w = flat[:cout * K].view(cin, k, k, cout).permute(3, 0, 1, 2).contiguous().requires_grad_(True)
            b = flat[cout * K:cout * K + cout].clone().requires_grad_(True)
            params[i] = (w, b, K)
            h = _act(torch, Fn.conv2d(h, w, b, stride=s, padding=p), act)
        elif e[0] == "maxpool":
            h = _act(torch, Fn.max_pool2d(h, e[1], e[2], e[3]), e[4] if len(e) > 4 else None)
        elif e[0] == "avgpool":
            h = _act(torch, Fn.avg_pool2d(h, e[1], e[2], e[3], count_include_pad=False), e[4] if len(e) > 4 else None)
        elif e[0] == "rnorm":
            _, k, a, bpow, act = e
            F_ = h.shape[1]
            sq = Fn.pad(h * h, (0, 0, 0, 0, k // 2, k - k // 2 - 1))
            Ssum = sum(sq[:, j:j + F_] for j in range(k))
            h = _act(torch, h * (1 + a * Ssum) ** (-bpow), act)
        else:
            cout = e[1]
            K = h.shape[1] * h.shape[2] * h.shape[3]
            flat = P[off:off + size].clone()
            w = flat[:cout * K].view(K, cout).clone().requires_grad_(True)
            b = flat[cout * K:cout * K + cout].clone().requires_grad_(True)
            params[i] = (w, b, K)
            h = h.reshape(batch, K) @ w + b
    out = n.model_output_layer(model)
    lf = out["loss_function"]
    if lf == "CROSS_ENTROPY_MULTINOMIAL":
        loss = Fn.cross_entropy(h, labels, reduction="sum")
        value = loss
    elif lf == "CROSS_ENTROPY_BINARY":                     # the derivative is sigma(h) - t where t >= 0
        care = targets >= 0
        tt = torch.where(care, targets, torch.zeros_like(targets))
        loss = (Fn.binary_cross_entropy_with_logits(h, tt, reduction="none") * care).sum()
        y = torch.sigmoid(h)
        value = torch.where(care, -tt * torch.log(y + 1e-10) - (1 - tt) * torch.log(1 - y + 1e-10), torch.zeros_like(y)).sum()
    elif lf == "CROSS_ENTROPY_MULTINOMIAL_DISTRIBUTED":   # the derivative is softmax(h) - t (the targets sum to 1)
        loss = -(targets * Fn.log_softmax(h, 1)).sum()
        value = -(targets * torch.log(torch.softmax(h, 1) + 1e-10)).sum()
    else:
        loss = 0.5 * ((h - targets) ** 2).sum()
        value = loss
    loss.backward()
    return float(value.detach()), params


@pytest.mark.parametrize("model", sorted(MIRRORS))
def test_backprop_matches_float64_autograd(env, model):
    """the chain's backward ops with logistic units (sigma' fused into conv dgrads, as passes after pooling and response
    norm) and each output loss, against an independent float64 autograd model with the same parameters, at batch 128"""
    _, lib, _, net = env
    for mode, tol in (("fp32", 2e-5), ("tf32", 5e-2), ("bf16", 1.5e-1)):
        lib.set_precision(mode)
        batch = 128
        n = net.Net(model, batch, seed=7)
        g = torch.Generator(device="cuda").manual_seed(11)
        n.input_tensor().normal_(generator=g)
        labels, targets = _targets(n, model, batch, g)
        n.fprop(False); n.bprop()
        loss = n.loss()
        ref_loss, params = _mirror(n, model, batch, labels, targets)
        assert abs(loss - ref_loss) / abs(ref_loss) < {"fp32": 1e-5, "tf32": 2e-3, "bf16": 1e-2}[mode], (mode, loss, ref_loss)
        G = n.grads_tensor().double()
        edges = n.edges()
        for i, (w, b, K) in params.items():
            off = edges[i][2]
            cout = b.shape[0]
            gw = G[off:off + cout * K].view(K, cout)
            if w.dim() == 4:
                gw = gw.view(w.shape[1], w.shape[2], w.shape[3], cout).permute(3, 0, 1, 2)
            gb = G[off + cout * K:off + cout * K + cout]
            for nm, mine, ref in (("w", gw, w.grad / batch), ("b", gb, b.grad / batch)):
                if mode == "fp32":
                    err = ((mine - ref).abs().max() / ref.abs().mean().clamp_min(1e-12)).item()
                else:
                    err = ((mine - ref).norm() / ref.norm().clamp_min(1e-12)).item()
                assert err < tol, (model, mode, edges[i][0], nm, err)
        n.close()


@pytest.mark.parametrize("model", ["logcheck", "gradcheck+squared-error", "gradcheck+binary-ce", "gradcheck+soft-targets"])
def test_grad_check(env, model):
    """the reference's run_grad_check criterion (mean scaled difference < 0.01 at the best epsilon) on every edge, except
    logcheck's conv1: its derivative passes four sigma' factors, and in float32 no epsilon of {1e-2, 3e-3, 1e-3} gets both
    the truncation error of the central difference and the rounding noise of the summed loss below 1 % there (0.017 - 0.054
    measured over batches 16 - 256 and two seeds on an H100).  Its gradient is checked against float64 autograd instead
    (test_backprop_matches_float64_autograd[logcheck]); here it must stay within 10 %"""
    _, lib, _, net = env
    lib.set_precision("fp32")
    n = net.Net(model, 16, seed=3, grad_checker=True)
    try:
        res = n.grad_check(seed=6)
        assert len(res) == 3
        for name, eps, dw, db in res:
            bar = 0.1 if (model, name) == ("logcheck", "input:conv1") else 0.01
            assert dw < bar and db < bar, (model, res)
    finally:
        n.close()


@pytest.mark.parametrize("model", ["tiny", "lenet+binary-ce", "tiny+soft-targets", "lenet+squared-error"])
def test_net_metric(env, model):
    _, lib, _, net = env
    lib.set_precision("tf32")
    batch = 96
    n = net.Net(model, batch, seed=2)
    try:
        g = torch.Generator(device="cuda").manual_seed(4)
        n.input_tensor().normal_(generator=g)
        labels, targets = _targets(n, model, batch, g)
        n.fprop(False)
        y = n.output_tensor().double().view(-1, batch).T.cpu().numpy()
        out = n.model_output_layer(model)
        metric = n.metric()
        if out["performance_metric"] == "CLASSIFICATION_MULTINOMIAL":
            ref = R.classification_multinomial(np.float32(y), labels.cpu().numpy()).sum()
            assert metric == ref
        elif out["performance_metric"] == "CLASSIFICATION_BINARY":
            ref = R.classification_binary(np.float32(y), np.float32(targets.cpu().numpy())).sum()
            assert abs(metric - ref) <= 1e-4 * batch
        else:
            code = R.SQUARED_ERROR if out["performance_metric"] == "SQUARED_ERROR" else R.CE_DISTRIBUTED
            _, _, v, v_bar = R.loss_ref(code, y, targets.cpu().numpy())
            assert abs(metric - v.sum()) <= v_bar.sum() + 1e-6 * abs(v.sum())
            assert metric == n.loss()                   # the loss is its own metric here (weight 1)
    finally:
        n.close()


def test_alexnet_logistic_runs_are_bit_identical():
    def run():
        r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "staging_worker.py"), "params", "alexnet+logistic",
                            "64", "3"], capture_output=True, text=True, timeout=900,
                           env={k: v for k, v in os.environ.items() if k != "CONVNET_B200_STAGE_VERIFY"})
        lines = [ln for ln in r.stdout.splitlines() if ln.startswith("PARAMS")]
        assert r.returncode == 0 and lines, (r.returncode, r.stdout[-1000:], r.stderr[-1500:])
        return lines[-1]
    a = run()
    assert all(math.isfinite(float(v)) for v in a.split()[2:])
    assert a == run()


def test_binary_ce_bf16_copies_verify():
    """CONVNET_B200_STAGE_VERIFY=1: every staged bf16 copy a lenet+binary-ce step uses equals a fresh conversion"""
    env = dict(os.environ, CONVNET_B200_STAGE_VERIFY="1")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "staging_worker.py"), "train", "lenet+binary-ce", "128",
                        "3"], capture_output=True, text=True, timeout=900, env=env)
    assert r.returncode == 0 and "VERIFY-TRAIN-OK" in r.stdout, (r.returncode, r.stdout[-1500:], r.stderr[-1500:])


@pytest.mark.parametrize("model,mode", [("tiny+bn+logistic", "bf16"), ("tiny+bn+logistic", "fp32"),
                                        ("lenet+binary-ce", "bf16"), ("tiny+soft-targets", "tf32")])
def test_training_reduces_the_loss(env, model, mode):
    _, lib, _, net = env
    lib.set_precision(mode)
    batch = 64
    n = net.Net(model, batch, seed=1)
    try:
        g = torch.Generator(device="cuda").manual_seed(0)
        n.input_tensor().normal_(generator=g)
        _targets(n, model, batch, g)
        losses = [n.train_step(True) / batch for _ in range(60)]
        assert all(math.isfinite(v) for v in losses)
        assert min(losses[30:]) < 0.9 * losses[0], losses[::6]
    finally:
        n.close()


def test_data_parallel_binary_ce_replicas_identical(tmp_path):
    """2 ranks of lenet+binary-ce over NCCL: the replicas stay bit-identical"""
    ngpu = torch.cuda.device_count()
    if ngpu < 2:
        pytest.skip("needs >= 2 GPUs")
    code = r"""
import os, sys, json, torch, torch.distributed as dist
sys.path.insert(0, %r)
from convnet_b200 import lib
from convnet_b200.net import Net, dp_unique_id
rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
torch.cuda.set_device(local)
dist.init_process_group("nccl", device_id=torch.device("cuda", local))
lib.load(); lib.set_precision("bf16")
net = Net("lenet+binary-ce", 64, seed=7)
idt = torch.zeros(128, dtype=torch.uint8, device="cuda")
if rank == 0:
    idt.copy_(torch.frombuffer(bytearray(dp_unique_id()), dtype=torch.uint8))
dist.broadcast(idt, 0)
net.dp_init(rank, world, bytes(idt.cpu().numpy().tobytes()), 4096)
g = torch.Generator(device="cuda").manual_seed(rank)
for s in range(3):
    net.input_tensor().normal_(generator=g)
    net.targets_tensor().copy_((torch.rand(net.targets_tensor().numel(), device="cuda", generator=g) < 0.5).float())
    net.train_step(False)
torch.cuda.synchronize()
p = net.params_tensor().clone()
gathered = [torch.empty_like(p) for _ in range(world)]
dist.all_gather(gathered, p)
if rank == 0:
    print(json.dumps({"identical": all(torch.equal(gathered[0], t) for t in gathered)}), flush=True)
net.close()
dist.destroy_process_group()
""" % ROOT
    worker = tmp_path / "binary_ce_dp_worker.py"
    worker.write_text(code)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
           "--master-addr", "127.0.0.1", "--master-port", "29523", str(worker)]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900)
    line = [ln for ln in r.stdout.splitlines() if ln.startswith("{")]
    assert r.returncode == 0 and line, (r.returncode, r.stdout[-2000:], r.stderr[-2000:])
    assert json.loads(line[-1])["identical"]
