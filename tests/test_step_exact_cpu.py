"""The step auditor (tests/step_exact.py) without a GPU: it passes a float32 torch step of `tiny` and `gradcheck` (and
of `tiny` with dropout on its 1x1 layer, with logistic units, with each target-trained output layer, with Adagrad or
RMSProp, on a frozen trunk, and of `logcheck`, `tiednet` and a small 3-D net), and it fails every single injected fault, naming the layer
and quantity.

The snapshot is made the way the net makes one: torch float32 forward and autograd backward in the library's layouts,
with the fusion plan's semantics (each layer's derivative is the loss gradient at its pre-activation, ReLU' or sigma'
and the dropout mask applied; weight and bias gradients scaled by 1 / batch, a tie group's summed over its members; the
output derivative p - onehot or y - t, 0 at don't-care binary targets), then the optimizer step of every trained weight
and bias tensor.  Frozen edges get no gradient (the sentinel stays), no step, and the layers they write no derivative."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as tF

import abi_rest_exact as ax
import conv_exact as cx
import loss_ref as lr
import opt_rules as opt
import step_exact as se
from convnet_b200 import net


def _nchw(flat, N, C, H, W):
    return cx._act(flat, N, W, H, C)


def _frames(h, T):
    """(N, C*T, H, W) with frames as channel blocks -> (N, C, T, H, W)"""
    N, CT, H, W = h.shape
    return h.view(N, T, CT // T, H, W).transpose(1, 2)


def _unframes(z):
    """(N, C, T, H, W) -> (N, C*T, H, W), frame t at channels [C*t, C*t + C)"""
    N, C, T, H, W = z.shape
    return z.transpose(1, 2).reshape(N, T * C, H, W)


def _flat(t):
    return cx._unact(t).contiguous()


def _rnorm(x, k, alpha, beta, blocked):
    """x (N, C, H, W) float32: x * (1 + alpha * sum of squares over the channel window)^-beta"""
    C = x.shape[1]
    sq = x * x
    if blocked:
        j = torch.arange(C)
        lo = (j // k) * k
        hi = torch.clamp(lo + k, max=C)
    else:
        a = k // 2
        j = torch.arange(C)
        lo, hi = torch.clamp(j - a, min=0), torch.clamp(j + k - a, max=C)
    S = torch.stack([sq[:, int(lo[c]):int(hi[c])].sum(1) for c in range(C)], 1)
    return x * (1.0 + alpha * S) ** -beta


def simulate(model, N, seed=0, seeds=None, lr_scale=1.0, fprop_operands=None, fault=None):
    """a Snapshot of one float32 step of `model` (a step_exact.Model).  seeds: per layer dropout seed (default: drawn);
    fprop_operands: {edge index: operand-model kind} rounds that edge's fprop operands like a tensor-core path;
    fault: 'relu_deriv' takes ReLU' instead of sigma' at every logistic layer, 'labels_deriv' makes a soft-target
    output derivative against one-hot labels, 'adagrad_twice' adds the squared gradient to the Adagrad state twice,
    'frame_offset' starts the frame windows of every 3-D conv one frame apart instead of stride_t, 'drop_last_window'
    leaves the last frame window of every 3-D pool unwritten (0)"""
    g = torch.Generator().manual_seed(seed)
    m = model
    L = len(m.layers)
    params = torch.zeros(m.total, dtype=torch.float32)
    hist = torch.zeros(m.total, dtype=torch.float32)
    for k, e in enumerate(m.edges):
        if e.kind in se.WEIGHTED:
            gg = m.conv_geo(e, N)
            (w0, w1), bs = m.weight_slices(k, N)
            params[w0:w1] = torch.randn(w1 - w0, generator=g) / math.sqrt(gg.K)
            hist[w0:w1] = torch.randn(w1 - w0, generator=g) * 1e-3
            if bs:
                params[bs[0]:bs[1]] = torch.randn(bs[1] - bs[0], generator=g) * 0.1
                hist[bs[0]:bs[1]] = torch.randn(bs[1] - bs[0], generator=g) * 1e-3
    if seeds is None:
        seeds = [int(s) for s in torch.randint(1, 2 ** 62, (L,), generator=g)]
        seeds = [s if m.layers[i].dropprob > 0 else 0 for i, s in enumerate(seeds)]
    labels = torch.randint(0, m.layers[-1].C, (N,), generator=g)
    targets = None
    if m.loss != lr.CE_MULTINOMIAL:
        targets = se.make_targets(m.loss, N, m.layers[-1].floats(N) // N, g).reshape(-1)
    l0 = m.layers[0]
    x = torch.randn(l0.floats(N), generator=g)

    P = params.clone().requires_grad_(True)
    states, zs = [x], [None]
    h = _nchw(x, N, l0.C * l0.T, l0.H, l0.W)
    for k, e in enumerate(m.edges):
        s, d = m.layers[e.src], m.layers[e.dst]
        if e.kind in se.WEIGHTED:
            gg = m.conv_geo(e, N)
            (w0, w1), bs = m.weight_slices(k, N)
            W, b = P[w0:w1], P[bs[0]:bs[1]]
            xin = h
            if fprop_operands and k in fprop_operands:
                kind = fprop_operands[k]
                W = cx.MODELS[kind](W.detach()) + (W - W.detach())
                xin = cx.MODELS[kind](h.detach()) + (h - h.detach())
            if e.kind == "FC":
                z = (_flat(xin).view(-1, N).t() @ W.view(gg.K, gg.Cout) + b).view(N, d.C, 1, 1)
            elif s.T > 1:                   # filter column c + Cin*dt: channel c of window frame dt
                wt = W.view(gg.kt, gg.Cin, gg.ky, gg.kx, gg.Cout).permute(4, 1, 0, 2, 3)
                st_t = 1 if fault == "frame_offset" else gg.st_t
                z = tF.conv3d(_frames(xin, s.T), wt, b, stride=(st_t, gg.sy, gg.sx), padding=(0, gg.py, gg.px))
                z = _unframes(z[:, :, :d.T])
            else:
                wt = W.view(gg.Cin, gg.ky, gg.kx, gg.Cout).permute(3, 0, 1, 2)
                z = tF.conv2d(xin, wt, b, stride=(gg.sy, gg.sx), padding=(gg.py, gg.px))
        elif e.kind == "RGBTOYUV":
            z = torch.einsum("ij,njhw->nihw", torch.tensor(ax.YUV, dtype=torch.float32), h)
        elif e.kind == "UPSAMPLE":
            f = int(e.cfg["sample_factor"])
            z = h.repeat_interleave(f, 2).repeat_interleave(f, 3)
        elif e.kind == "DOWNSAMPLE":
            f = int(e.cfg["sample_factor"])
            z = tF.avg_pool2d(h, f, f)
        elif e.kind in ("MAXPOOL", "AVERAGE_POOL") and s.T > 1:
            pg = m.pool_geo(e, N)
            win = dict(kernel_size=(pg.kt, pg.ky, pg.kx), stride=(pg.st_t, pg.sy, pg.sx), padding=(pg.pt, pg.py, pg.px))
            assert e.kind == "AVERAGE_POOL" or not any(win["padding"]) and all(          # windows that do not overlap
                st == k or k == n for st, k, n in zip(win["stride"], win["kernel_size"], (s.T, s.H, s.W)))
            z = (_MaxPool3dTies.apply(_frames(h, s.T), win["kernel_size"]) if e.kind == "MAXPOOL" else
                 tF.avg_pool3d(_frames(h, s.T), count_include_pad=False, **win))
            if fault == "drop_last_window":         # the last frame window never computed
                z = torch.cat([z[:, :, :-1], torch.zeros_like(z[:, :, -1:])], 2)
            z = _unframes(z)
        elif e.kind == "MAXPOOL":
            pg = m.pool_geo(e, N)
            z = tF.max_pool2d(h, (pg.ky, pg.kx), (pg.sy, pg.sx), (pg.py, pg.px))
        elif e.kind == "AVERAGE_POOL":
            pg = m.pool_geo(e, N)
            z = tF.avg_pool2d(h, (pg.ky, pg.kx), (pg.sy, pg.sx), (pg.py, pg.px), count_include_pad=False)
        else:
            c = e.cfg
            kk = int(np.float32(c["frac_of_filters_response_norm"]) * np.float32(s.C))
            z = _rnorm(h, kk, se.f32(c["add_scale"]), se.f32(c["pow_scale"]), bool(c["response_norm_in_blocks"]))
        if z.requires_grad:                 # (not the RGBTOYUV output: nothing below it is trained)
            z.retain_grad()
        zs.append(z)
        if d.act == "RECTIFIED_LINEAR":
            h = torch.relu(z)
        elif d.act in ("SOFTMAX", "SOFTMAX_DIST"):
            h = torch.softmax(z, 1)
        elif d.act == "LOGISTIC" and fault == "relu_deriv" and e.dst < L - 1:
            h = _LogisticReluDeriv.apply(z)
        elif d.act == "LOGISTIC":
            h = torch.sigmoid(z)
        else:
            h = z
        if d.dropprob > 0:
            kept = cx.dropout_kept(d.floats(N), np.float32(d.dropprob), seeds[e.dst])
            mask = torch.from_numpy(kept).float() * se.dropout_scale(d.dropprob)
            h = h * _nchw(mask, N, d.C * d.T, d.H, d.W)
        states.append(_flat(h.detach()))
    C = m.layers[-1].floats(N) // N           # output features (units x pixels), image fastest like the targets
    p = _flat(h.detach()).view(C, N).t()
    t = None if targets is None else targets.view(C, N).t()
    if fault == "labels_deriv":
        t = None
    # the output derivative at the pre-activation: y - onehot, y - t (don't-care entries 0), times the loss weight
    dz = p - (tF.one_hot(labels, C).float() if t is None else t)
    if m.loss == lr.CE_BINARY:
        dz = torch.where(targets.view(C, N).t() >= 0, dz, torch.zeros_like(dz))
    dz = dz * m.loss_weight
    _, _, v, _ = lr.loss_ref(m.loss, p.double().numpy(), t=None if targets is None else targets.view(C, N).t().numpy(),
                             labels=labels.numpy(), weight=m.loss_weight)
    loss = float(m.loss_weight * v.sum())
    zs[-1].backward(_nchw(dz.t().reshape(-1), N, m.layers[-1].C * m.layers[-1].T, m.layers[-1].H, m.layers[-1].W))
    derivs = [None] + [_flat(z.grad) if m.receives_deriv(i + 1) else None for i, z in enumerate(zs[1:])]
    grads = torch.full((m.total,), float("nan"))
    grads.view(torch.int32).fill_(se.SENTINEL)
    for k, e in enumerate(m.edges):
        if e.kind in se.WEIGHTED and k >= m.frozen:
            (w0, w1), bs = m.weight_slices(k, N)
            grads[w0:w1] = P.grad[w0:w1] / N
            grads[bs[0]:bs[1]] = P.grad[bs[0]:bs[1]] / N
    opt_state = {}
    p_after, h_after = params.clone(), hist.clone()
    adaptive = any(se.RULES[m.edges[k].cfg[key][0].get("optimizer_type", "STOCHASTIC_GRADIENT_DESCENT")] != opt.SGD
                   for k in range(len(m.edges)) if m.edges[k].kind in se.WEIGHTED and m.owner[k] == k
                   for key in ("weight_optimizer", "bias_optimizer"))
    s_before = (torch.rand(m.total, generator=g) + 0.5) if adaptive else None
    s_after = None if s_before is None else s_before.clone()
    for k, e in enumerate(m.edges):
        if e.kind not in se.WEIGHTED or k < m.frozen or m.owner[k] != k:      # (a tie group is updated once)
            continue
        opt_state[k] = {}
        (w0, w1), bs = m.weight_slices(k, N)
        for which, (a, b) in (("weights", (w0, w1)), ("bias", bs)):
            cfg = net.model_edge_optimizer(m.name, k, which)
            eps, mom = net.optimizer_schedule(cfg, 0)
            eps = se.f32(eps * lr_scale)
            opt_state[k][which] = {"step": 0, "epsilon": eps, "momentum": mom}
            rule = {0: opt.SGD, 2: opt.ADAGRAD, 3: opt.RMSPROP}[cfg["optimizer_type"]]     # (proto OptimizerType)
            param = cfg["adagrad_delta"] if rule == opt.ADAGRAD else cfg["rms_prop_factor"]
            st = None if rule == opt.SGD else s_before[a:b].numpy()
            if fault == "adagrad_twice" and rule == opt.ADAGRAD:
                st = opt.adagrad_state(st, grads[a:b].numpy(), param)
            w, hh, st = opt.opt_update(params[a:b].numpy(), hist[a:b].numpy(), st, grads[a:b].numpy(), rule, lr=eps,
                                       mom=mom, l2=max(cfg["l2_decay"], 0.0), clip=max(cfg["gradient_clip"], 0.0),
                                       param=param, scale=opt.adagrad_scale(0))
            p_after[a:b], h_after[a:b] = torch.from_numpy(w), torch.from_numpy(hh)
            if st is not None:
                s_after[a:b] = torch.from_numpy(st)
    return se.Snapshot(N, labels, states, derivs, params, hist, grads, p_after, h_after, loss, seeds, opt_state,
                       targets, s_before, s_after)


class _MaxPool3dTies(torch.autograd.Function):
    """3-D max pooling over non-overlapping windows whose backward gives the gradient to EVERY element equal to its
    window's maximum, as the reference's undo does (torch's picks one; ReLU layers tie at 0, often a whole window)"""

    @staticmethod
    def forward(ctx, x, k):
        z = tF.max_pool3d(x, k, k)
        ctx.save_for_backward(x, z)
        ctx.k = k
        return z

    @staticmethod
    def backward(ctx, dz):
        x, z = ctx.saved_tensors
        up = lambda t: t.repeat_interleave(ctx.k[0], 2).repeat_interleave(ctx.k[1], 3).repeat_interleave(  # noqa: E731
            ctx.k[2], 4)[:, :, :x.shape[2], :x.shape[3], :x.shape[4]]
        return torch.where(x == up(z), up(dz), torch.zeros_like(x)), None


class _LogisticReluDeriv(torch.autograd.Function):
    """sigma forward, ReLU' backward (a logistic layer whose derivative pass takes the ReLU rule)"""

    @staticmethod
    def forward(ctx, z):
        y = torch.sigmoid(z)
        ctx.save_for_backward(y)
        return y

    @staticmethod
    def backward(ctx, dy):
        y, = ctx.saved_tensors
        return dy * (y > 0).float()


def _sample_dropout_model(tmp_path):
    path = str(tmp_path / "updowndrop.pbtxt")
    with open(path, "w") as f:
        f.write(se.sample_dropout_text())
    return path


def _dropout_model(tmp_path):
    """tiny with dropout 0.25 on its 1x1 layer nin1 (a ReLU layer below a conv edge: fused dropout, folded scale)"""
    t = net.model_text("tiny")
    i = t.index('name: "nin1"')
    j = t.index("dropprob: 0", i)
    t = t[:j] + "dropprob: 0.25" + t[j + len("dropprob: 0"):]
    path = str(tmp_path / "tinydrop.pbtxt")
    with open(path, "w") as f:
        f.write(t)
    return path


@pytest.fixture(scope="module")
def drop_model(tmp_path_factory):
    path = _dropout_model(tmp_path_factory.mktemp("model"))
    return se.load_model(path, 32)


def _audit(model, snap, mode="fp32"):
    return se.Auditor(model, mode).audit(snap)


@pytest.mark.parametrize("name,N", [("tiny", 32), ("gradcheck", 32)])
def test_auditor_passes_a_float32_step(name, N):
    m = se.load_model(name, N)
    rows = _audit(m, simulate(m, N))
    for r in rows:
        print(r)
    assert not se.failures(rows), "\n".join(map(str, se.failures(rows)))
    kinds = {(r.quantity) for r in rows}
    assert {"fprop", "dgrad", "wgrad", "bias_grad", "undo", "softmax", "output_deriv", "loss", "update_weights",
            "history_bias"} <= kinds


def test_auditor_passes_dropout_step(drop_model):
    s = simulate(drop_model, 32)
    assert s.seeds[4] != 0 and drop_model.layers[4].name == "nin1"
    rows = _audit(drop_model, s)
    assert not se.failures(rows), "\n".join(map(str, se.failures(rows)))


def _layer_index(m, name):
    return [l.name for l in m.layers].index(name)


def _edge_index(m, name):
    return [l.name for l in m.layers].index(name) - 1


def _bump(t, i, rel=2.0 ** -8):
    t[i] = t[i] * (1 + rel) if t[i] != 0 else 1e-3


def _nonzero(t):
    return int(torch.nonzero(t)[len(torch.nonzero(t)) // 2])


def _flip_lsb(t, i):
    v = t[i:i + 1].view(torch.int32)
    v ^= 1


def _caught(m, s, layer, qty, mode="fp32"):
    fails = se.failures(_audit(m, s, mode))
    assert (layer, qty) in {(r.layer, r.quantity) for r in fails}, (layer, qty, [str(r) for r in fails])


FAULTS = ["state", "deriv", "wgrad", "bias_grad", "param", "history", "bias_twice"]


@pytest.mark.parametrize("fault", FAULTS)
def test_single_element_faults_are_caught(drop_model, fault):
    m = drop_model
    s = simulate(m, 32)
    k = _edge_index(m, "conv2")
    (w0, w1), bs = m.weight_slices(k, 32)
    if fault == "state":
        t = s.states[_layer_index(m, "conv2")]
        _bump(t, _nonzero(t))
        _caught(m, s, "conv2", "fprop")
    elif fault == "deriv":
        t = s.derivs[_layer_index(m, "rnorm1")]
        _bump(t, _nonzero(t))
        _caught(m, s, "rnorm1", "dgrad")
    elif fault == "wgrad":
        _bump(s.grads, w0 + 7)
        _caught(m, s, m.edges[k].name, "wgrad")
    elif fault == "bias_grad":
        _bump(s.grads, bs[0] + 3)
        _caught(m, s, m.edges[k].name, "bias_grad")
    elif fault == "param":
        _flip_lsb(s.params_after, w0 + 11)
        _caught(m, s, m.edges[k].name, "update_weights")
    elif fault == "history":
        _flip_lsb(s.hist_after, bs[0] + 1)
        _caught(m, s, m.edges[k].name, "history_bias")
    else:                                   # the bias gradient summed twice (side lane and pool undo both adding)
        kc = _edge_index(m, "conv1")
        _, b1 = m.weight_slices(kc, 32)
        s.grads[b1[0]:b1[1]] *= 2
        _caught(m, s, m.edges[kc].name, "bias_grad")


def test_dropout_scale_left_out_of_folded_dgrad(drop_model):
    m = drop_model
    s = simulate(m, 32)
    i = _layer_index(m, "nin1")
    s.derivs[i] /= se.dropout_scale(m.layers[i].dropprob)
    _caught(m, s, "nin1", "dgrad")


def test_dropout_mask_from_wrong_seed(drop_model):
    m = drop_model
    s = simulate(m, 32)
    i = _layer_index(m, "nin1")
    wrong = list(s.seeds)
    wrong[i] += 1
    bad = simulate(m, 32, seeds=wrong)
    bad.seeds = s.seeds
    _caught(m, bad, "nin1", "fprop")


def test_dgrad_from_updated_weights(drop_model):
    """the dgrad of conv2 into nin1 recomputed with the weights after the step (a filter bank rebuilt too early)"""
    m = drop_model
    s = simulate(m, 32, lr_scale=10.0)
    k = _edge_index(m, "conv2")
    i = m.edges[k].src
    g = m.conv_geo(m.edges[k], 32)
    (w0, w1), _ = m.weight_slices(k, 32)
    ok = se.Auditor(m, "fp32").dgrad(s, k)[0]
    assert ok.ok, str(ok)
    e = cx.expect("dgrad", g, s.derivs[i + 1], s.params_after[w0:w1], "fp32", so=se.dropout_scale(0.25),
                  mask=s.states[i])
    s.derivs[i] = e.ref.to(torch.float32)
    _caught(m, s, "nin1", "dgrad")


def test_bf16_operand_truncated_instead_of_rounded():
    """conv2's fprop on the bf16 path (Cin 24, N 32): operands rounded to nearest pass, truncated ones fail"""
    m = se.load_model("tiny", 32)
    k = _edge_index(m, "conv2")
    assert cx.conv_path("fprop", m.conv_geo(m.edges[k], 32), "bf16") == "tc-bf16"
    good = simulate(m, 32, fprop_operands={k: "bf16"})
    r, control = se.Auditor(m, "bf16").fprop(good, k)
    assert r.ok and control.ok, (str(r), str(control))
    bad = simulate(m, 32, fprop_operands={k: "bf16_trunc"})
    r = se.Auditor(m, "bf16").fprop(bad, k)[0]
    assert not r.ok and (r.layer, r.quantity) == ("conv2", "fprop"), str(r)


# the kinds beyond SGD chains of ReLU / linear layers with a softmax output: logistic units, the target-trained output
# layers, the adaptive optimizers and frozen trunks
NEW_KINDS = [("tiny+logistic", 32), ("logcheck", 32), ("tiny+squared-error", 32), ("tiny+binary-ce", 32),
             ("tiny+soft-targets", 32), ("tiny+adagrad", 32), ("tiny+rmsprop", 32), ("tiny+finetune", 32),
             ("tiny+logistic+adagrad+finetune", 32), ("tiednet", 8), ("updowncheck", 32), ("updown", 2)]


@pytest.mark.parametrize("name,N", NEW_KINDS)
def test_auditor_passes_new_kinds(name, N):
    m = se.load_model(name, N)
    rows = _audit(m, simulate(m, N))
    assert not se.failures(rows), "\n".join(map(str, se.failures(rows)))
    kinds = {r.quantity for r in rows}
    assert {"output_deriv", "loss"} <= kinds
    if "adagrad" in name or "rmsprop" in name:
        assert {"state_weights", "state_bias"} <= kinds
    if "finetune" in name:
        assert {"frozen_params", "frozen_history", "frozen_grads", "frozen_deriv"} <= kinds
        assert not any(r.quantity in ("dgrad", "undo") and r.layer in ("conv1", "pool1", "rnorm1", "nin1", "conv2")
                       for r in rows)


def test_sigma_deriv_replaced_by_relu_deriv():
    """logcheck with ReLU' (1 everywhere on a logistic layer) where sigma' belongs: the dgrad of the 1x1 edge into rnorm1
    and the undos into the logistic pooling layers fail"""
    m = se.load_model("logcheck", 32)
    s = simulate(m, 32, fault="relu_deriv")
    _caught(m, s, "rnorm1", "dgrad")
    _caught(m, s, "pool1", "undo")


def test_sigma_left_out_of_logistic_fprop():
    m = se.load_model("tiny+logistic", 32)
    s = simulate(m, 32)
    i = _layer_index(m, "conv2")
    k = _edge_index(m, "conv2")
    e = cx.expect("fprop", m.conv_geo(m.edges[k], 32), s.states[i - 1], se.Auditor(m, "fp32").weights(
        s.params_before, k, 32)[0], "fp32", bias=se.Auditor(m, "fp32").weights(s.params_before, k, 32)[1])
    s.states[i] = e.ref.to(torch.float32)
    _caught(m, s, "conv2", "fprop")


@pytest.mark.parametrize("name", ["tiny+squared-error", "tiny+binary-ce", "tiny+soft-targets"])
def test_output_derivative_against_labels(name):
    """the output derivative taken against one-hot labels instead of the layer's float targets"""
    m = se.load_model(name, 32)
    _caught(m, simulate(m, 32, fault="labels_deriv"), "output", "output_deriv")


def test_binary_dont_care_targets_get_a_derivative():
    m = se.load_model("tiny+binary-ce", 32)
    s = simulate(m, 32)
    care = s.targets >= 0
    assert 0 < int((~care).sum()) < care.numel() // 4
    i = int(torch.nonzero(~care)[0])
    s.derivs[-1][i] = s.states[-1][i] - 0.5
    _caught(m, s, "output", "output_deriv")


def test_adagrad_state_updated_twice():
    m = se.load_model("tiny+adagrad", 32)
    _caught(m, simulate(m, 32, fault="adagrad_twice"), m.edges[_edge_index(m, "conv2")].name, "state_weights")


def test_frozen_weight_changed_by_one_ulp():
    m = se.load_model("tiny+finetune", 32)
    assert m.frozen == 6 and m.trained_offset == m.offsets[6]
    s = simulate(m, 32)
    k = _edge_index(m, "conv2")
    (w0, _), _ = m.weight_slices(k, 32)
    _flip_lsb(s.params_after, w0 + 5)
    _caught(m, s, m.edges[k].name, "frozen_params")


@pytest.mark.parametrize("name,which", [("tiny+adagrad", "weights"), ("tiny+adagrad", "bias"),
                                        ("tiny+rmsprop", "weights"), ("tiny+rmsprop", "bias")])
def test_adaptive_state_off_by_one_ulp(name, which):
    m = se.load_model(name, 32)
    s = simulate(m, 32)
    k = _edge_index(m, "nin1")
    (w0, _), bs = m.weight_slices(k, 32)
    _flip_lsb(s.state_after, (w0 if which == "weights" else bs[0]) + 1)
    _caught(m, s, m.edges[k].name, "state_" + which)


@pytest.mark.parametrize("qty", ["frozen_history", "frozen_state"])
def test_frozen_history_or_state_changed_by_one_ulp(qty):
    m = se.load_model("tiny+logistic+adagrad+finetune", 32)
    s = simulate(m, 32)
    k = _edge_index(m, "nin1")
    (w0, _), _ = m.weight_slices(k, 32)
    _flip_lsb(s.hist_after if qty == "frozen_history" else s.state_after, w0 + 3)
    _caught(m, s, m.edges[k].name, qty)


def test_frozen_gradient_written():
    m = se.load_model("tiny+finetune", 32)
    s = simulate(m, 32)
    k = _edge_index(m, "conv1")
    (w0, _), _ = m.weight_slices(k, 32)
    s.grads[w0 + 2] = 0.0
    _caught(m, s, m.edges[k].name, "frozen_grads")
    s = simulate(m, 32)
    s.derivs[_layer_index(m, "nin1")] = torch.zeros_like(s.states[_layer_index(m, "nin1")])
    _caught(m, s, "nin1", "frozen_deriv")


def test_tie_group_missing_a_member():
    """tiednet's conv group (conv1:conv2 with pool2:conv3 and conv3:conv4) trained on two of its three wgrads"""
    m = se.load_model("tiednet", 8)
    s = simulate(m, 8)
    assert not se.failures(_audit(m, s))
    o = _edge_index(m, "conv2")
    assert m.group(o) == [1, 3, 4] and m.owner[4] == o
    e = m.edges[4]
    (w0, w1), _ = m.weight_slices(4, 8)
    assert m.weight_slices(o, 8)[0] == (w0, w1)
    miss = cx.expect("wgrad", m.conv_geo(e, 8), s.states[e.src], s.derivs[e.dst], "fp32", so=1.0 / 8)
    s.grads[w0:w1] -= miss.ref.to(torch.float32)
    _caught(m, s, m.edges[o].name, "wgrad")


@pytest.fixture(scope="module")
def sample_drop_model(tmp_path_factory):
    path = _sample_dropout_model(tmp_path_factory.mktemp("model"))
    return se.load_model(path, 32)


def test_auditor_passes_sampling_dropout_step(sample_drop_model):
    m = sample_drop_model
    s = simulate(m, 32)
    assert s.seeds[_layer_index(m, "down1")] and s.seeds[_layer_index(m, "up4")]
    rows = _audit(m, s)
    assert not se.failures(rows), "\n".join(map(str, se.failures(rows)))
    assert {("down1", "fprop"), ("down1", "dgrad"), ("up4", "fprop"), ("up4", "dgrad"), ("conv3", "undo")} <= {
        (r.layer, r.quantity) for r in rows}


def test_sampling_dropout_faults(sample_drop_model):
    """a dropout scale left out of the DOWNSAMPLE and UPSAMPLE fprops, and the dropout fold left out of the DOWNSAMPLE
    undo into conv3"""
    m = sample_drop_model
    for name in ("down1", "up4"):
        s = simulate(m, 32)
        s.states[_layer_index(m, name)] /= se.dropout_scale(0.25)
        _caught(m, s, name, "fprop")
    s = simulate(m, 32)
    s.derivs[_layer_index(m, "conv3")] /= se.dropout_scale(0.25)
    _caught(m, s, "conv3", "undo")


def test_upsample_backward_without_f2():
    """the derivative into conv2 (below up2, f = 3) as the block mean instead of the block sum"""
    m = se.load_model("updowncheck", 32)
    s = simulate(m, 32)
    s.derivs[_layer_index(m, "conv2")] /= 9
    _caught(m, s, "conv2", "undo")


def test_yuv_row_swapped():
    """RGBTOYUV with its U and V rows exchanged"""
    m = se.load_model("updown", 2)
    s = simulate(m, 2)
    y = s.states[_layer_index(m, "yuv")].view(3, -1)
    s.states[_layer_index(m, "yuv")] = y[[0, 2, 1]].reshape(-1).clone()
    _caught(m, s, "yuv", "fprop")
    s = simulate(m, 2)
    s.derivs[_layer_index(m, "yuv")] = torch.zeros_like(s.states[_layer_index(m, "yuv")])
    _caught(m, s, "yuv", "no_deriv")


def test_tie_group_bias_missing_a_member():
    """tiednet's FC pair (fc5:fc6 tied to fc6:fc7): the bias gradient from the owner's column sum alone"""
    m = se.load_model("tiednet", 8)
    s = simulate(m, 8)
    o = _edge_index(m, "fc7")
    assert m.group(o) == [6, 7]
    e = m.edges[6]
    d = m.layers[e.dst]
    _, bs = m.weight_slices(o, 8)
    miss = s.derivs[e.dst].double().view(d.C, -1).sum(1) / 8
    s.grads[bs[0]:bs[1]] -= miss.to(torch.float32)
    _caught(m, s, m.edges[o].name, "bias_grad")


@pytest.fixture(scope="module")
def video_model(tmp_path_factory):
    path = str(tmp_path_factory.mktemp("model") / "video.pbtxt")
    with open(path, "w") as f:
        f.write(se.video_text())
    return se.load_model(path, 4)


def test_auditor_passes_3d_step(video_model):
    """the small 3-D net: a conv with frame windows of 2, one of 3 at stride_t 2, 3-D max, average and global pools"""
    m = video_model
    assert [l.T for l in m.layers] == [8, 7, 7, 3, 2, 1, 1]
    rows = _audit(m, simulate(m, 4))
    assert not se.failures(rows), "\n".join(map(str, se.failures(rows)))
    got = {(r.layer, r.quantity) for r in rows}
    assert {("conv2", "fprop"), ("pool1", "dgrad"), ("pool1:conv2", "wgrad"), ("pool1:conv2", "bias_grad"),
            ("pool2", "fprop"), ("conv2", "undo"), ("pool3", "fprop"), ("pool2", "undo")} <= got
    assert "sum over 3 frames" in [r for r in rows if (r.layer, r.quantity) == ("pool1:conv2", "bias_grad")][0].detail


def test_3d_conv_frame_offset_without_stride_t(video_model):
    """conv2's frame windows started one frame apart instead of stride_t = 2 frames"""
    _caught(video_model, simulate(video_model, 4, fault="frame_offset"), "conv2", "fprop")


def test_3d_pool_drops_its_last_frame_window(video_model):
    """the last frame window of the 3-D max pool (pool1: 7 frames) and average pool (pool2: 2 windows of 2 frames)
    never written"""
    s = simulate(video_model, 4, fault="drop_last_window")
    _caught(video_model, s, "pool1", "fprop")
    _caught(video_model, s, "pool2", "fprop")


@pytest.mark.parametrize("name", ["tiny+bn", "lcnet", "tiedcheck", "localcheck"])
def test_unsupported_models_raise(name):
    with pytest.raises(se.Unsupported):
        se.load_model(name, 32)
