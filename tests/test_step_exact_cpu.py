"""The step auditor (tests/step_exact.py) without a GPU: it passes a float32 torch step of `tiny` and `gradcheck` (and
of `tiny` with dropout on its 1x1 layer), and it fails every single injected fault, naming the layer and quantity.

The snapshot is made the way the net makes one: torch float32 forward and autograd backward in the library's layouts,
with the fusion plan's semantics (each layer's derivative is the loss gradient at its pre-activation, ReLU' and the
dropout mask applied; weight and bias gradients scaled by 1 / batch; the output derivative p - onehot), then the SGD
step of every weight and bias tensor."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as tF

import conv_exact as cx
import opt_rules as opt
import step_exact as se
from convnet_b200 import net


def _nchw(flat, N, C, H, W):
    return cx._act(flat, N, W, H, C)


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


def simulate(model, N, seed=0, seeds=None, lr_scale=1.0, fprop_operands=None):
    """a Snapshot of one float32 step of `model` (a step_exact.Model).  seeds: per layer dropout seed (default: drawn);
    fprop_operands: {edge index: operand-model kind} rounds that edge's fprop operands like a tensor-core path"""
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
    l0 = m.layers[0]
    x = torch.randn(l0.floats(N), generator=g)

    P = params.clone().requires_grad_(True)
    states, zs = [x], [None]
    h = _nchw(x, N, l0.C, l0.H, l0.W)
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
            else:
                wt = W.view(gg.Cin, gg.ky, gg.kx, gg.Cout).permute(3, 0, 1, 2)
                z = tF.conv2d(xin, wt, b, stride=(gg.sy, gg.sx), padding=(gg.py, gg.px))
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
        z.retain_grad()
        zs.append(z)
        if d.act == "RECTIFIED_LINEAR":
            h = torch.relu(z)
        elif d.act == "SOFTMAX":
            h = torch.softmax(z, 1)
        else:
            h = z
        if d.dropprob > 0:
            kept = cx.dropout_kept(d.floats(N), np.float32(d.dropprob), seeds[e.dst])
            mask = torch.from_numpy(kept).float() * se.dropout_scale(d.dropprob)
            h = h * _nchw(mask, N, d.C, d.H, d.W)
        states.append(_flat(h.detach()))
    p = h.detach().reshape(N, -1)
    onehot = tF.one_hot(labels, p.shape[1]).float()
    loss = float(-torch.log(p[torch.arange(N), labels]).sum())
    zs[-1].backward((p - onehot).reshape(zs[-1].shape))
    derivs = [None] + [_flat(z.grad) for z in zs[1:]]
    grads = torch.zeros(m.total, dtype=torch.float32)
    for k, e in enumerate(m.edges):
        if e.kind in se.WEIGHTED:
            (w0, w1), bs = m.weight_slices(k, N)
            grads[w0:w1] = P.grad[w0:w1] / N
            grads[bs[0]:bs[1]] = P.grad[bs[0]:bs[1]] / N
    opt_state = {}
    p_after, h_after = params.clone(), hist.clone()
    for k, e in enumerate(m.edges):
        if e.kind not in se.WEIGHTED:
            continue
        opt_state[k] = {}
        (w0, w1), bs = m.weight_slices(k, N)
        for which, (a, b) in (("weights", (w0, w1)), ("bias", bs)):
            cfg = net.model_edge_optimizer(m.name, k, which)
            eps, mom = net.optimizer_schedule(cfg, 0)
            eps = se.f32(eps * lr_scale)
            opt_state[k][which] = {"step": 0, "epsilon": eps, "momentum": mom}
            w, hh, _ = opt.opt_update(params[a:b].numpy(), hist[a:b].numpy(), None, grads[a:b].numpy(), lr=eps,
                                      mom=mom, l2=max(cfg["l2_decay"], 0.0), clip=max(cfg["gradient_clip"], 0.0))
            p_after[a:b], h_after[a:b] = torch.from_numpy(w), torch.from_numpy(hh)
    return se.Snapshot(N, labels, states, derivs, params, hist, grads, p_after, h_after, loss, seeds, opt_state)


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


@pytest.mark.parametrize("name", ["tiny+bn", "lcnet", "tiednet", "logcheck", "c3d"])
def test_unsupported_models_raise(name):
    with pytest.raises(se.Unsupported):
        se.load_model(name, 32)
