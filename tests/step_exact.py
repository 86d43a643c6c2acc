"""The step auditor: every call of one training step of a chain net, teacher-forced against float64.

A training step (ConvNet::TrainOneBatch) is a chain of library calls whose inputs are the outputs of other calls.  A
free-running float64 mirror of the whole step drifts from the net (one flipped ReLU or max-pool decision moves every
layer above it), so its bar has to be loose.  This auditor instead takes a Snapshot of one real step — the input, the
parameters and momentum history before it, every layer's state and derivative and the gradients and parameters after
it — and computes each call's expected output in float64 from the values that call actually consumed: the stored state
below it, the stored derivative above it and the parameters BEFORE the step, each rounded by the operand model of the
path the call takes (conv_exact.conv_path).  No decision can flip, so every call is held to the per-element bar of its
kernel test:

  conv / 1x1 / FC fprop (bias, ReLU, dropout)   conv_exact.expect("fprop")                      |err| <= 2^-16 S
  conv / 1x1 / FC dgrad (ReLU' mask, dropout     conv_exact.expect("dgrad", so = dropout scale)  |err| <= 2^-16 S
    scale of the layer below)
  wgrad (scale_gradients / batch)               conv_exact.expect("wgrad")                      |err| <= 2^-16 S
  bias gradient                                 elementwise_exact.bias_grad (side-lane column sum) or
                                                pool_exact.bias_grad (summed by the pool undo above, sums_bias_below)
  max / avg pool, response norm, their undos    pool_exact (max forward bit-exact)
  softmax output                                the fc8 logits modelled like any FC fprop: the state must lie within
                                                p_j (d_j + sum_k p_k d_k) + the softmax bar of elementwise_exact,
                                                d_j = 2^-16 S_j the logit's bar
  output derivative, per-image loss             loss_ref.loss_ref on the net's own output state
  the returned loss                             weight * fp32 cnb_sum of the per-image values:
                                                sum_n vbar_n + (ceil(N/256) + 11) u sum_n |v_n|  (+ u for the weight)
  update                                        opt_rules.opt_update bit for bit (+ apply_norm for norm rules)

Dropout is checked inside the fprop of the layer that draws it: the keep mask of element i is
float32(hash(seed + i)) * 2^-32 >= p with the seed the net reported for the step (Net.dropout_seed), whether the edge's
epilogue applies it or a separate pass does (then the pass's product adds one rounding, far inside the bar).

Tensor-core calls are also controls: their output must FAIL against the wrong operand models of their precision
(conv_exact.CONTROLS), or the audit is too weak to see a rounding or bf16-twin fault and says so.

Layer and edge kinds the auditor does not restate raise Unsupported: batch normalisation, logistic units, LOCAL and
tied edges, 3-D layers.
"""
import dataclasses
import math
import re

import numpy as np
import torch

import conv_exact as cx
import elementwise_exact as ex
import loss_ref as lr
import opt_rules as opt
import pool_exact as px
from convnet_b200.abi import num_modules

U = 2.0 ** -24
WEIGHTED = ("CONVOLUTIONAL", "CONV_ONETOONE", "FC")


class Unsupported(ValueError):
    pass


# ---------------------------------------------------------------------------------------------------------------------
# the model, read from its text proto (net.model_text)
# ---------------------------------------------------------------------------------------------------------------------
def _value(v):
    v = v.strip()
    if v.startswith('"'):
        return v[1:-1]
    if v in ("true", "false"):
        return v == "true"
    if re.fullmatch(r"[-+0-9.eE]+|inf|-inf|nan", v):
        return float(v)
    return v


def parse_text(text):
    """{"layer": [dict], "edge": [dict], ...} of a config::Model text proto; nested blocks are dicts"""
    root, stack = {}, []
    cur = root
    for line in text.splitlines():
        line = line.strip()
        if not line or line.startswith("#"):
            continue
        if line.endswith("{"):
            d = {}
            cur.setdefault(line[:-1].strip(), []).append(d)
            stack.append(cur)
            cur = d
        elif line == "}":
            cur = stack.pop()
        else:
            k, v = line.split(":", 1)
            cur[k.strip()] = _value(v)
    return root


@dataclasses.dataclass
class LayerGeo:
    name: str
    C: int
    W: int
    H: int
    act: str
    dropprob: float
    cfg: dict

    def floats(self, N):
        return N * self.W * self.H * self.C


@dataclasses.dataclass
class EdgeGeo:
    name: str
    kind: str
    cfg: dict
    src: int
    dst: int


def f32(v):
    return float(np.float32(v))


def dropout_scale(p):
    return float(np.float32(1.0) / (np.float32(1.0) - np.float32(p)))


class Model:
    """geometry, parameter offsets and fusion plan of a model (host-only calls)"""

    def __init__(self, name, text, layout, fusion):
        m = parse_text(text)
        self.name = name
        layers, edges = m.get("layer", []), m.get("edge", [])
        if len(layers) != len(edges) + 1:
            raise Unsupported("%s: not a chain" % name)
        for lc in layers:
            if lc.get("batch_normalize"):
                raise Unsupported("%s: layer %s is batch-normalised" % (name, lc["name"]))
            if lc["activation"] not in ("LINEAR", "RECTIFIED_LINEAR", "SOFTMAX"):
                raise Unsupported("%s: layer %s has activation %s" % (name, lc["name"], lc["activation"]))
            if lc.get("dropprob", 0) > 0 and lc["activation"] != "RECTIFIED_LINEAR":
                raise Unsupported("%s: dropout on the non-ReLU layer %s" % (name, lc["name"]))
        inp = layers[0]
        if int(inp.get("image_size_t", 1)) != 1:
            raise Unsupported("%s: 3-D layers" % name)
        out = layers[-1]
        if out["activation"] != "SOFTMAX" or out.get("loss_function") != "CROSS_ENTROPY_MULTINOMIAL":
            raise Unsupported("%s: output layer %s / %s" % (name, out["activation"], out.get("loss_function")))
        self.loss_weight = f32(out.get("loss_function_weight", 1.0))
        W, H = int(inp["image_size_x"]), int(inp["image_size_y"])
        self.layers = [LayerGeo(inp["name"], int(inp["num_channels"]), W, H, inp["activation"], 0.0, inp)]
        self.edges = []
        for i, e in enumerate(edges):
            kind = e["edge_type"]
            if e.get("tied_to"):
                raise Unsupported("%s: edge %s is tied" % (name, e.get("name") or e["dest"]))
            if kind not in WEIGHTED + ("MAXPOOL", "AVERAGE_POOL", "RESPONSE_NORM"):
                raise Unsupported("%s: edge type %s" % (name, kind))
            if int(e.get("kernel_size_t", 1)) != 1 or int(e.get("padding_t", 0)) != 0:
                raise Unsupported("%s: 3-D edge" % name)
            if kind == "CONVOLUTIONAL" and not e.get("shared_bias", True):
                raise Unsupported("%s: unshared conv bias" % name)
            lc = layers[i + 1]
            src = self.layers[i]
            if kind == "FC":
                w, h = 1, 1
            elif kind in ("CONVOLUTIONAL", "MAXPOOL", "AVERAGE_POOL"):
                ky = int(e["kernel_size_y"]) if e["kernel_size_y"] > 0 else src.H
                kx = int(e["kernel_size_x"]) if e["kernel_size_x"] > 0 else src.W
                w = num_modules(src.W, kx, int(e["stride_x"]), int(e["padding_x"]))
                h = num_modules(src.H, ky, int(e["stride_y"]), int(e["padding_y"]))
            else:
                w, h = src.W, src.H
            self.layers.append(LayerGeo(lc["name"], int(lc["num_channels"]), w, h, lc["activation"],
                                        float(lc.get("dropprob", 0.0)), lc))
            self.edges.append(EdgeGeo(e.get("name") or "%s:%s" % (e["source"], e["dest"]), kind, e, i, i + 1))
        self.offsets = layout["edge_offsets"]
        self.total = layout["total"]
        self.plan = fusion["edges"]
        self.passes = fusion["layers"]

    def conv_geo(self, e, N):
        s, d = self.layers[e.src], self.layers[e.dst]
        c = e.cfg
        if e.kind == "FC":
            return cx.Geo(N, 1, 1, s.W * s.H * s.C, d.C, 1, 1)
        if e.kind == "CONV_ONETOONE":
            return cx.Geo(N, s.W, s.H, s.C, d.C, 1, 1)
        return cx.Geo(N, s.W, s.H, s.C, d.C, int(c["kernel_size_y"]), int(c["kernel_size_x"]), int(c["stride_y"]),
                      int(c["stride_x"]), int(c["padding_y"]), int(c["padding_x"]))

    def pool_geo(self, e, N):
        s, c = self.layers[e.src], e.cfg
        ky = int(c["kernel_size_y"]) if c["kernel_size_y"] > 0 else s.H
        kx = int(c["kernel_size_x"]) if c["kernel_size_x"] > 0 else s.W
        return px.PG(N, s.W, s.H, s.C, ky, kx, int(c["stride_y"]), int(c["stride_x"]), int(c["padding_y"]),
                     int(c["padding_x"]))

    def weight_slices(self, k, N):
        """(weights, bias) index ranges of weighted edge k in the flat buffers"""
        g = self.conv_geo(self.edges[k], N)
        o = self.offsets[k]
        nw = g.Cout * g.K
        has_bias = not self.edges[k].cfg.get("has_no_bias", False)
        return (o, o + nw), ((o + nw, o + nw + g.Cout) if has_bias else None)


def load_model(name, batch):
    from convnet_b200 import net
    return Model(name, net.model_text(name), net.model_param_layout(name, batch), net.model_fusion(name, batch))


# ---------------------------------------------------------------------------------------------------------------------
# the snapshot of one step
# ---------------------------------------------------------------------------------------------------------------------
@dataclasses.dataclass
class Snapshot:
    N: int
    labels: torch.Tensor          # int, N
    states: list                  # per layer, flat fp32 after the step (states[0] = the input)
    derivs: list                  # per layer, flat fp32 after the step (derivs[0] = None)
    params_before: torch.Tensor
    hist_before: torch.Tensor
    grads: torch.Tensor
    params_after: torch.Tensor
    hist_after: torch.Tensor
    loss: float
    seeds: list                   # per layer: the dropout seed of the step (0: none)
    opt_state: dict               # edge index -> {"weights": {step, epsilon, momentum}, "bias": {...}} before the step


@dataclasses.dataclass
class Row:
    layer: str                    # layer or edge name
    quantity: str
    ok: bool
    worst: float                  # worst |err| / bar (conv calls: |err| / (2^-16 S)); updates: inexact elements
    detail: str

    def __str__(self):
        return "%-28s %-14s %-4s worst=%.3e %s" % (self.layer, self.quantity, "ok" if self.ok else "FAIL", self.worst,
                                                    self.detail)


def _conv_row(name, qty, op, g, y, e, kind, controls, a=None, b=None, kw=None):
    """[the check of a conv call] + [its control] for a tensor-core call: the output must fail against every wrong
    operand model of its precision, else the check could not see a rounding or bf16-twin fault"""
    v = cx.check(op, g, y, e)
    rows = [Row(name, qty, v.ok, v.worst_ratio / cx.BAR, "model=%s %s" % (kind, v.where if not v.ok else ""))]
    if controls and kind != "fp32":
        weak = [w for w in cx.CONTROLS[kind] if cx.check(op, g, y, cx.expect(op, g, a, b, w, **kw)).ok]
        rows.append(Row(name, qty + "_control", not weak, 0.0, "also passes against %s: too weak to see a rounding "
                        "fault" % ", ".join(weak) if weak else "fails against %s" % ", ".join(cx.CONTROLS[kind])))
    return rows


def _px_row(name, qty, y, e):
    v = px.check(y, e)
    return Row(name, qty, v.ok, v.worst, v.where)


class Auditor:
    def __init__(self, model, mode, controls=True):
        self.m, self.mode, self.controls = model, mode, controls

    # ---- conv / 1x1 / FC
    def kind(self, op, g):
        return cx.PATH_MODEL[cx.conv_path(op, g, self.mode)]

    def weights(self, params, k, N):
        (w0, w1), bs = self.m.weight_slices(k, N)
        return params[w0:w1], (params[bs[0]:bs[1]] if bs else None)

    def fprop(self, s, k):
        m, e = self.m, self.m.edges[k]
        g = m.conv_geo(e, s.N)
        dst = m.layers[e.dst]
        W, b = self.weights(s.params_before, k, s.N)
        kind = self.kind("fprop", g)
        relu = dst.act == "RECTIFIED_LINEAR"
        drop = (f32(dst.dropprob), dropout_scale(dst.dropprob), s.seeds[e.dst]) if dst.dropprob > 0 else None
        kw = dict(bias=b, relu=relu, drop=drop)
        ex_ = cx.expect("fprop", g, s.states[e.src], W, kind, **kw)
        if dst.act == "SOFTMAX":
            return [self.softmax(s, g, ex_, dst)]
        return _conv_row(dst.name, "fprop", "fprop", g, s.states[e.dst], ex_, kind, self.controls, s.states[e.src], W,
                         kw)

    def softmax(self, s, g, e, dst):
        """the output state against the float64 softmax of the modelled logits, the logit bar propagated"""
        C = dst.C
        z = e.ref.view(C, s.N)
        d = (cx.BAR * e.S).view(C, s.N)
        p = torch.softmax(z, 0)
        prop = p * (d + (p * d).sum(0, keepdim=True))
        sm = ex.softmax(e.ref.to(torch.float32), s.N, C)
        bar = prop.reshape(-1) + sm.bar
        return _px_row(dst.name, "softmax", s.states[-1], px.Expect(p.reshape(-1), bar, sm.exact))

    def dgrad(self, s, k, params=None):
        m, e = self.m, self.m.edges[k]
        g = m.conv_geo(e, s.N)
        src = m.layers[e.src]
        W, _ = self.weights(s.params_before if params is None else params, k, s.N)
        kind = self.kind("dgrad", g)
        mask = s.states[e.src] if src.act == "RECTIFIED_LINEAR" else None
        so = dropout_scale(src.dropprob) if src.dropprob > 0 else 1.0
        kw = dict(so=so, mask=mask)
        ex_ = cx.expect("dgrad", g, s.derivs[e.dst], W, kind, **kw)
        return _conv_row(src.name, "dgrad", "dgrad", g, s.derivs[e.src], ex_, kind, self.controls, s.derivs[e.dst],
                         W, kw)

    def wgrad(self, s, k):
        m, e = self.m, self.m.edges[k]
        g = m.conv_geo(e, s.N)
        kind = self.kind("wgrad", g)
        so = f32(f32(e.cfg.get("scale_gradients", 1.0)) / s.N)
        (w0, w1), _ = m.weight_slices(k, s.N)
        kw = dict(so=so)
        ex_ = cx.expect("wgrad", g, s.states[e.src], s.derivs[e.dst], kind, **kw)
        return _conv_row(e.name, "wgrad", "wgrad", g, s.grads[w0:w1], ex_, kind, self.controls, s.states[e.src],
                         s.derivs[e.dst], kw)

    def bias_grad(self, s, k):
        m, e = self.m, self.m.edges[k]
        _, bs = m.weight_slices(k, s.N)
        dst = m.layers[e.dst]
        rows = s.N * dst.W * dst.H
        so = f32(f32(e.cfg.get("scale_gradients", 1.0)) / s.N)
        y = s.grads[bs[0]:bs[1]]
        zero = torch.zeros(dst.C, dtype=torch.float32, device=y.device)
        above = m.edges[e.dst] if e.dst < len(m.edges) else None
        if above is not None and m.plan[e.dst]["sums_bias_below"] and m.plan[k]["offers_bias_grad"]:
            pg = m.pool_geo(above, s.N)
            relu = m.plan[e.dst]["down_act"] == 1
            br = px.pool_undo_branch(pg, above.kind == "MAXPOOL", mask="input" if relu else None,
                                     cached=above.kind == "MAXPOOL")
            per_thread, slices = px.bias_depth(br, pg)
            exp = px.bias_grad(s.derivs[e.dst], rows, dst.C, 1, zero, 0.0, so, per_thread, slices)
            how = "pool-undo sum (%s)" % br.name
        else:
            exp = ex.bias_grad(s.derivs[e.dst], rows, dst.C, zero, 0.0, so)
            how = "column sum"
        r = _px_row(e.name, "bias_grad", y, exp)
        r.detail = how + " " + r.detail
        return r

    # ---- pooling and response normalisation
    def pool_fprop(self, s, k):
        m, e = self.m, self.m.edges[k]
        dst = m.layers[e.dst]
        x = s.states[e.src]
        if e.kind == "RESPONSE_NORM":
            F, c = m.layers[e.src].C, e.cfg
            kk = int(np.float32(c["frac_of_filters_response_norm"]) * np.float32(F))
            exp = px.rnorm_fwd(x, F, kk, f32(c["add_scale"]), f32(c["pow_scale"]),
                               bool(c.get("response_norm_in_blocks", False)), relu=dst.act == "RECTIFIED_LINEAR")
        else:
            exp = px.pool_fwd(m.pool_geo(e, s.N), x, e.kind == "MAXPOOL")
            if dst.act == "RECTIFIED_LINEAR":
                exp = px.Expect(exp.ref.clamp_min(0.0), exp.bar, exp.exact)
        if dst.dropprob > 0:
            raise Unsupported("dropout on the pooling layer %s" % dst.name)
        return _px_row(dst.name, "fprop", s.states[e.dst], exp)

    def pool_undo(self, s, k):
        m, e = self.m, self.m.edges[k]
        src = m.layers[e.src]
        mask = s.states[e.src] if src.act == "RECTIFIED_LINEAR" else None
        if src.dropprob > 0:
            raise Unsupported("dropout below the pooling edge %s" % e.name)
        if e.kind == "RESPONSE_NORM":
            F, c = src.C, e.cfg
            kk = int(np.float32(c["frac_of_filters_response_norm"]) * np.float32(F))
            exp = px.rnorm_undo(s.derivs[e.dst], s.states[e.src], F, kk, f32(c["add_scale"]), f32(c["pow_scale"]),
                                bool(c.get("response_norm_in_blocks", False)))
            if mask is not None:
                drop = ~(mask > 0)
                exp = px.Expect(torch.where(drop, torch.zeros_like(exp.ref), exp.ref),
                                torch.where(drop, torch.zeros_like(exp.bar), exp.bar), exp.exact)
        elif e.kind == "MAXPOOL":
            exp = px.max_undo(m.pool_geo(e, s.N), s.states[e.src], s.derivs[e.dst], s.states[e.dst], mask=mask)
        else:
            exp = px.avg_undo(m.pool_geo(e, s.N), s.derivs[e.dst], mask=mask)
        return _px_row(src.name, "undo", s.derivs[e.src], exp)

    # ---- output layer
    def output(self, s):
        m = self.m
        C, N = m.layers[-1].C, s.N
        y = s.states[-1].to(torch.float64).view(C, N).t().cpu().numpy()
        labels = s.labels.cpu().numpy()
        d, d_bar, v, v_bar = lr.loss_ref(lr.CE_MULTINOMIAL, y, labels=labels, weight=m.loss_weight)
        dev = s.states[-1].device
        t = lambda a: torch.from_numpy(np.ascontiguousarray(a.T).reshape(-1)).to(dev)  # noqa: E731
        rows = [_px_row(m.layers[-1].name, "output_deriv", s.derivs[-1],
                        px.Expect(t(d), t(d_bar), torch.zeros(N * C, dtype=torch.bool, device=dev)))]
        # the returned loss: weight * cnb_sum of the N per-image fp32 values, each within v_bar of v
        ref = m.loss_weight * v.sum()
        bar = abs(m.loss_weight) * (v_bar.sum() + (ex.cdiv(N, ex.BLOCK) + 11) * U * np.abs(v).sum()) + U * abs(ref)
        err = abs(s.loss - ref)
        rows.append(Row(m.layers[-1].name, "loss", bool(err <= bar), err / bar if bar > 0 else 0.0,
                        "loss=%r ref=%r bar=%.3e" % (s.loss, ref, bar)))
        return rows

    # ---- update
    def update(self, s, k):
        m, e = self.m, self.m.edges[k]
        (w0, w1), bs = m.weight_slices(k, s.N)
        rows = []
        for which, sl, key in (("weights", (w0, w1), "weight_optimizer"), ("bias", bs, "bias_optimizer")):
            if sl is None:
                continue
            c = e.cfg[key][0]
            if c.get("optimizer_type", "STOCHASTIC_GRADIENT_DESCENT") != "STOCHASTIC_GRADIENT_DESCENT":
                raise Unsupported("%s: optimizer %s" % (e.name, c["optimizer_type"]))
            st = s.opt_state[k][which]
            a, b = sl
            if st["step"] < int(c.get("start_optimization_after", 0)):
                w_new, h_new = s.params_before[a:b].cpu().numpy(), s.hist_before[a:b].cpu().numpy()
            else:
                w_new, h_new, _ = opt.opt_update(s.params_before[a:b].cpu().numpy(), s.hist_before[a:b].cpu().numpy(),
                                                 None, s.grads[a:b].cpu().numpy(), lr=st["epsilon"],
                                                 mom=st["momentum"], l2=max(c.get("l2_decay", 0.0), 0.0),
                                                 clip=max(c.get("gradient_clip", -1.0), 0.0))
            near = np.zeros(b - a, bool)
            if which == "weights" and (c.get("weight_norm_constraint", 0) > 0 or c.get("weight_norm_limit", 0) > 0):
                mode, val = ((opt.CONSTRAINT, c["weight_norm_constraint"]) if c.get("weight_norm_constraint", 0) > 0
                             else (opt.LIMIT, c["weight_norm_limit"]))
                rows_ = m.conv_geo(e, s.N).Cout
                w_new, bite = opt.apply_norm(w_new, rows_, mode, f32(val))
                near = np.broadcast_to(bite, (len(w_new) // rows_, rows_)).reshape(-1)
            for qty, got, want in (("update_" + which, s.params_after[a:b], w_new), ("history_" + which,
                                                                                    s.hist_after[a:b], h_new)):
                g = got.cpu().numpy()
                same = g.view(np.int32) == np.asarray(want, np.float32).view(np.int32)
                if qty.startswith("update") and near.any():
                    same = same | (near & (np.abs(g.astype(np.float64) - want) <= 8 * U * np.abs(want)))
                nbad = int((~same).sum())
                where = ""
                if nbad:
                    i = int(np.flatnonzero(~same)[0])
                    where = "first bad element %d: got=%r want=%r" % (i, float(g[i]), float(want[i]))
                rows.append(Row(e.name, qty, nbad == 0, float(nbad), "%d inexact %s" % (nbad, where)))
        return rows

    # ---- the whole step
    def audit(self, s):
        m = self.m
        for i, l in enumerate(m.layers):
            if s.states[i].numel() != l.floats(s.N):
                raise AssertionError("layer %s: %d floats, the model's geometry gives %d" % (
                    l.name, s.states[i].numel(), l.floats(s.N)))
        rows = []
        for k, e in enumerate(m.edges):
            if e.kind in WEIGHTED:
                rows += self.fprop(s, k)
                if e.src > 0:
                    rows += self.dgrad(s, k)
                rows += self.wgrad(s, k)
                if not e.cfg.get("has_no_bias", False):
                    rows.append(self.bias_grad(s, k))
                rows += self.update(s, k)
            else:
                rows.append(self.pool_fprop(s, k))
                if e.src > 0:
                    rows.append(self.pool_undo(s, k))
        rows += self.output(s)
        return rows


def failures(rows):
    return [r for r in rows if not r.ok]


# ---------------------------------------------------------------------------------------------------------------------
# a snapshot of a real step (needs a GPU)
# ---------------------------------------------------------------------------------------------------------------------
SENTINEL = 0x7FC0DEAD        # NaN bits written into every derivative and gradient before the audited step


def run_step(n, model, warmup):
    """`warmup` training steps of Net `n`, then the audited one: returns its Snapshot and the names of the tensors in
    which the step left a sentinel NaN.  Call n.params_tensor() only here: the library drops every staged bf16 copy
    and filter bank when it hands out the parameter pointer, which would change the step being audited."""
    P, Hs, G = n.params_tensor(), n.history_tensor(), n.grads_tensor()
    for _ in range(warmup):
        assert math.isfinite(n.train_step(True))
    torch.cuda.synchronize()
    L = len(model.layers)
    seeds = [int(n.dropout_seed(i)) for i in range(L)]
    opt_state = {k: n.optimizer_state(k) for k, e in enumerate(model.edges) if e.kind in WEIGHTED}
    p0, h0 = P.clone(), Hs.clone()
    for i in range(1, L):
        n.layer_deriv(i).view(torch.int32).fill_(SENTINEL)
    G.view(torch.int32).fill_(SENTINEL)
    torch.cuda.synchronize()
    loss = n.train_step(True)
    torch.cuda.synchronize()
    s = Snapshot(n.batch_size, n.labels_tensor().clone(), [n.layer_state(i).clone() for i in range(L)],
                 [None] + [n.layer_deriv(i).clone() for i in range(1, L)], p0, h0, G.clone(), P.clone(), Hs.clone(),
                 loss, seeds, opt_state)
    left = ["deriv %s" % model.layers[i].name for i in range(1, L) if bool(torch.isnan(s.derivs[i]).any())]
    for k, e in enumerate(model.edges):
        if e.kind in WEIGHTED:
            (w0, w1), bs = model.weight_slices(k, s.N)
            for what, t in (("grad", s.grads), ("param", s.params_after), ("history", s.hist_after)):
                for a, b in ((w0, w1), bs or (0, 0)):
                    if bool(torch.isnan(t[a:b]).any()):
                        left.append("%s %s[%d:%d]" % (what, e.name, a, b))
    return s, left


def audit_case(name, batch, mode, warmup, boost=None, seed=1234):
    """build `name` as bench.py does (seed 1234, N(0, 1) input, uniform labels), optionally raise the weight learning
    rate of some edges ({edge name: epsilon}) before the warm-up, run and audit step number `warmup` in precision
    `mode`.  Returns (rows, tensors the step left NaN in, stale-weight rows): for each boosted edge the share of its bf16
    weight copies the step changed, and its dgrad checked against the weights before and AFTER the step (the second
    must fail)."""
    from convnet_b200 import lib
    from convnet_b200.net import Net
    lib.set_precision(mode)
    model = load_model(name, batch)
    n = Net(name, batch, seed=seed)
    try:
        for edge, eps in (boost or {}).items():
            w = n.optimizer_state(edge)
            n.set_optimizer(edge, weights=dict(_sgd_config(model, edge), epsilon=eps))
            assert n.optimizer_state(edge)["weights"]["step"] == w["weights"]["step"]
        g = torch.Generator(device="cuda").manual_seed(seed)
        n.input_tensor().normal_(generator=g)
        n.labels_tensor().copy_(torch.randint(0, n.num_classes, (batch,), device="cuda", generator=g,
                                              dtype=torch.int32))
        s, left = run_step(n, model, warmup)
        a = Auditor(model, mode)
        rows = a.audit(s)
        stale = []
        for edge in boost or {}:
            k = [e.name for e in model.edges].index(edge)
            (w0, w1), _ = model.weight_slices(k, batch)
            b0 = s.params_before[w0:w1].to(torch.bfloat16)
            b1 = s.params_after[w0:w1].to(torch.bfloat16)
            share = float((b0.view(torch.int16) != b1.view(torch.int16)).float().mean())
            stale.append((edge, share, a.dgrad(s, k)[0], a.dgrad(s, k, params=s.params_after)[0]))
        return rows, left, stale
    finally:
        n.close()


def _sgd_config(model, edge):
    """the weight optimizer block of `edge` as OptimizerConfig fields"""
    from convnet_b200.net import OptimizerConfig
    c = model.edges[[e.name for e in model.edges].index(edge)].cfg["weight_optimizer"][0]
    names = [f[0] for f in OptimizerConfig._fields_]
    return {k: (int(v) if isinstance(v, float) and k in ("epsilon_decay_timescale", "momentum_transition_timescale",
                                                         "start_optimization_after") else v)
            for k, v in c.items() if k in names}
