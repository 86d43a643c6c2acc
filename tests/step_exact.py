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
  output derivative, per-image loss             loss_ref.loss_ref on the net's own output state (and targets)
  the returned loss                             weight * fp32 cnb_sum of the per-image values:
                                                sum_n vbar_n + (ceil(N/256) + 11) u sum_n |v_n|  (+ u for the weight)
  update                                        opt_rules.opt_update bit for bit (+ apply_norm for norm rules)

Logistic units (LOGISTIC hidden layers, the LOGISTIC output layer): sigma of the modelled pre-activation, whether the
conv or pool epilogue applies it or a separate pass does; sigma' <= 1/4, so the bar is 1/4 of the call's bar plus
loss_ref.sigmoid_bar.  The derivative into a logistic layer, from a dgrad or a pool undo, is the modelled one times
s(1 - s) of the stored state s: bar times s(1 - s) plus loss_ref.logistic_deriv_bar.

Output layers: SOFTMAX + CROSS_ENTROPY_MULTINOMIAL on labels; LINEAR + SQUARED_ERROR, LOGISTIC + CROSS_ENTROPY_BINARY
(targets < 0 are don't-care: derivative exactly 0) and SOFTMAX_DIST + CROSS_ENTROPY_MULTINOMIAL_DISTRIBUTED on the
float targets the Snapshot carries.

Optimizers: STOCHASTIC_GRADIENT_DESCENT, ADAGRAD_SGD and RMSPROP_SGD; parameters, momentum history and the adaptive state
(Net.adaptive_state_tensor) must equal opt_rules.opt_update(rule=...) bit for bit.

Tied edges: a tied edge's fprop and dgrad use its owner's weights before the step.  The group's weight gradient is the
sum of its members' wgrads in back-propagation order (S: the members' S plus the partial sum each later member adds to),
its bias gradient the sum of their column sums, and the group is updated once.

Sampling and colour edges (DESIGN.md 5, "Sampling and colour edges"): UPSAMPLE fprop is replication (exact), its
derivative the f x f block sum, pool_exact.pool_fwd(avg, so = f^2) on the big image; DOWNSAMPLE fprop is the f x f
average pool, its derivative pool_exact.avg_undo.  ReLU, sigma and dropout follow in fprop, the ReLU' mask and the dropout
fold (one more rounding) in the derivative, as for every pooling edge; the bias gradient of a conv below a sampling edge
summed by its derivative call uses that call's row-slice depth (pool_exact.bias_depth).  RGBTOYUV fprop is
abi_rest_exact.rgb_to_yuv; the layer it writes has no derivative, and the edge above it no dgrad.

Frozen trunks (block_backprop): frozen edges get fprop rows only.  Their slice of the parameters, history and adaptive
state is bit-identical after the step, their slice of the gradient buffer still holds the sentinel, and the hidden
layers they write have no derivative.

3-D layers (c3d): frames stack as channel blocks (channel c + C*t).  A 3-D conv is conv_exact's 3-D Geo (T, kt, st_t:
frame window f reads frames [f st_t, f st_t + kt)), its bias added to every output frame and its bias gradient the sum of
one column sum per output frame (the first writing, the others adding, as in a tie group); max / average pools are
pool_exact's 3-D PG (kernel_size / kernel_size_t 0: the whole image / clip), and an FC edge reads every frame.

Dropout is checked inside the fprop of the layer that draws it: the keep mask of element i is
float32(hash(seed + i)) * 2^-32 >= p with the seed the net reported for the step (Net.dropout_seed), whether the edge's
epilogue applies it or a separate pass does (then the pass's product adds one rounding, far inside the bar).

Tensor-core calls are also controls: their output must FAIL against the wrong operand models of their precision
(conv_exact.CONTROLS), or the audit is too weak to see a rounding or bf16-twin fault and says so.

Not audited, raising Unsupported: batch-normalised layers, LOCAL edges and CONVOLUTIONAL edges with an unshared bias,
dropout on non-ReLU layers (its keep mask cannot be read back from the state), other output layers and optimizers, nets
that are not chains, and on 3-D layers every edge but CONVOLUTIONAL, MAXPOOL, AVERAGE_POOL and FC.
"""
import dataclasses
import math
import re

import numpy as np
import torch

import abi_rest_exact as ax
import conv_exact as cx
import elementwise_exact as ex
import loss_ref as lr
import opt_rules as opt
import pool_exact as px
from convnet_b200.abi import num_modules

U = 2.0 ** -24
WEIGHTED = ("CONVOLUTIONAL", "CONV_ONETOONE", "FC")
SAMPLING = ("UPSAMPLE", "DOWNSAMPLE", "RGBTOYUV")
# the output layers (activation, loss function) the auditor restates, and their loss_ref code
OUTPUTS = {("SOFTMAX", "CROSS_ENTROPY_MULTINOMIAL"): lr.CE_MULTINOMIAL, ("LINEAR", "SQUARED_ERROR"): lr.SQUARED_ERROR,
           ("LOGISTIC", "CROSS_ENTROPY_BINARY"): lr.CE_BINARY,
           ("SOFTMAX_DIST", "CROSS_ENTROPY_MULTINOMIAL_DISTRIBUTED"): lr.CE_DISTRIBUTED}
RULES = {"STOCHASTIC_GRADIENT_DESCENT": opt.SGD, "ADAGRAD_SGD": opt.ADAGRAD, "RMSPROP_SGD": opt.RMSPROP}
SENTINEL = 0x7FC0DEAD        # NaN bits written into every derivative and gradient before the audited step


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
    T: int = 1                    # frames (3-D layers stack them as channel blocks, channel c + C*t)

    def floats(self, N):
        return N * self.W * self.H * self.C * self.T


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
        inp = layers[0]
        for lc in layers:
            if lc.get("batch_normalize"):
                raise Unsupported("%s: layer %s is batch-normalised" % (name, lc["name"]))
            if lc["activation"] not in ("LINEAR", "RECTIFIED_LINEAR", "LOGISTIC") and lc is not layers[-1]:
                raise Unsupported("%s: layer %s has activation %s" % (name, lc["name"], lc["activation"]))
            if lc.get("dropprob", 0) > 0 and lc["activation"] != "RECTIFIED_LINEAR":
                raise Unsupported("%s: dropout on the non-ReLU layer %s" % (name, lc["name"]))
        out = layers[-1]
        self.loss = OUTPUTS.get((out["activation"], out.get("loss_function")))
        if self.loss is None:
            raise Unsupported("%s: output layer %s / %s" % (name, out["activation"], out.get("loss_function")))
        self.loss_weight = f32(out.get("loss_function_weight", 1.0))
        W, H = int(inp["image_size_x"]), int(inp["image_size_y"])
        self.layers = [LayerGeo(inp["name"], int(inp["num_channels"]), W, H, inp["activation"], 0.0, inp,
                                int(inp.get("image_size_t", 1)))]
        self.edges = []
        for i, e in enumerate(edges):
            kind = e["edge_type"]
            if kind not in WEIGHTED + ("MAXPOOL", "AVERAGE_POOL", "RESPONSE_NORM") + SAMPLING:
                raise Unsupported("%s: edge type %s" % (name, kind))
            if kind == "CONVOLUTIONAL" and not e.get("shared_bias", True):
                raise Unsupported("%s: unshared conv bias" % name)
            lc = layers[i + 1]
            src = self.layers[i]
            if src.T > 1 and kind not in ("CONVOLUTIONAL", "FC", "MAXPOOL", "AVERAGE_POOL"):
                raise Unsupported("%s: %s edge on the 3-D layer %s" % (name, kind, src.name))
            t = src.T
            if kind == "FC":
                w, h, t = 1, 1, 1
            elif kind in ("CONVOLUTIONAL", "MAXPOOL", "AVERAGE_POOL"):
                ky = int(e["kernel_size_y"]) if e["kernel_size_y"] > 0 else src.H
                kx = int(e["kernel_size_x"]) if e["kernel_size_x"] > 0 else src.W
                w = num_modules(src.W, kx, int(e["stride_x"]), int(e["padding_x"]))
                h = num_modules(src.H, ky, int(e["stride_y"]), int(e["padding_y"]))
                kt = int(e.get("kernel_size_t", 1)) if e.get("kernel_size_t", 1) > 0 else src.T
                t = num_modules(src.T, kt, int(e.get("stride_t", 1)), int(e.get("padding_t", 0)))
            elif kind == "UPSAMPLE":
                f = int(e.get("sample_factor", 1))
                w, h = src.W * f, src.H * f
            elif kind == "DOWNSAMPLE":
                f = int(e.get("sample_factor", 1))
                w, h = src.W // f, src.H // f
            else:
                w, h = src.W, src.H
            self.layers.append(LayerGeo(lc["name"], int(lc["num_channels"]), w, h, lc["activation"],
                                        float(lc.get("dropprob", 0.0)), lc, t))
            self.edges.append(EdgeGeo(e.get("name") or "%s:%s" % (e["source"], e["dest"]), kind, e, i, i + 1))
        # tie groups: owner[k] is the edge whose parameters weighted edge k uses (tied_to names it), and the group's
        # parameters sit at the slice of its lowest member (Net.model_ties)
        names = [x.name for x in self.edges]
        self.owner = [names.index(x.cfg["tied_to"]) if x.cfg.get("tied_to") else k for k, x in enumerate(self.edges)]
        # block_backprop freezes its edge and every edge below it (Net: fine-tuning)
        self.frozen = max([i + 1 for i, e in enumerate(edges) if e.get("block_backprop")], default=0)
        # the layer an RGBTOYUV edge writes receives no derivative either
        self.yuv = {x.dst for x in self.edges if x.kind == "RGBTOYUV"}
        self.offsets = layout["edge_offsets"]
        self.total = layout["total"]
        self.trained_offset = self.offsets[self.frozen] if self.frozen else 0
        self.plan = fusion["edges"]
        self.passes = fusion["layers"]

    def conv_geo(self, e, N):
        s, d = self.layers[e.src], self.layers[e.dst]
        c = e.cfg
        if e.kind == "FC":
            return cx.Geo(N, 1, 1, s.W * s.H * s.C * s.T, d.C, 1, 1)
        if e.kind == "CONV_ONETOONE":
            return cx.Geo(N, s.W, s.H, s.C, d.C, 1, 1)
        return cx.Geo(N, s.W, s.H, s.C, d.C, int(c["kernel_size_y"]), int(c["kernel_size_x"]), int(c["stride_y"]),
                      int(c["stride_x"]), int(c["padding_y"]), int(c["padding_x"]), T=s.T,
                      kt=int(c.get("kernel_size_t", 1)), st_t=int(c.get("stride_t", 1)))

    def group(self, k):
        """the weighted edges that share edge k's parameters (edge k alone when untied), in chain order"""
        return [j for j, e in enumerate(self.edges) if e.kind in WEIGHTED and self.owner[j] == self.owner[k]]

    def receives_deriv(self, i):
        """layer i gets a derivative: not the input layer, and no hidden layer a frozen edge writes"""
        return i > self.frozen and i not in self.yuv

    def sample_geo(self, e, N):
        """the f x f, stride f average-pool geometry of a sampling edge: on its input for DOWNSAMPLE (fprop, and its undo
        as the derivative), on its output for UPSAMPLE (whose derivative is the block sum, the average times f^2)"""
        f = int(e.cfg.get("sample_factor", 1))
        big = self.layers[e.src if e.kind == "DOWNSAMPLE" else e.dst]
        return px.PG(N, big.W, big.H, big.C, f, f, f, f, 0, 0), f

    def pool_geo(self, e, N):
        s, c = self.layers[e.src], e.cfg
        ky = int(c["kernel_size_y"]) if c["kernel_size_y"] > 0 else s.H
        kx = int(c["kernel_size_x"]) if c["kernel_size_x"] > 0 else s.W
        kt = int(c.get("kernel_size_t", 1)) if c.get("kernel_size_t", 1) > 0 else s.T    # (0: the whole clip)
        return px.PG(N, s.W, s.H, s.C, ky, kx, int(c["stride_y"]), int(c["stride_x"]), int(c["padding_y"]),
                     int(c["padding_x"]), s.T, kt, int(c.get("stride_t", 1)), int(c.get("padding_t", 0)))

    def weight_slices(self, k, N):
        """(weights, bias) index ranges of weighted edge k in the flat buffers"""
        g = self.conv_geo(self.edges[k], N)
        o = self.offsets[self.group(k)[0]]
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
    targets: torch.Tensor = None  # the output layer's float targets (column-major like its state); None: labels
    state_before: torch.Tensor = None   # adaptive optimizer state (Net.adaptive_state_tensor); None: SGD only
    state_after: torch.Tensor = None


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


def _conv_row(name, qty, op, g, y, make, kind, controls):
    """[the check of a conv call against make(kind), its cx.Expect under operand model `kind`] + [its control] for a
    tensor-core call: the output must fail against every wrong operand model of its precision, else the check could not
    see a rounding or bf16-twin fault"""
    v = cx.check(op, g, y, make(kind))
    rows = [Row(name, qty, v.ok, v.worst_ratio / cx.BAR, "model=%s %s" % (kind, v.where if not v.ok else ""))]
    if controls and kind != "fp32":
        weak = [w for w in cx.CONTROLS[kind] if cx.check(op, g, y, make(w)).ok]
        rows.append(Row(name, qty + "_control", not weak, 0.0, "also passes against %s: too weak to see a rounding "
                        "fault" % ", ".join(weak) if weak else "fails against %s" % ", ".join(cx.CONTROLS[kind])))
    return rows


def _sigmoid(e):
    """sigma of a pool_exact.Expect: the bar scaled by sigma' <= 1/4, plus sigma's own (loss_ref.sigmoid_bar)"""
    sig = torch.sigmoid(e.ref)
    return px.Expect(sig, e.bar / 4 + 6 * U * sig + 2.0 ** -126, torch.zeros_like(e.exact))


def _logistic_deriv(e, state):
    """a pool_exact.Expect times s(1 - s) of the logistic layer's stored state s, plus the bar of that product
    (loss_ref.logistic_deriv_bar)"""
    sl = state[:e.ref.numel()].to(torch.float64)
    ds = sl * (1 - sl)
    ref = e.ref * ds
    return px.Expect(ref, e.bar * ds + 3 * U * ref.abs() + 2.0 ** -148, torch.zeros_like(e.exact))


def _dropout(e, layer, seed):
    """the keep mask of a pooling or sampling layer's dropout on a pool_exact.Expect: dropped elements exactly 0, kept
    ones times the scale (one more rounding)"""
    n = e.ref.numel()
    kept = torch.from_numpy(cx.dropout_kept(n, np.float32(layer.dropprob), seed)).to(e.ref.device)
    scale = dropout_scale(layer.dropprob)
    ref = torch.where(kept, e.ref * scale, torch.zeros_like(e.ref))
    bar = torch.where(kept, e.bar * scale + U * ref.abs(), torch.zeros_like(e.bar))
    return px.Expect(ref, bar, torch.zeros_like(e.exact))


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
        kw = dict(bias=b, relu=relu, drop=drop, logistic=dst.act == "LOGISTIC")
        make = lambda kd: cx.expect("fprop", g, s.states[e.src], W, kd, **kw)  # noqa: E731
        if dst.act in ("SOFTMAX", "SOFTMAX_DIST"):
            return [self.softmax(s, g, make(kind), dst)]
        return _conv_row(dst.name, "fprop", "fprop", g, s.states[e.dst], make, kind, self.controls)

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
        lmask = s.states[e.src] if src.act == "LOGISTIC" else None
        so = dropout_scale(src.dropprob) if src.dropprob > 0 else 1.0
        kw = dict(so=so, mask=mask, lmask=lmask)
        make = lambda kd: cx.expect("dgrad", g, s.derivs[e.dst], W, kd, **kw)  # noqa: E731
        return _conv_row(src.name, "dgrad", "dgrad", g, s.derivs[e.src], make, kind, self.controls)

    def wgrad(self, s, k):
        """the weight gradient of edge k's tie group (edge k alone when untied): the sum of its members' wgrads, written by
        the first member in back-propagation order and accumulated by the others (scaleTargets 1), so S is the sum of
        the members' S plus the magnitude of the partial sum each later member adds to"""
        m, e = self.m, self.m.edges[k]
        members = m.group(k)[::-1]
        geos = [m.conv_geo(m.edges[j], s.N) for j in members]
        kinds = [self.kind("wgrad", g) for g in geos]
        kind = next((kd for kd in kinds if kd != "fp32"), "fp32")
        (w0, w1), _ = m.weight_slices(k, s.N)

        def make(kd):
            total = None
            for j, g, own in zip(members, geos, kinds):
                ej = m.edges[j]
                so = f32(f32(ej.cfg.get("scale_gradients", 1.0)) / s.N)
                x = cx.expect("wgrad", g, s.states[ej.src], s.derivs[ej.dst], kd if own != "fp32" else own, so=so)
                if total is not None:
                    x.S += total.ref.abs()
                    x.ref += total.ref
                    x.S += total.S
                total = x
            return total
        return _conv_row(e.name, "wgrad", "wgrad", geos[0], s.grads[w0:w1], make, kind, self.controls)

    def bias_grad(self, s, k):
        m, e = self.m, self.m.edges[k]
        _, bs = m.weight_slices(k, s.N)
        dst = m.layers[e.dst]
        rows = s.N * dst.W * dst.H
        so = f32(f32(e.cfg.get("scale_gradients", 1.0)) / s.N)
        y = s.grads[bs[0]:bs[1]]
        zero = torch.zeros(dst.C, dtype=torch.float32, device=y.device)
        above = m.edges[e.dst] if e.dst < len(m.edges) else None
        if len(m.group(k)) > 1 or dst.T > 1:
            # a tie group or a 3-D layer: one column sum per member (in back-propagation order) and per output frame,
            # on the side lane (no such edge hands its bias gradient to a pool undo, ConvNet::PlanFusion), the first
            # writing the gradient and each later one adding to the stored partial (st = 1): its bar covers that
            # addition (the st * b0 term), and the partial's own error carries over unscaled, so the bars add
            assert not any(m.plan[j]["offers_bias_grad"] for j in m.group(k)), "%s offers its bias gradient" % e.name
            exp = None
            for j in m.group(k)[::-1]:
                ej = m.edges[j]
                dj = m.layers[ej.dst]
                soj = f32(f32(ej.cfg.get("scale_gradients", 1.0)) / s.N)
                per = s.N * dj.W * dj.H
                for t in range(dj.T):
                    b0 = zero if exp is None else exp.ref.to(torch.float32)
                    x = ex.bias_grad(s.derivs[ej.dst][t * per * dj.C:(t + 1) * per * dj.C], per, dj.C, b0,
                                     0.0 if exp is None else 1.0, soj)
                    exp = x if exp is None else px.Expect(exp.ref + (x.ref - b0.to(torch.float64)), exp.bar + x.bar,
                                                          x.exact)
            how = "tie group sum" if len(m.group(k)) > 1 else "sum over %d frames" % dst.T
        elif above is not None and m.plan[e.dst]["sums_bias_below"] and m.plan[k]["offers_bias_grad"]:
            relu = m.plan[e.dst]["down_act"] == 1
            if above.kind == "UPSAMPLE":          # the block sum is a forward average pool on the big image
                pg, f = m.sample_geo(above, s.N)
                br = px.pool_fwd_branch(pg, False, so=float(f * f), epi=True)
            else:
                pg = m.sample_geo(above, s.N)[0] if above.kind == "DOWNSAMPLE" else m.pool_geo(above, s.N)
                br = px.pool_undo_branch(pg, above.kind == "MAXPOOL", mask="input" if relu else None,
                                         cached=above.kind == "MAXPOOL", epi=True)
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
            if e.kind == "RGBTOYUV":
                exp = ax.rgb_to_yuv(x[:3 * dst.W * dst.H * s.N])
            elif e.kind == "UPSAMPLE":            # replication of every pixel into its f x f block: exact
                f = int(e.cfg.get("sample_factor", 1))
                src = m.layers[e.src]
                big = x.to(torch.float64).view(src.C, src.H, src.W, s.N).repeat_interleave(f, 1).repeat_interleave(f, 2)
                exp = px.Expect(big.reshape(-1), torch.zeros(big.numel(), dtype=torch.float64, device=x.device),
                                torch.ones(big.numel(), dtype=torch.bool, device=x.device))
            elif e.kind == "DOWNSAMPLE":
                exp = px.pool_fwd(m.sample_geo(e, s.N)[0], x, False)
            else:
                exp = px.pool_fwd(m.pool_geo(e, s.N), x, e.kind == "MAXPOOL")
            if dst.act == "RECTIFIED_LINEAR":
                exp = px.Expect(exp.ref.clamp_min(0.0), exp.bar, exp.exact)
        if dst.act == "LOGISTIC":
            exp = _sigmoid(exp)
        if dst.dropprob > 0:
            exp = _dropout(exp, dst, s.seeds[e.dst])
        return _px_row(dst.name, "fprop", s.states[e.dst], exp)

    def pool_undo(self, s, k):
        m, e = self.m, self.m.edges[k]
        src = m.layers[e.src]
        mask = s.states[e.src] if src.act == "RECTIFIED_LINEAR" else None
        # the dropout fold of the layer below: its scale, one more rounding (the ReLU' mask of the dropped-out state
        # zeroes the dropped elements)
        so = dropout_scale(src.dropprob) if src.dropprob > 0 else 1.0
        if e.kind == "UPSAMPLE":
            pg, f = m.sample_geo(e, s.N)
            exp = px.pool_fwd(pg, s.derivs[e.dst], False, so=float(f * f))
            if mask is not None:
                drop = ~(mask[:exp.ref.numel()] > 0)
                exp = px.Expect(torch.where(drop, torch.zeros_like(exp.ref), exp.ref),
                                torch.where(drop, torch.zeros_like(exp.bar), exp.bar), exp.exact & ~drop)
        elif e.kind == "DOWNSAMPLE":
            exp = px.avg_undo(m.sample_geo(e, s.N)[0], s.derivs[e.dst], mask=mask)
        elif e.kind == "RESPONSE_NORM":
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
        if so != 1.0:
            ref = exp.ref * so
            exp = px.Expect(ref, exp.bar * so + U * ref.abs(), torch.zeros_like(exp.exact))
        if src.act == "LOGISTIC":
            exp = _logistic_deriv(exp, s.states[e.src])
        return _px_row(src.name, "undo", s.derivs[e.src], exp)

    # ---- output layer
    def output(self, s):
        m = self.m
        N = s.N
        C = m.layers[-1].floats(N) // N        # output features: units x pixels
        y = s.states[-1].to(torch.float64).view(C, N).t().cpu().numpy()
        if m.loss == lr.CE_MULTINOMIAL:
            d, d_bar, v, v_bar = lr.loss_ref(m.loss, y, labels=s.labels.cpu().numpy(), weight=m.loss_weight)
        else:
            t = s.targets[:N * C].to(torch.float64).view(C, N).t().cpu().numpy()
            d, d_bar, v, v_bar = lr.loss_ref(m.loss, y, t=t, weight=m.loss_weight)
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
            rule = RULES.get(c.get("optimizer_type", "STOCHASTIC_GRADIENT_DESCENT"))
            if rule is None:
                raise Unsupported("%s: optimizer %s" % (e.name, c["optimizer_type"]))
            st = s.opt_state[k][which]
            a, b = sl
            started = st["step"] >= int(c.get("start_optimization_after", 0))
            s_old = None if rule == opt.SGD else s.state_before[a:b].cpu().numpy()
            # (before its start an Adagrad tensor accumulates its state only; the other rules do nothing)
            if not started and rule != opt.ADAGRAD:
                w_new, h_new = s.params_before[a:b].cpu().numpy(), s.hist_before[a:b].cpu().numpy()
                s_new = s_old
            else:
                param = c.get("adagrad_delta", 1.0) if rule == opt.ADAGRAD else c.get("rms_prop_factor", 0.0)
                w_new, h_new, s_new = opt.opt_update(
                    s.params_before[a:b].cpu().numpy(), s.hist_before[a:b].cpu().numpy(), s_old,
                    s.grads[a:b].cpu().numpy(), rule, lr=st["epsilon"], mom=st["momentum"],
                    l2=max(c.get("l2_decay", 0.0), 0.0), clip=max(c.get("gradient_clip", -1.0), 0.0), param=param,
                    scale=opt.adagrad_scale(st["step"]), state_only=not started)
            near = np.zeros(b - a, bool)
            if which == "weights" and (c.get("weight_norm_constraint", 0) > 0 or c.get("weight_norm_limit", 0) > 0):
                mode, val = ((opt.CONSTRAINT, c["weight_norm_constraint"]) if c.get("weight_norm_constraint", 0) > 0
                             else (opt.LIMIT, c["weight_norm_limit"]))
                rows_ = m.conv_geo(e, s.N).Cout
                w_new, bite = opt.apply_norm(w_new, rows_, mode, f32(val))
                near = np.broadcast_to(bite, (len(w_new) // rows_, rows_)).reshape(-1)
            checks = [("update_" + which, s.params_after[a:b], w_new), ("history_" + which, s.hist_after[a:b], h_new)]
            if s_new is not None:
                checks.append(("state_" + which, s.state_after[a:b], s_new))
            for qty, got, want in checks:
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

    # ---- a frozen edge (block_backprop): forward only
    def frozen(self, s, k):
        """the edge's slice of the parameters, momentum history and adaptive state is bit-identical after the step, its
        slice of the gradient buffer still holds the sentinel (nothing wrote it), and the layer it writes has no
        derivative"""
        m, e = self.m, self.m.edges[k]
        a, b = m.offsets[k], (m.offsets[k + 1] if k + 1 < len(m.offsets) else m.total)
        rows = [Row(m.layers[e.dst].name, "frozen_deriv", s.derivs[e.dst] is None,
                    0.0, "" if s.derivs[e.dst] is None else "the frozen layer has a derivative")]
        if b == a:
            return rows
        pairs = [("frozen_params", s.params_after, s.params_before), ("frozen_history", s.hist_after, s.hist_before)]
        if s.state_before is not None:
            pairs.append(("frozen_state", s.state_after, s.state_before))
        sentinel = torch.full((m.total,), SENTINEL, dtype=torch.int32, device=s.grads.device).view(torch.float32)
        pairs.append(("frozen_grads", s.grads, sentinel))
        for qty, got, want in pairs:
            bad = got[a:b].view(torch.int32) != want[a:b].view(torch.int32)
            nbad = int(bad.sum())
            where = "first changed element %d" % (a + int(torch.nonzero(bad)[0])) if nbad else ""
            rows.append(Row(e.name, qty, nbad == 0, float(nbad), "%d changed %s" % (nbad, where)))
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
            if k < m.frozen:
                rows += self.fprop(s, k) if e.kind in WEIGHTED else [self.pool_fprop(s, k)]
                rows += self.frozen(s, k)
            elif e.kind in WEIGHTED:
                rows += self.fprop(s, k)
                if m.receives_deriv(e.src):
                    rows += self.dgrad(s, k)
                if m.owner[k] != k:           # a tied edge: its group's gradient and update are audited at the owner
                    continue
                rows += self.wgrad(s, k)
                if not e.cfg.get("has_no_bias", False):
                    rows.append(self.bias_grad(s, k))
                rows += self.update(s, k)
            else:
                rows.append(self.pool_fprop(s, k))
                if m.receives_deriv(e.src):
                    rows.append(self.pool_undo(s, k))
                if e.kind == "RGBTOYUV":
                    d = s.derivs[e.dst]
                    rows.append(Row(m.layers[e.dst].name, "no_deriv", d is None, 0.0,
                                    "" if d is None else "the RGBTOYUV output has a derivative"))
        rows += self.output(s)
        return rows


def failures(rows):
    return [r for r in rows if not r.ok]


# ---------------------------------------------------------------------------------------------------------------------
# a snapshot of a real step (needs a GPU)
# ---------------------------------------------------------------------------------------------------------------------


def run_step(n, model, warmup):
    """`warmup` training steps of Net `n`, then the audited one: returns its Snapshot and the names of the tensors in
    which the step left a sentinel NaN.  Call n.params_tensor() only here: the library drops every staged bf16 copy
    and filter bank when it hands out the parameter pointer, which would change the step being audited."""
    P, Hs, G = n.params_tensor(), n.history_tensor(), n.grads_tensor()
    assert n.trained_offset == model.trained_offset, (n.trained_offset, model.trained_offset)
    for _ in range(warmup):
        assert math.isfinite(n.train_step(True))
    torch.cuda.synchronize()
    L = len(model.layers)
    seeds = [int(n.dropout_seed(i)) for i in range(L)]
    opt_state = {k: n.optimizer_state(k) for k, e in enumerate(model.edges)
                 if e.kind in WEIGHTED and k >= model.frozen and model.owner[k] == k}
    A = n.adaptive_state_tensor()
    p0, h0, a0 = P.clone(), Hs.clone(), (None if A is None else A.clone())
    derivs = [None] + [n.layer_deriv(i) for i in range(1, L)]
    for d in derivs:
        if d is not None:
            d.view(torch.int32).fill_(SENTINEL)
    G.view(torch.int32).fill_(SENTINEL)
    torch.cuda.synchronize()
    loss = n.train_step(True)
    torch.cuda.synchronize()
    T = n.targets_tensor()
    s = Snapshot(n.batch_size, n.labels_tensor().clone(), [n.layer_state(i).clone() for i in range(L)],
                 [None if d is None else d.clone() for d in derivs], p0, h0, G.clone(), P.clone(), Hs.clone(),
                 loss, seeds, opt_state, None if T is None else T.clone(), a0, None if A is None else A.clone())
    left = ["deriv %s" % model.layers[i].name for i in range(1, L)
            if s.derivs[i] is not None and bool(torch.isnan(s.derivs[i]).any())]
    for k, e in enumerate(model.edges):
        if e.kind in WEIGHTED and k >= model.frozen:        # (a frozen slice keeps the sentinel: Auditor.frozen)
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
        T = n.targets_tensor()
        if T is not None:
            T.copy_(make_targets(model.loss, batch, T.numel() // batch, g).reshape(-1))
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


def make_targets(loss, N, C, g):
    """float targets (C, N) (column-major, image fastest) of an output layer trained on them: N(0, 1) regression
    targets; binary targets in {0, 1} with about one in eight -1 (don't care); a distribution over the classes per image
    (soft targets)"""
    dev = g.device
    if loss == lr.SQUARED_ERROR:
        return torch.randn(C, N, device=dev, generator=g)
    if loss == lr.CE_BINARY:
        t = (torch.rand(C, N, device=dev, generator=g) < 0.5).float()
        return torch.where(torch.rand(C, N, device=dev, generator=g) < 0.125, torch.full_like(t, -1.0), t)
    assert loss == lr.CE_DISTRIBUTED
    return torch.softmax(2 * torch.randn(C, N, device=dev, generator=g), 0)


def sample_dropout_text():
    """updowncheck with ReLU and dropout 0.25 on down1 and up4, the layers a DOWNSAMPLE and an UPSAMPLE write (fused into
    the average-pool row kernels in fprop), and on conv3, the layer below the DOWNSAMPLE down3 (its dropout folded into
    the sampling edge's derivative), as a model-file text"""
    from convnet_b200 import net
    t = net.model_text("updowncheck")
    for name in ("down1", "up4", "conv3"):
        i = t.index('name: "%s"' % name)
        j = t.index("activation: LINEAR", i)
        t = t[:j] + "activation: RECTIFIED_LINEAR" + t[j + len("activation: LINEAR"):]
        j = t.index("dropprob: 0", i)
        t = t[:j] + "dropprob: 0.25" + t[j + len("dropprob: 0"):]
    return t


def video_text():
    """a small 3-D net as a model-file text: 16 x 16 clips of 8 frames and 4 channels; conv1 (kt 2) and a 2 x 2 max pool
    within frames, conv2 with frame windows of 3 at stride_t 2 (overlapping: its dgrad sums two windows on every second
    frame), a 2 x 2 average pool with overlapping frame windows of 2 at stride_t 1 and c3d's global max pool
    (kernel_size 0, kernel_size_t 0) under an FC softmax.  At N 16 every conv call of bf16 mode takes the bf16 tensor
    cores."""
    return """name: "video"
seed: 42
default_weight_optimizer { epsilon: 0.01 final_momentum: 0.9 }
default_bias_optimizer { epsilon: 0.01 final_momentum: 0.9 }
layer { name: "input" num_channels: 4 image_size_y: 16 image_size_x: 16 image_size_t: 8 }
layer { name: "conv1" num_channels: 16 activation: RECTIFIED_LINEAR }
layer { name: "pool1" num_channels: 16 }
layer { name: "conv2" num_channels: 32 activation: RECTIFIED_LINEAR }
layer { name: "pool2" num_channels: 32 }
layer { name: "pool3" num_channels: 32 }
layer { name: "output" num_channels: 10 activation: SOFTMAX }
edge { source: "input" dest: "conv1" edge_type: CONVOLUTIONAL kernel_size: 3 padding: 1 kernel_size_t: 2
       shared_bias: true initialization: DENSE_UNIFORM_SQRT_FAN_IN }
edge { source: "conv1" dest: "pool1" edge_type: MAXPOOL kernel_size: 2 stride: 2 }
edge { source: "pool1" dest: "conv2" edge_type: CONVOLUTIONAL kernel_size: 3 padding: 1 kernel_size_t: 3 stride_t: 2
       shared_bias: true initialization: DENSE_UNIFORM_SQRT_FAN_IN }
edge { source: "conv2" dest: "pool2" edge_type: AVERAGE_POOL kernel_size: 2 stride: 2 kernel_size_t: 2 }
edge { source: "pool2" dest: "pool3" edge_type: MAXPOOL kernel_size: 0 kernel_size_t: 0 }
edge { source: "pool3" dest: "output" edge_type: FC initialization: DENSE_UNIFORM_SQRT_FAN_IN }
"""


def _sgd_config(model, edge):
    """the weight optimizer block of `edge` as OptimizerConfig fields"""
    from convnet_b200.net import OptimizerConfig
    c = model.edges[[e.name for e in model.edges].index(edge)].cfg["weight_optimizer"][0]
    names = [f[0] for f in OptimizerConfig._fields_]
    return {k: (int(v) if isinstance(v, float) and k in ("epsilon_decay_timescale", "momentum_transition_timescale",
                                                         "start_optimization_after") else v)
            for k, v in c.items() if k in names}
