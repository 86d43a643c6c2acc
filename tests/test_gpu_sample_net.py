"""Nets with UPSAMPLE, DOWNSAMPLE and RGBTOYUV edges on the GPU: updowncheck passes run_grad_check; the RGBTOYUV layer
holds RGBToYUV's output, receives no derivative and the edge above it runs no dgrad; the dropout fusions on layers
written by both sampling edges train bit-identically to the separate passes; updown trains from its model_text
bit-identically to the built-in; updowncheck's and a reduced updown's states, derivatives and gradients against float64
autograd in fp32, tf32 and bf16; sampling on a 3-D layer; a 2-rank data-parallel run (skipped on one GPU)."""
import json
import math
import os
import subprocess
import sys

import pytest
import torch

from convnet_b200 import net as N

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_updowncheck_passes_grad_check():
    n = N.Net("updowncheck", 8, seed=5, grad_checker=True)
    try:
        res = n.grad_check(seed=3)
    finally:
        n.close()
    assert len(res) == 5      # the four convs and the FC
    assert all(dw < 0.01 and db < 0.01 for _, _, dw, db in res), res


SMALL = """name: "small-updown"
seed: 11
layer { name: "input" num_channels: 3 image_size_y: 16 image_size_x: 16 }
layer { name: "yuv" num_channels: 3 }
layer { name: "c1" num_channels: 8 activation: RECTIFIED_LINEAR }
layer { name: "d1" num_channels: 8 activation: RECTIFIED_LINEAR dropprob: 0.25 }
layer { name: "c2" num_channels: 16 activation: RECTIFIED_LINEAR }
layer { name: "u2" num_channels: 16 activation: RECTIFIED_LINEAR dropprob: 0.25 }
layer { name: "output" num_channels: 3 loss_function: SQUARED_ERROR performance_metric: SQUARED_ERROR }
edge { source: "input" dest: "yuv" edge_type: RGBTOYUV }
edge { source: "yuv" dest: "c1" edge_type: CONVOLUTIONAL kernel_size: 3 padding: 1 shared_bias: true }
edge { source: "c1" dest: "d1" edge_type: DOWNSAMPLE sample_factor: 2 }
edge { source: "d1" dest: "c2" edge_type: CONVOLUTIONAL kernel_size: 3 padding: 1 shared_bias: true }
edge { source: "c2" dest: "u2" edge_type: UPSAMPLE sample_factor: 2 }
edge { source: "u2" dest: "output" edge_type: CONVOLUTIONAL kernel_size: 3 padding: 1 shared_bias: true }
"""


def _write(tmp_path, text, name="net.pbtxt"):
    p = tmp_path / name
    p.write_text(text)
    return str(p)


def test_yuv_layer_state_and_no_derivative(tmp_path):
    from convnet_b200 import lib
    from convnet_b200.matrix import CUDAMatrix
    path = _write(tmp_path, SMALL)
    n = N.Net(path, 8, seed=2)
    try:
        torch.manual_seed(1)
        n.input_tensor().normal_()
        n.fprop(True)
        torch.cuda.synchronize()
        x = CUDAMatrix(8, 16 * 16 * 3, (8, 16, 16, 3), storage=n.input_tensor().clone())
        y = CUDAMatrix(8, 16 * 16 * 3, (8, 16, 16, 3))
        lib.load().RGBToYUV(x.p_mat, y.p_mat)
        torch.cuda.synchronize()
        assert torch.equal(n.layer_state(1), y.storage)
        assert n.layer_deriv(0) is None and n.layer_deriv(1) is None and n.layer_deriv(2) is not None
        n.bprop()
        torch.cuda.synchronize()
        assert torch.isfinite(n.grads_tensor()).all() and n.grads_tensor().abs().sum() > 0
    finally:
        n.close()


def _params_run(path, **env):
    e = dict(os.environ, **env)
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "staging_worker.py"), "params", path, "16", "3"],
                       capture_output=True, text=True, timeout=1200, env=e)
    assert r.returncode == 0, r.stderr[-2000:]
    return [l for l in r.stdout.splitlines() if l.startswith("PARAMS")][-1]


def test_dropout_fusions_train_bit_identically(tmp_path):
    """ReLU + dropout on the layers DOWNSAMPLE (d1) and UPSAMPLE (u2) write: the fused dropout and the dropout fold against
    the mask tensor and its passes, three bf16 training steps each"""
    path = _write(tmp_path, SMALL)
    plan = N.model_fusion(path)
    assert plan["edges"][2]["dropout_up"] and plan["edges"][4]["dropout_up"]
    assert plan["edges"][3]["scale_down"] and plan["edges"][5]["scale_down"]
    fused = _params_run(path)
    plain = _params_run(path, CONVNET_B200_NO_FUSED_DROPOUT="1", CONVNET_B200_NO_DROPOUT_FOLD="1")
    assert fused == plain


def _train(model, steps=2):
    n = N.Net(model, 16, seed=4)
    try:
        g = torch.Generator(device="cuda").manual_seed(9)
        n.input_tensor().copy_(torch.randn(n.input_floats, device="cuda", generator=g))
        n.targets_tensor().copy_(torch.randn(n.targets_tensor().numel(), device="cuda", generator=g))
        losses = [n.train_step(True) for _ in range(steps)]
        torch.cuda.synchronize()
        return losses, n.params_tensor().clone()
    finally:
        n.close()


def test_updown_trains_from_its_model_text(tmp_path):
    a_loss, a = _train("updown")
    b_loss, b = _train(_write(tmp_path, N.model_text("updown")))
    assert all(math.isfinite(v) for v in a_loss) and a_loss == b_loss and torch.equal(a, b)


# the float64 restatements: per layer after the input, (kind, channels, activation, factor); "conv" is 3x3 padding 1 with a
# shared bias, "fc" an FC edge into a softmax output
REDUCED = [("yuv", 3, "linear", 0), ("conv", 8, "relu", 0), ("down", 8, "relu", 2), ("conv", 16, "relu", 0),
           ("up", 16, "relu", 2), ("conv", 3, "linear", 0)]
UPDOWNCHECK = [("conv", 8, "linear", 0), ("down", 8, "linear", 3), ("conv", 8, "linear", 0), ("up", 8, "logistic", 3),
               ("conv", 6, "linear", 0), ("down", 6, "linear", 2), ("conv", 6, "linear", 0), ("up", 6, "linear", 2),
               ("fc", 5, "softmax", 0)]
# relative L2 bars of test_gpu_local_net.py (tf32 / bf16), and fp32's for states and derivatives
BARS = {"fp32": (1e-4, 1e-3), "tf32": (5e-2, 5e-2), "bf16": (1.5e-1, 1.5e-1)}
LOSS_BARS = {"fp32": 1e-5, "tf32": 2e-3, "bf16": 1e-2}


def _rel(a, b):
    return ((a - b).norm() / b.norm().clamp_min(1e-30)).item()


def _mirror(n, spec, B, first):
    """the net's forward pass and loss in float64 on its own parameters and on the state of layer `first` (the input, or
    the layer RGBTOYUV writes); returns {layer: (state, pre-activation)}, {edge: (w, b)} and the loss"""
    import torch.nn.functional as F
    params = n.params_tensor().double()
    offs = [e[2] for e in n.edges()]
    C, S = (3, 16) if first == 1 else (4, 6)
    x = n.layer_state(first).double().view(C, S, S, B).permute(3, 0, 1, 2)
    layers, weights = {}, {}
    for k, (kind, cout, act, f) in enumerate(spec, start=1):
        if k <= first:
            continue
        o = offs[k - 1]
        if kind == "conv":
            cin = x.shape[1]
            w = params[o:o + cout * 9 * cin].view(cin, 3, 3, cout).permute(3, 0, 1, 2).clone().requires_grad_(True)
            b = params[o + cout * 9 * cin:o + cout * 9 * cin + cout].clone().requires_grad_(True)
            weights[k - 1] = (w, b)
            pre = F.conv2d(x, w, b, padding=1)
        elif kind == "fc":
            K = x[0].numel()
            w = params[o:o + cout * K].view(K, cout).clone().requires_grad_(True)
            b = params[o + cout * K:o + cout * K + cout].clone().requires_grad_(True)
            weights[k - 1] = (w, b)
            pre = x.reshape(B, K) @ w + b
        elif kind == "down":
            pre = F.avg_pool2d(x, f)
        else:
            pre = x.repeat_interleave(f, 2).repeat_interleave(f, 3)
        pre.retain_grad()
        x = {"relu": F.relu, "logistic": torch.sigmoid, "linear": lambda v: v, "softmax": lambda v: v}[act](pre)
        layers[k] = (x, pre)
    if spec[-1][2] == "softmax":
        labels = n.labels_tensor().long()
        loss = F.cross_entropy(x, labels, reduction="sum")
    else:
        t = n.targets_tensor().double().view(x.shape[1], x.shape[2], x.shape[3], B).permute(3, 0, 1, 2)
        loss = 0.5 * ((x - t) ** 2).sum()
    loss.backward()
    return layers, weights, loss.item()


@pytest.mark.parametrize("mode", ["fp32", "tf32", "bf16"])
@pytest.mark.parametrize("model", ["reduced-updown", "updowncheck"])
def test_backprop_matches_float64_autograd(tmp_path, model, mode):
    """one training forward and backward pass (no dropout): the loss, every layer's state and derivative and every
    weight and bias gradient against float64 autograd on the net's own parameters, in fp32, tf32 and bf16 — in bf16 the
    convs read the bf16 twins the sampling kernels write"""
    from convnet_b200 import lib
    B = 32
    lib.set_precision(mode)
    name = _write(tmp_path, SMALL.replace(" dropprob: 0.25", "")) if model == "reduced-updown" else "updowncheck"
    spec = REDUCED if model == "reduced-updown" else UPDOWNCHECK
    n = N.Net(name, B, seed=6)
    try:
        g = torch.Generator(device="cuda").manual_seed(3)
        n.input_tensor().copy_(torch.randn(n.input_floats, device="cuda", generator=g))
        if n.targets_tensor() is not None:
            n.targets_tensor().copy_(torch.randn(n.targets_tensor().numel(), device="cuda", generator=g))
        else:
            n.labels_tensor().copy_(torch.randint(0, n.num_classes, (B,), device="cuda", generator=g, dtype=torch.int32))
        n.fprop(True)
        n.bprop()
        torch.cuda.synchronize()
        loss = n.loss()
        layers, weights, ref_loss = _mirror(n, spec, B, 1 if model == "reduced-updown" else 0)
        assert abs(loss - ref_loss) / ref_loss < LOSS_BARS[mode], (mode, loss, ref_loss)
        bar_act, bar_grad = BARS[mode]
        for k, (state, pre) in layers.items():
            if k < len(spec):                    # (the output's state is the softmax / linear result: the loss covers it)
                got = n.layer_state(k).double().view(*state.shape[1:], B).permute(3, 0, 1, 2)
                assert _rel(got, state.detach()) < bar_act, (mode, "state", k)
            gd = n.layer_deriv(k).double().view(*pre.shape[1:], B).permute(3, 0, 1, 2) if pre.dim() == 4 else \
                n.layer_deriv(k).double().view(-1, B).t()
            assert _rel(gd, pre.grad) < bar_act, (mode, "deriv", k)
        G = n.grads_tensor().double()
        offs = [e[2] for e in n.edges()]
        for i, (w, b) in weights.items():
            o = offs[i]
            if w.dim() == 4:
                cout, cin = w.shape[0], w.shape[1]
                gw = G[o:o + cout * 9 * cin].view(cin, 3, 3, cout).permute(3, 0, 1, 2)
                gb = G[o + cout * 9 * cin:o + cout * 9 * cin + cout]
            else:
                K, cout = w.shape
                gw, gb = G[o:o + cout * K].view(K, cout), G[o + cout * K:o + cout * K + cout]
            assert _rel(gw, w.grad / B) < bar_grad, (mode, i, "w")     # the net averages over the images
            assert _rel(gb, b.grad / B) < bar_grad, (mode, i, "b")
    finally:
        n.close()
        lib.set_precision("fp32")


def _bprop_launches(path):
    from convnet_b200 import lib
    L = lib.load()
    n = N.Net(path, 8, seed=2)
    try:
        n.input_tensor().normal_()
        n.fprop(True); n.bprop()                 # (the first step learns the conv paths)
        n.fprop(True)
        torch.cuda.synchronize()
        L.convnet_b200_reset_launch_count()
        n.bprop()
        torch.cuda.synchronize()
        return int(L.convnet_b200_launch_count())
    finally:
        n.close()


def test_conv_above_the_yuv_layer_runs_no_dgrad(tmp_path):
    """the conv above the RGBTOYUV layer launches exactly what the same conv above the input layer launches (wgrad and
    bias gradient, no dgrad); the same net with a 1x1 conv in place of RGBTOYUV launches that conv's dgrad too"""
    from convnet_b200 import lib
    lib.set_precision("fp32")
    yuv = _bprop_launches(_write(tmp_path, SMALL, "yuv.pbtxt"))
    no_yuv = SMALL.replace('layer { name: "yuv" num_channels: 3 }\n', "").replace(
        'edge { source: "input" dest: "yuv" edge_type: RGBTOYUV }\n', "").replace('source: "yuv"', 'source: "input"')
    direct = _bprop_launches(_write(tmp_path, no_yuv, "direct.pbtxt"))
    one_by_one = _bprop_launches(_write(tmp_path, SMALL.replace("edge_type: RGBTOYUV", "edge_type: CONV_ONETOONE"), "c.pbtxt"))
    assert yuv == direct and one_by_one > yuv, (yuv, direct, one_by_one)


THREE_D = """name: "updown-3d"
seed: 5
layer { name: "input" num_channels: 4 image_size_y: 8 image_size_x: 8 image_size_t: 2 }
layer { name: "c" num_channels: 6 activation: RECTIFIED_LINEAR }
layer { name: "d" num_channels: 6 }
layer { name: "u" num_channels: 6 }
layer { name: "output" num_channels: 5 activation: SOFTMAX }
edge { source: "input" dest: "c" edge_type: CONVOLUTIONAL kernel_size: 3 padding: 1 shared_bias: true }
edge { source: "c" dest: "d" edge_type: DOWNSAMPLE sample_factor: 2 }
edge { source: "d" dest: "u" edge_type: UPSAMPLE sample_factor: 2 }
edge { source: "u" dest: "output" edge_type: FC }
"""


def test_sampling_on_a_3d_layer(tmp_path):
    """frames folded into the planes: on a 2-frame layer DOWNSAMPLE averages and UPSAMPLE replicates within each
    (channel, frame) plane, and their derivatives are the block sum and d / 4 under the ReLU' mask of the conv layer"""
    from convnet_b200 import lib
    import torch.nn.functional as F
    lib.set_precision("fp32")
    B = 8
    n = N.Net(_write(tmp_path, THREE_D), B, seed=3)
    try:
        n.input_tensor().normal_()
        n.labels_tensor().copy_(torch.randint(0, 5, (B,), device="cuda", dtype=torch.int32))
        n.fprop(True)
        n.bprop()
        torch.cuda.synchronize()
        planes = lambda t, S: t.double().view(12, S, S, B).permute(3, 0, 1, 2)          # 6 channels x 2 frames
        c, d, u = planes(n.layer_state(1), 8), planes(n.layer_state(2), 4), planes(n.layer_state(3), 8)
        assert torch.allclose(d, F.avg_pool2d(c, 2), rtol=1e-6, atol=1e-7)
        assert torch.equal(u, d.repeat_interleave(2, 2).repeat_interleave(2, 3))
        dc, dd, du = planes(n.layer_deriv(1), 8), planes(n.layer_deriv(2), 4), planes(n.layer_deriv(3), 8)
        # the block sum of four fp32 terms: within 4 roundings of the sum of their magnitudes
        err = (dd - 4 * F.avg_pool2d(du, 2)).abs()
        assert (err <= 2.4e-7 * 4 * F.avg_pool2d(du.abs(), 2) + 1e-30).all(), err.max().item()
        # d / 4 is exact: the ReLU'-masked derivative of the conv layer is exactly the replicated quarter
        assert torch.equal(dc, dd.repeat_interleave(2, 2).repeat_interleave(2, 3) / 4 * (c > 0))
        assert dd.abs().sum() > 0
    finally:
        n.close()


def test_data_parallel_sampling_net_matches_single_rank():
    """tests/dp_worker.py on updowncheck (both sampling edges at factors 2 and 3, no dropout): bit-identical replicas,
    equal to the 1-rank run on the global batch"""
    ngpu = torch.cuda.device_count()
    if ngpu < 2:
        pytest.skip("needs >= 2 GPUs")
    world = 2 if ngpu < 4 else 4
    env = dict(os.environ, DP_MODEL="updowncheck", DP_BATCH="32", DP_PRECISION="fp32", MASTER_ADDR="127.0.0.1")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(world),
           "--master-addr", "127.0.0.1", "--master-port", "29523", os.path.join(ROOT, "tests", "dp_worker.py")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=1200, env=env)
    line = [ln for ln in r.stdout.splitlines() if ln.startswith("{")]
    assert r.returncode == 0 and line, (r.returncode, r.stdout[-2000:], r.stderr[-2000:])
    res = json.loads(line[-1])
    assert res["ok"]
    for b in res["results"]:
        assert b["bit_identical_across_ranks"] and b["rel_diff_vs_1rank_global_batch"] < 1e-5 and b["max_param_change"] > 0
