"""GPU tests of batch normalisation (cnb_bn_stats / cnb_bn_apply / cnb_bn_backward, Layer::ApplyBatchNormalization and
its derivative in host/convnet.cc, the "+bn" models): the kernels against a float64 numpy restatement, the whole net
against float64 PyTorch autograd, the running statistics, the update paths, the grad check, training, bf16 coherence
and data-parallel replicas."""
import json
import math
import os
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SHAPES = [(128, 4096), (32 * 55 * 55, 16), (100 * 25 * 25, 48)]       # (N * pixels, channels)


@pytest.fixture(scope="module")
def env():
    import torch
    assert torch.cuda.is_available()
    from convnet_b200 import lib, net
    L = lib.load(); net.load_host()
    yield torch, lib, L, net
    lib.set_precision("fp32")


def _rel(got, ref):
    got = np.asarray(got, dtype=np.float64)
    return float(np.abs(got - ref).max() / max(np.abs(ref).max(), 1e-30))


@pytest.mark.parametrize("n,C", SHAPES)
def test_kernels_match_float64(env, n, C):
    torch, lib, L, _ = env
    lib.set_precision("fp32")
    g = torch.Generator(device="cuda").manual_seed(n + C)
    # channels with an offset far from 0 and different scales: the variance must be taken about the mean
    x = (torch.randn(C, n, device="cuda", generator=g) * (torch.rand(C, 1, device="cuda", generator=g) * 2 + 0.1)
         + torch.randn(C, 1, device="cuda", generator=g) * 4).reshape(-1)
    d = torch.randn(C * n, device="cuda", generator=g)
    gamma = torch.rand(C, device="cuda", generator=g) + 0.5
    beta = torch.randn(C, device="cuda", generator=g)
    run = torch.cat([torch.randn(C, device="cuda", generator=g), torch.rand(C, device="cuda", generator=g) + 0.5])
    bm, bs = torch.empty(C, device="cuda"), torch.empty(C, device="cuda")
    eps, f = 1e-5, 0.9
    X, D = x.double().view(C, n).cpu().numpy(), d.double().view(C, n).cpu().numpy()
    G, B, R = gamma.double().cpu().numpy(), beta.double().cpu().numpy(), run.double().cpu().numpy()

    rm, rs = run[:C].clone(), run[C:].clone()
    L.cnb_bn_stats(x.data_ptr(), n, C, eps, f, bm.data_ptr(), bs.data_ptr(), rm.data_ptr(), rs.data_ptr())
    mu = X.mean(1)
    sig = np.sqrt(((X - mu[:, None]) ** 2).mean(1) + eps)
    assert _rel(bm.cpu(), mu) < 1e-5 and _rel(bs.cpu(), sig) < 1e-5
    assert _rel(rm.cpu(), f * R[:C] + (1 - f) * mu) < 1e-5 and _rel(rs.cpu(), f * R[C:] + (1 - f) * sig) < 1e-5

    for train in (True, False):
        m_, s_ = (bm, bs) if train else (run[:C], run[C:])
        M, S = (mu, sig) if train else (R[:C], R[C:])
        xh = (X - M[:, None]) / S[:, None]
        for relu in (0, 1):
            y = torch.empty_like(x)
            L.cnb_bn_apply(x.data_ptr(), y.data_ptr(), n, C, gamma.data_ptr(), beta.data_ptr(), m_.data_ptr(), s_.data_ptr(), relu)
            Y = G[:, None] * xh + B[:, None]
            assert _rel(y.view(C, n).cpu(), np.maximum(Y, 0) if relu else Y) < 1e-5, (train, relu)
        dx, gg, gb = d.clone(), torch.empty(C, device="cuda"), torch.empty(C, device="cuda")
        L.cnb_bn_backward(dx.data_ptr(), x.data_ptr(), n, C, gamma.data_ptr(), m_.data_ptr(), s_.data_ptr(), int(train),
                          gg.data_ptr(), gb.data_ptr())
        rb, rg = D.mean(1), (D * xh).mean(1)
        ref = (G / S)[:, None] * ((D - rb[:, None] - xh * rg[:, None]) if train else D)
        assert _rel(gb.cpu(), rb) < 1e-5 and _rel(gg.cpu(), rg) < 1e-5, train
        assert _rel(dx.view(C, n).cpu(), ref) < 1e-5, train

        # deterministic: a second run gives the same bits
        dx2, gg2, gb2 = d.clone(), torch.empty(C, device="cuda"), torch.empty(C, device="cuda")
        L.cnb_bn_backward(dx2.data_ptr(), x.data_ptr(), n, C, gamma.data_ptr(), m_.data_ptr(), s_.data_ptr(), int(train),
                          gg2.data_ptr(), gb2.data_ptr())
        assert torch.equal(dx, dx2) and torch.equal(gg, gg2) and torch.equal(gb, gb2)
    bm2, bs2 = torch.empty(C, device="cuda"), torch.empty(C, device="cuda")
    L.cnb_bn_stats(x.data_ptr(), n, C, eps, f, bm2.data_ptr(), bs2.data_ptr(), None, None)
    assert torch.equal(bm, bm2) and torch.equal(bs, bs2)


def test_bf16_twins_equal_the_rounded_outputs():
    env_ = dict(os.environ, CONVNET_B200_STAGE_VERIFY="1")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "bn_worker.py"), "twin"], capture_output=True, text=True,
                       timeout=600, env=env_)
    assert r.returncode == 0 and "BN-TWIN-OK" in r.stdout, (r.returncode, r.stdout[-1500:], r.stderr[-1500:])


# float64 autograd mirror of "tiny+bn": tests/test_gpu_net.py's "tiny" with batch normalisation before the ReLU of conv1,
# nin1 and conv2.  spec entries as there, "conv" with a trailing bn flag
TINY_BN = [("conv", 16, 3, 1, 1, True, True), ("maxpool", 3, 2, 1), ("rnorm", 8, 0.01, 0.75, True),
           ("conv", 24, 1, 1, 0, True, True), ("conv", 16, 3, 2, 1, True, True), ("avgpool", 2, 2, 0), ("fc", 10)]


def _mirror(torch, n, batch, running=None, eps=1e-5):
    """loss, {edge: (w, b, K)}, {layer: (gamma, beta, pixels)}, {layer: (mean, sigma)} of the batch.  running: {layer:
    (mean, sigma)} -> the test-mode transform"""
    import torch.nn.functional as Fn
    P = n.params_tensor().double()
    edges = n.edges()
    bn_off = {i: off for i, _, _, off in n.bn_layers()}
    params, bnp, stats = {}, {}, {}
    h = n.input_tensor().double().view(8, 12, 12, batch).permute(3, 0, 1, 2).contiguous()
    for i, e in enumerate(TINY_BN):
        if e[0] == "conv":
            _, cout, k, s, p, relu, bn = e
            off, size = edges[i][2], edges[i][3]
            K = h.shape[1] * k * k
            flat = P[off:off + size]
            w = flat[:cout * K].view(K, cout).view(h.shape[1], k, k, cout).permute(3, 0, 1, 2).contiguous().requires_grad_(True)
            b = flat[cout * K:cout * K + cout].clone().requires_grad_(True)
            params[i] = (w, b, K)
            h = Fn.conv2d(h, w, b, stride=s, padding=p)
            if bn:
                o = bn_off[i + 1]
                ga = P[o:o + cout].clone().requires_grad_(True)
                be = P[o + cout:o + 2 * cout].clone().requires_grad_(True)
                bnp[i + 1] = (ga, be, h.shape[2] * h.shape[3])
                if running is None:
                    stats[i + 1] = (h.mean((0, 2, 3)).detach(), (h.var((0, 2, 3), unbiased=False) + eps).sqrt().detach())
                    h = Fn.batch_norm(h, None, None, ga, be, training=True, eps=eps)
                else:
                    m, sg = running[i + 1]
                    h = (h - m[None, :, None, None]) / sg[None, :, None, None] * ga[None, :, None, None] + be[None, :, None, None]
            h = torch.relu(h) if relu else h
        elif e[0] == "maxpool":
            h = Fn.max_pool2d(h, e[1], e[2], e[3])
        elif e[0] == "avgpool":
            h = Fn.avg_pool2d(h, e[1], e[2], e[3], count_include_pad=False)
        elif e[0] == "rnorm":
            _, k, a, bpow, relu = e
            F_ = h.shape[1]
            sq = Fn.pad(h * h, (0, 0, 0, 0, k // 2, k - k // 2 - 1))
            h = h * (1 + a * sum(sq[:, j:j + F_] for j in range(k))) ** (-bpow)
            h = torch.relu(h) if relu else h
        elif e[0] == "fc":
            cout, K = e[1], h.shape[1] * h.shape[2] * h.shape[3]
            off, size = edges[i][2], edges[i][3]
            flat = P[off:off + size]
            w = flat[:cout * K].view(K, cout).clone().requires_grad_(True)
            b = flat[cout * K:cout * K + cout].clone().requires_grad_(True)
            params[i] = (w, b, K)
            h = h.reshape(batch, K) @ w + b
    probs = torch.softmax(h, 1)
    loss = Fn.cross_entropy(h, n.labels_tensor().long(), reduction="sum")
    loss.backward()
    return loss.item(), params, bnp, stats, probs.detach()


def _compare_grads(torch, n, batch, params, bnp, mode, tol, train):
    G = n.grads_tensor().double()
    edges = n.edges()
    bn_off = {i: off for i, _, _, off in n.bn_layers()}
    checks = []
    for i, (w, b, K) in params.items():
        off, cout = edges[i][2], b.shape[0]
        gw = G[off:off + cout * K].view(K, cout)
        if w.dim() == 4:
            gw = gw.view(w.shape[1], w.shape[2], w.shape[3], cout).permute(3, 0, 1, 2)
        gb = G[off + cout * K:off + cout * K + cout]
        checks.append((edges[i][0] + " w", gw, w.grad / batch, None))
        # the bias of an edge that feeds a training-mode BN layer has gradient 0 (the batch mean absorbs it): both sides
        # are rounding noise, measured against the scale of that edge's weight gradient instead
        absorbed = train and (i + 1) in bn_off
        checks.append((edges[i][0] + " b", gb, b.grad / batch, (w.grad / batch).abs().mean() if absorbed else None))
    for l, (ga, be, pix) in bnp.items():
        o, c = bn_off[l], ga.shape[0]
        nn = batch * pix                                      # gamma / beta: the reference's 1 / (N * pixels)
        checks += [("layer %d gamma" % l, G[o:o + c], ga.grad / nn, None), ("layer %d beta" % l, G[o + c:o + 2 * c], be.grad / nn, None)]
    for name, mine, ref, scale in checks:
        if scale is not None:
            err = ((mine - ref).abs().max() / scale).item()
        elif mode == "fp32":
            err = ((mine - ref).abs().max() / ref.abs().mean().clamp_min(1e-12)).item()
        else:
            err = ((mine - ref).norm() / ref.norm().clamp_min(1e-12)).item()
        assert err < tol, (mode, name, err)


def _tiny_bn(torch, net, batch, seed=7, data_seed=11):
    n = net.Net("tiny+bn", batch, seed=seed)
    g = torch.Generator(device="cuda").manual_seed(data_seed)
    n.input_tensor().normal_(generator=g)
    n.labels_tensor().copy_(torch.randint(0, n.num_classes, (batch,), device="cuda", generator=g, dtype=torch.int32))
    return n


def test_backprop_matches_float64_autograd(env):
    """training-mode forward and backward of "tiny+bn" against float64 autograd with F.batch_norm (biased variance, eps
    inside the square root), at the tolerances of test_gpu_net.py::test_backprop_matches_float64_autograd"""
    torch, lib, _, net = env
    for mode, tol in (("fp32", 2e-5), ("tf32", 5e-2), ("bf16", 1.5e-1)):
        lib.set_precision(mode)
        batch = 32
        n = _tiny_bn(torch, net, batch)
        assert [l[1] for l in n.bn_layers()] == ["conv1", "nin1", "conv2"]
        n.fprop(True); n.bprop()
        loss = n.loss()
        ref_loss, params, bnp, stats, _ = _mirror(torch, n, batch)
        assert abs(loss - ref_loss) / ref_loss < {"fp32": 1e-5, "tf32": 2e-3, "bf16": 1e-2}[mode]
        _compare_grads(torch, n, batch, params, bnp, mode, tol, True)
        n.close()


def test_running_statistics_and_test_mode(env):
    """three training steps, then: the running statistics follow mu = f*mu + (1-f)*batch mean (sigma likewise, from 0 / 1)
    over the batch statistics of every step; the batch statistics of a fourth training fprop match the mirror's; a
    test-mode fprop matches the mirror's eval transform, and a test-mode bprop its gradients"""
    torch, lib, _, net = env
    lib.set_precision("fp32")
    batch, f = 32, 0.98
    n = _tiny_bn(torch, net, batch, data_seed=3)
    layers = [l[0] for l in n.bn_layers()]
    run = {l: (np.zeros(n.bn_state(l)["gamma"].numel()), np.ones(n.bn_state(l)["gamma"].numel())) for l in layers}

    def follow():
        for l in layers:
            s = n.bn_state(l)
            m, sg = run[l]
            run[l] = (f * m + (1 - f) * s["batch_mean"].double().cpu().numpy(),
                      f * sg + (1 - f) * s["batch_sigma"].double().cpu().numpy())

    for _ in range(3):
        n.train_step(False)
        follow()
    n.fprop(True)
    follow()
    _, _, _, stats, _ = _mirror(torch, n, batch)
    for l in layers:
        s = n.bn_state(l)
        assert _rel(s["batch_mean"].cpu(), stats[l][0].cpu().numpy()) < 1e-5
        assert _rel(s["batch_sigma"].cpu(), stats[l][1].cpu().numpy()) < 1e-5
        assert _rel(s["running_mean"].cpu(), run[l][0]) < 1e-5 and _rel(s["running_sigma"].cpu(), run[l][1]) < 1e-5
        assert not torch.equal(s["gamma"], torch.ones_like(s["gamma"]))                # gamma trained
    n.fprop(False)
    out = n.output_tensor().view(10, batch).t().double()
    n.bprop()
    running = {l: (n.bn_state(l)["running_mean"].double(), n.bn_state(l)["running_sigma"].double()) for l in layers}
    _, params, bnp, _, probs = _mirror(torch, n, batch, running=running)
    assert ((out - probs).abs().max() / probs.abs().max()).item() < 1e-5
    _compare_grads(torch, n, batch, params, bnp, "fp32", 2e-5, False)
    st = n.bn_optimizer_state(layers[0])
    assert st["gamma"]["step"] == 3 and st["beta"]["step"] == 3
    n.close()


def test_eager_and_stand_alone_updates_agree(env):
    torch, lib, _, net = env
    lib.set_precision("bf16")
    a, b = _tiny_bn(torch, net, 32), _tiny_bn(torch, net, 32)
    for n in (a, b):
        n.set_bn_optimizer("conv2", gamma={"epsilon": 0.02, "initial_momentum": 0.5, "final_momentum": 0.9,
                                           "momentum_transition_timescale": 3}, beta={"epsilon": 0.005, "gradient_clip": 0.01})
    for _ in range(3):
        a.train_step(False)
        b.fprop(True); b.bprop(); b.update()
    torch.cuda.synchronize()
    assert torch.equal(a.params_tensor(), b.params_tensor())
    assert a.bn_optimizer_state("conv2") == b.bn_optimizer_state("conv2")
    fresh = _tiny_bn(torch, net, 32)
    p0 = fresh.params_tensor().clone()
    fresh.close()
    for _, _, c, o in a.bn_layers():
        assert not torch.equal(a.params_tensor()[o:o + 2 * c], p0[o:o + 2 * c])
    with pytest.raises(ValueError):
        a.set_bn_optimizer("conv2", gamma={"epsilon": 0.01, "weight_norm_limit": 1.0})
    with pytest.raises(KeyError):
        a.bn_state("pool1")
    a.close(); b.close()
    lib.set_precision("fp32")


def test_grad_check_passes_on_bn_net(env):
    """run_grad_check (test-mode forward, so the finite differences see the running-statistics transform) on
    "gradcheck+bn", at the bound "gradcheck" meets"""
    torch, lib, _, net = env
    lib.set_precision("fp32")
    for seed in (1, 5):
        n = net.Net("gradcheck+bn", 8, seed=3, grad_checker=True)
        res = n.grad_check(seed=seed)
        n.close()
        assert len(res) == 3
        for name, eps, dw, db in res:
            assert dw < 5e-4 and db < 5e-4, (seed, res)


@pytest.mark.parametrize("model,batch", [("tiny+bn", 32), ("lenet+bn", 100)])
def test_training_reduces_the_loss(env, model, batch):
    torch, lib, _, net = env
    lib.set_precision("bf16")
    n = net.Net(model, batch, seed=1)
    g = torch.Generator(device="cuda").manual_seed(0)
    n.input_tensor().normal_(generator=g)
    n.labels_tensor().copy_(torch.randint(0, 10, (batch,), device="cuda", generator=g, dtype=torch.int32))
    losses = [n.train_step(True) / batch for _ in range(40)]
    n.close()
    lib.set_precision("fp32")
    assert all(math.isfinite(v) for v in losses)
    assert min(losses[20:]) < 0.8 * losses[0], losses[::5]


def test_alexnet_bn_step_keeps_bf16_copies_coherent():
    """tests/staging_worker.py "train" under CONVNET_B200_STAGE_VERIFY=1: every staged copy the BN passes write or
    invalidate is checked at its next use"""
    env_ = dict(os.environ, CONVNET_B200_STAGE_VERIFY="1")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "staging_worker.py"), "train", "alexnet+bn", "8", "2"],
                       capture_output=True, text=True, timeout=900, env=env_)
    assert r.returncode == 0 and "VERIFY-TRAIN-OK" in r.stdout, (r.returncode, r.stdout[-1500:], r.stderr[-1500:])


def test_data_parallel_replicas_stay_bit_identical():
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr",
           "127.0.0.1", "--master-port", "29521", os.path.join(ROOT, "tests", "bn_worker.py"), "dp", "lenet+bn", "32"]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, env=dict(os.environ, MASTER_ADDR="127.0.0.1"))
    line = [ln for ln in r.stdout.splitlines() if ln.startswith("{")]
    assert r.returncode == 0 and line, (r.returncode, r.stdout[-2000:], r.stderr[-2000:])
    res = json.loads(line[-1])
    assert res["identical"] and res["gammas_moved"], res
