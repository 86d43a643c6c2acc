"""The Adagrad and RMSProp optimizers on the GPU (cnb_opt_update_multi, ADAGRAD_SGD / RMSPROP_SGD): the kernel against the
float32 restatement of tests/opt_rules.py bit for bit, the state against the reference's (tests/golden/ref_opt.npz), and
nets trained with the rules against a numpy replay of their recorded gradients."""
import ctypes as ct
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import opt_rules as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu


class CnbOptTensor(ct.Structure):           # include/convnet_b200_ext.h
    _fields_ = [("w", ct.c_void_p), ("hist", ct.c_void_p), ("grad", ct.c_void_p), ("n", ct.c_longlong),
                ("lr", ct.c_float), ("momentum", ct.c_float), ("l2", ct.c_float), ("clip", ct.c_float),
                ("rows", ct.c_int), ("norm_mode", ct.c_int), ("norm_value", ct.c_float)]


class CnbOptTensorEx(ct.Structure):
    _fields_ = [("t", CnbOptTensor), ("rule", ct.c_int), ("state_only", ct.c_int), ("state", ct.c_void_p),
                ("rule_param", ct.c_float), ("scale", ct.c_float)]


def _ex(spec, w, h, g, s):
    t = CnbOptTensor(w.data_ptr(), h.data_ptr(), g.data_ptr(), w.numel(), spec["lr"], spec["mom"], spec["l2"], spec["clip"],
                     spec["rows"], spec["mode"], spec["value"])
    return CnbOptTensorEx(t, spec["rule"], int(spec.get("state_only", False)), s.data_ptr() if s is not None else None,
                          spec.get("param", 0.0), spec.get("scale", 1.0))


def _bits(a):
    return np.asarray(a, np.float32).view(np.uint32)


def _check(tag, spec, host, dev):
    """h and s bit for bit; w bit for bit outside the rows a norm rule rescales, there within 2e-6"""
    w0, h0, g0, s0 = host
    w, h, s = (None if t is None else t.cpu().numpy() for t in dev)
    rw, rh, rs = R.opt_update(w0, h0, s0, g0, spec["rule"], spec["lr"], spec["mom"], spec["l2"], spec["clip"],
                              spec.get("param", 0.0), spec.get("scale", 1.0), spec.get("state_only", False))
    assert np.array_equal(_bits(h), _bits(rh)), tag
    if rs is not None:
        assert np.array_equal(_bits(s), _bits(rs)), tag
    if spec.get("state_only"):
        assert np.array_equal(_bits(w), _bits(w0)), tag
        return
    fw, bite = R.apply_norm(rw, spec["rows"], spec["mode"], spec["value"])
    rows = spec["rows"] if spec["mode"] else 1
    nrm = np.sqrt((rw.astype(np.float64).reshape(-1, rows) ** 2).sum(axis=0))
    exact = ~bite & (np.abs(nrm / max(spec["value"], 1e-30) - 1) > 1e-5) if spec["mode"] else np.ones(rows, bool)
    wm, fm = w.reshape(-1, rows), fw.reshape(-1, rows)
    assert np.array_equal(_bits(wm[:, exact]), _bits(fm[:, exact])), tag
    np.testing.assert_allclose(w, fw, rtol=2e-6, atol=1e-30, err_msg=tag)
    if spec["mode"]:
        assert bite.any() or spec["value"] >= 1e3, tag


def _make(torch, gen, rows, K, rule, offset=0, zero_rows=()):
    n = rows * K
    buf = [torch.empty(n + offset, device="cuda") for _ in range(4)]
    w, h, g, s = (b[offset:] for b in buf)
    w.copy_(torch.randn(n, device="cuda", generator=gen) * 0.3)
    h.copy_(torch.randn(n, device="cuda", generator=gen) * 0.01)
    g.copy_(torch.randn(n, device="cuda", generator=gen) * 0.05)
    s.copy_(torch.rand(n, device="cuda", generator=gen) * 0.2 + (1.0 if rule == R.RMSPROP else 0.5))
    for r in zero_rows:                          # exact zero gradients: the 0 / 0 of the reference
        g.view(K, rows)[:, r] = 0
    g[: min(n, 7)] = 0
    return w, h, g, (s if rule != R.SGD else None), buf


def test_kernel_matches_the_float32_restatement():
    import torch
    from convnet_b200 import lib
    L = lib.load()
    gen = torch.Generator(device="cuda").manual_seed(7)
    # (rows, K, clip, l2, mode, value, offset): Cout not a multiple of 4, Cout > 4096 (vector tiles), a 1-row bias, K = 1,
    # an unaligned pointer (scalar path), chunks with a tail
    shapes = [(1001, 37, 0.0, 5e-4, R.LIMIT, None, 0), (4100, 9, 0.0, 5e-4, R.LIMIT, None, 0),
              (256, 1, 0.0, 0.0, R.CONSTRAINT, 1.0, 0), (130, 70, 0.02, 0.0, R.CONSTRAINT, 2.0, 0),
              (1, 700, 0.0, 0.0, R.LIMIT, None, 0), (1, 10001, 0.03, 5e-4, R.NONE, 0.0, 0),
              (96, 363, 0.0, 0.0, R.NONE, 0.0, 0), (96, 363, 0.01, 1e-3, R.NONE, 0.0, 1), (64, 33, 0.0, 0.0, R.LIMIT, None, 1)]
    rules = [(R.ADAGRAD, {"param": 1.0, "scale": R.adagrad_scale(3)}), (R.ADAGRAD, {"param": 0.0, "scale": 1.0}),
             (R.ADAGRAD, {"param": 0.5, "scale": R.adagrad_scale(1), "state_only": True}),
             (R.RMSPROP, {"param": 0.9}), (R.RMSPROP, {"param": 0.0}), (R.SGD, {})]
    specs, host, dev, keep = [], [], [], []
    for k, (rows, K, clip, l2, mode, value, off) in enumerate(shapes):
        for rule, extra in rules:
            w, h, g, s, buf = _make(torch, gen, rows, K, rule, off, zero_rows=(3,) if rows > 3 else ())
            spec = dict(lr=0.01 if rule == R.SGD else 0.002, mom=0.7, l2=l2, clip=clip, rows=rows, mode=mode,
                        value=value or 0.0, rule=rule, **extra)
            if value is None:                    # a limit that bites on about half of the rows
                rw, _, _ = R.opt_update(w.cpu().numpy(), h.cpu().numpy(), None if s is None else s.cpu().numpy(),
                                        g.cpu().numpy(), rule, spec["lr"], spec["mom"], l2, clip, extra.get("param", 0.0),
                                        extra.get("scale", 1.0))
                nrm = np.sqrt((rw.astype(np.float64).reshape(-1, rows) ** 2).sum(axis=0))
                spec["value"] = float(np.median(nrm)) * (0.5 if rows == 1 else 1.0001)
            specs.append(spec)
            host.append(tuple(None if t is None else t.cpu().numpy() for t in (w, h, g, s)))
            dev.append((w, h, g, s))
            keep.append(buf)
    sgd_copy = [(w.clone(), h.clone(), g.clone()) for (w, h, g, s), sp in zip(dev, specs) if sp["rule"] == R.SGD]
    arr = (CnbOptTensorEx * len(specs))(*[_ex(sp, *d) for sp, d in zip(specs, dev)])
    before = L.convnet_b200_launch_count()
    L.cnb_opt_update_multi(arr, len(specs))
    launches = L.convnet_b200_launch_count() - before
    sgd_specs = [sp for sp in specs if sp["rule"] == R.SGD]
    plain = (CnbOptTensor * len(sgd_specs))(*[_ex(sp, w, h, g, None).t for sp, (w, h, g) in zip(sgd_specs, sgd_copy)])
    L.cnb_sgd_update_multi(plain, len(sgd_specs))
    torch.cuda.synchronize()
    assert launches == 2 * ((len(specs) + 47) // 48)     # update + rescale per 48 tensors, every rule in the same launches
    for k, (sp, hs, d) in enumerate(zip(specs, host, dev)):
        tag = "tensor %d rows %d mode %d rule %d %s" % (k, sp["rows"], sp["mode"], sp["rule"], sp.get("param"))
        _check(tag, sp, hs, (d[0], d[1], d[3]))
    for (w, h, g, s), (wc, hc, _) in zip([d for d, sp in zip(dev, specs) if sp["rule"] == R.SGD], sgd_copy):
        assert torch.equal(w, wc) and torch.equal(h, hc)     # the SGD rule: cnb_sgd_update_multi's bits


def test_state_after_one_update_equals_the_reference():
    import torch
    from convnet_b200 import lib
    L = lib.load()
    z = np.load(os.path.join(ROOT, "tests", "golden", "ref_opt.npz"))
    names = sorted(k[:-4] for k in z.files if k.endswith("_out"))
    specs, dev = [], []
    for name in names:
        s0, g0, p = z[name + "_s"], z[name + "_g"], float(z[name + "_param"])
        n = s0.size
        w, h = torch.zeros(n, device="cuda"), torch.zeros(n, device="cuda")
        g, s = torch.from_numpy(g0).cuda(), torch.from_numpy(s0).cuda()
        rule = R.ADAGRAD if name.startswith("adagrad") else R.RMSPROP
        specs.append(dict(lr=0.0, mom=0.0, l2=0.0, clip=0.0, rows=1, mode=R.NONE, value=0.0, rule=rule, param=p))
        dev.append((w, h, g, s))
    arr = (CnbOptTensorEx * len(specs))(*[_ex(sp, *d) for sp, d in zip(specs, dev)])
    L.cnb_opt_update_multi(arr, len(specs))
    torch.cuda.synchronize()
    for name, (w, h, g, s) in zip(names, dev):
        assert np.array_equal(_bits(s.cpu().numpy()), _bits(z[name + "_out"])), name
        zero = g == 0                                        # 0 / 0 gives a zero step, not NaN
        assert (h[zero] == 0).all() and (w[zero] == 0).all(), name


@pytest.mark.parametrize("rule", [R.ADAGRAD, R.RMSPROP])
def test_update_refreshes_the_staged_bf16_weights(rule):
    import torch
    from convnet_b200 import conv_gemm as cg
    from convnet_b200 import lib
    from convnet_b200.abi import GetConvDesc
    from convnet_b200.matrix import CUDAMatrix
    L = lib.load()
    lib.set_precision("bf16")
    try:
        N, W, Cin, Cout = 128, 8, 64, 64
        d = GetConvDesc(Cin, Cout, 3, 3, 1, 1, 1, 1)
        x = CUDAMatrix(N, W * W * Cin, (N, W, W, Cin)); x.storage.normal_()
        w = CUDAMatrix(Cout, 9 * Cin, (Cout, 3, 3, Cin)); w.storage.normal_().mul_(0.05)
        h, g = torch.zeros_like(w.storage), torch.randn_like(w.storage)
        s = torch.ones_like(w.storage)
        L.convnet_b200_bf16_stage(w.ptr, w.storage.numel())
        t = CnbOptTensor(w.ptr, h.data_ptr(), g.data_ptr(), w.storage.numel(), 0.01, 0.9, 0.0, 0.0, Cout, R.CONSTRAINT, 1.0)
        ex = CnbOptTensorEx(t, rule, 0, s.data_ptr(), 1.0 if rule == R.ADAGRAD else 0.9, 1.0)
        L.cnb_opt_update_multi(ct.byref(ex), 1)
        assert L.convnet_b200_bf16_is_staged(w.ptr, w.storage.numel()) == 1
        z1 = CUDAMatrix(N, W * W * Cout, (N, W, W, Cout)); cg.convUp(x, w, z1, d)
        L.convnet_b200_bf16_invalidate(w.ptr)
        z2 = CUDAMatrix(N, W * W * Cout, (N, W, W, Cout)); cg.convUp(x, w, z2, d)
        assert torch.equal(z1.storage, z2.storage)
        assert not torch.equal(s, torch.ones_like(s))
    finally:
        L.convnet_b200_bf16_invalidate(None)
        lib.set_precision("fp32")


def _net(model, seed=5, batch=16):
    import torch
    from convnet_b200.net import Net
    n = Net(model, batch, seed=seed)
    g = torch.Generator(device="cuda").manual_seed(9)
    n.input_tensor().copy_(torch.randn(n.input_floats, device="cuda", generator=g))
    n.labels_tensor().copy_(torch.randint(0, n.num_classes, (batch,), device="cuda", generator=g, dtype=torch.int32))
    return n


ADA = {"optimizer_type": "ADAGRAD_SGD", "adagrad_delta": 0.5, "epsilon": 0.02, "epsilon_decay": "INVERSE_T",
       "epsilon_decay_timescale": 2, "initial_momentum": 0.3, "final_momentum": 0.9, "momentum_transition_timescale": 3,
       "start_optimization_after": 2, "l2_decay": 0.001}
RMS = {"optimizer_type": "RMSPROP_SGD", "rms_prop_factor": 0.9, "epsilon": 0.001, "epsilon_decay": "EXPONENTIAL",
       "epsilon_decay_timescale": 4, "initial_momentum": 0.5, "final_momentum": 0.9, "momentum_transition_timescale": 2,
       "gradient_clip": 0.05, "start_optimization_after": 1}
SGD = {"epsilon": 0.01, "final_momentum": 0.9}
# model -> {edge: (weights, bias)}, the output channels of each weighted edge
PLANS = {"tiny": ({0: (ADA, RMS), 3: (RMS, SGD), 4: (SGD, ADA), 6: (ADA, ADA)}, {0: 16, 3: 24, 4: 16, 6: 10}),
         "lenet": ({0: (RMS, ADA), 2: (ADA, SGD), 4: (RMS, RMS)}, {0: 48, 2: 128, 4: 10})}


def _configure(n, plan):
    for e, (w, b) in plan.items():
        n.set_optimizer(e, weights=w, bias=b)


def _replay(model, rounds=4):
    """the net's updates against opt_update on its recorded gradients, bit for bit (no norm rules here)"""
    import torch
    from convnet_b200 import net as N
    plan, couts = PLANS[model]
    n = _net(model)
    assert n.adaptive_state_tensor() is None                   # SGD only so far: no state buffer
    _configure(n, plan)
    edges = n.edges()
    p = n.params_tensor().cpu().numpy()
    hist = np.zeros_like(p)
    state = n.adaptive_state_tensor().cpu().numpy()
    for e, (wc, bc) in plan.items():                         # the starts: adagrad_delta, 1
        off, size = edges[e][2], edges[e][3]
        nw = size - couts[e]
        for lo, hi, c in ((off, off + nw, wc), (off + nw, off + size, bc)):
            start = {"ADAGRAD_SGD": c.get("adagrad_delta", 1.0), "RMSPROP_SGD": 1.0}.get(c.get("optimizer_type"))
            if start is not None:
                assert (state[lo:hi] == np.float32(start)).all()
    try:
        for rnd in range(rounds):
            n.fprop(True); n.bprop(); torch.cuda.synchronize()
            p0, g0 = n.params_tensor().cpu().numpy(), n.grads_tensor().cpu().numpy()
            n.update(); torch.cuda.synchronize()
            p1, s1 = n.params_tensor().cpu().numpy(), n.adaptive_state_tensor().cpu().numpy()
            expect, expect_s = p0.copy(), state.copy()
            for e, (wc, bc) in plan.items():
                off, size = edges[e][2], edges[e][3]
                nw = size - couts[e]
                for lo, hi, c in ((off, off + nw, wc), (off + nw, off + size, bc)):
                    rule = {"ADAGRAD_SGD": R.ADAGRAD, "RMSPROP_SGD": R.RMSPROP}.get(c.get("optimizer_type"), R.SGD)
                    started = rnd >= c.get("start_optimization_after", 0)
                    if not started and rule != R.ADAGRAD:
                        continue
                    eps, mom = N.optimizer_schedule(c, rnd)
                    param = c.get("adagrad_delta", 1.0) if rule == R.ADAGRAD else c.get("rms_prop_factor", 0.0)
                    w, h, s = R.opt_update(p0[lo:hi], hist[lo:hi], state[lo:hi] if rule != R.SGD else None, g0[lo:hi],
                                           rule, eps, mom, c.get("l2_decay", 0.0), c.get("gradient_clip", -1.0), param,
                                           R.adagrad_scale(rnd), state_only=not started)
                    expect[lo:hi], hist[lo:hi] = w, h
                    if s is not None:
                        expect_s[lo:hi] = s
            assert np.array_equal(_bits(p1), _bits(expect)), "%s round %d" % (model, rnd)
            assert np.array_equal(_bits(s1), _bits(expect_s)), "%s round %d state" % (model, rnd)
            state = s1
        return p1
    finally:
        n.close()


@pytest.mark.parametrize("model", ["tiny", "lenet"])
def test_trajectory_matches_the_numpy_replay(model):
    _replay(model)


@pytest.mark.parametrize("model", ["tiny", "lenet"])
def test_eager_and_stand_alone_updates_agree(model):
    import torch
    a, b = _net(model), _net(model)
    try:
        for n in (a, b):
            _configure(n, PLANS[model][0])
        for _ in range(4):
            a.train_step(False)
            b.fprop(True); b.bprop(); b.update()
        torch.cuda.synchronize()
        assert torch.equal(a.params_tensor(), b.params_tensor())
        assert torch.equal(a.adaptive_state_tensor(), b.adaptive_state_tensor())
    finally:
        a.close(); b.close()


def test_switching_rules_restarts_only_that_state():
    import torch
    n = _net("tiny")
    try:
        n.set_optimizer(0, weights=dict(RMS, start_optimization_after=0), bias=ADA)
        n.set_optimizer(6, weights=RMS)
        for _ in range(3):
            n.train_step(False)
        edges = n.edges()
        off3, size3 = edges[3][2], edges[3][3]
        nw3 = size3 - 24
        s_before, p_before = n.adaptive_state_tensor().clone(), n.params_tensor().clone()
        n.set_optimizer(3, weights=RMS)                        # SGD -> RMSProp: the slice starts at 1
        s = n.adaptive_state_tensor()
        assert (s[off3:off3 + nw3] == 1).all()
        mask = torch.ones_like(s, dtype=torch.bool); mask[off3:off3 + nw3] = False
        assert torch.equal(s[mask], s_before[mask]) and torch.equal(n.params_tensor(), p_before)
        n.train_step(False)
        n.set_optimizer(3, weights=dict(ADA, adagrad_delta=0.25))      # RMSProp -> Adagrad: delta
        s_mid = n.adaptive_state_tensor().clone()
        assert (s_mid[off3:off3 + nw3] == 0.25).all()
        n.set_optimizer(3, weights=dict(ADA, adagrad_delta=0.25, epsilon=0.5))   # same rule and delta: the state stays
        assert torch.equal(n.adaptive_state_tensor(), s_mid)
        n.train_step(False)
        assert torch.isfinite(n.params_tensor()).all()
    finally:
        n.close()


def test_bn_rmsprop_trains_gamma_and_beta():
    import torch
    n = _net("tiny+bn+rmsprop", batch=32)
    try:
        layers = n.bn_layers()
        assert layers
        losses = [n.train_step(True) for _ in range(30)]
        assert np.isfinite(losses).all() and losses[-1] < losses[0], losses
        st = n.bn_state(layers[0][0])
        assert not torch.equal(st["gamma"], torch.ones_like(st["gamma"]))
        off, c = layers[0][3], layers[0][2]
        assert not torch.equal(n.adaptive_state_tensor()[off:off + 2 * c], torch.ones(2 * c, device="cuda"))
    finally:
        n.close()


@pytest.mark.parametrize("model", ["tiny+adagrad", "tiny+rmsprop"])
def test_data_parallel_replicas_stay_bit_identical(model):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    env = dict(os.environ, DP_MODEL=model, DP_BATCH="32", MASTER_ADDR="127.0.0.1")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
           "--master-addr", "127.0.0.1", "--master-port", "29523", os.path.join(ROOT, "tests", "dp_worker.py")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, env=env)
    line = [ln for ln in r.stdout.splitlines() if ln.startswith("{")]
    assert r.returncode == 0 and line, (r.returncode, r.stdout[-2000:], r.stderr[-2000:])
    res = json.loads(line[-1])
    assert res["ok"]
    for b in res["results"]:
        assert b["bit_identical_across_ranks"] and b["rel_diff_vs_1rank_global_batch"] < 1e-5


def test_bf16_copies_stay_coherent_under_rmsprop():
    """tests/staging_worker.py "train" under CONVNET_B200_STAGE_VERIFY=1: an update that left the bf16 twin or the prebuilt
    dgrad banks behind the fp32 weights aborts there"""
    env = dict(os.environ, CONVNET_B200_STAGE_VERIFY="1")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "staging_worker.py"), "train", "alexnet+rmsprop",
                        "32", "3"], capture_output=True, text=True, timeout=900, env=env)
    assert r.returncode == 0 and "VERIFY-TRAIN-OK" in r.stdout, (r.returncode, r.stdout[-1500:], r.stderr[-1500:])


def test_alexnet_adaptive_models_keep_a_finite_loss():
    import torch
    from convnet_b200 import lib
    from convnet_b200.net import Net
    lib.set_precision("bf16")
    try:
        for model in ("alexnet+adagrad", "alexnet+rmsprop"):
            n = Net(model, 16, seed=11)
            n.input_tensor().normal_()
            n.labels_tensor().copy_(torch.randint(0, n.num_classes, (16,), device="cuda", dtype=torch.int32))
            losses = [n.train_step(True) for _ in range(5)]
            assert np.isfinite(losses).all(), (model, losses)
            assert torch.isfinite(n.adaptive_state_tensor()).all(), model
            n.close()
    finally:
        lib.set_precision("fp32")
