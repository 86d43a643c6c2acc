"""The reference's SGD step on the GPU (cnb_sgd_update_multi, host optimizer schedules): the kernel against a numpy
restatement of SGDOptimizer::Optimize (src/optimizer.cc:174-200) + kNormLimitRowwise (cudamat_kernels.cu:1549-1569),
trajectories of a net under Net.set_optimizer, and the "+ref-optimizer" models end to end."""
import ctypes as ct
import json
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu


class CnbOptTensor(ct.Structure):           # include/convnet_b200_ext.h
    _fields_ = [("w", ct.c_void_p), ("hist", ct.c_void_p), ("grad", ct.c_void_p), ("n", ct.c_longlong),
                ("lr", ct.c_float), ("momentum", ct.c_float), ("l2", ct.c_float), ("clip", ct.c_float),
                ("rows", ct.c_int), ("norm_mode", ct.c_int), ("norm_value", ct.c_float)]


NONE, LIMIT, CONSTRAINT = 0, 1, 2


def ref_update(w, h, g, lr, mom, l2, clip, rows, mode, value):
    """float64 restatement; returns (w, h)"""
    w, h, g = (np.asarray(a, np.float64) for a in (w, h, g))
    g = g + l2 * w
    if clip > 0:
        g = np.clip(g, -clip, clip)
    h = mom * h + lr * g
    w = w - h
    if mode:
        m = w.reshape(-1, rows)                   # [K, rows]: row r = elements r + rows*k
        nrm = np.sqrt((m * m).sum(axis=0))
        scale = np.ones_like(nrm)
        bite = (nrm > 0) & ((nrm > value) if mode == LIMIT else True)
        scale[bite] = value / nrm[bite]
        w = (m * scale).reshape(-1)
    return w, h


def _run(L, specs, tensors):
    arr = (CnbOptTensor * len(specs))()
    for k, (s, (w, h, g)) in enumerate(zip(specs, tensors)):
        arr[k] = CnbOptTensor(w.data_ptr(), h.data_ptr(), g.data_ptr(), w.numel(), s["lr"], s["mom"], s["l2"], s["clip"],
                              s["rows"], s["mode"], s["value"])
    L.cnb_sgd_update_multi(arr, len(specs))


def test_update_kernel_matches_the_reference_step():
    import torch
    from convnet_b200 import lib
    L = lib.load()
    gen = torch.Generator(device="cuda").manual_seed(3)
    # (rows, K, clip, l2, mode, value): Cout not a multiple of 4, Cout > 4096 (vector path), K = 1, a 1-row bias
    shapes = [(1001, 37, 0.0, 5e-4, LIMIT, None), (4100, 9, 0.0, 5e-4, LIMIT, None), (4100, 9, 0.0, 0.0, LIMIT, 1e3),
              (256, 1, 0.0, 0.0, CONSTRAINT, 1.0), (130, 70, 0.02, 0.0, CONSTRAINT, 2.0), (1, 700, 0.0, 0.0, LIMIT, None),
              (1, 10001, 0.03, 5e-4, NONE, 0.0), (96, 363, 0.0, 0.0, NONE, 0.0)]
    specs, host, dev = [], [], []
    for rows, K, clip, l2, mode, value in shapes:
        n = rows * K
        w = torch.randn(n, device="cuda", generator=gen) * 0.3
        h = torch.randn(n, device="cuda", generator=gen) * 0.01
        g = torch.randn(n, device="cuda", generator=gen)
        if mode == CONSTRAINT:                     # a dead unit: norm 0 before and after
            w.view(K, rows)[:, 3] = 0; h.view(K, rows)[:, 3] = 0; g.view(K, rows)[:, 3] = 0
        s = dict(lr=0.01, mom=0.7, l2=l2, clip=clip, rows=rows, mode=mode, value=value or 0.0)
        if value is None:                          # a limit that bites on about half of the rows (on the 1-row bias)
            wn, _ = ref_update(w.cpu().numpy(), h.cpu().numpy(), g.cpu().numpy(), **dict(s, mode=NONE))
            s["value"] = float(np.median(np.sqrt((wn.reshape(-1, rows) ** 2).sum(axis=0)))) * (0.5 if rows == 1 else 1)
        specs.append(s)
        host.append([t.cpu().numpy() for t in (w, h, g)])
        dev.append((w, h, g))
    plain = [(w.clone(), h.clone(), g.clone()) for w, h, g in dev]
    _run(L, specs, dev)
    _run(L, [dict(s, mode=NONE) for s in specs], plain)
    torch.cuda.synchronize()
    for s, (w0, h0, g0), (w, h, _), (wp, _, _) in zip(specs, host, dev, plain):
        rw, rh = ref_update(w0, h0, g0, **s)
        tag = "rows %d mode %d" % (s["rows"], s["mode"])
        w, h, wp = w.cpu().numpy(), h.cpu().numpy(), wp.cpu().numpy()
        np.testing.assert_allclose(h, rh, rtol=1e-6, atol=1e-8, err_msg=tag)
        np.testing.assert_allclose(w, rw, rtol=1e-6, atol=1e-7, err_msg=tag)
        norms = np.sqrt((wp.astype(np.float64).reshape(-1, s["rows"]) ** 2).sum(axis=0))
        got = np.sqrt((w.astype(np.float64).reshape(-1, s["rows"]) ** 2).sum(axis=0))
        if s["mode"] == LIMIT:
            under = norms <= s["value"] * (1 - 1e-6)
            assert (under.any() or s["rows"] == 1) and (s["value"] == 1e3 or (~under).any()), tag
            assert np.array_equal(w.reshape(-1, s["rows"])[:, under], wp.reshape(-1, s["rows"])[:, under]), tag
            assert (got <= s["value"] * (1 + 1e-6)).all(), tag
        elif s["mode"] == CONSTRAINT:
            live = norms > 0
            np.testing.assert_allclose(got[live], s["value"], atol=1e-5, err_msg=tag)
            assert (w.reshape(-1, s["rows"])[:, ~live] == 0).all(), tag
        else:
            assert np.array_equal(w, wp), tag          # no norm rule: the same bits as the plain call


def test_rescale_refreshes_the_staged_bf16_weights():
    """a constrained conv filter bank staged in bf16: after the update + rescale, a conv that reads the refreshed copy
    equals one that converts the final fp32 weights itself"""
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
        L.convnet_b200_bf16_stage(w.ptr, w.storage.numel())
        t = CnbOptTensor(w.ptr, h.data_ptr(), g.data_ptr(), w.storage.numel(), 0.01, 0.9, 0.0, 0.0, Cout, CONSTRAINT, 1.0)
        L.cnb_sgd_update_multi(ct.byref(t), 1)
        assert L.convnet_b200_bf16_is_staged(w.ptr, w.storage.numel()) == 1
        z1 = CUDAMatrix(N, W * W * Cout, (N, W, W, Cout)); cg.convUp(x, w, z1, d)
        L.convnet_b200_bf16_invalidate(w.ptr)
        z2 = CUDAMatrix(N, W * W * Cout, (N, W, W, Cout)); cg.convUp(x, w, z2, d)
        assert torch.equal(z1.storage, z2.storage)
        norms = w.storage.view(-1, Cout).double().pow(2).sum(0).sqrt()
        assert torch.allclose(norms, torch.ones_like(norms), atol=1e-5)
    finally:
        L.convnet_b200_bf16_invalidate(None)
        lib.set_precision("fp32")


# tiny's weighted edges: (edge index, output channels)
TINY = [(0, 16), (3, 24), (4, 16), (6, 10)]
TINY_OPT = {"epsilon": 0.05, "epsilon_decay": "INVERSE_T", "epsilon_decay_timescale": 2, "initial_momentum": 0.3,
            "final_momentum": 0.9, "momentum_transition_timescale": 3, "gradient_clip": 0.02,
            "start_optimization_after": 1, "l2_decay": 0.001}


def _configure_tiny(net, limit):
    for e, _ in TINY:
        w = dict(TINY_OPT)
        if e == 3:
            w["weight_norm_constraint"] = 1.5
        elif e == 6:
            w["weight_norm_limit"] = limit
        net.set_optimizer(e, weights=w, bias=dict(TINY_OPT))


def _tiny_net(seed=5):
    import torch
    from convnet_b200.net import Net
    n = Net("tiny", 16, seed=seed)
    g = torch.Generator(device="cuda").manual_seed(9)
    n.input_tensor().copy_(torch.randn(n.input_floats, device="cuda", generator=g))
    n.labels_tensor().copy_(torch.randint(0, n.num_classes, (16,), device="cuda", generator=g, dtype=torch.int32))
    return n


def test_tiny_trajectory_matches_numpy():
    import torch
    from convnet_b200 import net as N
    n = _tiny_net()
    edges = n.edges()
    p = n.params_tensor().cpu().numpy()
    fc_off, fc_size = edges[6][2], edges[6][3]
    fc_norms = np.sqrt((p[fc_off:fc_off + fc_size - 10].reshape(-1, 10).astype(np.float64) ** 2).sum(axis=0))
    limit = float(np.median(fc_norms))                 # bites on some rows from the first update on
    _configure_tiny(n, limit)
    hist = np.zeros_like(p, dtype=np.float64)
    try:
        for rnd in range(3):
            for e, _ in TINY:
                st = n.optimizer_state(e)
                assert st["weights"]["step"] == rnd and st["bias"]["step"] == rnd
            n.fprop(True); n.bprop(); torch.cuda.synchronize()
            p0, g0 = n.params_tensor().cpu().numpy(), n.grads_tensor().cpu().numpy()
            n.update(); torch.cuda.synchronize()
            p1 = n.params_tensor().cpu().numpy()
            expect = p0.astype(np.float64).copy()
            for e, cout in TINY:
                off, size = edges[e][2], edges[e][3]
                nw = size - cout
                for lo, hi, rows, which in ((off, off + nw, cout, "w"), (off + nw, off + size, 1, "b")):
                    if rnd < TINY_OPT["start_optimization_after"]:
                        continue
                    eps, mom = N.optimizer_schedule(TINY_OPT, rnd)
                    mode, value = NONE, 0.0
                    if which == "w" and e == 3:
                        mode, value = CONSTRAINT, 1.5
                    elif which == "w" and e == 6:
                        mode, value = LIMIT, limit
                    w, h = ref_update(p0[lo:hi], hist[lo:hi], g0[lo:hi], eps, mom, TINY_OPT["l2_decay"],
                                      TINY_OPT["gradient_clip"], rows, mode, value)
                    expect[lo:hi], hist[lo:hi] = w, h
            np.testing.assert_allclose(p1, expect, rtol=1e-5, atol=1e-7, err_msg="round %d" % rnd)
            if rnd == 0:
                assert np.array_equal(p1, p0)              # start_optimization_after = 1: the first update is skipped
        for e, _ in TINY:
            assert n.optimizer_state(e)["weights"]["step"] == 3
        fc = p1[fc_off:fc_off + fc_size - 10].reshape(-1, 10).astype(np.float64)
        assert (np.sqrt((fc ** 2).sum(axis=0)) <= limit * (1 + 1e-6)).all()
        # ReduceLearningRate scales the base epsilon of both optimizers
        before = n.optimizer_state(0)
        n.reduce_learning_rate(0.5)
        after = n.optimizer_state(0)
        for k in ("weights", "bias"):
            assert after[k]["epsilon"] == pytest.approx(0.5 * before[k]["epsilon"], rel=1e-6)
            assert after[k]["momentum"] == before[k]["momentum"]
    finally:
        n.close()


def test_eager_and_stand_alone_updates_agree():
    import torch
    a, b = _tiny_net(), _tiny_net()
    try:
        for n in (a, b):
            _configure_tiny(n, 0.5)
        for _ in range(3):
            a.train_step(False)
            b.fprop(True); b.bprop(); b.update()
        torch.cuda.synchronize()
        assert torch.equal(a.params_tensor(), b.params_tensor())
        assert a.optimizer_state(6) == b.optimizer_state(6)
    finally:
        a.close(); b.close()


def test_alexnet_ref_optimizer_keeps_the_norm_rules():
    import torch
    from convnet_b200 import lib
    from convnet_b200.net import Net
    lib.set_precision("bf16")
    try:
        n = Net("alexnet+ref-optimizer", 8, seed=11)
        n.input_tensor().normal_()
        n.labels_tensor().copy_(torch.randint(0, n.num_classes, (8,), device="cuda", dtype=torch.int32))
        losses = [n.train_step(True) for _ in range(3)]
        assert np.isfinite(losses).all(), losses
        p, edges = n.params_tensor(), n.edges()
        outs = {4: 256, 8: 768, 10: 768, 11: 384, 13: 1024, 14: 512, 16: 4096, 17: 4096, 18: 1000}
        for e, cout in outs.items():
            off, size = edges[e][2], edges[e][3]
            w = p[off:off + size - cout].view(-1, cout).double()
            norms = w.pow(2).sum(0).sqrt()
            if e < 16:
                assert torch.allclose(norms, torch.ones_like(norms), atol=1e-5), (e, norms.min().item(), norms.max().item())
            else:
                assert (norms <= 4 * (1 + 1e-6)).all(), (e, norms.max().item())
        assert n.optimizer_state(16)["weights"]["step"] == 3
        n.close()
    finally:
        lib.set_precision("fp32")


def test_bf16_copies_stay_coherent_under_the_reference_optimizer():
    """tests/staging_worker.py "train" under CONVNET_B200_STAGE_VERIFY=1 (see test_gpu_staging.py): a rescale that left the
    bf16 twin or the prebuilt dgrad banks behind the fp32 weights aborts there"""
    env = dict(os.environ, CONVNET_B200_STAGE_VERIFY="1")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "staging_worker.py"), "train", "alexnet+ref-optimizer",
                        "32", "3"], capture_output=True, text=True, timeout=900, env=env)
    assert r.returncode == 0 and "VERIFY-TRAIN-OK" in r.stdout, (r.returncode, r.stdout[-1500:], r.stderr[-1500:])


def test_data_parallel_replicas_stay_bit_identical_with_norm_rules():
    """tests/dp_worker.py on lenet+ref-optimizer (FC weight_norm_limit 4, l2 on every weight): bit-identical replicas"""
    import torch
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    env = dict(os.environ, DP_MODEL="lenet+ref-optimizer", DP_BATCH="32", MASTER_ADDR="127.0.0.1")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
           "--master-addr", "127.0.0.1", "--master-port", "29519", os.path.join(ROOT, "tests", "dp_worker.py")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, env=env)
    line = [ln for ln in r.stdout.splitlines() if ln.startswith("{")]
    assert r.returncode == 0 and line, (r.returncode, r.stdout[-2000:], r.stderr[-2000:])
    res = json.loads(line[-1])
    assert res["ok"]
    for b in res["results"]:
        assert b["bit_identical_across_ranks"] and b["rel_diff_vs_1rank_global_batch"] < 1e-5
