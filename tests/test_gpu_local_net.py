"""The host's LOCAL edge at net level on the GPU: back-prop of nets with local edges against a float64 PyTorch autograd
mirror (one unfolded GEMM per module) that shares the native parameters, in fp32, tf32 and bf16 at batch 128 (where the
local edges run on the tensor cores); the weight norm rule on a local edge (a row = one output channel across all
modules); and the data-parallel sync of nets with local edges (2+ GPUs).

Parameter layout of a local edge (host/edge.h LocalEdge): [Cout x (K*modules + modules)] column-major — weight (o, k, m)
at o + Cout*(k + K*m), k = tx + kx*(ty + ky*c); then the bias, whose entry j = m + modules*o belongs to output column j."""
import json
import math
import os
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def env():
    import torch
    assert torch.cuda.is_available()
    from convnet_b200 import lib, net
    lib.load(); net.load_host()
    yield torch, lib, net
    lib.set_precision("tf32")


# spec entries: ("conv", cout, k, stride, pad, relu) | ("local", cout, k, stride, pad, relu) | ("maxpool", k, s, p) |
#               ("avgpool", k, s, p) | ("fc", cout, relu, dropprob)
NETS = {
    "lcnet": dict(cin=3, size=96, spec=[("conv", 64, 5, 2, 2, True), ("maxpool", 3, 2, 1), ("conv", 128, 3, 1, 1, True),
                                        ("maxpool", 3, 2, 1), ("local", 128, 3, 1, 1, True), ("local", 128, 3, 1, 0, True),
                                        ("fc", 1024, True, 0.5), ("fc", 1000, False, 0.0)]),
    "localcheck": dict(cin=4, size=8, spec=[("local", 8, 3, 1, 1, False), ("avgpool", 2, 1, 0), ("local", 8, 3, 2, 0, False),
                                            ("fc", 5, False, 0.0)]),
}


def _mirror(torch, n, batch, model):
    """float64 forward + backward of the native net's current parameters after a TRAINING forward (the dropout of a layer
    is taken from the native state); returns (summed loss, {edge: (kind, w, b)})"""
    import torch.nn.functional as Fn
    cfg = NETS[model]
    P = n.params_tensor().double()
    edges = n.edges()
    params = {}
    C, S = cfg["cin"], cfg["size"]
    h = n.input_tensor().double().view(C, S, S, batch).permute(3, 0, 1, 2).contiguous()       # [N, C, H, W]
    for i, e in enumerate(cfg["spec"]):
        off, size = edges[i][2], edges[i][3]
        flat = P[off:off + size]
        if e[0] == "conv":
            _, cout, k, s, p, relu = e
            cin = h.shape[1]
            K = cin * k * k
            w = flat[:cout * K].view(cin, k, k, cout).permute(3, 0, 1, 2).contiguous().requires_grad_(True)
            b = flat[cout * K:cout * K + cout].clone().requires_grad_(True)
            params[i] = ("conv", w, b)
            h = Fn.conv2d(h, w, b, stride=s, padding=p)
            h = torch.relu(h) if relu else h
        elif e[0] == "local":
            _, cout, k, s, p, relu = e
            cin = h.shape[1]
            K = cin * k * k
            my = (h.shape[2] + 2 * p - k) // s + 1
            mx = (h.shape[3] + 2 * p - k) // s + 1
            M = mx * my
            w = flat[:cout * K * M].view(M, K, cout).permute(0, 2, 1).contiguous().requires_grad_(True)   # [M, cout, K]
            b = flat[cout * K * M:cout * K * M + cout * M].view(cout, M).clone().requires_grad_(True)     # [cout, M]
            params[i] = ("local", w, b)
            cols = Fn.unfold(h, (k, k), padding=p, stride=s)                      # [N, K, M], K = c*k*k + ty*k + tx
            h = (torch.einsum("mok,nkm->nom", w, cols) + b).view(batch, cout, my, mx)
            h = torch.relu(h) if relu else h
        elif e[0] == "maxpool":
            h = Fn.max_pool2d(h, e[1], e[2], e[3])
        elif e[0] == "avgpool":
            h = Fn.avg_pool2d(h, e[1], e[2], e[3], count_include_pad=False)
        elif e[0] == "fc":                                     # features flattened as x + W*(y + H*c)
            _, cout, relu, drop = e
            K = h[0].numel()
            w = flat[:cout * K].view(K, cout).clone().requires_grad_(True)
            b = flat[cout * K:cout * K + cout].clone().requires_grad_(True)
            params[i] = ("fc", w, b)
            h = h.reshape(batch, K) @ w + b
            h = torch.relu(h) if relu else h
            if drop:                   # the units the native training step kept: non-zero in its (ReLU'd, dropped) state
                kept = n.layer_state(i + 1).view(cout, batch).t() != 0
                h = h * kept.double() * (1.0 / (1.0 - drop))
    loss = Fn.cross_entropy(h, n.labels_tensor().long(), reduction="sum")
    loss.backward()
    return loss.item(), params


def _native_grads(G, off, kind, w, b):
    """the native gradient of an edge in the mirror's shapes"""
    if kind == "conv":
        cout, cin, k, _ = w.shape
        K = cin * k * k
        return G[off:off + cout * K].view(cin, k, k, cout).permute(3, 0, 1, 2), G[off + cout * K:off + cout * K + cout]
    if kind == "local":
        M, cout, K = w.shape
        gw = G[off:off + cout * K * M].view(M, K, cout).permute(0, 2, 1)
        return gw, G[off + cout * K * M:off + cout * K * M + cout * M].view(cout, M)
    K, cout = w.shape
    return G[off:off + cout * K].view(K, cout), G[off + cout * K:off + cout * K + cout]


@pytest.mark.parametrize("model", sorted(NETS))
def test_local_backprop_matches_float64_autograd(env, model):
    """LocalEdge::ComputeUp (with the fused per-feature bias + ReLU), ComputeDown (ReLU' mask), ComputeOuter
    (scale_gradients / batch, bias sum on the side lane) and every other backward op of the chain, at batch 128, against
    float64 autograd on the same parameters"""
    torch, lib, net = env
    batch = 128
    # fp32 per-entry bar, relative to the mean |gradient|: 1e-3 — fc5:output's entries are sums over 128 images that
    # largely cancel, so fp32 accumulation reaches 2.3e-4 of the mean there (relative L2 1.6e-6); a wrong index or
    # layout gives errors of order 1
    for mode, tol in (("fp32", 1e-3), ("tf32", 5e-2), ("bf16", 1.5e-1)):
        lib.set_precision(mode)
        n = net.Net(model, batch, seed=7)
        g = torch.Generator(device="cuda").manual_seed(11)
        n.input_tensor().normal_(generator=g)
        n.labels_tensor().copy_(torch.randint(0, n.num_classes, (batch,), device="cuda", generator=g, dtype=torch.int32))
        n.fprop(True); n.bprop()                 # training forward: lcnet's fc5 dropout is on (see _mirror)
        torch.cuda.synchronize()
        loss = n.loss()
        ref_loss, params = _mirror(torch, n, batch, model)
        assert abs(loss - ref_loss) / ref_loss < {"fp32": 1e-5, "tf32": 2e-3, "bf16": 1e-2}[mode], (mode, loss, ref_loss)
        G = n.grads_tensor().double()
        edges = n.edges()
        # fp32: every entry of the edges from the last max-pool down to the loss (the local edges among them) matches.  The
        # edges in front of a max-pool are held to relative L2 only: at batch 128 lcnet's pools have 19 M windows, and the
        # few whose fp32 and float64 maxima differ route single gradients elsewhere (lcnet fp32, on an H100: conv1 / conv2
        # worst entry 8e-3 / 2e-3 of the mean, relative L2 3e-4 / 4e-5; local3 .. fc5 worst entry <= 5e-5)
        last_pool = max([j for j, e in enumerate(NETS[model]["spec"]) if e[0] == "maxpool"], default=-1)
        for i, (kind, w, b) in params.items():
            gw, gb = _native_grads(G, edges[i][2], kind, w, b)
            for name, mine, ref in (("w", gw, w.grad / batch), ("b", gb, b.grad / batch)):   # scale_gradients / batch
                bar = tol
                if mode == "fp32" and i >= last_pool:        # exact arithmetic: every entry matches
                    err = ((mine - ref).abs().max() / ref.abs().mean().clamp_min(1e-12)).item()
                else:                   # relative L2 (operand rounding flips a few ReLU / max-pool decisions)
                    err = ((mine - ref).norm() / ref.norm().clamp_min(1e-12)).item()
                    bar = 1e-3 if mode == "fp32" else tol
                assert err < bar, (mode, edges[i][0], name, err)
        n.close()


def test_local_paths_at_batch_128(env):
    """the mirror test above runs the local edges of lcnet on the tensor cores in tf32 / bf16: the untied calls of one
    training step at batch 128 take the tensor-core paths"""
    torch, lib, net = env
    from convnet_b200 import conv_gemm as cg
    from convnet_b200.abi import GetConvDesc
    from convnet_b200.matrix import CUDAMatrix
    for mode in ("tf32", "bf16"):
        lib.set_precision(mode)
        d = GetConvDesc(128, 128, 3, 3, 1, 1, 1, 1)
        x = CUDAMatrix(128, 144 * 128, (128, 12, 12, 128)); x.storage.normal_()
        w = CUDAMatrix(128, 1152 * 144, (128, 3, 3, 128 * 144)); w.storage.normal_()
        y = CUDAMatrix(128, 144 * 128, (128, 12, 12, 128))
        cg.localUp(x, w, y, d)
        assert lib.last_conv_path() == "tc-" + mode


def test_weight_norm_limit_on_a_local_edge_is_per_output_channel(env):
    """weight_norm_limit on a local edge: a row is one output channel o across ALL modules (Cout rows of K*modules
    columns), the bias untouched — numpy restatement; a per-(channel, module) reading gives a different result"""
    torch, lib, net = env
    lib.set_precision("tf32")
    n = net.Net("lcnet", 128, seed=3)
    try:
        edge = "pool2:local3"
        i = [e[0] for e in n.edges()].index(edge)
        _, _, off, size = n.edges()[i]
        Cout, K, M = 128, 1152, 144
        P = n.params_tensor()
        with torch.no_grad():                                     # spread the row norms: row o scaled by (1 + o/32)
            P[off:off + Cout * K * M].view(K * M, Cout).mul_(1 + torch.arange(Cout, device="cuda") / 32.0)
        before = P[off:off + size].double().cpu().numpy()
        W = before[:Cout * K * M].reshape(K * M, Cout).T             # [Cout, K*M]
        norms = np.sqrt((W * W).sum(1))
        limit = float(np.median(norms))
        # epsilon 0, no momentum: the update changes nothing but the norm rule (the gradients are zero anyway)
        n.set_optimizer(edge, weights={"epsilon": 0.0, "final_momentum": 0.0, "weight_norm_limit": limit},
                        bias={"epsilon": 0.0, "final_momentum": 0.0})
        n.update()
        torch.cuda.synchronize()
        after = n.params_tensor()[off:off + size].double().cpu().numpy()
        scale = np.where(norms > np.float32(limit), np.float32(limit) / norms, 1.0)
        expect = (W * scale[:, None]).T.reshape(-1)
        got = after[:Cout * K * M]
        assert 0 < (scale < 1).sum() < Cout
        np.testing.assert_allclose(got, expect, rtol=2e-6, atol=0)
        assert np.array_equal(after[Cout * K * M:], before[Cout * K * M:])       # the bias: one row, no norm rule
        Wm = before[:Cout * K * M].reshape(M, K, Cout)                            # per (o, m) rows: what it must NOT do
        nm = np.sqrt((Wm * Wm).sum(1))
        per_module = (Wm * np.where(nm > limit, limit / nm, 1.0)[:, None, :]).reshape(-1)
        assert not np.allclose(got, per_module, rtol=1e-3)
    finally:
        n.close()


def _dp(model, batch, precision):
    import torch
    ngpu = torch.cuda.device_count()
    if ngpu < 2:
        pytest.skip("needs >= 2 GPUs")
    world = 2 if ngpu < 4 else 4
    env = dict(os.environ, DP_MODEL=model, DP_BATCH=str(batch), DP_PRECISION=precision, MASTER_ADDR="127.0.0.1")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(world),
           "--master-addr", "127.0.0.1", "--master-port", "29519", os.path.join(ROOT, "tests", "dp_worker.py")]
    return subprocess.run(cmd, capture_output=True, text=True, timeout=1200, env=env)


def test_data_parallel_local_net_matches_single_rank():
    """tests/dp_worker.py on a net with local edges and no dropout: bit-identical replicas, equal to the 1-rank run on the
    global batch.  tf32 at 128 images per rank: local2 runs on the tensor cores (local1, Cin 4, on the CUDA cores)"""
    r = _dp("localcheck", 128, "tf32")
    line = [ln for ln in r.stdout.splitlines() if ln.startswith("{")]
    assert r.returncode == 0 and line, (r.returncode, r.stdout[-2000:], r.stderr[-2000:])
    res = json.loads(line[-1])
    assert res["ok"]
    for b in res["results"]:
        assert b["bit_identical_across_ranks"] and b["rel_diff_vs_1rank_global_batch"] < 1e-5 and b["max_param_change"] > 0


def test_data_parallel_lcnet_replicas_identical():
    """lcnet over NCCL at 128 images per rank, bf16: the replicas stay bit-identical (bench.py asserts it and reports it).
    Not compared with a 1-rank run: fc5's dropout is seeded with the rank (as the reference seeds each process with
    seed + rank), so a 2-rank step draws different masks from a 1-rank step on the concatenated batch."""
    import torch
    ngpu = torch.cuda.device_count()
    if ngpu < 2:
        pytest.skip("needs >= 2 GPUs")
    world = 2 if ngpu < 4 else 4
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(world), "--master-addr",
           "127.0.0.1", "--master-port", "29521", os.path.join(ROOT, "bench.py"), "--gpus", str(world), "--model", "lcnet",
           "--steps", "5", "--warmup", "2", "--no-cpu-baseline", "--no-cfg3"]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=1200, cwd=ROOT)
    line = [ln for ln in r.stdout.splitlines() if ln.startswith("{")]
    assert r.returncode == 0 and line, (r.returncode, r.stdout[-2000:], r.stderr[-2000:])
    res = json.loads(line[-1])
    assert res["replicas_identical"] and math.isfinite(res["last_loss"])
