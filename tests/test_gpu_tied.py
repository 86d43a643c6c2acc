"""Tied edges on the GPU (EdgeConfig::tied_to): tiednet against its untied twin — the same model written without tied_to,
each tied edge given a copy of its owner's weights and bias.

1. Forward: the two nets compute bit-identical outputs (fp32, tf32, bf16).
2. Gradients: the shared gradient is the twin's per-edge gradients summed in back-propagation order (highest edge
   first).  The first contribution of a step overwrites the gradient and the later ones accumulate.  Both accumulating
   epilogues compute fl(fl(so*acc) + old) — the wgrad kernels' scaleTargets = 1 store and the side lane's bias column
   sum (SumRows) — so the sum is bit-identical.  The one exception is the twin's own bias summation: where the twin
   hands a member's bias gradient to the pool-undo above it (which a tie group does not), the twin sums it in another
   order, and that bias is held to 1e-5 of its largest element.
3. Update: one train_step under SGD with momentum and under RMSProp is the rule (tests/opt_rules.py) applied once to the
   summed gradient, with the owner's optimizer.
4. Grad check: every owner of tiedcheck passes the reference's < 0.01 bar.
5. Checkpoints: 2 steps, save, load into a fresh net, 2 steps equals 4 steps, bit for bit (bf16, fp32).
6. Dgrad banks (bf16): after warm-up, a training step builds the three geometries' banks of the shared conv filters in
   the prestage behind the update only, never inside a dgrad call; every layer derivative equals the twin's bit for bit.
7. Data parallel (2+ GPUs): replicas of tiednet hold bit-identical parameters after several steps.
"""
import json
import os
import re
import subprocess
import sys

import numpy as np
import pytest

from opt_rules import RMSPROP, SGD, opt_update

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BATCH = 128                                      # the conv edges run on the tensor cores from here


@pytest.fixture(scope="module")
def env():
    import torch
    assert torch.cuda.is_available()
    from convnet_b200 import lib, net
    lib.load(); net.load_host()
    yield torch, lib, net
    lib.set_precision("tf32")


def twin_file(N, tmp_path, model):
    p = tmp_path / "twin.pbtxt"
    p.write_text(re.sub(r'\n *tied_to: "[^"]*"', "", N.model_text(model)))
    return str(p)


def fill_inputs(torch, n, seed=3):
    g = torch.Generator(device="cuda").manual_seed(seed)
    n.input_tensor().normal_(generator=g)
    n.labels_tensor().copy_(torch.randint(0, n.num_classes, (n.batch_size,), device="cuda", generator=g, dtype=torch.int32))


def copy_into_twin(torch, tied, twin):
    """the twin's parameters: every edge's slice from the tied net's slice for that edge (its owner's for a tied edge)"""
    tp, wp = tied.params_tensor(), twin.params_tensor()
    for (name, _, off, size), (name2, _, off2, size2) in zip(tied.edges(), twin.edges()):
        assert name == name2
        if size2:
            wp[off2:off2 + size2].copy_(tp[off:off + size2])
    twin.input_tensor().copy_(tied.input_tensor())
    twin.labels_tensor().copy_(tied.labels_tensor())
    torch.cuda.synchronize()


def pair(env, tmp_path, model="tiednet", precision="fp32", batch=BATCH):
    torch, lib, N = env
    lib.set_precision(precision)
    tied = N.Net(model, batch, seed=11)
    twin = N.Net(twin_file(N, tmp_path, model), batch, seed=11)
    fill_inputs(torch, tied)
    copy_into_twin(torch, tied, twin)
    return tied, twin


def groups(N, net):
    """{owner index: [edge indices of the group, in chain order]}"""
    names = [e[0] for e in net.edges()]
    out = {}
    for tied, owner in N.model_ties(net.model).items():
        o = names.index(owner)
        out.setdefault(o, [o]).append(names.index(tied))
    return {o: sorted(m) for o, m in out.items()}


@pytest.mark.parametrize("precision", ["fp32", "tf32", "bf16"])
def test_forward_matches_the_twin_bit_for_bit(env, tmp_path, precision):
    torch, lib, N = env
    tied, twin = pair(env, tmp_path, precision=precision)
    for n in (tied, twin):
        n.fprop(train=False)
    torch.cuda.synchronize()
    assert torch.equal(tied.output_tensor(), twin.output_tensor())
    # a tied edge owns no parameters; it reports its owner's slice
    e = tied.edges()
    assert [x[3] for x in e][3:5] == [0, 0] and e[3][2] == e[4][2] == e[1][2] and e[6][3] == 0 and e[6][2] == e[7][2]
    tied.close(); twin.close()


@pytest.mark.parametrize("precision", ["fp32", "tf32", "bf16"])
def test_shared_gradient_is_the_sum_in_backprop_order(env, tmp_path, precision):
    torch, lib, N = env
    tied, twin = pair(env, tmp_path, precision=precision)
    for n in (tied, twin):
        n.fprop(train=True)                      # the dropout masks hang on the layer names: the same in both nets
        n.bprop()
    torch.cuda.synchronize()
    assert torch.equal(tied.output_tensor(), twin.output_tensor())
    g, tg = tied.grads_tensor().cpu().numpy(), twin.grads_tensor().cpu().numpy()
    te, handoff = twin.edges(), N.model_fusion(twin.model)["edges"]
    for owner, members in groups(N, tied).items():
        name, _, off, size = tied.edges()[owner]
        nw = len(N.model_initial_weights(tied.model, owner))                    # weights first, then the bias
        got = g[off:off + size]
        parts = [tg[te[m][2]:te[m][2] + size] for m in reversed(members)]       # back-propagation order
        want = parts[0].copy()
        for p in parts[1:]:
            want = (want + p).astype(np.float32)
        tol = np.zeros(size)                                                    # fl(fl(so*acc) + old): bit for bit
        if any(handoff[m]["offers_bias_grad"] for m in members):
            tol[nw:] = 1e-5 * np.abs(want[nw:]).max()
        diff = np.abs(got.astype(np.float64) - want)
        for part, sl in (("weight", slice(0, nw)), ("bias", slice(nw, size))):
            bad = diff[sl] > tol[sl]
            assert not bad.any(), (precision, name, part, int(bad.sum()), float(diff[sl].max()))
    tied.close(); twin.close()


@pytest.mark.parametrize("rule", ["sgd", "rmsprop"])
def test_one_update_of_the_shared_tensors(env, tmp_path, rule):
    torch, lib, N = env
    lib.set_precision("fp32")
    model = "tiednet" if rule == "sgd" else "tiednet+rmsprop"
    net = N.Net(model, 32, seed=5)
    fill_inputs(torch, net)
    p0 = net.params_tensor().cpu().numpy().copy()
    net.train_step()
    torch.cuda.synchronize()
    p1, h1, g = (t.cpu().numpy() for t in (net.params_tensor(), net.history_tensor(), net.grads_tensor()))
    for owner, members in groups(N, net).items():
        name, _, off, size = net.edges()[owner]
        o = N.model_edge_optimizer(model, owner, "weights")
        assert net.optimizer_state(owner)["weights"]["step"] == 1
        for m in members:
            if m != owner:
                with pytest.raises(ValueError, match=re.escape(name)):
                    net.optimizer_state(m)
                with pytest.raises(ValueError, match=re.escape(name)):
                    net.set_optimizer(m, weights={"epsilon": 0.1})
        sl = slice(off, off + size)
        s0 = np.ones(size, np.float32) if rule == "rmsprop" else None
        w, h, _ = opt_update(p0[sl], np.zeros(size, np.float32), s0, g[sl], rule=RMSPROP if rule == "rmsprop" else SGD,
                             lr=o["epsilon"], mom=o["final_momentum"], l2=o["l2_decay"], param=o["rms_prop_factor"])
        np.testing.assert_allclose(h1[sl], h, rtol=1e-6, atol=1e-8, err_msg=name)
        np.testing.assert_allclose(p1[sl], w, rtol=1e-6, atol=1e-7, err_msg=name)
        assert np.abs(p1[sl] - p0[sl]).max() > 0
    net.close()


def test_grad_check_of_every_tie_group(env):
    torch, lib, N = env
    lib.set_precision("fp32")
    net = N.Net("tiedcheck", 16, seed=2, grad_checker=True)
    res = {name: (dw, db) for name, eps, dw, db in net.grad_check(seed=1)}
    owners = set(N.model_ties("tiedcheck").values())
    assert owners <= set(res), res
    for name, (dw, db) in res.items():
        assert dw < 0.01 and db < 0.01, (name, dw, db)
    net.close()


@pytest.mark.parametrize("precision", ["bf16", "fp32"])
def test_checkpoint_resumes_bit_for_bit(env, tmp_path, precision):
    torch, lib, N = env
    lib.set_precision(precision)

    def fresh():
        n = N.Net("tiednet", 64, seed=7)
        fill_inputs(torch, n, seed=9)
        return n

    a = fresh()
    for _ in range(4):
        a.train_step()
    b = fresh()
    for _ in range(2):
        b.train_step()
    path = str(tmp_path / "tied.ckpt")
    b.save(path)
    b.close()
    c = fresh()
    c.load(path)
    for _ in range(2):
        c.train_step()
    torch.cuda.synchronize()
    assert torch.equal(a.params_tensor(), c.params_tensor())
    assert torch.equal(a.history_tensor(), c.history_tensor())
    # the records: owners only
    from checkpoint_format import read
    names = list(read(path))
    assert "conv1:conv2:weight" in names and "fc6:fc7:weight" in names
    assert not any(n.startswith(("pool2:conv3:", "conv3:conv4:", "fc5:fc6:")) for n in names)
    a.close(); c.close()


def test_checkpoint_of_a_differently_tied_model_is_refused(env, tmp_path):
    torch, lib, N = env
    lib.set_precision("fp32")
    tied = N.Net("tiednet", 32, seed=1)
    path = str(tmp_path / "tied.ckpt")
    tied.save(path)
    twin = N.Net(twin_file(N, tmp_path, "tiednet"), 32, seed=1)
    before = twin.params_tensor().clone()
    with pytest.raises(ValueError, match="record 'pool2:conv3:weight'"):
        twin.load(path)
    assert torch.equal(before, twin.params_tensor())
    twin.save(str(tmp_path / "twin.ckpt"))
    with pytest.raises(ValueError, match="record"):
        tied.load(str(tmp_path / "twin.ckpt"))
    tied.close(); twin.close()


def test_dgrad_banks_are_built_behind_the_update_only(env, tmp_path):
    torch, lib, N = env
    tied, twin = pair(env, tmp_path, precision="bf16")
    L = lib.load()
    for _ in range(3):                           # warm-up: paths learnt, banks prestaged
        tied.train_step()
    torch.cuda.synchronize()
    inside, behind = L.convnet_b200_dgrad_bank_builds(0), L.convnet_b200_dgrad_bank_builds(1)
    tied.train_step()
    torch.cuda.synchronize()
    # conv1:conv2 at 32 x 32, pool2:conv3 at 16 x 16, conv3:conv4 with stride 2: three sets of banks of one filter tensor
    assert L.convnet_b200_dgrad_bank_builds(0) == inside
    assert L.convnet_b200_dgrad_bank_builds(1) - behind == 3
    # a backward pass on the same weights: every layer derivative equals the twin's, whose edges each have their own
    # filters (the copy goes through params_tensor(), which drops every staged copy, so both nets rebuild their banks).
    # The twin first takes as many steps as the tied net: the dropout masks follow the step count
    for _ in range(4):
        twin.train_step()
    copy_into_twin(torch, tied, twin)
    for n in (tied, twin):
        n.fprop(train=True)
        n.bprop()
    torch.cuda.synchronize()
    assert torch.equal(tied.output_tensor(), twin.output_tensor())
    for i in range(1, len(tied.edges()) + 1):
        assert torch.equal(tied.layer_deriv(i), twin.layer_deriv(i)), i
    tied.close(); twin.close()


def test_data_parallel_replicas_stay_identical():
    import torch
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    world = 2 if n < 4 else 4
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(world),
           "--master-addr", "127.0.0.1", "--master-port", "29531", os.path.join(ROOT, "tests", "tied_dp_worker.py")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, env=dict(os.environ, MASTER_ADDR="127.0.0.1"))
    line = [l for l in r.stdout.splitlines() if l.startswith("{")]
    assert r.returncode == 0 and line, (r.returncode, r.stdout[-2000:], r.stderr[-2000:])
    res = json.loads(line[-1])
    assert res["bit_identical_across_ranks"] and res["max_param_change"] > 0, res
