"""Checkpoints and Polyak averaging on the device (host/checkpoint.cc, cnb_polyak_average).

- Resume bit for bit: train 3 steps, save, train 3 more and save (A); a fresh net built with another seed loads the first
  file, trains the same 3 steps and saves (B).  A and B are the same bytes and the last 3 losses are equal.
- Contents: the records (read by tests/checkpoint_format.py) equal the net's tensors and step counts.
- An edge with has_no_bias: its bias optimizer answers and takes settings but never steps, the file holds no bias
  records, and a resumed net trains on bit for bit.
- Refusals: another model's checkpoint and a truncated file raise ValueError naming a record; the net is unchanged.
- Staging: train steps after load / load_polyak_weights / load_current_weights under CONVNET_B200_STAGE_VERIFY=1.
- Polyak: the average of a wrapped ring equals a float32 restatement of the reference's loop in slot order, fprop follows
  it, the restore is exact and training afterwards equals a run that never inserted.
- PRETRAINED: an FC edge takes weights, bias, history and steps from another net's checkpoint.
- Data parallel (2 ranks): rank 0 saves, every rank loads and resumes as an uninterrupted run would.
"""
import json
import os
import struct
import subprocess
import sys

import numpy as np
import pytest
import torch

import checkpoint_format as CF
from convnet_b200 import lib
from convnet_b200.net import Net, model_text

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu


def batches(net, steps, seed=99):
    g = torch.Generator(device="cuda").manual_seed(seed)
    B = net.batch_size
    return [(torch.randn(net.input_floats, device="cuda", generator=g),
             torch.randint(0, net.num_classes, (B,), device="cuda", generator=g, dtype=torch.int32)) for _ in range(steps)]


@pytest.fixture(autouse=True)
def hygiene():
    L = lib.load()
    prec = L.convnet_b200_get_conv_precision()
    try:
        yield
    finally:
        L.convnet_b200_set_conv_precision(prec)
        L.convnet_b200_bf16_invalidate(None)


def feed(net, x):
    """a write the library cannot see: the input's staged bf16 copy is dropped"""
    net.input_tensor().copy_(x)
    lib.load().convnet_b200_bf16_invalidate(net.input_tensor().data_ptr())


def train(net, data):
    out = []
    for x, y in data:
        feed(net, x)
        net.labels_tensor().copy_(y)
        out.append(net.train_step(True))
    torch.cuda.synchronize()
    return [struct.pack("<f", v) for v in out]


def same_files(a, b):
    with open(a, "rb") as fa, open(b, "rb") as fb:
        while True:
            x, y = fa.read(1 << 24), fb.read(1 << 24)
            if x != y:
                return False
            if not x:
                return True


def bits(t):
    return t.detach().view(torch.int32).clone()


RESUME = [("lenet+ref-optimizer", "bf16", 32), ("lenet+ref-optimizer", "fp32", 32), ("tiny+bn+rmsprop", "bf16", 32),
          ("tiny+bn+rmsprop", "fp32", 32), ("tiny+adagrad", "bf16", 32), ("tiny+adagrad", "fp32", 32),
          ("lcnet", "bf16", 32), ("lcnet", "fp32", 32), ("alexnet", "bf16", 16)]


@pytest.mark.parametrize("model,prec,batch", RESUME)
def test_resume_bit_for_bit(tmp_path, model, prec, batch):
    lib.set_precision(prec)
    a = Net(model, batch, seed=5)
    data = batches(a, 6)
    tune = model.startswith("lenet")
    if tune:                                          # the settings in force are saved, not the ones the net was built with
        a.reduce_learning_rate(0.5)
        a.set_optimizer(0, weights={"epsilon": 0.003, "initial_momentum": 0.5, "final_momentum": 0.95,
                                    "momentum_transition_timescale": 50})
    train(a, data[:3])
    first, pa, pb = str(tmp_path / "first.ckpt"), str(tmp_path / "a.ckpt"), str(tmp_path / "b.ckpt")
    a.save(first)
    la = train(a, data[3:])
    a.save(pa)
    state_a = [a.optimizer_state(e[0]) for e in a.edges() if e[3] > 0] if tune else None
    a.close()
    b = Net(model, batch, seed=1234)
    b.load(first)
    os.remove(first)
    assert b.iteration == 3
    lb = train(b, data[3:])
    b.save(pb)
    if tune:
        assert [b.optimizer_state(e[0]) for e in b.edges() if e[3] > 0] == state_a
    b.close()
    try:
        assert la == lb
        assert same_files(pa, pb)
    finally:
        os.remove(pa)
        os.remove(pb)


def test_contents(tmp_path):
    lib.set_precision("bf16")
    n = Net("tiny+bn+rmsprop", 32, seed=9)
    train(n, batches(n, 2))
    path = str(tmp_path / "c.ckpt")
    n.save(path)
    rec = CF.read(path)
    p, h, s = (t.cpu().numpy() for t in (n.params_tensor(), n.history_tensor(), n.adaptive_state_tensor()))
    assert rec["__current_iter__"][0] == 2 and rec["__seed__"][0] == 9 and rec["__model__"] == model_text("tiny+bn+rmsprop").replace(
        "seed: 42", "seed: 9")
    seen = {"__model__", "__current_iter__", "__seed__"}

    def tensor(prefix, off, n_, step):
        for suffix, buf in (("", p), ("_gradient_history", h), ("_rms_history", s)):
            assert rec[prefix + suffix].view(np.int32).tolist() == buf[off:off + n_].view(np.int32).tolist(), prefix + suffix
            seen.add(prefix + suffix)
        assert rec[prefix + "_step"].tolist() == [step]
        seen.add(prefix + "_step")
    for name, _, off, size in n.edges():
        if size == 0:
            continue
        nw = rec[name + ":weight"].size
        assert nw + rec[name + ":bias"].size == size
        st = n.optimizer_state(name)
        tensor(name + ":weight", off, nw, st["weights"]["step"])
        tensor(name + ":bias", off + nw, size - nw, st["bias"]["step"])
    for i, lname, c, off in n.bn_layers():
        bn, st = n.bn_state(i), n.bn_optimizer_state(i)
        tensor(lname + ":gamma", off, c, st["gamma"]["step"])
        tensor(lname + ":beta", off + c, c, st["beta"]["step"])
        for k in ("running_mean", "running_sigma"):
            assert rec[lname + ":" + k].view(np.int32).tolist() == bn[k].cpu().numpy().view(np.int32).tolist()
            seen.add(lname + ":" + k)
    assert seen == set(rec)
    n.close()


def test_edge_without_bias(tmp_path):
    lib.set_precision("bf16")
    path = str(tmp_path / "nobias.pbtxt")
    text = model_text("tiny")
    assert "has_no_bias: false" in text
    open(path, "w").write(text.replace("has_no_bias: false", "has_no_bias: true", 1))
    a = Net(path, 32, seed=5)
    name = [e[0] for e in a.edges() if e[3] > 0][0]   # the first weighted edge carries the first has_no_bias line
    data = batches(a, 4)
    train(a, data[:2])
    st = a.optimizer_state(name)
    assert st["weights"]["step"] == 2 and st["bias"]["step"] == 0
    a.set_optimizer(name, bias={"epsilon": 0.5})
    assert a.optimizer_state(name)["bias"] == {"step": 0, "epsilon": 0.5, "momentum": 0.0}
    first, pa, pb = str(tmp_path / "first.ckpt"), str(tmp_path / "a.ckpt"), str(tmp_path / "b.ckpt")
    a.save(first)
    rec = CF.read(first)
    assert name + ":weight" in rec and not [r for r in rec if r.startswith(name + ":bias")]
    la = train(a, data[2:])
    a.save(pa)
    a.close()
    b = Net(path, 32, seed=77)
    b.load(first)
    lb = train(b, data[2:])
    b.save(pb)
    b.close()
    assert la == lb
    assert same_files(pa, pb)


def test_refusals_leave_the_net_unchanged(tmp_path, capfd):
    lib.set_precision("bf16")
    other = Net("tiny", 32, seed=2)
    train(other, batches(other, 1))
    foreign = str(tmp_path / "tiny.ckpt")
    other.save(foreign)
    other.close()
    n = Net("lenet", 32, seed=3)
    train(n, batches(n, 2))
    mine = str(tmp_path / "lenet.ckpt")
    n.save(mine)
    before, hist, it = bits(n.params_tensor()), bits(n.history_tensor()), n.iteration
    data = open(mine, "rb").read()
    cut = str(tmp_path / "cut.ckpt")
    open(cut, "wb").write(data[:len(data) - 1000])
    for path in (foreign, cut):
        with pytest.raises(ValueError, match="record"):
            n.load(path)
        assert torch.equal(bits(n.params_tensor()), before) and torch.equal(bits(n.history_tensor()), hist)
        assert n.iteration == it
    n.load(mine)                                      # still loads its own file afterwards
    assert torch.equal(bits(n.params_tensor()), before)
    n.close()


def test_staging_coherent_after_loads(tmp_path):
    env = dict(os.environ, CONVNET_B200_STAGE_VERIFY="1")
    for model in ("lenet", "tiny"):
        r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "checkpoint_worker.py"), "staging", str(tmp_path), model],
                           capture_output=True, text=True, timeout=900, env=env)
        assert r.returncode == 0 and "VERIFY-CHECKPOINT-OK" in r.stdout, (model, r.stdout[-2000:], r.stderr[-2000:])


def polyak_file(tmp_path, base, queue=3):
    path = str(tmp_path / "polyak.pbtxt")
    open(path, "w").write(model_text(base).replace("seed: 42\n", "seed: 42\npolyak_after: 1\npolyak_queue_size: %d\n" % queue, 1))
    return path


@pytest.mark.parametrize("prec", ["bf16", "fp32"])
def test_polyak_average_restore_and_training(tmp_path, prec):
    lib.set_precision(prec)
    path, B = polyak_file(tmp_path, "tiny"), 32
    n = Net(path, B, seed=5)
    data = batches(n, 7)
    with pytest.raises(ValueError):
        n.load_current_weights()
    with pytest.raises(ValueError):
        n.load_polyak_weights()                      # nothing inserted yet
    snaps = []
    for k in range(5):                                # Q = 3: the ring wraps
        train(n, data[k:k + 1])
        snaps.append(n.params_tensor().cpu().numpy().copy())
        n.polyak_insert()
    assert n.polyak_count == 3
    slots = [snaps[3], snaps[4], snaps[2]]            # storage order, not insertion order
    want = np.zeros_like(slots[0])
    for s in slots:
        want = (want + s).astype(np.float32)
    want = (want / np.float32(3)).astype(np.float32)
    current = bits(n.params_tensor())
    n.load_polyak_weights()
    assert n.params_tensor().cpu().numpy().view(np.int32).tolist() == want.view(np.int32).tolist()
    x = data[6][0]
    feed(n, x)
    n.fprop(False)
    out = bits(n.output_tensor())
    avg = str(tmp_path / "avg.ckpt")
    n.save(avg)
    fresh = Net(path, B, seed=77)
    fresh.load(avg)
    feed(fresh, x)
    fresh.fprop(False)
    assert torch.equal(bits(fresh.output_tensor()), out)
    fresh.close()
    n.load_current_weights()
    assert torch.equal(bits(n.params_tensor()), current)
    after = train(n, data[5:7])
    plain = Net(path, B, seed=5)                      # the same run without any insert
    train(plain, data[:5])
    assert train(plain, data[5:7]) == after
    assert torch.equal(bits(plain.params_tensor()), bits(n.params_tensor()))
    plain.close()
    n.close()


def test_polyak_kernel_minus_zero_and_tail():
    L = lib.load()
    k, n = 3, 1001                                    # a tail beyond the float4 groups
    q = torch.randn(k, 1004, device="cuda")
    q[:, 5] = -0.0
    out = torch.empty(n, device="cuda")
    L.cnb_polyak_average(out.data_ptr(), q.data_ptr(), n, 1004, k)
    torch.cuda.synchronize()
    h = q.cpu().numpy()
    want = np.zeros(n, np.float32)
    for s in range(k):
        want = (want + h[s, :n]).astype(np.float32)
    want = (want / np.float32(k)).astype(np.float32)
    assert out.cpu().numpy().view(np.int32).tolist() == want.view(np.int32).tolist()
    assert out[5].item() == 0.0 and not np.signbit(out[5].item())


def test_pretrained_edge_on_the_device(tmp_path):
    lib.set_precision("bf16")
    src = Net("tiny", 32, seed=4)
    train(src, batches(src, 2))
    ckpt = str(tmp_path / "src.ckpt")
    src.save(ckpt)
    src.close()
    rec = CF.read(ckpt)
    text = model_text("tiny")
    head, last = text.rsplit("edge {", 1)
    name = "%s:%s" % tuple(l.split('"')[1] for l in last.splitlines() if l.startswith(("  source:", "  dest:")))
    last = "\n".join(l for l in last.splitlines() if not l.startswith("  initialization:"))
    last = last.replace("  has_no_bias:", '  initialization: PRETRAINED\n  pretrained_model: "%s"\n  has_no_bias:' % ckpt, 1)
    path = str(tmp_path / "pre.pbtxt")
    open(path, "w").write(head + "edge {" + last + "\n")
    n = Net(path, 32, seed=8)
    off, size = [(e[2], e[3]) for e in n.edges() if e[0] == name][0]
    p, h = n.params_tensor().cpu().numpy(), n.history_tensor().cpu().numpy()
    wb = np.concatenate([rec[name + ":weight"], rec[name + ":bias"]])
    hb = np.concatenate([rec[name + ":weight_gradient_history"], rec[name + ":bias_gradient_history"]])
    assert wb.size == size
    assert p[off:off + size].view(np.int32).tolist() == wb.view(np.int32).tolist()
    assert h[off:off + size].view(np.int32).tolist() == hb.view(np.int32).tolist()
    st = n.optimizer_state(name)
    assert st["weights"]["step"] == 2 and st["bias"]["step"] == 2
    loss = struct.unpack("<f", train(n, batches(n, 1))[0])[0]
    assert np.isfinite(loss)
    n.close()


def test_data_parallel_resume(tmp_path):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    env = dict(os.environ, DP_MODEL="lenet", DP_CKPT=str(tmp_path / "dp.ckpt"), MASTER_ADDR="127.0.0.1")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", "29531", os.path.join(ROOT, "tests", "checkpoint_worker.py"), "dp"]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, env=env)
    line = [l for l in r.stdout.splitlines() if l.startswith("{")]
    assert r.returncode == 0 and line, (r.returncode, r.stdout[-2000:], r.stderr[-2000:])
    assert json.loads(line[-1])["ok"]
