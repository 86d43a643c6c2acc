"""Fine-tuning on a frozen trunk on the device (block_backprop, subnets, "+finetune").

1. Frozen stays frozen: several training steps leave the frozen prefix of the parameters, the momentum history and the
   adaptive state bit for bit as they were, never write the frozen prefix of the gradient buffer (filled with NaN), give
   no derivative to the frozen layers, and in bf16 build no dgrad filter bank after the first step.
2. The head learns what it would anyway: after one step from the same seed, the gradients and parameters of the trained
   edges of X+finetune are bit-identical to those of X.
3. A subnet PRETRAINED from a checkpoint: its trunk computes the saved lenet's test-mode features bit for bit, and its
   new head trains bit-identically to a head-only net that reads those features as its input layer.
4. Checkpoints: 2 steps, save, load, 2 steps equals 4 steps, bit for bit (tiny+bn+finetune).
5. Polyak: load_polyak_weights leaves the frozen range bit for bit.
6. Buckets: the gradient buckets cover the trained range only; with 2+ GPUs, replicas of tiny+finetune stay
   bit-identical and match one rank on the global batch (tests/dp_worker.py).
"""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import checkpoint_format as ckpt

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def env():
    import torch
    from convnet_b200 import lib
    from convnet_b200 import net as N
    lib.load()
    yield torch, lib, N
    lib.set_precision("tf32")


def feed(torch, net, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    net.input_tensor().copy_(torch.randn(net.input_floats, device="cuda", generator=g))
    net.labels_tensor().copy_(torch.randint(0, net.num_classes, (net.batch_size,), device="cuda", generator=g,
                                            dtype=torch.int32))


def frozen_layers(N, net):
    names = N.model_frozen(net.model)["layers"]
    return [i for i in range(net.H.cnb_net_num_layers(net.h)) if net.H.cnb_net_layer_name(net.h, i).decode() in names]


@pytest.mark.parametrize("model,batch,prec", [("lenet+finetune", 32, "fp32"), ("lenet+finetune", 32, "tf32"),
                                              ("lenet+finetune", 32, "bf16"), ("lenet+rmsprop+finetune", 32, "tf32"),
                                              ("alexnet+finetune", 128, "bf16")])
def test_frozen_stays_frozen(env, model, batch, prec):
    torch, lib, N = env
    lib.set_precision(prec)
    net = N.Net(model, batch, seed=3)
    off = net.trained_offset
    assert 0 < off < net.num_params
    net.grads_tensor()[:off].fill_(float("nan"))
    state = net.adaptive_state_tensor()
    start = [t[:off].clone() for t in (net.params_tensor(), net.history_tensor()) + ((state,) if state is not None else ())]
    L = lib.load()
    feed(torch, net, 1)
    net.train_step()
    torch.cuda.synchronize()
    builds = L.convnet_b200_dgrad_bank_builds(0) + L.convnet_b200_dgrad_bank_builds(1)
    head = net.params_tensor()[off:].clone()
    losses = []
    for s in range(3):
        feed(torch, net, 2 + s)
        losses.append(net.train_step())
    torch.cuda.synchronize()
    now = [net.params_tensor()[:off], net.history_tensor()[:off]] + ([state[:off]] if state is not None else [])
    for a, b in zip(start, now):
        assert torch.equal(a, b)
    assert torch.isnan(net.grads_tensor()[:off]).all()
    assert np.isfinite(losses).all() and not torch.equal(head, net.params_tensor()[off:])
    layers = frozen_layers(N, net)
    assert layers and all(net.layer_deriv(i) is None for i in layers)
    assert net.layer_deriv(layers[-1] + 1) is not None
    assert L.convnet_b200_dgrad_bank_builds(0) + L.convnet_b200_dgrad_bank_builds(1) == builds
    frozen_edge = N.model_frozen(model)["edges"][0]
    with pytest.raises(ValueError, match="block_backprop"):
        net.set_optimizer(frozen_edge, weights={"epsilon": 0.1})
    assert net.optimizer_state(frozen_edge)["weights"]["step"] == 0
    net.close()


@pytest.mark.parametrize("base,batch", [("lenet", 32), ("alexnet", 128)])
@pytest.mark.parametrize("prec", ["fp32", "tf32", "bf16"])
def test_the_head_learns_what_it_would_anyway(env, base, batch, prec):
    torch, lib, N = env
    lib.set_precision(prec)
    full, tuned = N.Net(base, batch, seed=5), N.Net(base + "+finetune", batch, seed=5)
    off = tuned.trained_offset
    assert torch.equal(full.params_tensor(), tuned.params_tensor())
    for net in (full, tuned):
        feed(torch, net, 11)
        net.train_step()
    torch.cuda.synchronize()
    assert torch.equal(full.grads_tensor()[off:], tuned.grads_tensor()[off:])
    assert torch.equal(full.params_tensor()[off:], tuned.params_tensor()[off:])
    assert not torch.equal(full.params_tensor()[:off], tuned.params_tensor()[:off])
    full.close()
    tuned.close()


def write(tmp_path, name, text):
    p = tmp_path / name
    p.write_text(text)
    return str(p)


# the new head on lenet's trunk: 3 x 3 x 128 features -> 64 -> 10
HEAD_LAYERS = ('layer { name: "hidden" num_channels: 64 activation: RECTIFIED_LINEAR }\n'
               'layer { name: "output" num_channels: 10 activation: SOFTMAX }\n'
               'default_weight_optimizer { epsilon: 0.01 final_momentum: 0.9 }\n'
               'default_bias_optimizer { epsilon: 0.01 final_momentum: 0.9 }\n')


@pytest.mark.parametrize("prec", ["fp32", "tf32", "bf16"])
def test_a_subnet_from_a_checkpoint(env, tmp_path, prec):
    torch, lib, N = env
    lib.set_precision(prec)
    B, steps = 32, 3
    lenet = N.Net("lenet", B, seed=9)
    for s in range(3):
        feed(torch, lenet, 20 + s)
        lenet.train_step()
    saved = str(tmp_path / "lenet.ckpt")
    lenet.save(saved)
    trunk_file = write(tmp_path, "lenet.pbtxt", N.model_text("lenet"))
    model = write(tmp_path, "net.pbtxt", 'name: "tuned"\nseed: 1\n'
                  'layer { name: "data" num_channels: 1 image_size_y: 28 image_size_x: 28 }\n' + HEAD_LAYERS +
                  'subnet { name: "lenet" model_file: "%s" parameters_file: "%s" block_backprop: true\n'
                  '  remove_layer: "output" merge_layer { subnet_layer: "input" net_layer: "data" } }\n'
                  'edge { source: "lenet_hidden2_maxpool" dest: "hidden" edge_type: FC }\n'
                  'edge { source: "hidden" dest: "output" edge_type: FC }\n' % (trunk_file, saved))
    tuned = N.Net(model, B, seed=4)
    off, trunk = tuned.trained_offset, 4                   # layer 4: lenet_hidden2_maxpool
    assert torch.equal(tuned.params_tensor()[:off], lenet.params_tensor()[:off])
    # the head-only net: the features are its input layer, its initial weights the tuned net's (PRETRAINED)
    records = {}
    for k, edge in enumerate(("feat:hidden", "hidden:output")):
        w = np.array(N.model_initial_weights(model, 4 + k, seed=4 + 17 * (4 + k)), np.float32)
        rows = 64 if k == 0 else 10
        for kind, v in (("weight", w), ("bias", np.zeros(rows, np.float32))):
            records["%s:%s" % (edge, kind)] = v
            records["%s:%s_gradient_history" % (edge, kind)] = np.zeros(v.size, np.float32)
            records["%s:%s_step" % (edge, kind)] = 0
    init = str(tmp_path / "head.ckpt")
    ckpt.write(init, records)
    head_model = write(tmp_path, "head.pbtxt", 'name: "head"\nseed: 1\n'
                       'layer { name: "feat" num_channels: 128 image_size_y: 3 image_size_x: 3 }\n' + HEAD_LAYERS +
                       ''.join('edge { source: "%s" dest: "%s" edge_type: FC initialization: PRETRAINED '
                               'pretrained_model: "%s" }\n' % (s, d, init) for s, d in (("feat", "hidden"), ("hidden", "output"))))
    head = N.Net(head_model, B, seed=4)
    assert torch.equal(tuned.params_tensor()[off:], head.params_tensor())
    for s in range(steps):
        feed(torch, tuned, 30 + s)
        lenet.input_tensor().copy_(tuned.input_tensor())
        lenet.fprop(train=False)
        tuned.train_step()
        assert torch.equal(tuned.layer_state(trunk), lenet.layer_state(trunk))
        head.input_tensor().copy_(tuned.layer_state(trunk))
        head.labels_tensor().copy_(tuned.labels_tensor())
        head.train_step()
        torch.cuda.synchronize()
        assert torch.equal(tuned.params_tensor()[off:], head.params_tensor()), s
        assert torch.equal(tuned.layer_state(6), head.layer_state(2)), s
    for net in (lenet, tuned, head):
        net.close()


def test_checkpoint_resume_is_bit_exact(env, tmp_path):
    torch, lib, N = env
    lib.set_precision("tf32")
    model, B = "tiny+bn+finetune", 32
    straight = N.Net(model, B, seed=6)
    for s in range(4):
        feed(torch, straight, 40 + s)
        straight.train_step()
    first = N.Net(model, B, seed=6)
    for s in range(2):
        feed(torch, first, 40 + s)
        first.train_step()
    mid = str(tmp_path / "mid.ckpt")
    first.save(mid)
    resumed = N.Net(model, B, seed=99)
    resumed.load(mid)
    for s in range(2, 4):
        feed(torch, resumed, 40 + s)
        resumed.train_step()
    a, b = str(tmp_path / "a.ckpt"), str(tmp_path / "b.ckpt")
    straight.save(a)
    resumed.save(b)
    assert open(a, "rb").read() == open(b, "rb").read()
    for net in (straight, first, resumed):
        net.close()


def test_polyak_leaves_the_frozen_range_alone(env, tmp_path):
    torch, lib, N = env
    lib.set_precision("tf32")
    path = write(tmp_path, "polyak.pbtxt", N.model_text("tiny+finetune").replace(
        "seed: 42\n", "seed: 42\npolyak_after: 1\npolyak_queue_size: 3\n", 1))
    net = N.Net(path, 32, seed=8)
    off = net.trained_offset
    for s in range(3):
        feed(torch, net, 50 + s)
        net.train_step()
        net.polyak_insert()
    before = net.params_tensor().clone()
    net.load_polyak_weights()
    torch.cuda.synchronize()
    after = net.params_tensor()
    assert torch.equal(before[:off], after[:off])
    assert not torch.equal(before[off:], after[off:])
    net.load_current_weights()
    assert torch.equal(before, net.params_tensor())
    net.close()


def test_buckets_cover_the_trained_range_only(env):
    torch, lib, N = env
    lib.set_precision("tf32")
    for model in ("alexnet+finetune", "tiny+finetune"):
        net = N.Net(model, 32, seed=2)
        feed(torch, net, 60)
        trace = net.trace_step()
        mb = sum(b["MB"] for b in trace["buckets"])          # (each rounded to 3 decimals)
        assert abs(mb - (net.num_params - net.trained_offset) * 4e-6) <= 5e-4 * len(trace["buckets"]), (model, trace)
        net.close()


def test_data_parallel_replicas(env):
    torch, lib, N = env
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    world = 2 if n < 4 else 4
    env_vars = dict(os.environ, DP_MODEL="tiny+finetune", DP_BATCH="32", MASTER_ADDR="127.0.0.1")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(world),
           "--master-addr", "127.0.0.1", "--master-port", "29531", os.path.join(ROOT, "tests", "dp_worker.py")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, env=env_vars)
    line = [ln for ln in r.stdout.splitlines() if ln.startswith("{")]
    assert r.returncode == 0 and line, (r.returncode, r.stdout[-2000:], r.stderr[-2000:])
    res = json.loads(line[-1])
    assert res["ok"]
    for b in res["results"]:
        assert b["bit_identical_across_ranks"] and b["rel_diff_vs_1rank_global_batch"] < 1e-5 and b["max_param_change"] > 0
