"""The training loop on the GPU (Net.train, Net.validate, host/train.cc): the loop against a hand-written Python loop over
get_batch / train_step / metric / validate / reduce_learning_rate / save with the same schedule (parameters, histories,
epsilons, logged values and checkpoints all bit-identical), Polyak validation and twins, resuming from a loop
checkpoint, Validate against the running mean of per-batch metrics, and the command-line app."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import checkpoint_format
from convnet_b200 import net as N
from test_train_loop_cpu import cmod, due, model_file

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
f32 = np.float32
# image side and crop per model: the data set is stored 2 pixels larger than the input layer
SIZES = {"tiny": (8, 12), "lenet": (1, 28), "tiny+bn": (8, 12)}


def dataset(base, n, classes, seed):
    C, G = SIZES[base]
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(n, C, G + 2, G + 2, generator=g).pin_memory(),
            torch.randint(0, classes, (n,), generator=g, dtype=torch.int32))


def feeds(base, batch, classes, seed):
    """(training handler, validation handler): random crops and mirrors in a shuffled order, and centre crops"""
    G = SIZES[base][1]
    ti, tl = dataset(base, 6 * batch, classes, seed)
    vi, vl = dataset(base, 3 * batch + 5, classes, seed + 1)        # the 5 left over are dropped
    train = N.DataHandler(ti, tl, batch_size=batch, chunk_size=4 * batch, gpu_image_size=G, translate=True, flip=True,
                          randomize_gpu=True, seed=seed)
    valid = N.DataHandler(vi, vl, batch_size=batch, gpu_image_size=G, seed=seed)
    return train, valid


def schedule_of(path):
    s = N.model_schedule(path)
    s.update(N.model_polyak(path) or {"polyak_after": 0, "polyak_queue_size": 0})
    return s


def hand_loop(n, path, train, valid, base):
    """src/convnet.cc:921-1006 written out over the public calls: the events Net.train gives, and the files it writes"""
    s, batch = schedule_of(path), n.batch_size
    polyak = s["polyak_after"] > 0 and s["polyak_queue_size"] > 0
    events, slots, hist, dont, counter = [], [], [], 0, n.lr_reduce_counter

    def save():
        n.save(base + ".ckpt")
        if polyak:
            if n.polyak_count:
                n.load_polyak_weights(); n.save(base + ".ckptpolyak"); n.load_current_weights()
            else:
                n.save(base + ".ckptpolyak")

    for i in range(n.iteration, s["max_iter"]):
        it = i + 1
        train.get_batch(n)
        n.train_step(want_loss=False)
        slots.append(f32(n.metric()))
        if cmod(it, s["print_after"]) == 0:
            total = f32(0)
            for v in slots:
                total = f32(total + v)
            events.append({"iteration": it, "kind": "train", "value": float(total / f32(s["print_after"] * batch)),
                           "lr_reduced": False, "polyak": False})
            slots = []
        if N.polyak_due(path, it):
            n.polyak_insert()
        if valid is not None and s["validate_after"] > 0 and cmod(it, s["validate_after"]) == 0:
            average = polyak and n.polyak_count > 0
            if average:
                n.load_polyak_weights()                        # and not restored: training continues from the average
            v = n.validate(valid)
            hist.append(v)
            reduce = False
            if f32(s["reduce_lr_factor"]) < 1.0 and due(hist, s["reduce_lr_num_steps"], s["reduce_lr_threshold"],
                                                        s["smaller_is_better"]) and counter < s["reduce_lr_max"]:
                dont -= 1
                if dont + 1 < 0:
                    dont, counter, reduce = s["reduce_lr_num_steps"], counter + 1, True
                    n.reduce_learning_rate(s["reduce_lr_factor"])
            events.append({"iteration": it, "kind": "valid", "value": v, "lr_reduced": reduce, "polyak": average})
        if cmod(it, s["save_after"]) == 0:
            save()
    if cmod(s["max_iter"], s["save_after"]) != 0:
        save()
    return events, counter


def edge_names(n):
    return [e[0] for e in n.edges() if e[3] > 0]


def assert_same_state(a, b):
    torch.cuda.synchronize()
    for t in ("params_tensor", "history_tensor"):
        assert torch.equal(getattr(a, t)(), getattr(b, t)()), t
    assert a.iteration == b.iteration
    for e in edge_names(a):
        assert a.optimizer_state(e) == b.optimizer_state(e), e


def assert_same_checkpoint(loop_file, hand_file, counter):
    x, y = checkpoint_format.read(loop_file), checkpoint_format.read(hand_file)
    assert x.pop("__lr_reduce_counter__", np.array([0]))[0] == counter
    assert list(x) == list(y)
    for k in x:
        assert (x[k] == y[k]) if isinstance(x[k], str) else np.array_equal(x[k].view(np.uint8), y[k].view(np.uint8)), k


LOOP = dict(max_iter=24, print_after=3, validate_after=4, save_after=10, reduce_lr_factor=0.5, reduce_lr_num_steps=2,
            reduce_lr_max=2, reduce_lr_threshold=1.0)


@pytest.mark.parametrize("base,batch", [("tiny", 16), ("lenet", 32)])
def test_loop_equals_the_hand_written_loop(tmp_path, base, batch):
    path = model_file(tmp_path, base=base, **LOOP)
    runs = {}
    for who in ("loop", "hand"):
        n = N.Net(path, batch, seed=5)
        train, valid = feeds(base, batch, n.num_classes, 11)
        if who == "loop":
            events = n.train(train, valid, checkpoint_dir=str(tmp_path / who), run_name="run")
            counter = n.lr_reduce_counter
        else:
            os.makedirs(tmp_path / who)
            events, counter = hand_loop(n, path, train, valid, str(tmp_path / who / "run"))
        runs[who] = (n, events, counter, train, valid)
    (a, ea, ca, *_), (b, eb, cb, *_) = runs["loop"], runs["hand"]
    assert ea == eb
    assert ca == cb >= 1 and any(e["lr_reduced"] for e in ea)
    assert [e["iteration"] for e in ea if e["kind"] == "train"] == list(range(3, 25, 3))
    assert_same_state(a, b)
    assert a.optimizer_state(edge_names(a)[0])["weights"]["epsilon"] < N.model_edge_optimizer(path, 0)["epsilon"]
    assert_same_checkpoint(tmp_path / "loop" / "run.ckpt", tmp_path / "hand" / "run.ckpt", ca)
    # the run files: the model at the start, one log line per print and per validation
    d = tmp_path / "loop"
    strip = lambda t: [l for l in t.split("\n") if not l.startswith("seed:")]      # the Net's seed, not the file's
    assert strip((d / "run.pbtxt").read_text()) == strip(N.model_text(path))
    train_log = (d / "run_train.log").read_text().split("\n")[:-1]
    assert [int(l.split()[0]) for l in train_log] == [e["iteration"] for e in ea if e["kind"] == "train"]
    assert [f32(l.split()[2]) for l in train_log] == [f32(e["value"]) for e in ea if e["kind"] == "train"]
    valid_log = (d / "run_valid.log").read_text().split("\n")[:-1]
    assert [(int(l.split()[0]), f32(l.split()[1])) for l in valid_log] == \
        [(e["iteration"], f32(e["value"])) for e in ea if e["kind"] == "valid"]
    assert not os.path.exists(d / "run.ckptpolyak")
    for n, _, _, t, v in runs.values():
        t.close(); v.close(); n.close()


def test_polyak_validation_and_twins(tmp_path):
    # inserts after every third step; validations every second step, the first one before any insert
    sched = dict(LOOP, max_iter=13, print_after=4, validate_after=2, save_after=6, polyak_after=3, polyak_queue_size=2)
    path = model_file(tmp_path, **sched)
    runs = {}
    for who in ("loop", "hand"):
        n = N.Net(path, 16, seed=2)
        train, valid = feeds("tiny", 16, n.num_classes, 3)
        if who == "loop":
            events = n.train(train, valid, checkpoint_dir=str(tmp_path / who), run_name="p")
        else:
            os.makedirs(tmp_path / who)
            events, _ = hand_loop(n, path, train, valid, str(tmp_path / who / "p"))
        runs[who] = (n, events, train, valid)
    (a, ea, *_), (b, eb, *_) = runs["loop"], runs["hand"]
    assert ea == eb
    valid_events = [e for e in ea if e["kind"] == "valid"]
    assert [e["polyak"] for e in valid_events] == [False] + [True] * 5       # the queue is empty at iteration 2 only
    assert_same_state(a, b)
    for f in ("p.ckpt", "p.ckptpolyak"):
        assert_same_checkpoint(tmp_path / "loop" / f, tmp_path / "hand" / f, a.lr_reduce_counter)
    twin, ckpt = (checkpoint_format.read(tmp_path / "loop" / f) for f in ("p.ckptpolyak", "p.ckpt"))
    w = [k for k in ckpt if k.endswith(":weight")][0]
    assert not np.array_equal(twin[w], ckpt[w])                  # the average of iterations 9 and 12, and iteration 13
    for n, _, t, v in runs.values():
        t.close(); v.close(); n.close()


def test_training_continues_from_the_polyak_average(tmp_path):
    """after a validation on the average, the parameters are the average (the reference does not restore them)"""
    path = model_file(tmp_path, max_iter=4, print_after=4, validate_after=4, save_after=100, polyak_after=2,
                      polyak_queue_size=2)
    n = N.Net(path, 16, seed=2)
    train, valid = feeds("tiny", 16, n.num_classes, 3)
    ref = N.Net(path, 16, seed=2)
    rt, rv = feeds("tiny", 16, n.num_classes, 3)
    n.train(train, valid, checkpoint_dir=str(tmp_path), run_name="c")
    for it in range(1, 5):
        rt.get_batch(ref); ref.train_step(want_loss=False)
        if N.polyak_due(path, it):
            ref.polyak_insert()
    ref.load_polyak_weights()
    torch.cuda.synchronize()
    assert n.polyak_count == 2
    assert torch.equal(n.params_tensor(), ref.params_tensor())
    for x in (train, valid, rt, rv, n, ref):
        x.close()


def test_resume_restores_the_counter_without_reducing_again(tmp_path):
    path = model_file(tmp_path, **LOOP)
    n = N.Net(path, 16, seed=5)
    train, valid = feeds("tiny", 16, n.num_classes, 11)
    n.train(train, valid, checkpoint_dir=str(tmp_path), run_name="r")
    counter, eps = n.lr_reduce_counter, {e: n.optimizer_state(e) for e in edge_names(n)}
    assert counter >= 1
    assert checkpoint_format.read(tmp_path / "r.ckpt")["__lr_reduce_counter__"][0] == counter
    longer = model_file(tmp_path, "longer.pbtxt", **dict(LOOP, max_iter=30))
    m = N.Net(longer, 16, seed=9)
    m.load(str(tmp_path / "r.ckpt"))
    assert m.iteration == 24 and m.lr_reduce_counter == counter
    assert {e: m.optimizer_state(e) for e in edge_names(m)} == eps            # the epsilons are not reduced again
    t2, v2 = feeds("tiny", 16, m.num_classes, 12)
    events = m.train(t2, v2, checkpoint_dir=str(tmp_path), run_name="r2")
    assert m.iteration == 30 and [e["iteration"] for e in events] == [27, 28, 30]
    assert m.lr_reduce_counter >= counter
    # a net the loop never reduced writes no counter record; loading such a file resets the counter
    fresh = N.Net(longer, 16, seed=9)
    fresh.save(str(tmp_path / "fresh.ckpt"))
    assert "__lr_reduce_counter__" not in checkpoint_format.read(tmp_path / "fresh.ckpt")
    m.load(str(tmp_path / "fresh.ckpt"))
    assert m.lr_reduce_counter == 0
    for x in (train, valid, t2, v2, n, m, fresh):
        x.close()


@pytest.mark.parametrize("base", ["tiny", "tiny+bn"])
def test_validate_is_the_running_mean_of_batch_metrics(base):
    batch = 16
    n = N.Net(base, batch, seed=4)
    train, valid = feeds(base, batch, n.num_classes, 21)
    for _ in range(5):                                             # running statistics away from their start
        train.get_batch(n); n.train_step(want_loss=False)
    bn = n.bn_layers()
    before = [n.bn_state(b[0])["running_mean"].clone() for b in bn]
    v = n.validate(valid)
    total = f32(0)
    valid.seek(0)
    for k in range(3):                                             # 3 * 16 + 5 images: the last 5 are dropped
        valid.get_batch(n)
        n.fprop(False)
        e = f32(n.metric())
        total = f32(f32(total * f32(k)) / f32(k + 1)) + f32(e / f32(batch * (k + 1)))
    assert v == float(total)
    if base == "tiny+bn":
        assert bn and all(torch.equal(x, n.bn_state(b[0])["running_mean"]) for x, b in zip(before, bn))
    other = N.DataHandler(*dataset(base, 40, n.num_classes, 1), batch_size=8, gpu_image_size=SIZES[base][1])
    with pytest.raises(ValueError, match="batch size"):
        n.validate(other)
    with pytest.raises(ValueError, match="batch size"):
        n.train(other)
    for x in (train, valid, other, n):
        x.close()


def test_command_line_app(tmp_path):
    probe = N.Net("tiny", 1)
    classes = probe.num_classes
    probe.close()
    for name, count, seed in (("train", 64, 1), ("valid", 40, 2)):
        images, labels = dataset("tiny", count, classes, seed)
        np.savez(tmp_path / (name + ".npz"), images=images.numpy(), labels=labels.numpy())
    blocks = """
train_dataset { batch_size: 16 randomize_gpu: true
  data_config { file_pattern: "x" layer_name: "input" can_translate: true can_flip: true gpu_image_size_y: 12 gpu_image_size_x: 12 } }
valid_dataset { batch_size: 16 data_config { file_pattern: "y" layer_name: "input" gpu_image_size_y: 12 gpu_image_size_x: 12 } }
"""
    path = model_file(tmp_path, "app.pbtxt", max_iter=8, print_after=2, validate_after=4, save_after=3)
    with open(path, "a") as f:
        f.write(blocks)
    out = tmp_path / "out"
    env = dict(os.environ, PYTHONPATH=ROOT)
    r = subprocess.run([sys.executable, "-m", "convnet_b200.train", path, "--train", str(tmp_path / "train.npz"),
                        "--valid", str(tmp_path / "valid.npz"), "--checkpoint-dir", str(out), "--seed", "3"],
                       cwd=str(tmp_path), env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr
    names = sorted(os.listdir(out))
    run = names[0][:-len(".ckpt")]
    assert run.startswith("tiny_") and names == [run + s for s in (".ckpt", ".pbtxt", "_train.log", "_valid.log")]
    assert len((out / (run + "_train.log")).read_text().split("\n")) == 5
    assert len((out / (run + "_valid.log")).read_text().split("\n")) == 3
    assert r.stdout.count("Train Acc") == 4 and r.stdout.count("Val Acc") == 2 and "End of training." in r.stdout
    # resumed from its checkpoint, it has nothing left to train and writes the final checkpoint again
    r2 = subprocess.run([sys.executable, "-m", "convnet_b200.train", path, "--train", str(tmp_path / "train.npz"),
                         "--checkpoint-dir", str(out / "again"), "--resume", str(out / (run + ".ckpt"))],
                        cwd=str(tmp_path), env=env, capture_output=True, text=True, timeout=600)
    assert r2.returncode == 0, r2.stderr
    assert "Train Acc" not in r2.stdout and any(f.endswith(".ckpt") for f in os.listdir(out / "again"))
