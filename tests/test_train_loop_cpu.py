"""CPU-only: the schedule of the training loop (Net.train, host/train.cc TrainSchedule) against a Python restatement of
the reference's Train loop (src/convnet.cc:921-1006, C++'s truncating %), CheckReduceLearningRate (reduce_lr_due)
against a numpy float32 restatement bit for bit, the schedule fields of a model (model_schedule) and the loop's
refusals."""
import itertools

import numpy as np
import pytest

from convnet_b200 import net as N

f32 = np.float32


def cmod(a, b):
    """C++'s a % b: the remainder takes the sign of a"""
    r = abs(a) % abs(b)
    return -r if a < 0 else r


def due(history, num_steps, threshold, smaller_is_better):
    """CheckReduceLearningRate (src/convnet.cc:799-817) in float32"""
    h = [f32(v) for v in history]
    if len(h) < num_steps:
        return False
    i, m1, m2 = len(h) - num_steps, f32(0), f32(0)
    for j in range(num_steps // 2):
        m1 = (m1 * f32(j)) / f32(j + 1) + h[i] / f32(j + 1)
        i += 1
    for j in range(num_steps - num_steps // 2):
        m2 = (m2 * f32(j)) / f32(j + 1) + h[i] / f32(j + 1)
        i += 1
    diff = m1 - m2 if smaller_is_better else m2 - m1
    return bool(diff < f32(threshold))


def restated_loop(s, values, start=0, counter=0):
    """src/convnet.cc:921-1006 over schedule `s` (a dict of Model fields) with the validation values `values` (None: no
    validation set): the records train_dry_run gives"""
    out, hist, dont, inserted = [], [], 0, 0
    pa, qs, va, sa = s["polyak_after"], s["polyak_queue_size"], s["validate_after"], s["save_after"]
    for i in range(start, s["max_iter"]):
        it, a = i + 1, set()
        if cmod(it, s["print_after"]) == 0:
            a.add("print")
        if pa > 0 and qs > 0 and cmod(it, pa) == 0 and (cmod(it, va) >= va - pa * qs or cmod(it, sa) >= sa - pa * qs):
            a.add("insert")
            inserted += 1
        if values is not None and va > 0 and cmod(it, va) == 0:
            a.add("validate")
            if pa > 0 and qs > 0 and inserted:
                a.add("polyak")
            hist.append(values[len(hist)])
            if f32(s["reduce_lr_factor"]) < 1.0:
                if due(hist, s["reduce_lr_num_steps"], s["reduce_lr_threshold"], s["smaller_is_better"]) and \
                        counter < s["reduce_lr_max"]:
                    dont -= 1
                    if dont + 1 < 0:
                        dont = s["reduce_lr_num_steps"]
                        counter += 1
                        a.add("lr_reduced")
        if cmod(it, sa) == 0:
            a.add("save")
        if a:
            out.append((it, a))
    if cmod(s["max_iter"], sa) != 0:
        out.append((s["max_iter"], {"save", "final"}))
    return out


DEFAULTS = dict(max_iter=-1, print_after=-1, validate_after=-1, save_after=-1, reduce_lr_factor=1.0,
                reduce_lr_threshold=0.0, reduce_lr_num_steps=0, reduce_lr_max=0, smaller_is_better=False,
                reduce_lr_layer_name="", checkpoint_dir="", polyak_after=0, polyak_queue_size=0)


def model_file(tmp_path, name="s.pbtxt", base="tiny", **fields):
    """model_text(base) with the Model fields `fields` in front"""
    head = []
    for k, v in fields.items():
        head.append('%s: "%s"' % (k, v) if isinstance(v, str) else "%s: %s" % (k, str(v).lower() if isinstance(v, bool) else v))
    p = tmp_path / name
    p.write_text("\n".join(head) + "\n" + N.model_text(base))
    return str(p)


def values(n, seed):
    """validation values that wander up and down, so that reductions come and go"""
    r = np.random.RandomState(seed)
    return [float(f32(v)) for v in 0.5 + np.cumsum(r.choice([-0.02, -0.01, 0.0, 0.01, 0.02], n))]


PERIODS = [(-1, 4, -1), (3, 4, 5), (5, 7, 3), (2, -1, 6), (4, 6, -3), (-3, 5, 10), (7, 0, 7)]


@pytest.mark.parametrize("polyak", [None, (1, 2), (2, 3), (3, 1)])
@pytest.mark.parametrize("print_after,validate_after,save_after", PERIODS)
def test_dry_run_matches_the_reference_loop(tmp_path, print_after, validate_after, save_after, polyak):
    if polyak and validate_after == 0:
        pytest.skip("the model reader refuses validate_after 0 with Polyak averaging on")
    s = dict(DEFAULTS, max_iter=31, print_after=print_after, validate_after=validate_after, save_after=save_after,
             reduce_lr_factor=0.5, reduce_lr_num_steps=2, reduce_lr_max=2)
    if polyak:
        s.update(polyak_after=polyak[0], polyak_queue_size=polyak[1])
    path = model_file(tmp_path, **{k: v for k, v in s.items() if k not in ("reduce_lr_layer_name", "checkpoint_dir")})
    vals = values(40, (print_after + 7 * save_after) % 1000)
    for start in (0, 13):
        for v in (vals, None):
            want = restated_loop(s, v, start)
            assert N.train_dry_run(path, v, iteration=start) == want
    if polyak is None:
        assert not any("insert" in a or "polyak" in a for _, a in N.train_dry_run(path, vals))
    else:
        assert any("insert" in a for _, a in N.train_dry_run(path, vals))


@pytest.mark.parametrize("num_steps,reduce_lr_max,counter,threshold,smaller", [
    (2, 3, 0, 0.0, False), (3, 1, 0, 0.0, True), (4, 10, 0, 0.005, False), (5, 2, 1, -0.01, True), (1, 4, 0, 0.0, False),
    (0, 2, 0, 0.0, False), (6, 0, 0, 0.0, False), (3, 5, 5, 0.0, False)])
def test_learning_rate_decisions(tmp_path, num_steps, reduce_lr_max, counter, threshold, smaller):
    """reduce_lr_max, the counter a checkpoint restores and dont_reduce_lr's short-circuit decide as in :986-994"""
    s = dict(DEFAULTS, max_iter=60, print_after=10, validate_after=2, save_after=30, reduce_lr_factor=0.25,
             reduce_lr_num_steps=num_steps, reduce_lr_max=reduce_lr_max, reduce_lr_threshold=threshold,
             smaller_is_better=smaller)
    path = model_file(tmp_path, **{k: v for k, v in s.items() if k not in ("reduce_lr_layer_name", "checkpoint_dir")})
    for seed in range(4):
        vals = values(30, seed)
        got = N.train_dry_run(path, vals, lr_reduce_counter=counter)
        assert got == restated_loop(s, vals, counter=counter)
        reductions = sum("lr_reduced" in a for _, a in got)
        assert reductions <= max(0, reduce_lr_max - counter)
    # a factor of 1 (the default) never reduces
    path1 = model_file(tmp_path, "one.pbtxt", **{k: v for k, v in dict(s, reduce_lr_factor=1.0).items()
                                                  if k not in ("reduce_lr_layer_name", "checkpoint_dir")})
    assert not any("lr_reduced" in a for _, a in N.train_dry_run(path1, values(30, 0)))


def test_reduce_lr_due_bit_for_bit():
    r = np.random.RandomState(5)
    checked = 0
    for num_steps, smaller in itertools.product([0, 1, 2, 3, 4, 5, 6, 7, 9], [False, True]):
        for trial in range(40):
            n = r.randint(0, 12)
            h = [float(f32(v)) for v in r.uniform(0, 1, n) * (10.0 ** r.randint(-3, 2))]
            for thr in (0.0, -0.01, 0.01, float(f32(r.uniform(-0.1, 0.1)))):
                assert N.reduce_lr_due(h, num_steps, thr, smaller) == due(h, num_steps, thr, smaller)
                checked += 1
            if len(h) >= num_steps and num_steps:
                # the threshold at the float32 difference itself and one ulp either side: the comparison is strict
                i, m1, m2 = len(h) - num_steps, f32(0), f32(0)
                for j in range(num_steps // 2):
                    m1 = (m1 * f32(j)) / f32(j + 1) + f32(h[i]) / f32(j + 1); i += 1
                for j in range(num_steps - num_steps // 2):
                    m2 = (m2 * f32(j)) / f32(j + 1) + f32(h[i]) / f32(j + 1); i += 1
                d = m1 - m2 if smaller else m2 - m1
                for thr in (d, np.nextafter(d, f32(np.inf)), np.nextafter(d, f32(-np.inf))):
                    assert N.reduce_lr_due(h, num_steps, float(thr), smaller) == due(h, num_steps, float(thr), smaller)
                assert not N.reduce_lr_due(h, num_steps, float(d), smaller)
                assert N.reduce_lr_due(h, num_steps, float(np.nextafter(d, f32(np.inf))), smaller)
    assert checked > 2000


def test_model_schedule_defaults_and_example_values(tmp_path):
    assert N.model_schedule("tiny") == DEFAULTS_SCHEDULE
    assert N.model_schedule(model_file(tmp_path, "plain.pbtxt")) == DEFAULTS_SCHEDULE
    # the schedule lines of examples/imagenet/CLS_net_20140801232522.pbtxt and examples/mnist-conv/net.pbtxt
    imagenet = dict(max_iter=10000000, print_after=100, save_after=2000, validate_after=2000, reduce_lr_factor=0.5,
                    reduce_lr_num_steps=4, reduce_lr_max=10, reduce_lr_threshold=0.0, checkpoint_dir="./")
    mnist = dict(max_iter=100000, print_after=1000, save_after=10000, validate_after=1000, reduce_lr_factor=0.5,
                 reduce_lr_num_steps=6, reduce_lr_max=10, reduce_lr_threshold=0.0, checkpoint_dir="./checkpoint_dir")
    for name, fields in (("imagenet.pbtxt", imagenet), ("mnist.pbtxt", mnist)):
        assert N.model_schedule(model_file(tmp_path, name, base="lenet", **fields)) == dict(DEFAULTS_SCHEDULE, **fields)
    other = dict(smaller_is_better=True, reduce_lr_layer_name="output", reduce_lr_threshold=0.25, print_after=-7)
    assert N.model_schedule(model_file(tmp_path, "o.pbtxt", **other)) == dict(DEFAULTS_SCHEDULE, **other)
    # model_text writes none of them: a model's text, and so a checkpoint's __model__, carries no schedule
    assert N.model_text(model_file(tmp_path, "m.pbtxt", base="lenet", **mnist)) == N.model_text("lenet")


DEFAULTS_SCHEDULE = {k: v for k, v in DEFAULTS.items() if k not in ("polyak_after", "polyak_queue_size")}


@pytest.mark.parametrize("fields,match", [
    (dict(max_iter=5, print_after=0), "field 'print_after'"),
    (dict(max_iter=5, save_after=0), "field 'save_after'"),
    (dict(max_iter=5, reduce_lr_layer_name="hidden"), "field 'reduce_lr_layer_name'"),
    (dict(max_iter=5, reduce_lr_layer_name="nosuch"), "field 'reduce_lr_layer_name'")])
def test_refusals_name_the_field(tmp_path, fields, match):
    with pytest.raises(ValueError, match=match):
        N.train_dry_run(model_file(tmp_path, **fields))
    # the model itself still reads: the refusal belongs to the loop
    assert N.model_schedule(model_file(tmp_path, **fields))["max_iter"] == 5


def test_a_validate_after_of_zero_never_validates(tmp_path):
    got = N.train_dry_run(model_file(tmp_path, max_iter=6, validate_after=0, save_after=3), [0.1] * 10)
    assert got == [(k, {"print"} | ({"save"} if k % 3 == 0 else set())) for k in range(1, 7)]


def test_more_validations_than_values_is_refused(tmp_path):
    with pytest.raises(ValueError, match="values"):
        N.train_dry_run(model_file(tmp_path, max_iter=6, validate_after=2), [0.1])
