"""CPU-only: the model-file side of checkpoints and Polyak averaging.

- polyak_after / polyak_queue_size are accepted together, reported by model_polyak and printed by model_text with the two
  periods the insertion rule reads; validate_after: 0 and save_after: 0 are refused while Polyak is on.
- polyak_due is the reference's insertion rule (src/convnet.cc:881-883, 965-967), restated here with C++'s truncating %.
- A PRETRAINED edge reads its checkpoint (written here by tests/checkpoint_format.py, an independent numpy writer):
  model_initial_weights gives its weights bit for bit, pretrained_edge_name picks another edge's records, and a missing
  file, a missing record or a wrong size is refused with the model file's line and the field.
"""
import itertools

import numpy as np
import pytest

import checkpoint_format as CF
from convnet_b200 import net as N

NET = """name: "ck"
seed: 7
%s
layer { name: "input" num_channels: 3 image_size_y: 8 image_size_x: 8 }
layer { name: "h" num_channels: 4 activation: RECTIFIED_LINEAR }
layer { name: "output" num_channels: 5 activation: SOFTMAX }
edge { source: "input" dest: "h" edge_type: CONVOLUTIONAL kernel_size: 3 }
edge { source: "h" dest: "output" edge_type: FC %s }
"""
FC_WEIGHTS, FC_BIAS = 5 * 6 * 6 * 4, 5     # the FC edge: 5 outputs of a 6 x 6 x 4 layer


def write(tmp_path, text, name="net.pbtxt"):
    p = tmp_path / name
    p.write_text(text)
    return str(p)


def refused(tmp_path, capfd, text, line, *words):
    path = write(tmp_path, text)
    capfd.readouterr()
    with pytest.raises(ValueError) as e:
        N.model_text(path)
    err = capfd.readouterr().err
    for text in (err, str(e.value)):
        assert "%s:%d:" % (path, line) in text, text
        for w in words:
            assert w in text, (w, text)


# ------------------------------------------------------------------------------------------------------ Polyak
def test_polyak_pair_is_accepted_and_round_trips(tmp_path):
    path = write(tmp_path, NET % ("polyak_after: 10 polyak_queue_size: 3 validate_after: -5", ""))
    assert N.model_polyak(path) == {"polyak_after": 10, "polyak_queue_size": 3, "validate_after": -5, "save_after": -1}
    text = N.model_text(path)
    for line in ("polyak_after: 10", "polyak_queue_size: 3", "validate_after: -5", "save_after: -1"):
        assert line in text.splitlines()
    again = write(tmp_path, text, "again.pbtxt")
    assert N.model_text(again) == text and N.model_polyak(again) == N.model_polyak(path)


def test_polyak_off_prints_nothing_new(tmp_path):
    plain = write(tmp_path, NET % ("", ""), "plain.pbtxt")
    assert N.model_polyak(plain) is None and N.model_polyak("alexnet") is None
    assert "polyak" not in N.model_text(plain) and "validate_after" not in N.model_text(plain)


@pytest.mark.parametrize("field", ["validate_after", "save_after"])
def test_zero_period_is_refused_with_polyak_on(tmp_path, capfd, field):
    refused(tmp_path, capfd, NET % ("polyak_after: 10 polyak_queue_size: 3\n%s: 0" % field, ""), 4, field)
    assert N.model_polyak(write(tmp_path, NET % ("%s: 0" % field, ""), "off.pbtxt")) is None   # no Polyak: read, unused


def trunc_rem(a, b):
    """C++'s a % b: the remainder of the quotient truncated towards zero"""
    q = abs(a) // abs(b)
    return a - b * (q if (a >= 0) == (b > 0) else -q)


def reference_due(pa, q, va, sa, it):
    """src/convnet.cc:881-883 and 965-967 with i + 1 = it"""
    start_val, start_save = va - pa * q, sa - pa * q
    return pa > 0 and trunc_rem(it, pa) == 0 and (trunc_rem(it, va) >= start_val or trunc_rem(it, sa) >= start_save)


def test_polyak_due_is_the_reference_rule(tmp_path):
    assert trunc_rem(-7, 5) == -2 and trunc_rem(7, -5) == 2 and (-7) % 5 == 3     # why the restatement is needed
    checked = fired = 0
    for k, (pa, q, va, sa) in enumerate(itertools.product([1, 3, 10], [1, 2, 4], [-1, -5, 7, 40], [-1, -3, 9, 100])):
        path = write(tmp_path, NET % ("polyak_after: %d polyak_queue_size: %d validate_after: %d save_after: %d"
                                      % (pa, q, va, sa), ""), "p%d.pbtxt" % k)
        for it in list(range(0, 130)) + [1000, 12345]:
            want = reference_due(pa, q, va, sa, it)
            assert N.polyak_due(path, it) == want, (pa, q, va, sa, it)
            checked += 1
            fired += want
    assert 0 < fired < checked
    assert not N.polyak_due(write(tmp_path, NET % ("", ""), "off.pbtxt"), 10)


def test_default_periods_insert_every_polyak_after_steps(tmp_path):
    path = write(tmp_path, NET % ("polyak_after: 4 polyak_queue_size: 2", ""))
    assert [it for it in range(1, 21) if N.polyak_due(path, it)] == [4, 8, 12, 16, 20]


# ------------------------------------------------------------------------------------------------------ PRETRAINED
def checkpoint(tmp_path, edge="h:output", skip=(), sizes=None, name="pre.ckpt"):
    rng = np.random.default_rng(3)
    sizes = sizes or {"weight": FC_WEIGHTS, "bias": FC_BIAS}
    rec = {}
    for t in ("weight", "bias"):
        rec["%s:%s" % (edge, t)] = rng.standard_normal(sizes[t]).astype(np.float32)
        rec["%s:%s_gradient_history" % (edge, t)] = rng.standard_normal(sizes[t]).astype(np.float32)
        rec["%s:%s_step" % (edge, t)] = 17
    rec["%s:weight" % edge][0] = -0.0
    for k in skip:
        del rec[k]
    path = str(tmp_path / name)
    CF.write(path, rec)
    return path, rec


def pretrained(ckpt, extra=""):
    return NET % ("", 'initialization: PRETRAINED pretrained_model: "%s"%s' % (ckpt, extra))


def test_pretrained_weights_come_from_the_file(tmp_path):
    ckpt, rec = checkpoint(tmp_path)
    path = write(tmp_path, pretrained(ckpt))
    got = np.array(N.model_initial_weights(path, 1), dtype=np.float32)
    assert got.view(np.int32).tolist() == rec["h:output:weight"].view(np.int32).tolist()
    text = N.model_text(path)
    assert "initialization: PRETRAINED" in text and 'pretrained_model: "%s"' % ckpt in text
    assert 'pretrained_edge_name: "h:output"' in text
    assert N.model_text(write(tmp_path, text, "again.pbtxt")) == text
    assert N.model_initial_weights(path, 0) == N.model_initial_weights(write(tmp_path, NET % ("", ""), "p.pbtxt"), 0)


def test_pretrained_edge_name_picks_another_edge(tmp_path):
    ckpt, rec = checkpoint(tmp_path, edge="old:top")
    path = write(tmp_path, pretrained(ckpt, ' pretrained_edge_name: "old:top"'))
    got = np.array(N.model_initial_weights(path, 1), dtype=np.float32)
    assert got.view(np.int32).tolist() == rec["old:top:weight"].view(np.int32).tolist()
    assert 'pretrained_edge_name: "old:top"' in N.model_text(path)


def test_pretrained_refusals(tmp_path, capfd):
    refused(tmp_path, capfd, pretrained(str(tmp_path / "none.ckpt")), 8, "pretrained_model", "none.ckpt", "cannot open")
    ckpt, _ = checkpoint(tmp_path, skip=("h:output:bias_step",), name="a.ckpt")
    refused(tmp_path, capfd, pretrained(ckpt), 8, "pretrained_model", "h:output:bias_step", "missing")
    ckpt, _ = checkpoint(tmp_path, sizes={"weight": FC_WEIGHTS + 1, "bias": FC_BIAS}, name="b.ckpt")
    refused(tmp_path, capfd, pretrained(ckpt), 8, "pretrained_model", "h:output:weight", str(FC_WEIGHTS + 1), str(FC_WEIGHTS))
    ckpt, _ = checkpoint(tmp_path, name="c.ckpt")
    refused(tmp_path, capfd, pretrained(ckpt, '\npretrained_edge_name: "x:y"'), 9, "pretrained_edge_name", "x:y:weight")
    bad = tmp_path / "bad.ckpt"
    bad.write_bytes(b"not a checkpoint")
    refused(tmp_path, capfd, pretrained(str(bad)), 8, "pretrained_model", "bad magic")
    refused(tmp_path, capfd, NET % ("", "initialization: PRETRAINED"), 8, "initialization", "PRETRAINED")
