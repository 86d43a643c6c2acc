"""CPU-only: fine-tuning on a frozen trunk, host logic without a GPU.

- block_backprop: which edges and layers are frozen (model_frozen), the refusals at the line of block_backprop, the FLOPs
  a frozen trunk leaves out, and "+finetune" / "+gradcheck" on the built-in models.
- Subnets (the reference's Model.subnet): renaming, merge_layer, remove_layer, num_channels_multiplier, nested subnets,
  parameters_file, block_backprop, start_optimization_after, the parent's default optimizers, tied_to renamed with its
  subnet, and every refusal with its file and line.  model_text writes the expanded model, which reads back to itself.
- Every built-in model and suffix combination keeps the model_text, parameter layout, fusion plan and flops_train it had
  before block_backprop existed (tests/golden/model_plans.json, tools/gen_model_plans_golden.py).
"""
import json
import os

import numpy as np
import pytest

import checkpoint_format as ckpt
from convnet_b200 import net as N

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def write(tmp_path, name, text):
    p = tmp_path / name
    p.write_text(text)
    return str(p)


def edge_blocks(text):
    """{source:dest: the edge block's text} of a model_text"""
    out = {}
    for block in text.split("edge {")[1:]:
        src = block.split('source: "')[1].split('"')[0]
        dst = block.split('dest: "')[1].split('"')[0]
        out[src + ":" + dst] = block
    return out


def refused(tmp_path, capfd, path, file, line, *words):
    capfd.readouterr()
    with pytest.raises(ValueError) as e:
        N.model_text(path)
    err = capfd.readouterr().err
    for text in (err, str(e.value)):
        assert "%s:%d:" % (file, line) in text, text
        for w in words:
            assert w in text, (w, text)


# ------------------------------------------------------------------------------------------------ built-in models
def test_models_without_block_backprop_keep_their_plans():
    import importlib.util
    spec = importlib.util.spec_from_file_location("gen", os.path.join(ROOT, "tools", "gen_model_plans_golden.py"))
    gen = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(gen)
    want = json.load(open(os.path.join(ROOT, "tests", "golden", "model_plans.json")))
    assert len(want) > 100
    for model, record in want.items():
        assert gen.plans(model) == record, model
        assert N.model_frozen(model) == {"edges": [], "layers": []}, model


def fc_flops(model, batch, edge, outputs):
    """2 N K M of an FC edge with M outputs, from its parameter count (K M weights, M biases)"""
    return 2.0 * batch * (N.model_edge_params(model, batch)[edge] - outputs)


@pytest.mark.parametrize("model,fc", [("lenet", {4: 10}), ("alexnet", {16: 4096, 17: 4096, 18: 1000})])
def test_finetune_freezes_the_trunk_below_the_lowest_fc_edge(model, fc):
    lowest = min(fc)
    frozen = N.model_frozen(model + "+finetune")
    assert len(frozen["edges"]) == lowest == len(frozen["layers"])
    text = N.model_text(model + "+finetune")
    blocks = list(edge_blocks(text).values())
    assert len(blocks) == max(fc) + 1
    assert [("block_backprop: true" in b) for b in blocks] == [k < lowest for k in range(len(blocks))]
    assert frozen["edges"] == list(edge_blocks(text))[:lowest]
    # the layout is the full model's; the fusion plan leaves every frozen layer without a derivative pass
    assert N.model_param_layout(model + "+finetune") == N.model_param_layout(model)
    fusion, full = N.model_fusion(model + "+finetune"), N.model_fusion(model)
    for k in range(len(blocks)):
        assert fusion["edges"][k]["up_act"] == full["edges"][k]["up_act"]
        assert fusion["edges"][k]["down_act"] == (0 if k <= lowest else full["edges"][k]["down_act"]), k
    assert not any(layer["deriv_pass"] for layer in fusion["layers"][:lowest + 1])
    # fprop of every edge, the wgrad of the FC edges, and the dgrad of every FC edge but the lowest
    batch = 128
    flops = N.model_flops(model + "+finetune", batch)
    want = flops["fprop"] + sum(fc_flops(model, batch, e, m) * (1 if e == lowest else 2) for e, m in fc.items())
    assert flops["fprop"] == N.model_flops(model, batch)["fprop"]
    assert flops["train"] == pytest.approx(want, rel=1e-12)
    assert flops["train"] < 0.4 * N.model_flops(model, batch)["train"]


def test_finetune_composes_and_refuses_a_model_without_fc(capfd):
    for model in ("alexnet+ref-optimizer+finetune", "tiny+bn+finetune", "tiny+finetune+gradcheck", "tiednet+finetune"):
        assert N.model_frozen(model)["edges"], model
    base = N.model_text("alexnet+ref-optimizer")
    assert N.model_text("alexnet+ref-optimizer+finetune").replace("  block_backprop: true\n", "") == base
    # gamma / beta of a frozen layer keep their place in the buffer
    assert N.model_param_layout("tiny+bn+finetune") == N.model_param_layout("tiny+bn")
    # +gradcheck flags the trained edges only; +finetune drops the flags of the edges it freezes
    for model in ("tiny+finetune+gradcheck", "tiny+finetune"):
        blocks = list(edge_blocks(N.model_text(model)).values())
        assert ["grad_check: true" in b for b in blocks] == [False] * 6 + [True]
    capfd.readouterr()
    with pytest.raises(ValueError):
        N.model_frozen("updown+finetune")
    assert "+finetune" in capfd.readouterr().err


# ------------------------------------------------------------------------------------------------ block_backprop
HEAD = 'name: "b"\nseed: 3\n'
# lines 3-8 the layers, 9-13 the edges (one per line)
CHAIN = HEAD + """layer { name: "input" num_channels: 4 image_size_y: 8 image_size_x: 8 }
layer { name: "c1" num_channels: 8 activation: RECTIFIED_LINEAR }
layer { name: "c2" num_channels: 8 activation: RECTIFIED_LINEAR }
layer { name: "p" num_channels: 8 }
layer { name: "f" num_channels: 16 activation: RECTIFIED_LINEAR }
layer { name: "output" num_channels: 10 activation: SOFTMAX }
edge { source: "input" dest: "c1" edge_type: CONVOLUTIONAL kernel_size: 3 padding: 1 }
edge { source: "c1" dest: "c2" edge_type: CONVOLUTIONAL kernel_size: 3 padding: 1 }
edge { source: "c2" dest: "p" edge_type: MAXPOOL kernel_size: 2 stride: 2 }
edge { source: "p" dest: "f" edge_type: FC }
edge { source: "f" dest: "output" edge_type: FC }
"""


def add(text, adds):
    lines = text.splitlines(keepends=True)
    for line, what in adds.items():
        lines[line - 1] = lines[line - 1].rstrip("\n").rstrip()[:-1] + " " + what + " }\n"
    return "".join(lines)


def test_block_backprop_freezes_the_edges_below(tmp_path):
    path = write(tmp_path, "n.pbtxt", add(CHAIN, {9: "block_backprop: true", 10: "block_backprop: true",
                                                  11: "block_backprop: true"}))
    assert N.model_frozen(path) == {"edges": ["input:c1", "c1:c2", "c2:p"], "layers": ["c1", "c2", "p"]}
    # a pooling edge below a blocked one needs no flag of its own
    path = write(tmp_path, "m.pbtxt", add(CHAIN, {9: "block_backprop: true", 10: "block_backprop: true"}))
    assert N.model_frozen(path) == {"edges": ["input:c1", "c1:c2"], "layers": ["c1", "c2"]}
    again = write(tmp_path, "again.pbtxt", N.model_text(path))
    assert N.model_text(again) == N.model_text(path)
    assert N.model_text(path).count("block_backprop: true") == 2
    # every edge frozen: the output layer keeps the derivative its loss writes
    path = write(tmp_path, "all.pbtxt", add(CHAIN, {k: "block_backprop: true" for k in (9, 10, 12, 13)}))
    assert N.model_frozen(path)["layers"] == ["c1", "c2", "p", "f"]
    assert N.model_flops(path, 8)["train"] == N.model_flops(path, 8)["fprop"]


@pytest.mark.parametrize("adds,line,words", [
    ({12: "block_backprop: true"}, 12, ["edge 'input:c1'", "below the blocked edge 'p:f'", "set block_backprop on it too"]),
    ({10: "block_backprop: true"}, 10, ["edge 'input:c1'", "below the blocked edge 'c1:c2'"]),
    ({9: "block_backprop: true grad_check: true"}, 9, ["grad_check on a frozen edge"]),
], ids=["below-an-fc", "below-a-conv", "grad-check"])
def test_block_backprop_refusals(tmp_path, capfd, adds, line, words):
    path = write(tmp_path, "n.pbtxt", add(CHAIN, adds))
    refused(tmp_path, capfd, path, path, line, "field 'block_backprop'", *words)
    with pytest.raises(ValueError):
        N.model_frozen(path)


def test_a_tie_group_is_frozen_or_trained_as_a_whole(tmp_path, capfd):
    path = write(tmp_path, "n.pbtxt", add(CHAIN.replace('"input" num_channels: 4', '"input" num_channels: 8'),
                                          {9: "block_backprop: true", 10: 'tied_to: "input:c1"'}))
    refused(tmp_path, capfd, path, path, 9, "field 'block_backprop'", "tie group")
    ok = write(tmp_path, "ok.pbtxt", add(CHAIN.replace('"input" num_channels: 4', '"input" num_channels: 8'),
                                         {9: "block_backprop: true", 10: 'tied_to: "input:c1" block_backprop: true'}))
    assert N.model_ties(ok) == {"c1:c2": "input:c1"} and len(N.model_frozen(ok)["edges"]) == 2


# ------------------------------------------------------------------------------------------------ subnets
# the subnet: a trunk with its own default optimizer (which the parent's replaces), lines 3-6 layers, 7-9 edges
SUB = """name: "trunk"
seed: 1
layer { name: "input" num_channels: 4 image_size_y: 8 image_size_x: 8 }
layer { name: "c1" num_channels: 8 activation: RECTIFIED_LINEAR }
layer { name: "p1" num_channels: 8 }
layer { name: "out" num_channels: 10 activation: SOFTMAX }
edge { source: "input" dest: "c1" edge_type: CONVOLUTIONAL kernel_size: 3 padding: 1 weight_optimizer { epsilon: 0.5 } }
edge { source: "c1" dest: "p1" edge_type: MAXPOOL kernel_size: 2 stride: 2 }
edge { source: "p1" dest: "out" edge_type: FC }
default_weight_optimizer { epsilon: 0.3 initial_momentum: 0.7 }
"""


def parent(sub_path, subnet="", extra=""):
    """lines 1-2 the head, 3-4 the layers, 5 the default optimizer, 6-8 the subnet block, 9 the new head's edge"""
    return ('name: "net"\nseed: 5\n'
            'layer { name: "data" num_channels: 4 image_size_y: 8 image_size_x: 8 }\n'
            'layer { name: "head" num_channels: 10 activation: SOFTMAX }\n'
            'default_weight_optimizer { epsilon: 0.01 l2_decay: 0.001 }\n'
            'subnet { name: "s" model_file: "%s"\n'
            '  merge_layer { subnet_layer: "input" net_layer: "data" } remove_layer: "out"\n'
            '  %s }\n'
            'edge { source: "s_p1" dest: "head" edge_type: FC }\n%s' % (sub_path, subnet, extra))


def test_subnet_expansion(tmp_path):
    sub = write(tmp_path, "sub.pbtxt", SUB)
    path = write(tmp_path, "net.pbtxt", parent(sub, "block_backprop: true start_optimization_after: 7 "
                                                    "num_channels_multiplier: 2"))
    text = N.model_text(path)
    assert "subnet" not in text
    assert [b.split('name: "')[1].split('"')[0] for b in text.split("layer {")[1:]] == ["data", "s_c1", "s_p1", "head"]
    assert 'name: "s_c1"\n  num_channels: 16' in text and 'name: "s_p1"\n  num_channels: 16' in text
    assert 'name: "data"\n  num_channels: 4' in text                 # the net's config of a merged layer
    edges = edge_blocks(text)
    assert list(edges) == ["data:s_c1", "s_c1:s_p1", "s_p1:head"]
    assert ["block_backprop: true" in b for b in edges.values()] == [True, True, False]
    assert N.model_frozen(path) == {"edges": ["data:s_c1", "s_c1:s_p1"], "layers": ["s_c1", "s_p1"]}
    w, b = N.model_edge_optimizer(path, 0, "weights"), N.model_edge_optimizer(path, 0, "bias")
    # the edge's own block over the PARENT's default (the subnet file's defaults are not applied); start_optimization_after
    # on both optimizers
    assert (w["epsilon"], w["l2_decay"], w["initial_momentum"], w["start_optimization_after"]) == \
        (0.5, np.float32(0.001), 0.0, 7)
    assert (b["epsilon"], b["start_optimization_after"]) == (0.0, 7)
    head = N.model_edge_optimizer(path, 2, "weights")
    assert (head["epsilon"], head["start_optimization_after"]) == (np.float32(0.01), 0)
    again = write(tmp_path, "again.pbtxt", text)
    assert N.model_text(again) == text


def test_start_optimization_after_zero_is_set_too(tmp_path):
    sub = write(tmp_path, "sub.pbtxt", SUB.replace("{ epsilon: 0.5 }", "{ epsilon: 0.5 start_optimization_after: 9 }"))
    assert N.model_edge_optimizer(write(tmp_path, "n.pbtxt", parent(sub)), 0)["start_optimization_after"] == 0


def test_nested_subnets_expand_first(tmp_path):
    sub = write(tmp_path, "sub.pbtxt", SUB)
    # the middle file holds the trunk as its subnet "in", its input merged into the middle's own input layer "x"
    mid = write(tmp_path, "mid.pbtxt", 'name: "mid"\nseed: 1\n'
                'layer { name: "x" num_channels: 4 image_size_y: 8 image_size_x: 8 }\n'
                'subnet { name: "in" model_file: "%s" merge_layer { subnet_layer: "input" net_layer: "x" } }\n' % sub)
    path = write(tmp_path, "net.pbtxt", parent(mid).replace('subnet_layer: "input"', 'subnet_layer: "x"')
                 .replace('remove_layer: "out"', 'remove_layer: "in_out"').replace('"s_p1"', '"s_in_p1"'))
    assert list(edge_blocks(N.model_text(path))) == ["data:s_in_c1", "s_in_c1:s_in_p1", "s_in_p1:head"]


def test_tied_to_is_renamed_with_its_subnet(tmp_path):
    sub = write(tmp_path, "sub.pbtxt", SUB.replace("num_channels: 4", "num_channels: 8").replace(
        'layer { name: "p1"', 'layer { name: "c2" num_channels: 8 activation: RECTIFIED_LINEAR }\nlayer { name: "p1"').replace(
        'edge { source: "c1" dest: "p1"', 'edge { source: "c1" dest: "c2" edge_type: CONVOLUTIONAL kernel_size: 3 padding: 1 '
        'tied_to: "input:c1" }\nedge { source: "c2" dest: "p1"'))
    path = write(tmp_path, "n.pbtxt", parent(sub).replace("num_channels: 4", "num_channels: 8"))
    assert N.model_ties(path) == {"s_c1:s_c2": "data:s_c1"}


def test_parameters_file_makes_every_edge_pretrained(tmp_path):
    sub = write(tmp_path, "sub.pbtxt", SUB)
    w = np.arange(8 * 36, dtype=np.float32) / 100
    records = {}
    for kind, n, v in (("weight", 8 * 36, w), ("bias", 8 * 64, np.ones(8 * 64, np.float32))):
        records["input:c1:" + kind] = v
        records["input:c1:%s_gradient_history" % kind] = np.zeros(n, np.float32)
        records["input:c1:%s_step" % kind] = 3
    params = str(tmp_path / "trunk.ckpt")
    ckpt.write(params, records)
    path = write(tmp_path, "n.pbtxt", parent(sub, 'parameters_file: "%s" block_backprop: true' % params))
    block = edge_blocks(N.model_text(path))["data:s_c1"]
    assert "initialization: PRETRAINED" in block and 'pretrained_model: "%s"' % params in block
    assert 'pretrained_edge_name: "input:c1"' in block
    assert np.array_equal(np.array(N.model_initial_weights(path, 0), np.float32), w)

def test_parameters_file_without_a_record(tmp_path, capfd):
    """a record the checkpoint lacks is named at the line of parameters_file"""
    sub = write(tmp_path, "sub.pbtxt", SUB)
    params = str(tmp_path / "trunk.ckpt")
    ckpt.write(params, {"input:c1:weight": np.zeros(8 * 36, np.float32)})
    path = write(tmp_path, "n.pbtxt", parent(sub, 'parameters_file: "%s"' % params))
    refused(tmp_path, capfd, path, path, 8, "edge 'data:s_c1'", "input:c1:weight_gradient_history")


SUBNET_REFUSALS = [
    ('merge_layer { subnet_layer: "nope" net_layer: "data" }', "net", 8, "field 'subnet_layer'", "no layer 'nope'"),
    ('merge_layer { subnet_layer: "c1" net_layer: "nope" }', "net", 8, "field 'net_layer'", "the net has no layer 'nope'"),
    ('remove_layer: "nope"', "net", 8, "field 'remove_layer'", "no layer 'nope'"),
    ("gpu_id_offset: 1", "net", 8, "field 'gpu_id_offset'"),
    ("num_channels_multiplier: 0", "net", 8, "field 'num_channels_multiplier'"),
]


@pytest.mark.parametrize("case", SUBNET_REFUSALS, ids=lambda c: c[0][:30])
def test_subnet_refusals(tmp_path, capfd, case):
    what, file, line, *words = case
    sub = write(tmp_path, "sub.pbtxt", SUB)
    path = write(tmp_path, "net.pbtxt", parent(sub, what))
    refused(tmp_path, capfd, path, path, line, "subnet 's'", *words)


def test_subnet_refusals_in_files(tmp_path, capfd):
    sub = write(tmp_path, "sub.pbtxt", SUB)
    # a renamed layer that the net already has: named at the subnet file's layer
    path = write(tmp_path, "net.pbtxt", parent(sub).replace('"head" num_channels', '"s_c1" num_channels: 8 }\n'
                                                           'layer { name: "head" num_channels'))
    refused(tmp_path, capfd, path, sub, 4, "becomes 's_c1'")
    # an error inside the subnet file: that file and line
    bad = write(tmp_path, "bad.pbtxt", SUB.replace('"p1" num_channels: 8', '"p1" num_channels: 8 gaussian_dropout: true'))
    refused(tmp_path, capfd, write(tmp_path, "n2.pbtxt", parent(bad)), bad, 5, "gaussian_dropout")
    # a file that cannot be read, or that contains itself
    refused(tmp_path, capfd, write(tmp_path, "n3.pbtxt", parent(str(tmp_path / "missing.pbtxt"))),
            str(tmp_path / "n3.pbtxt"), 6, "field 'model_file'", "cannot open")
    loop = str(tmp_path / "loop.pbtxt")
    write(tmp_path, "loop.pbtxt", parent(loop))
    refused(tmp_path, capfd, loop, loop, 6, "contains itself")
    # no merge: two layers without an incoming edge, not a single chain
    path = write(tmp_path, "n4.pbtxt", parent(sub).replace('merge_layer { subnet_layer: "input" net_layer: "data" } ', ""))
    capfd.readouterr()
    with pytest.raises(ValueError):
        N.model_text(path)
    assert "single chain" in capfd.readouterr().err
    # the subnet's block_backprop, refused below: a weighted edge of the net under the blocked trunk
    path = write(tmp_path, "n5.pbtxt", parent(sub, "block_backprop: true").replace(
        'layer { name: "data" num_channels: 4 image_size_y: 8 image_size_x: 8 }\n',
        'layer { name: "raw" num_channels: 4 image_size_y: 8 image_size_x: 8 }\n'
        'layer { name: "data" num_channels: 4 }\n') +
        'edge { source: "raw" dest: "data" edge_type: CONVOLUTIONAL kernel_size: 3 padding: 1 }\n')
    refused(tmp_path, capfd, path, path, 9, "edge 'raw:data'", "field 'block_backprop'", "below the blocked edge")
