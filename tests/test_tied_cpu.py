"""CPU-only: tied edges (the reference's Edge.tied_to), host logic without a GPU.

- Refusals: every tie the host cannot run raises ValueError and names the line of tied_to and what is wrong.
- Model files: tiednet, tiedcheck and a hand-written file with ties in both directions read back to the same model.
- The flat parameter buffer: a tied edge owns no floats, the group's one slice sits at its lowest edge, and the buffer is
  the untied twin's (the same model without tied_to) less the tied edges' slices.
- Buckets and fusion: the shared slice is carried by a bucket triggered at or below the group's lowest edge, and a tie
  group offers no bias-gradient hand-off, the rest of the plan being the twin's.
"""
import re

import pytest

from convnet_b200 import net as N

HEAD = 'name: "t"\nseed: 7\n'
# line 3 the input, 4-11 the layers, 12-19 the edges (one per line)
BASE = HEAD + """layer { name: "input" num_channels: 4 image_size_y: 12 image_size_x: 12 }
layer { name: "a" num_channels: 8 activation: RECTIFIED_LINEAR }
layer { name: "b" num_channels: 8 activation: RECTIFIED_LINEAR }
layer { name: "c" num_channels: 8 activation: RECTIFIED_LINEAR }
layer { name: "p" num_channels: 8 }
layer { name: "f1" num_channels: 16 activation: RECTIFIED_LINEAR }
layer { name: "f2" num_channels: 16 activation: RECTIFIED_LINEAR }
layer { name: "f3" num_channels: 16 activation: RECTIFIED_LINEAR }
layer { name: "output" num_channels: 10 activation: SOFTMAX }
edge { source: "input" dest: "a" edge_type: CONVOLUTIONAL kernel_size: 3 padding: 1 shared_bias: true }
edge { source: "a" dest: "b" edge_type: CONVOLUTIONAL kernel_size: 3 padding: 1 shared_bias: true }
edge { source: "b" dest: "c" edge_type: CONVOLUTIONAL kernel_size: 3 }
edge { source: "c" dest: "p" edge_type: MAXPOOL kernel_size: 2 stride: 2 }
edge { source: "p" dest: "f1" edge_type: FC }
edge { source: "f1" dest: "f2" edge_type: FC }
edge { source: "f2" dest: "f3" edge_type: FC }
edge { source: "f3" dest: "output" edge_type: FC }
"""
# b:c runs a:b's filters at padding 0 (a tie to a LOWER edge); f1:f2 runs f2:f3's weights (a tie to a HIGHER edge)
TIES = {14: 'shared_bias: true tied_to: "a:b"', 17: 'tied_to: "f2:f3"'}


def add(text, adds):
    lines = text.splitlines(keepends=True)
    for line, what in adds.items():
        lines[line - 1] = lines[line - 1].rstrip("\n").rstrip()[:-1] + " " + what + " }\n"
    return "".join(lines)


def write(tmp_path, text, name="net.pbtxt"):
    p = tmp_path / name
    p.write_text(text)
    return str(p)


def untied_twin(tmp_path, model, name="twin.pbtxt"):
    """the model with tied_to removed, as a file: each tied edge gets parameters of its own"""
    return write(tmp_path, re.sub(r'\n *tied_to: "[^"]*"', "", N.model_text(model)), name)


def padded(n):
    return (n + 127) // 128 * 128


# ------------------------------------------------------------------------------------------------------ refusals
# (what is added on which lines, the line the message names, words it contains)
REFUSALS = [
    ({14: 'tied_to: "x:y"'}, 14, "edge 'b:c'", "tied_to", "no edge 'x:y'"),
    ({13: 'tied_to: "b:c"', 14: 'tied_to: "a:b"'}, 13, "edge 'a:b'", "tied_to", "'b:c' is itself tied", "'a:b'"),
    ({16: 'tied_to: "c:p"'}, 16, "edge 'p:f1'", "tied_to", "'c:p' has no parameters"),
    ({16: 'tied_to: "a:b"'}, 16, "tied_to", "CONVOLUTIONAL", "FC", "edge_type"),
    ({15: 'tied_to: "a:b"'}, 15, "tied_to", "CONVOLUTIONAL", "MAXPOOL"),
    ({13: 'tied_to: "input:a"'}, 13, "tied_to", "(8, 3, 3, 8)", "(8, 3, 3, 4)"),
    ({17: 'tied_to: "p:f1"'}, 17, "tied_to", "(16, 1, 1, 16)", "(16, 1, 1, 200)"),
    ({14: 'tied_to: "a:b"'}, 14, "tied_to", "bias", "8 x 100 (one per output position)", "8 x 1 (shared_bias)"),
    ({14: 'shared_bias: true has_no_bias: true tied_to: "a:b"'}, 14, "tied_to", "none (has_no_bias)"),
    ({17: 'has_no_bias: true tied_to: "f2:f3"'}, 17, "tied_to", "none (has_no_bias)", "16 x 1"),
    ({14: 'shared_bias: true tied_to: "a:b" grad_check: true'}, 14, "tied_to", "grad_check", "'a:b'"),
]


@pytest.mark.parametrize("case", REFUSALS, ids=lambda c: "-".join(str(k) for k in c[0]) + ":" + list(c[0].values())[-1][:30])
def test_tie_refusals(tmp_path, capfd, case):
    adds, line, *words = case
    path = write(tmp_path, add(BASE, adds))
    capfd.readouterr()
    with pytest.raises(ValueError):
        N.model_text(path)
    err = capfd.readouterr().err
    assert "%s:%d:" % (path, line) in err, err
    for w in words:
        assert w in err, (w, err)
    with pytest.raises(ValueError):
        N.model_param_layout(path)


def test_tied_edge_may_differ_in_stride_padding_and_image_size(tmp_path):
    # b:c (12 x 12, padding 0) runs a:b's filters (12 x 12, padding 1); tiednet runs one conv at three geometries
    assert N.model_ties(write(tmp_path, add(BASE, TIES))) == {"b:c": "a:b", "f1:f2": "f2:f3"}
    assert N.model_ties("tiednet") == {"pool2:conv3": "conv1:conv2", "conv3:conv4": "conv1:conv2", "fc5:fc6": "fc6:fc7"}
    assert N.model_ties("tiedcheck") == {"c1:c2": "c0:c1", "o1:o2": "pool:o1", "l1:l2": "o2:l1", "f1:f2": "f2:f3"}
    assert N.model_ties("alexnet") == {} and N.model_ties("tiny") == {}


# ------------------------------------------------------------------------------------------------------ model files
def describe(model):
    n = len(N.model_param_layout(model)["edge_offsets"])
    return {"text": N.model_text(model), "layout": N.model_param_layout(model), "params": N.model_edge_params(model),
            "fusion": N.model_fusion(model), "ties": N.model_ties(model), "output": N.model_output_layer(model),
            "optimizers": [(N.model_edge_optimizer(model, e, "weights"), N.model_edge_optimizer(model, e, "bias"))
                           for e in range(n)]}


@pytest.mark.parametrize("model", ["tiednet", "tiedcheck", "hand-written"])
def test_round_trip(tmp_path, model):
    if model == "hand-written":
        model = write(tmp_path, add(BASE, TIES), "hand.pbtxt")
    path = write(tmp_path, N.model_text(model))
    assert describe(path) == describe(model)
    assert N.model_text(write(tmp_path, N.model_text(path), "again.pbtxt")) == N.model_text(model)


def test_model_text_of_a_tied_edge(tmp_path):
    blocks = N.model_text("tiednet").split("\nedge {")[1:]
    tied = [b for b in blocks if "tied_to" in b]
    assert len(tied) == 3
    for b in tied:                               # the owner's initialisation and optimizers apply: none are written
        for field in ("initialization", "init_wt", "init_bias", "pretrained", "weight_optimizer", "bias_optimizer"):
            assert field not in b, (field, b)
        assert "scale_gradients" in b and "has_no_bias" in b


def test_tied_edges_have_no_initial_weights_or_optimizers():
    for model in ("tiednet", "tiedcheck"):
        params = N.model_edge_params(model)
        tied = {m for o, members in groups(model).items() for m in members if m != o}
        for i, p in enumerate(params):
            own = p > 0                          # an edge with parameters of its own: not tied, not a pooling edge
            assert own == (i not in tied and N.model_edge_optimizer(model, i, "weights") is not None), i
            assert (N.model_initial_weights(model, i) is not None) == own, i
    assert len(N.model_initial_weights("tiednet", 1)) == 64 * 64 * 9


# ------------------------------------------------------------------------------------------------------ layout
def groups(model):
    """{owner index: [member indices]} of a model's tie groups"""
    ties = N.model_ties(model)
    names = re.findall(r'source: "([^"]*)"\n *dest: "([^"]*)"', N.model_text(model))
    names = ["%s:%s" % n for n in names]
    out = {}
    for i, n in enumerate(names):
        if n in ties:
            out.setdefault(names.index(ties[n]), [names.index(ties[n])]).append(i)
    return {o: sorted(m) for o, m in out.items()}


@pytest.mark.parametrize("model", ["tiednet", "tiedcheck", "hand-written"])
def test_parameter_layout(tmp_path, model):
    if model == "hand-written":
        model = write(tmp_path, add(BASE, TIES), "hand.pbtxt")
    twin = untied_twin(tmp_path, model)
    g = groups(model)
    assert g
    tied = sorted(set(m for o, members in g.items() for m in members if m != o))
    params, twin_params = N.model_edge_params(model), N.model_edge_params(twin)
    layout, twin_layout = N.model_param_layout(model), N.model_param_layout(twin)
    # a tied edge owns no floats; every other edge owns what its twin does
    for i, (p, q) in enumerate(zip(params, twin_params)):
        assert p == (0 if i in tied else q), (i, p, q)
    assert layout["total"] == twin_layout["total"] - sum(padded(twin_params[i]) for i in tied)
    offs = layout["edge_offsets"] + [layout["total"]]
    slot = [offs[i + 1] - offs[i] for i in range(len(params))]
    for owner, members in g.items():
        lo = members[0]                          # the group's lowest edge carries the owner's slice
        assert slot[lo] == padded(params[owner]), (owner, lo, slot)
        for m in members[1:]:
            assert slot[m] == 0
    # tiednet's FC tie is named by the lower edge: the slice is not at its owner
    if "tiednet" in str(model):
        assert slot[6] == padded(256 * 257) and slot[7] == 0


@pytest.mark.parametrize("model", ["tiednet", "tiedcheck"])
@pytest.mark.parametrize("bucket_floats", [1, 4096, 1 << 20, 1 << 30])
def test_buckets_carry_the_shared_slice_at_or_below_the_lowest_edge(model, bucket_floats):
    layout = N.model_param_layout(model)
    offs = layout["edge_offsets"] + [layout["total"]]
    slots = [offs[i + 1] - offs[i] for i in range(len(offs) - 1)]
    buckets, total = N.plan_buckets(slots, bucket_floats)
    assert total == layout["total"]
    for owner, members in groups(model).items():
        lo = members[0]
        a, b = offs[lo], offs[lo] + slots[lo]
        (carrier,) = [k for k in buckets if k[0] <= a and b <= k[1]]
        assert carrier[2] <= lo, (carrier, lo)


@pytest.mark.parametrize("model", ["tiednet", "tiedcheck", "hand-written"])
def test_tie_groups_offer_no_bias_hand_off(tmp_path, model):
    if model == "hand-written":
        model = write(tmp_path, add(BASE, TIES), "hand.pbtxt")
    plan, twin = N.model_fusion(model), N.model_fusion(untied_twin(tmp_path, model))
    grouped = {m for members in groups(model).values() for m in members}
    for i, (e, t) in enumerate(zip(plan["edges"], twin["edges"])):
        if i in grouped:
            assert not e["offers_bias_grad"]
            e, t = dict(e, offers_bias_grad=None), dict(t, offers_bias_grad=None)
        assert e == t, i
    assert plan["layers"] == twin["layers"]
    # tiednet: conv1:conv2 sits under the max-pool, which would sum its bias gradient if it were untied
    if model == "tiednet":
        assert twin["edges"][1]["offers_bias_grad"] and twin["edges"][2]["sums_bias_below"]


def test_gradcheck_suffix_skips_tied_edges():
    text = N.model_text("tiednet+gradcheck")
    for block in text.split("\nedge {")[1:]:
        if 'edge_type: MAXPOOL' in block:
            continue
        assert ("grad_check: true" in block) == ("tied_to" not in block), block
