"""CPU-only: the UPSAMPLE, DOWNSAMPLE and RGBTOYUV edges in model files and built-in models.

- sample_factor and the three edge types read, written and read back; shapes propagated (2-D and 3-D layers).
- Every refusal at the line of the field it names; a tie on a sampling edge refused with a message.
- The fusion plan and parameter layout of updown / updowncheck, and their composition with +bn, +rmsprop, +logistic.
"""
import pytest

from convnet_b200 import net as N

HEAD = 'name: "s"\nseed: 3\n'


def write(tmp_path, text, name="net.pbtxt"):
    p = tmp_path / name
    p.write_text(text)
    return str(p)


def chain(layers, edges, size=12, channels=4, t=1):
    """a chain model: input (channels x size x size x t), then `layers` [(name, channels, extra)], `edges` [extra] between
    consecutive layers; the last layer is a LINEAR SQUARED_ERROR output"""
    text = HEAD + 'layer { name: "input" num_channels: %d image_size_y: %d image_size_x: %d image_size_t: %d }\n' % (
        channels, size, size, t)
    names = ["input"]
    for k, (name, ch, extra) in enumerate(layers):
        out = " loss_function: SQUARED_ERROR performance_metric: SQUARED_ERROR" if k + 1 == len(layers) else ""
        text += 'layer { name: "%s" num_channels: %d%s%s }\n' % (name, ch, (" " + extra) if extra else "", out)
        names.append(name)
    for k, extra in enumerate(edges):
        text += 'edge { source: "%s" dest: "%s" %s }\n' % (names[k], names[k + 1], extra)
    return text


def refused(tmp_path, capfd, text, line, *words):
    path = write(tmp_path, text)
    capfd.readouterr()
    with pytest.raises(ValueError):
        N.model_text(path)
    err = capfd.readouterr().err
    assert "%s:%d:" % (path, line) in err, err
    for w in words:
        assert w in err, (w, err)
    with pytest.raises(ValueError):
        N.Net(path, 2)


CONV = "edge_type: CONVOLUTIONAL kernel_size: 3 padding: 1 shared_bias: true"
# input 4 x 12 x 12 -> conv 8 -> down 3 (4 x 4) -> conv 8 -> up 2 (8 x 8) -> conv 3 output.  Edge lines 9..13
UPDOWN = chain([("c1", 8, ""), ("d1", 8, ""), ("c2", 8, "activation: RECTIFIED_LINEAR"), ("u2", 8, ""), ("output", 3, "")],
               [CONV, "edge_type: DOWNSAMPLE sample_factor: 3", CONV, "edge_type: UPSAMPLE sample_factor: 2", CONV])


def edge_lines(text):
    return {l.split(":", 1)[0].strip(): l.split(":", 1)[1].strip() for l in text.splitlines() if l.startswith("  ")
            and not l.startswith("    ") and ":" in l}


def blocks(text, kind):
    return [edge_lines(b) for b in text.split("\n%s {" % kind)[1:]]


def test_sample_factor_round_trip(tmp_path):
    path = write(tmp_path, UPDOWN)
    text = N.model_text(path)
    edges = blocks(text, "edge")
    assert [e["edge_type"] for e in edges] == ["CONVOLUTIONAL", "DOWNSAMPLE", "CONVOLUTIONAL", "UPSAMPLE", "CONVOLUTIONAL"]
    assert (edges[1]["sample_factor"], edges[3]["sample_factor"]) == ("3", "2")
    assert "sample_factor" not in edges[0] and "kernel_size" not in edges[1]
    again = write(tmp_path, text, "again.pbtxt")
    assert N.model_text(again) == text
    assert N.model_param_layout(again) == N.model_param_layout(path)
    assert N.model_fusion(again) == N.model_fusion(path)
    # sampling edges have no parameters: 8 x (36 + 1), 8 x (72 + 1), 3 x (72 + 1)
    assert N.model_edge_params(path) == [8 * 37, 0, 8 * 73, 0, 3 * 73]


@pytest.mark.parametrize("model", ["updown", "updowncheck", "updown+bn", "updown+rmsprop", "updown+logistic",
                                   "updowncheck+rmsprop"])
def test_built_ins_round_trip(tmp_path, model):
    path = write(tmp_path, N.model_text(model))
    assert N.model_text(path) == N.model_text(model)
    assert N.model_param_layout(path) == N.model_param_layout(model)
    assert N.model_fusion(path) == N.model_fusion(model)


def test_rgbtoyuv_round_trip(tmp_path):
    text = chain([("yuv", 3, ""), ("c", 4, "activation: RECTIFIED_LINEAR"), ("output", 3, "")],
                 ["edge_type: RGBTOYUV", CONV, CONV], channels=3)
    path = write(tmp_path, text)
    assert blocks(N.model_text(path), "edge")[0] == {"source": '"input"', "dest": '"yuv"', "edge_type": "RGBTOYUV"}
    plan = N.model_fusion(path)
    # the layer RGBTOYUV writes receives no derivative: the conv above it has no act' to apply and nothing sums below it
    assert plan["edges"][1]["down_act"] == 0 and not plan["edges"][1]["sums_bias_below"]
    assert plan["edges"][0] == dict(up_act=0, down_act=0, dropout_up=False, scale_down=False, sums_bias_below=False,
                                    offers_bias_grad=False)


def test_shapes_propagate(tmp_path):
    # model_edge_params of the conv after each sampling edge is independent of the image size, so read the sizes through
    # an FC edge: its weights are (features in) x (features out)
    text = chain([("d", 4, ""), ("u", 4, ""), ("output", 2, "")],
                 ["edge_type: DOWNSAMPLE sample_factor: 2", "edge_type: UPSAMPLE sample_factor: 3", "edge_type: FC"])
    assert N.model_edge_params(write(tmp_path, text)) == [0, 0, 2 * (4 * 18 * 18 + 1)]        # 12 -> 6 -> 18
    # 3-D: the frames are kept, the spatial axes sampled (4 channels x 2 frames)
    text3 = chain([("d", 4, ""), ("u", 4, ""), ("output", 2, "")],
                  ["edge_type: DOWNSAMPLE sample_factor: 3", "edge_type: UPSAMPLE sample_factor: 2", "edge_type: FC"], t=2)
    assert N.model_edge_params(write(tmp_path, text3, "t.pbtxt")) == [0, 0, 2 * (4 * 8 * 8 * 2 + 1)]   # 12 -> 4 -> 8


def test_updown_fusion_plan():
    plan = N.model_fusion("updown")
    e = plan["edges"]
    # every conv under an UPSAMPLE offers its bias gradient; the UPSAMPLE dgrad sums it under the ReLU' mask
    for up in (6, 8):
        assert e[up - 1]["offers_bias_grad"] and e[up]["sums_bias_below"] and e[up]["down_act"] == 1
        assert e[up]["scale_down"]
    for down in (2, 4):
        assert e[down]["down_act"] == 1 and e[down]["sums_bias_below"]
    assert e[0]["up_act"] == 0 and e[1]["down_act"] == 0
    assert not any(l["activation_pass"] or l["deriv_pass"] for l in plan["layers"])
    assert N.model_param_layout("updown")["edge_offsets"][:3] == [0, 0, 1792]     # yuv has no parameters; conv1 3 x 3 x 3 -> 64


def test_updowncheck_logistic_layer_keeps_its_passes():
    plan = N.model_fusion("updowncheck")
    assert [e["down_act"] for e in plan["edges"]][4] == 2      # sigma' of up2 from the conv above it
    # the sampling kernels fuse ReLU only: sigma after the up-sampling stays the layer's own pass
    assert plan["edges"][3]["up_act"] == 0 and plan["layers"][4]["activation_pass"]
    assert N.model_text("updowncheck").count("grad_check: true") == 5      # the four convs and the FC


def test_bn_composes_but_not_on_the_yuv_layer():
    bn = N.model_param_layout("updown+bn")["bn_offsets"]
    assert bn[1] is None and all(bn[k] is not None for k in (2, 4, 6, 8, 10))


REFUSALS = [
    # (replace, by, line, words)
    ("sample_factor: 3", "sample_factor: 0", 10, "sample_factor", "below 1"),
    ("sample_factor: 2", "sample_factor: -1", 12, "sample_factor", "below 1"),
    ("sample_factor: 3", "sample_factor: 5", 10, "sample_factor", "divisible"),
    ('layer { name: "d1" num_channels: 8 }', 'layer { name: "d1" num_channels: 6 }', 10, "edge_type", "DOWNSAMPLE",
     "channel count"),
    ('layer { name: "u2" num_channels: 8 }', 'layer { name: "u2" num_channels: 5 }', 12, "edge_type", "UPSAMPLE",
     "channel count"),
    ("edge_type: UPSAMPLE sample_factor: 2", "edge_type: RGBTOYUV", 12, "edge_type", "RGBTOYUV", "input layer"),
]


@pytest.mark.parametrize("case", REFUSALS, ids=lambda c: c[1][:30])
def test_refusals(tmp_path, capfd, case):
    old, new, line, *words = case
    assert old in UPDOWN
    refused(tmp_path, capfd, UPDOWN.replace(old, new), line, *words)


def test_rgbtoyuv_refusals(tmp_path, capfd):
    base = lambda ch, t=1: chain([("yuv", ch, ""), ("output", 3, "")], ["edge_type: RGBTOYUV", CONV], channels=ch, t=t)
    refused(tmp_path, capfd, base(4), 6, "edge_type", "RGBTOYUV", "3 colour channels")
    refused(tmp_path, capfd, base(3, 2), 6, "edge_type", "RGBTOYUV", "3-D")
    bn = base(3).replace('layer { name: "yuv" num_channels: 3 }', 'layer { name: "yuv" num_channels: 3\n  batch_normalize: true }')
    refused(tmp_path, capfd, bn, 5, "layer 'yuv'", "batch_normalize", "RGBTOYUV")
    # into the output layer: it would receive no derivative, and its loss needs one
    refused(tmp_path, capfd, chain([("output", 3, "")], ["edge_type: RGBTOYUV"], channels=3), 5, "edge_type", "RGBTOYUV",
            "output layer")
    softmax = HEAD + 'layer { name: "input" num_channels: 3 image_size_y: 4 image_size_x: 4 }\n' + \
        'layer { name: "output" num_channels: 3 activation: SOFTMAX }\n' + \
        'edge { source: "input" dest: "output" edge_type: RGBTOYUV }\n'
    refused(tmp_path, capfd, softmax, 5, "edge_type", "RGBTOYUV", "output layer")


def test_tie_on_a_sampling_edge_is_refused(tmp_path, capfd):
    text = UPDOWN.replace("edge_type: UPSAMPLE sample_factor: 2", 'edge_type: UPSAMPLE sample_factor: 2 tied_to: "c1:d1"')
    refused(tmp_path, capfd, text, 12, "tied_to", "has no parameters")
    old = 'dest: "c2" ' + CONV + ' }'
    assert old in UPDOWN
    refused(tmp_path, capfd, UPDOWN.replace(old, old[:-1] + 'tied_to: "c2:u2" }'), 11, "tied_to", "edge 'c2:u2' has no parameters")
