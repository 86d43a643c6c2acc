"""CPU-only: model files, the reference's config::Model text protos (examples/*/net.pbtxt).

- Round trip: model_text(name) written to a file builds the same model as `name` (same text, parameter layout, fusion
  plan, BN layers, output layer and optimizers) for the built-ins and suffixed names.
- Semantics, one small file per rule: the proto's defaults and presence rules for the geometry, the default optimizers'
  MergeFrom (gamma with the weight default, beta with the bias default), graph order, the ignored is_input / is_output,
  the initialisation rules and init_bias.
- Refusals: what the host cannot run, malformed syntax and unknown fields raise ValueError and name the line and field
  on stderr.
- The reference's own example files, where the reference tree exists.
"""
import math
import os

import numpy as np
import pytest

from convnet_b200 import net as N

ROUND_TRIP = ["alexnet", "alexnet+ref-optimizer+bn", "lenet", "lenet+ref-optimizer", "lcnet", "c3d", "tiny",
              "tiny+bn+rmsprop", "gradcheck", "logcheck", "tiny+bn+gradcheck", "alexnet+soft-targets", "localcheck",
              "alexnet+logistic", "tiny+adagrad", "lenet+binary-ce", "tiny+squared-error"]


def write(tmp_path, text, name="net.pbtxt"):
    p = tmp_path / name
    p.write_text(text)
    return str(p)


def edge_optimizers(model):
    out, n = [], len(N.model_param_layout(model)["edge_offsets"])
    for e in range(n):
        out.append((N.model_edge_optimizer(model, e, "weights"), N.model_edge_optimizer(model, e, "bias")))
    return out


def describe(model):
    return {"text": N.model_text(model), "layout": N.model_param_layout(model), "params": N.model_edge_params(model),
            "fusion": N.model_fusion(model), "bn": N.model_bn_layers(model), "output": N.model_output_layer(model),
            "optimizers": edge_optimizers(model)}


@pytest.mark.parametrize("model", ROUND_TRIP)
def test_round_trip(tmp_path, model):
    path = write(tmp_path, N.model_text(model))
    assert describe(path) == describe(model)


def test_suffixes_compose_with_a_file(tmp_path):
    path = write(tmp_path, N.model_text("tiny"))
    for suffix in ("+bn", "+rmsprop", "+bn+adagrad", "+logistic", "+soft-targets", "+gradcheck"):
        assert N.model_text(path + suffix) == N.model_text("tiny" + suffix)
        assert N.model_param_layout(path + suffix) == N.model_param_layout("tiny" + suffix)


def test_floats_read_back_bit_exactly(tmp_path):
    values = [0.1, 1e-5, 3.4028234663852886e38, 1.401298464324817e-45, -0.0, 0.0005, 1 / 3, 2.5e-8]
    blocks = "".join("layer { name: \"l%d\" num_channels: 4 dropprob: %r }\n" % (k, v) for k, v in enumerate(values))
    edges = "".join("edge { source: \"l%d\" dest: \"l%d\" }\n" % (k, k + 1) for k in range(len(values) - 1))
    text = "name: \"f\" seed: 1\n" + blocks + edges
    path = write(tmp_path, text.replace("dropprob: %r }\n" % values[-1], "activation: SOFTMAX }\n"))
    once = N.model_text(path)
    assert N.model_text(write(tmp_path, once, "again.pbtxt")) == once
    got = [float(l.split(":")[1]) for l in once.splitlines() if l.strip().startswith("dropprob")][:-1]
    assert [np.float32(g).tobytes() for g in got] == [np.float32(v).tobytes() for v in values[:-1]]


# ------------------------------------------------------------------------------------------------------ semantics
HEAD = 'name: "t"\nseed: 7\n'
INPUT = 'layer { name: "input" num_channels: 4 image_size_y: 12 image_size_x: 12 }\n'
OUT = 'layer { name: "output" num_channels: 10 activation: SOFTMAX }\n'


def edge_block(text, dest):
    """the lines of the edge block into `dest` in a model_text"""
    for block in text.split("\nedge {")[1:]:
        if 'dest: "%s"' % dest in block:
            return {l.split(":")[0].strip(): l.split(":", 1)[1].strip() for l in block.splitlines() if ":" in l and "{" not in l
                    and l.startswith("  ") and not l.startswith("    ")}
    raise KeyError(dest)


def test_geometry_falls_back_only_when_absent(tmp_path):
    text = HEAD + INPUT + 'layer { name: "c" num_channels: 8 }\nlayer { name: "p" num_channels: 8 }\n' + OUT + """
edge { source: "input" dest: "c" edge_type: CONVOLUTIONAL kernel_size: 5 kernel_size_y: 3 stride: 2 stride_x: 1
       padding: 2 padding_y: 0 shared_bias: true }
edge { source: "c" dest: "p" edge_type: MAXPOOL }
edge { source: "p" dest: "output" edge_type: FC }
"""
    path = write(tmp_path, text)
    c = edge_block(N.model_text(path), "c")
    assert (c["kernel_size_y"], c["kernel_size_x"], c["kernel_size_t"]) == ("3", "5", "1")
    assert (c["stride_y"], c["stride_x"], c["stride_t"]) == ("2", "1", "1")
    assert (c["padding_y"], c["padding_x"], c["padding_t"]) == ("0", "2", "0")
    # 12 x 12 -> (12 - 3) / 2 + 1 = 5 rows, (12 + 4 - 5) / 1 + 1 = 12 columns; the pool without kernel_size (-1) is global
    p = edge_block(N.model_text(path), "p")
    assert (p["kernel_size"], p["kernel_size_y"], p["kernel_size_x"]) == ("-1", "-1", "-1")
    assert N.model_edge_params(path) == [8 * (3 * 5 * 4 + 1), 0, 10 * (8 + 1)]


def test_proto_defaults_shared_bias_and_response_norm(tmp_path):
    text = HEAD + INPUT + 'layer { name: "c" num_channels: 8 }\n' + OUT + """
edge { source: "input" dest: "c" edge_type: CONVOLUTIONAL kernel_size: 3 }
edge { source: "c" dest: "output" edge_type: FC }
"""
    path = write(tmp_path, text)
    # shared_bias defaults to false: one bias per output position (10 x 10 modules)
    assert N.model_edge_params(path)[0] == 8 * (3 * 3 * 4 + 100)
    e = edge_block(N.model_text(path), "c")
    assert (e["shared_bias"], e["initialization"], e["init_wt"], e["init_bias"]) == ("false", "DENSE_GAUSSIAN_SQRT_FAN_IN", "1", "0")
    rn = HEAD + INPUT + 'layer { name: "r" num_channels: 4 }\n' + OUT + """
edge { source: "input" dest: "r" edge_type: RESPONSE_NORM frac_of_filters_response_norm: 0.5 }
edge { source: "r" dest: "output" edge_type: FC }
"""
    r = edge_block(N.model_text(write(tmp_path, rn, "rn.pbtxt")), "r")
    assert (r["add_scale"], r["pow_scale"], r["frac_of_filters_response_norm"]) == ("0", "0", "0.5")


def test_default_optimizers_merge_field_by_field(tmp_path):
    text = HEAD + """
default_weight_optimizer { epsilon: 0.1 l2_decay: 0.001 final_momentum: 0.9 }
default_bias_optimizer { epsilon: 0.2 final_momentum: 0.5 }
""" + INPUT + 'layer { name: "h" num_channels: 8 activation: RECTIFIED_LINEAR batch_normalize: true ' \
        'gamma_optimizer { epsilon: 0.03 } beta_optimizer { l2_decay: 0.25 } }\n' + OUT + """
edge { source: "input" dest: "h" edge_type: CONV_ONETOONE weight_optimizer { epsilon: 0.05 } }
edge { source: "h" dest: "output" edge_type: FC bias_optimizer { optimizer_type: RMSPROP_SGD rms_prop_factor: 0.9 } }
"""
    path = write(tmp_path, text)
    w0, b0 = N.model_edge_optimizer(path, 0, "weights"), N.model_edge_optimizer(path, 0, "bias")
    assert (w0["epsilon"], w0["l2_decay"], w0["final_momentum"]) == (pytest.approx(0.05), pytest.approx(0.001), pytest.approx(0.9))
    assert (b0["epsilon"], b0["final_momentum"], b0["l2_decay"]) == (pytest.approx(0.2), 0.5, 0.0)
    w1, b1 = N.model_edge_optimizer(path, 1, "weights"), N.model_edge_optimizer(path, 1, "bias")
    assert w1["epsilon"] == pytest.approx(0.1) and w1["optimizer_type"] == 0
    assert (b1["epsilon"], b1["final_momentum"], b1["optimizer_type"]) == (pytest.approx(0.2), 0.5, 3)
    assert b1["rms_prop_factor"] == pytest.approx(0.9)
    # gamma merges with the default WEIGHT optimizer, beta with the default BIAS optimizer
    (bn,) = N.model_bn_layers(path)
    g, b = bn["gamma_optimizer"], bn["beta_optimizer"]
    assert (g["epsilon"], g["l2_decay"], g["final_momentum"]) == (pytest.approx(0.03), pytest.approx(0.001), pytest.approx(0.9))
    assert (b["epsilon"], b["l2_decay"], b["final_momentum"]) == (pytest.approx(0.2), 0.25, 0.5)


def test_graph_order_and_is_input_do_not_matter(tmp_path):
    text = N.model_text("tiny")
    layers = ["layer {" + b for b in text.split("layer {")[1:]]
    layers[-1], edges_tail = layers[-1].split("edge {", 1)
    edges = ["edge {" + b for b in ("edge {" + edges_tail).split("edge {")[1:]]
    head = text.split("layer {")[0]
    shuffled = head + "".join(edges[::-1][:3]) + "".join(layers[::-1]) + "".join(edges[::-1][3:])
    # the deprecated flags are not read: the graph decides input and output
    shuffled = shuffled.replace('name: "conv1"\n', 'name: "conv1"\n  is_input: true\n  is_output: true\n', 1)
    shuffled = shuffled.replace('name: "input"\n', 'name: "input"\n  is_output: true\n', 1)
    path = write(tmp_path, shuffled)
    assert describe(path) == describe("tiny")


INIT_NET = HEAD + INPUT + 'layer { name: "h" num_channels: 64 }\n' + OUT + """
edge { source: "input" dest: "h" edge_type: CONVOLUTIONAL kernel_size: 5 shared_bias: true %s }
edge { source: "h" dest: "output" edge_type: FC }
"""


@pytest.mark.parametrize("rule,init_wt,std", [
    ("DENSE_GAUSSIAN", 0.02, 0.02),
    ("DENSE_GAUSSIAN_SQRT_FAN_IN", 2.0, 2.0 / 10.0),                  # fan-in 5 x 5 x 4 = 100
    ("DENSE_UNIFORM", 0.3, 0.3 * 2 / math.sqrt(12)),                 # U(-0.5, 0.5) x 2 init_wt
    ("DENSE_UNIFORM_SQRT_FAN_IN", 1.0, 2 / math.sqrt(100 / 3.0) / math.sqrt(12)),
])
def test_initialisation_rules(tmp_path, rule, init_wt, std):
    path = write(tmp_path, INIT_NET % ("initialization: %s init_wt: %r" % (rule, init_wt)))
    w = np.array(N.model_initial_weights(path, 0, seed=3), np.float64)
    assert w.size == 64 * 100
    # 6400 samples: the sample std is within 3 % of the rule's (> 7 standard errors), the mean within 5 % of it
    assert abs(w.std() / std - 1) < 0.03, (w.std(), std)
    assert abs(w.mean()) < 0.05 * std
    if rule.startswith("DENSE_UNIFORM"):
        half = std * math.sqrt(3)                                  # the range is +-half
        assert w.max() <= half and w.min() >= -half and w.max() > 0.99 * half and w.min() < -0.99 * half
    else:
        assert abs((w ** 4).mean() / w.var() ** 2 - 3) < 0.3       # kurtosis of a Gaussian


def test_constant_initialisation_takes_init_wt_as_given(tmp_path):
    for v in (0.0, 0.25, -1.5):
        path = write(tmp_path, INIT_NET % ("initialization: CONSTANT init_wt: %r" % v))
        assert set(N.model_initial_weights(path, 0)) == {np.float32(v)}


def test_init_bias_is_read_and_written(tmp_path):
    path = write(tmp_path, INIT_NET % "init_bias: 1.0 initialization: DENSE_UNIFORM_SQRT_FAN_IN")
    assert edge_block(N.model_text(path), "h")["init_bias"] == "1"
    assert edge_block(N.model_text(path), "output")["init_bias"] == "0"


def test_built_in_models_keep_their_initialisation():
    w = np.array(N.model_initial_weights("tiny", 0, seed=42))
    bound = 2 / math.sqrt(8 * 9 / 3.0) / 2                            # conv1: fan-in 8 x 3 x 3, uniform
    assert w.size == 16 * 72 and np.abs(w).max() <= bound and np.abs(w).max() > 0.98 * bound
    assert edge_block(N.model_text("lcnet"), "local3")["init_wt"] == "12"
    assert edge_block(N.model_text("alexnet"), "hidden1_conv")["initialization"] == "DENSE_UNIFORM_SQRT_FAN_IN"


def test_driver_only_fields_are_read_and_ignored(tmp_path):
    extra = """max_iter: 10 print_after: 1 display_after: 1 display: true save_after: 5 validate_after: 5
checkpoint_dir: './ckpt' timestamp: ["1", "2"] reduce_lr_factor: 0.5 reduce_lr_threshold: 0 reduce_lr_num_steps: 3
reduce_lr_max: 2 reduce_lr_layer_name: "output" smaller_is_better: false print_weights: false localizer: false
image_size: 256 patch_size: 224
train_dataset { data_config { file_pattern: "x.h5" layer_name: "input" can_flip: true } batch_size: 128 }
valid_dataset < data_config: [{ file_pattern: "y.h5" layer_name: "input" }] >
"""
    base = INIT_NET % "partial_sum: 4 display: true"
    path = write(tmp_path, base.replace(HEAD, HEAD + extra))
    assert N.model_text(path) == N.model_text(write(tmp_path, INIT_NET % "", "plain.pbtxt"))


def test_syntax_variants(tmp_path):
    text = """# a comment
name: 'sy\\x6Etax' ; seed: 0x7,
layer: { name: "in" "put" num_channels: 4 image_size_y: 8 image_size_x: 8 }   # ':' before '{'
layer < name: "h" num_channels: 6 dropprob: .25 activation: 2 >
layer { name: "output", num_channels: 3; activation: SOFTMAX loss_function_weight: 2.5e-1f }
edge { source: "input" dest: "h" edge_type: CONV_ONETOONE init_wt: 1E0 has_no_bias: True }
edge { source: "h" dest: "output" grad_check: t grad_check_num_params: 3 grad_check_epsilon: [1e-2, 1e-3]
       grad_check_epsilon: 1e-4 }
"""
    t = N.model_text(write(tmp_path, text))
    assert 'name: "syntax"' in t and "seed: 7" in t and 'name: "input"' in t
    assert "dropprob: 0.25" in t and "activation: RECTIFIED_LINEAR" in t and "loss_function_weight: 0.25" in t
    assert edge_block(t, "h")["has_no_bias"] == "true"
    assert edge_block(t, "output")["grad_check_epsilon"] == "[0.01, 0.001, 0.0001]"


# ------------------------------------------------------------------------------------------------------ refusals
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


CHAIN = HEAD + INPUT + 'layer { name: "h" num_channels: 8 activation: RECTIFIED_LINEAR }\n' + OUT + \
    'edge { source: "input" dest: "h" edge_type: CONVOLUTIONAL kernel_size: 3 }\n' + \
    'edge { source: "h" dest: "output" edge_type: FC }\n'
# (what is added, where, the line the message names, words it contains); line 6 is the first edge, 7 the second
REFUSALS = [
    ('layer { name: "x" num_channels: 2 }\nedge { source: "h" dest: "x" }\n', "end", 9, "single chain"),
    ('layer { name: "a" num_channels: 2 }\nlayer { name: "b" num_channels: 2 }\nedge { source: "a" dest: "b" }\n'
     'edge { source: "b" dest: "a" }\n', "end", 8, "layer 'a'", "single chain"),
    ('edge { source: "input" dest: "nowhere" }\n', "end", 8, "dest", "no layer"),
    ('subnet { name: "s" model_file: "m.pbtxt" }\n', "end", 8, "subnet"),
    ("tied_to: \"input:h\"", 6, 6, "tied_to"),
    ("source_slice: \"x\"", 6, 6, "source_slice"),
    ("dest_slice: \"x\"", 7, 7, "dest_slice"),
    ("gpu_id: 1", 6, 6, "gpu_id"),
    ("block_backprop: true", 7, 7, "block_backprop"),
    ("initialization: SPARSE_GAUSSIAN", 6, 6, "initialization", "SPARSE_GAUSSIAN"),
    ("initialization: PRETRAINED", 7, 7, "initialization", "PRETRAINED"),
    ("weight_optimizer { nesterov_momentum: true }", 6, 6, "nesterov_momentum"),
    ("bias_optimizer { shared_prior: true }", 6, 6, "shared_prior"),
    ("weight_optimizer { shared_prior_cost: 0.5 }", 7, 7, "shared_prior_cost"),
    ("weight_optimizer { shared_prior_file: \"p.h5\" }", 7, 7, "shared_prior_file"),
    ("weight_optimizer { lbfgs_memory: 5 }", 6, 6, "lbfgs_memory"),
    ("weight_optimizer { optimizer_type: LBFGS }", 6, 6, "weight_optimizer", "LBFGS is not supported"),
    ("weight_optimizer { epsilon_decay_timescale: 10 }", 6, 6, "weight_optimizer", "epsilon_decay"),
]
LAYER_REFUSALS = [
    ("gaussian_dropout: true", 4, "gaussian_dropout"),
    ("gpu_id: 2", 4, "gpu_id"),
    ('layer_slice { name: "s" }', 4, "layer_slice"),
    ('tied_data: "input"', 4, "tied_data"),
    ("batch_normalize: true gamma_optimizer { weight_norm_limit: 1 }", 4, "gamma_optimizer", "weight_norm_limit"),
]


def add_to_line(text, line, what):
    lines = text.splitlines(keepends=True)
    lines[line - 1] = lines[line - 1].rstrip("\n").rstrip()[:-1] + " " + what + " }\n"
    return "".join(lines)


@pytest.mark.parametrize("case", REFUSALS, ids=lambda c: c[0][:40])
def test_refusals(tmp_path, capfd, case):
    what, where, line, *words = case
    text = CHAIN + what if where == "end" else add_to_line(CHAIN, where, what)
    refused(tmp_path, capfd, text, line, *words)


@pytest.mark.parametrize("case", LAYER_REFUSALS, ids=lambda c: c[0][:40])
def test_layer_refusals(tmp_path, capfd, case):
    what, line, *words = case
    refused(tmp_path, capfd, add_to_line(CHAIN, line, what), line, "layer 'h'", *words)


@pytest.mark.parametrize("edge_type", ["UPSAMPLE", "DOWNSAMPLE", "RGBTOYUV"])
def test_edge_type_refusals(tmp_path, capfd, edge_type):
    refused(tmp_path, capfd, CHAIN.replace("edge_type: FC", "edge_type: " + edge_type), 7, "edge 'h:output'", "edge_type",
            edge_type)


def test_softmax_on_a_hidden_layer_keeps_its_message(tmp_path, capfd):
    refused(tmp_path, capfd, CHAIN.replace("activation: RECTIFIED_LINEAR", "activation: SOFTMAX"), 4, "layer 'h'",
            "SOFTMAX / SOFTMAX_DIST is an output activation")


def test_model_level_refusals(tmp_path, capfd):
    for field in ("polyak_after: 100", "polyak_queue_size: 3"):
        refused(tmp_path, capfd, CHAIN.replace("seed: 7\n", "seed: 7\n" + field + "\n"), 3, field.split(":")[0])


def test_output_layer_refusals_keep_their_message(tmp_path, capfd):
    text = CHAIN.replace('activation: SOFTMAX }', 'activation: SOFTMAX\n  loss_function: HINGE_LINEAR }')
    refused(tmp_path, capfd, text, 6, "layer 'output'", "loss_function HINGE_LINEAR is not supported")


def test_response_norm_window_below_one_channel(tmp_path, capfd):
    text = HEAD + INPUT + 'layer { name: "r" num_channels: 4 }\n' + OUT + \
        'edge { source: "input" dest: "r" edge_type: RESPONSE_NORM\n  frac_of_filters_response_norm: 0.2 }\n' + \
        'edge { source: "r" dest: "output" edge_type: FC }\n'
    refused(tmp_path, capfd, text, 7, "frac_of_filters_response_norm", "below one channel")
    refused(tmp_path, capfd, text.replace("\n  frac_of_filters_response_norm: 0.2", ""), 6, "frac_of_filters_response_norm")


def test_edge_that_leaves_no_output(tmp_path, capfd):
    # 12 x 12 input, 20 x 20 kernel: (12 - 20) / 1 + 1 = -7 modules
    refused(tmp_path, capfd, CHAIN.replace("kernel_size: 3", "kernel_size: 20"), 6, "edge 'input:h'", "no output",
            "-7 x -7 x 1")
    # only y is too large: 12 + 2 - 15 < 0
    refused(tmp_path, capfd, CHAIN.replace("kernel_size: 3", "kernel_size: 3 kernel_size_y: 15 padding: 1"), 6,
            "edge 'input:h'", "no output")
    # a pooling window beyond the image; a temporal kernel on a 2-D layer
    pool = HEAD + INPUT + 'layer { name: "p" num_channels: 4 }\n' + OUT + \
        'edge { source: "input" dest: "p" edge_type: MAXPOOL kernel_size: 13 }\n' + \
        'edge { source: "p" dest: "output" edge_type: FC }\n'
    refused(tmp_path, capfd, pool, 6, "edge 'input:p'", "no output")
    refused(tmp_path, capfd, CHAIN.replace("kernel_size: 3", "kernel_size: 3 kernel_size_t: 2"), 6, "edge 'input:h'",
            "10 x 10 x 0 modules")


@pytest.mark.parametrize("edge_type", ["MAXPOOL", "AVERAGE_POOL", "RESPONSE_NORM"])
def test_pool_and_rnorm_keep_the_channel_count(tmp_path, capfd, edge_type):
    text = HEAD + INPUT + 'layer { name: "p" num_channels: 8 }\n' + OUT + \
        'edge { source: "input" dest: "p" edge_type: %s kernel_size: 3 frac_of_filters_response_norm: 0.5 }\n' % edge_type + \
        'edge { source: "p" dest: "output" edge_type: FC }\n'
    refused(tmp_path, capfd, text, 6, "edge 'input:p'", "channel count", "has 4 channels and the destination 8")
    N.model_text(write(tmp_path, text.replace("num_channels: 8", "num_channels: 4"), "ok.pbtxt"))


def test_padding_refusals(tmp_path, capfd):
    refused(tmp_path, capfd, CHAIN.replace("kernel_size: 3", "kernel_size: 3 padding_y: -1"), 6, "padding_y", "negative")
    refused(tmp_path, capfd, CHAIN.replace("kernel_size: 3", "kernel_size: 3 padding: -1"), 6, "'padding'", "negative")
    # the 3-D conv kernels take no temporal padding
    refused(tmp_path, capfd, CHAIN.replace("kernel_size: 3", "kernel_size: 3 padding_t: 1"), 6, "edge 'input:h'",
            "padding_t 1 is not supported")


def test_explicit_geometry_is_not_a_fallback(tmp_path):
    # kernel_size_y: 0 on a pool is present, so it is used: global in y (the reference's has_kernel_size_y), not 3
    text = HEAD + INPUT + 'layer { name: "p" num_channels: 4 }\n' + OUT + \
        'edge { source: "input" dest: "p" edge_type: MAXPOOL kernel_size: 3 stride: 3 kernel_size_y: 0 }\n' + \
        'edge { source: "p" dest: "output" edge_type: FC }\n'
    path = write(tmp_path, text)
    p = edge_block(N.model_text(path), "p")
    assert (p["kernel_size"], p["kernel_size_y"], p["kernel_size_x"]) == ("3", "0", "3")
    # y: one global window; x: (12 - 3) / 3 + 1 = 4 windows; 4 channels
    assert N.model_edge_params(path) == [0, 10 * (1 * 4 * 4 + 1)]
    assert N.model_text(write(tmp_path, N.model_text(path), "again.pbtxt")) == N.model_text(path)


SYNTAX = [
    ("unknown field", CHAIN.replace("kernel_size: 3", "kernel_size: 3\n kernal_size: 3"), 7, "kernal_size", "unknown field"),
    ("wrong type", CHAIN.replace("kernel_size: 3", "kernel_size: \"3\""), 6, "kernel_size", "integer"),
    ("float for an int", CHAIN.replace("kernel_size: 3", "kernel_size: 3.5"), 6, "kernel_size", "integer"),
    ("bad enum", CHAIN.replace("edge_type: FC", "edge_type: FULL"), 7, "edge_type", "FULL"),
    ("bad bool", CHAIN.replace("kernel_size: 3", "kernel_size: 3 shared_bias: yes"), 6, "shared_bias"),
    ("missing colon", CHAIN.replace("kernel_size: 3", "kernel_size 3"), 6, "kernel_size", "expected ':'"),
    ("unclosed block", CHAIN[:-2], 7, "not closed"),
    ("unclosed string", CHAIN.replace('dest: "h"', 'dest: "h'), 6, "string"),
    ("twice", CHAIN.replace("kernel_size: 3", "kernel_size: 3 kernel_size: 5"), 6, "kernel_size", "twice"),
    ("list for a scalar", CHAIN.replace("kernel_size: 3", "kernel_size: [3, 5]"), 6, "kernel_size", "not repeated"),
    ("missing seed", CHAIN.replace("seed: 7\n", ""), 1, "seed", "required"),
    ("missing source", CHAIN.replace('source: "h" ', ""), 7, "source", "required"),
    ("int32 range", CHAIN.replace("kernel_size: 3", "kernel_size: 4294967296"), 6, "kernel_size", "int32"),
    ("stray symbol", CHAIN.replace("seed: 7", "seed: 7 }"), 2, "field name"),
]


@pytest.mark.parametrize("case", SYNTAX, ids=lambda c: c[0])
def test_syntax_errors(tmp_path, capfd, case):
    _, text, line, *words = case
    refused(tmp_path, capfd, text, line, *words)


def test_missing_file_and_other_names():
    with pytest.raises(ValueError):
        N.model_text("/nonexistent/net.pbtxt")
    with pytest.raises(ValueError):
        N.model_text("no-such-model")
    assert N.model_text("tiny").startswith('name: "tiny"\nseed: 42\n')


# ------------------------------------------------------------------------------------------------------ the reference's files
REF = "/root/reference/examples"
needs_ref = pytest.mark.skipif(not os.path.isdir(REF), reason="the reference tree is not on this machine")


def blocks(text):
    """model_text -> {("layer" | "edge", name or dest): the block's lines}, and the model-level lines"""
    out, head = {}, []
    cur = None
    for l in text.splitlines():
        if l in ("layer {", "edge {"):
            cur = [l]
        elif cur is None:
            head.append(l)
        else:
            cur.append(l)
            if l == "}":
                key = next(x for x in cur if x.startswith("  name:" if cur[0] == "layer {" else "  dest:"))
                out[(cur[0][:-2], key.split('"')[1])] = cur
                cur = None
    return out, head


def assert_same_apart_from(path, model, differences):
    """the file builds `model`, apart from its name, its seed and the initialisation fields listed in `differences`
    ({edge dest: {field: (value in the file, value of the built-in)}})"""
    (fb, fhead), (mb, mhead) = blocks(N.model_text(path)), blocks(N.model_text(model))
    assert [l.split(":")[0] for l in fhead] == [l.split(":")[0] for l in mhead] == ["name", "seed"]
    assert fb.keys() == mb.keys()
    for key in fb:
        f, m = list(fb[key]), list(mb[key])
        for field, (in_file, in_model) in differences.get(key[1] if key[0] == "edge" else None, {}).items():
            assert "  %s: %s" % (field, in_file) in f and "  %s: %s" % (field, in_model) in m, (key, field)
            f.remove("  %s: %s" % (field, in_file))
            m.remove("  %s: %s" % (field, in_model))
        assert f == m, key
    for fn in (N.model_param_layout, N.model_edge_params, N.model_fusion, N.model_bn_layers, N.model_output_layer,
               edge_optimizers):
        assert fn(path) == fn(model), fn.__name__


@needs_ref
def test_reference_mnist_conv_is_lenet_with_its_optimizers():
    assert_same_apart_from(os.path.join(REF, "mnist-conv", "net.pbtxt"), "lenet+ref-optimizer",
                           {"hidden2_conv": {"init_bias": ("1", "0")}})


@needs_ref
def test_reference_imagenet_net_is_alexnet_with_its_optimizers():
    assert_same_apart_from(os.path.join(REF, "imagenet", "CLS_net_20140801232522.pbtxt"), "alexnet+ref-optimizer",
                           {"hidden2_conv": {"init_bias": ("1", "0")}, "hidden4_conv": {"init_bias": ("1", "0")},
                            "hidden5_conv": {"init_bias": ("1", "0")}, "output": {"init_wt": ("0.1", "1")}})


@needs_ref
def test_reference_mnist_ff_loads():
    path = os.path.join(REF, "mnist-ff", "net.pbtxt")
    assert N.model_edge_params(path) == [1024 * 785, 1024 * 1025, 10 * 1025]
    assert N.model_edge_optimizer(path, 0, "weights")["weight_norm_limit"] == 2.0
    assert N.model_output_layer(path)["loss_function"] == "CROSS_ENTROPY_MULTINOMIAL"
