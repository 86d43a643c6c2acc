"""Logistic units and the output layers' loss functions and metrics, host side (no GPU): the model suffixes and how they
compose, ConvNet's refusals, the static output-layer description, and the float64 restatements of tests/loss_ref.py pinned
to the reference's own CPU library (tests/golden/ref_loss.npz, tools/gen_loss_golden.py)."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import loss_ref as R  # noqa: E402
from convnet_b200 import net as N  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden", "ref_loss.npz")
REF_LIB = os.path.join(ROOT, "oracle", "_ref", "libeigenmat_ref.so")

SOFTMAX_OUT = {"activation": "SOFTMAX", "loss_function": "CROSS_ENTROPY_MULTINOMIAL",
               "performance_metric": "CLASSIFICATION_MULTINOMIAL", "loss_function_weight": 1.0, "labels": True}


@pytest.mark.parametrize("model", ["alexnet", "lenet", "tiny", "gradcheck", "lcnet", "c3d", "alexnet+ref-optimizer"])
def test_existing_models_keep_the_softmax_output(model):
    assert N.model_output_layer(model) == SOFTMAX_OUT
    assert N.Net.model_output_layer(model) == SOFTMAX_OUT


@pytest.mark.parametrize("suffix,act,loss,metric", [
    ("+squared-error", "LINEAR", "SQUARED_ERROR", "SQUARED_ERROR"),
    ("+binary-ce", "LOGISTIC", "CROSS_ENTROPY_BINARY", "CLASSIFICATION_BINARY"),
    ("+soft-targets", "SOFTMAX_DIST", "CROSS_ENTROPY_MULTINOMIAL_DISTRIBUTED", "CROSS_ENTROPY_MULTINOMIAL_DISTRIBUTED")])
@pytest.mark.parametrize("base", ["lenet", "tiny", "gradcheck", "tiny+bn", "lenet+logistic", "alexnet+ref-optimizer+rmsprop"])
def test_output_suffixes(base, suffix, act, loss, metric):
    d = N.model_output_layer(base + suffix)
    assert d == {"activation": act, "loss_function": loss, "performance_metric": metric, "loss_function_weight": 1.0,
                 "labels": False}
    # the output layer keeps its width: the same parameters
    assert N.model_param_layout(base + suffix) == N.model_param_layout(base)


@pytest.mark.parametrize("model", ["alexnet", "lenet", "tiny", "lcnet", "c3d", "tiny+bn", "alexnet+ref-optimizer",
                                   "tiny+adagrad", "lenet+rmsprop", "tiny+gradcheck", "tiny+bn+adagrad"])
def test_logistic_keeps_the_parameter_layout(model):
    assert N.model_param_layout(model + "+logistic") == N.model_param_layout(model)
    assert N.model_edge_params(model + "+logistic") == N.model_edge_params(model)
    assert N.model_output_layer(model + "+logistic") == SOFTMAX_OUT


def test_logistic_composes_with_the_other_suffixes():
    # the suffixes apply in either order and keep their own effects
    for a, b in (("tiny+bn+logistic", "tiny+logistic+bn"), ("tiny+logistic+adagrad", "tiny+adagrad+logistic"),
                 ("tiny+logistic+gradcheck", "tiny+gradcheck+logistic")):
        assert N.model_param_layout(a) == N.model_param_layout(b)
    assert [x["name"] for x in N.model_bn_layers("tiny+bn+logistic")] == [x["name"] for x in N.model_bn_layers("tiny+bn")]
    assert N.model_edge_optimizer("tiny+logistic+adagrad", 0)["optimizer_type"] == 2
    assert N.model_edge_optimizer("alexnet+ref-optimizer+logistic", 0)["momentum_transition_timescale"] == 2000


def test_logcheck_is_gradcheck_with_logistic_units():
    assert N.model_param_layout("logcheck") == N.model_param_layout("gradcheck")
    assert N.model_output_layer("logcheck") == SOFTMAX_OUT
    assert N.model_output_layer("logcheck+squared-error")["loss_function"] == "SQUARED_ERROR"


@pytest.mark.parametrize("model,message", [
    ("tiny+binary-ce+soft-targets", "one output suffix only"),
    ("lenet+squared-error+squared-error", "one output suffix only"),
    ("gradcheck+logistic", "+logistic finds no RECTIFIED_LINEAR hidden layer"),
    ("tiny+logistic+logistic", "+logistic finds no RECTIFIED_LINEAR hidden layer")])
def test_refusals(model, message, capfd):
    with pytest.raises(ValueError) as e:
        N.model_param_layout(model)
    assert message in capfd.readouterr().err
    assert message in str(e.value)


# tiny's model text with fields of one layer changed; the refusal names the line of `field`
@pytest.mark.parametrize("layer,changes,field,message", [
    ("nin1", {"activation": "SOFTMAX"}, "activation", "layer 'nin1': SOFTMAX / SOFTMAX_DIST is an output activation"),
    ("output", {"loss_function": "HINGE_LINEAR"}, "loss_function",
     "layer 'output': loss_function HINGE_LINEAR is not supported"),
    ("output", {"performance_metric": "HINGE_QUADRATIC"}, "performance_metric",
     "layer 'output': performance_metric HINGE_QUADRATIC is not supported"),
    # a labels output with a per-feature loss; a per-feature output with the labels metric
    ("output", {"loss_function": "SQUARED_ERROR"}, "loss_function",
     "layer 'output': loss_function SQUARED_ERROR reads a float target per feature, but this output layer's activation "
     "has integer labels"),
    ("output", {"activation": "LOGISTIC", "loss_function": "CROSS_ENTROPY_BINARY"}, "performance_metric",
     "layer 'output': performance_metric CLASSIFICATION_MULTINOMIAL reads integer labels, but this output layer's "
     "activation has a float target per feature"),
    ("output", {"activation": "LOGISTIC", "loss_function": "CLASSIFICATION_BINARY"}, "loss_function",
     "layer 'output': loss_function CLASSIFICATION_BINARY has no derivative to train with")])
def test_refusals_in_a_model_file(tmp_path, capfd, layer, changes, field, message):
    lines = N.model_text("tiny").splitlines(keepends=True)
    k, at = lines.index('  name: "%s"\n' % layer), {}
    while lines[k] != "}\n":
        name = lines[k].split(":")[0].strip()
        if name in changes:
            lines[k] = "  %s: %s\n" % (name, changes[name])
        at[name] = k + 1
        k += 1
    path = tmp_path / "tiny.pbtxt"
    path.write_text("".join(lines))
    with pytest.raises(ValueError) as e:
        N.model_param_layout(str(path))
    assert "%s:%d: %s" % (path, at[field], message) in capfd.readouterr().err
    assert "%s:%d: %s" % (path, at[field], message) in str(e.value)


def test_loss_codes_follow_the_proto():
    assert N.LOSS_FUNCTIONS.index("CROSS_ENTROPY_MULTINOMIAL") == 2 == R.CE_MULTINOMIAL
    assert N.LOSS_FUNCTIONS.index("CLASSIFICATION_BINARY") == 6 == R.CLASS_BINARY
    assert N.LOSS_FUNCTIONS.index("HINGE_QUADRATIC") == 8


# ---- the float64 restatements against the reference's CPU library (eigenmat), as stored
def test_restatements_match_the_reference_goldens():
    z = np.load(GOLDEN)
    # apply_sigmoid computes 1 / (1 + exp(-x)) in float: within the sigmoid bar of the exact value
    assert np.all(np.abs(z["sigmoid"] - R.sigmoid(z["x"])) <= R.sigmoid_bar(z["x"]))
    # d * s * (1 - s), float
    assert np.all(np.abs(z["logistic_deriv"] - R.logistic_deriv(z["d"], z["s"])) <= R.logistic_deriv_bar(z["d"], z["s"]))
    # the CROSS_ENTROPY_BINARY derivative: 0 on don't-care targets, y - t (exact in float here) elsewhere
    g, _, _ = R.loss_terms(R.CE_BINARY, z["y"], z["t"])
    assert np.array_equal(z["logistic_grad"].astype(np.float64), g.astype(np.float32).astype(np.float64))
    assert np.all(z["logistic_grad"][z["t"] < 0] == 0)
    # -q log(p + 1e-10): the per-element terms of CROSS_ENTROPY_MULTINOMIAL_DISTRIBUTED
    _, terms, mags = R.loss_terms(R.CE_DISTRIBUTED, z["p"], z["q"])
    assert np.all(np.abs(z["cross_entropy"] - terms) <= 8 * R.U * mags)
    # the Bernoulli cross-entropy (CROSS_ENTROPY_BINARY's value here) on the t >= 0 entries
    tb = np.maximum(z["t"], 0)
    _, terms, mags = R.loss_terms(R.CE_BINARY, z["y"], tb)
    assert np.all(np.abs(z["cross_entropy_bernoulli"] - terms) <= 8 * R.U * mags)
    # the metrics decide exactly as the reference does
    assert np.array_equal(R.classification_multinomial(z["p"], z["labels"]), z["softmax_correct"])
    assert np.allclose(R.classification_binary(z["y"], z["t"]), z["logistic_correct"], rtol=2 * R.U, atol=0)
    assert z["logistic_correct"][3] == 0          # the image without a target


def test_restatements_catch_wrong_rules():
    z = np.load(GOLDEN)
    # a sigmoid of the wrong sign, a derivative without the (1 - s), a metric that counts don't-cares
    assert not np.all(np.abs(z["sigmoid"] - R.sigmoid(-z["x"])) <= R.sigmoid_bar(-z["x"]))
    assert not np.all(np.abs(z["logistic_deriv"] - z["d"] * z["s"]) <= R.logistic_deriv_bar(z["d"], z["s"]))
    t = np.maximum(z["t"], 0)
    assert not np.allclose(R.classification_binary(z["y"], t), z["logistic_correct"])


@pytest.mark.skipif(not os.path.exists(REF_LIB), reason="the reference's CPU library is not built here")
def test_goldens_regenerate_from_the_reference_library():
    import gen_loss_golden
    fresh, stored = gen_loss_golden.generate(REF_LIB), np.load(GOLDEN)
    assert sorted(fresh) == sorted(stored.files)
    for k in stored.files:
        assert np.array_equal(fresh[k], stored[k]), k
