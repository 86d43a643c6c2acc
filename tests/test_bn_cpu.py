"""CPU-only: the "+bn" models (batch normalisation, proto/convnet_config.proto:56-61) — which layers they normalise, the
gamma / beta optimizers they derive, the refusals, and the flat parameter layout (host logic, no device memory)."""
import numpy as np
import pytest

from convnet_b200 import net as N

f32 = np.float32
pad = lambda v: (v + 127) // 128 * 128

# hidden layers written by a conv, 1x1 or FC edge (models.cc)
ALEX_BN = ["hidden1_conv", "hidden2_conv", "hidden2_conv_nin1", "hidden3_conv", "hidden3_conv_nin1", "hidden4_conv",
           "hidden4_conv_nin1", "hidden4_conv_nin2", "hidden5_conv", "hidden5_conv_nin1", "hidden5_conv_nin2", "hidden6",
           "hidden7"]


def test_bn_models_normalise_every_hidden_layer_a_weighted_edge_writes():
    assert [l["name"] for l in N.model_bn_layers("alexnet+bn")] == ALEX_BN
    assert [l["name"] for l in N.model_bn_layers("lenet+bn")] == ["hidden1_conv", "hidden2_conv"]
    assert [l["name"] for l in N.model_bn_layers("tiny+bn")] == ["conv1", "nin1", "conv2"]
    assert [l["name"] for l in N.model_bn_layers("gradcheck+bn")] == ["conv1", "nin1"]
    for base in ("alexnet", "lenet", "tiny", "gradcheck", "c3d"):
        assert N.model_bn_layers(base) == []
    l = N.model_bn_layers("alexnet+bn")[0]
    assert (l["layer"], l["channels"]) == (1, 96)
    assert l["bn_f"] == f32(0.98) and l["bn_epsilon"] == f32(1e-5)             # the proto's defaults


def test_bn_suffix_composes():
    for m in ("tiny+bn", "lenet+bn", "alexnet+bn", "gradcheck+bn", "alexnet+ref-optimizer+bn", "lenet+ref-optimizer+bn",
              "tiny+bn+gradcheck", "alexnet+bn+gradcheck"):
        assert N.model_bn_layers(m), m
    assert [l["name"] for l in N.model_bn_layers("tiny+bn+gradcheck")] == ["conv1", "nin1", "conv2"]


@pytest.mark.parametrize("model", ["c3d+bn", "alexnet+bn+ref-optimizer", "tiny+bn+bn", "nosuchnet+bn", "tiny+ref-optimizer+bn"])
def test_unsupported_bn_models_are_refused(model, capfd):
    with pytest.raises(ValueError):
        N.model_bn_layers(model)
    with pytest.raises(ValueError):
        N.model_param_layout(model)
    if model == "c3d+bn":
        assert "3-D" in capfd.readouterr().err


def test_norm_rules_on_gamma_and_beta_are_refused(capfd):
    N.check_bn_optimizer({"epsilon": 0.01, "final_momentum": 0.9})
    for rule in ({"weight_norm_limit": 4.0}, {"weight_norm_constraint": 1.0}):
        with pytest.raises(ValueError):
            N.check_bn_optimizer(dict({"epsilon": 0.01}, **rule))
    assert "norm" in capfd.readouterr().err
    with pytest.raises(ValueError):
        N.check_bn_optimizer({"epsilon": 0.01, "epsilon_decay_timescale": 10})      # as for any optimizer


def _plain(d):
    return {k: float(v) for k, v in N.OptimizerConfig.from_dict(d).to_dict().items()}


def test_gamma_and_beta_take_the_writing_edges_optimizers_without_l2_and_norm_rules():
    layers = {l["name"]: l for l in N.model_bn_layers("alexnet+ref-optimizer+bn")}
    ramp = {"epsilon": f32(0.01), "initial_momentum": f32(0.5), "final_momentum": f32(0.9),
            "momentum_transition_timescale": 2000}
    for name, l in layers.items():
        edge = l["layer"] - 1
        w, b = N.model_edge_optimizer("alexnet+ref-optimizer", edge), N.model_edge_optimizer("alexnet+ref-optimizer", edge, "bias")
        want_g = dict(w, l2_decay=0.0, weight_norm_limit=0.0, weight_norm_constraint=0.0)
        want_b = dict(b, l2_decay=0.0, weight_norm_limit=0.0, weight_norm_constraint=0.0)
        assert l["gamma_optimizer"] == want_g and l["beta_optimizer"] == want_b, name
        assert l["gamma_optimizer"] == _plain(ramp), name
    # hidden3_conv's edge has l2 0.0005, hidden2_conv_nin1's a norm constraint, hidden6's a norm limit: all cleared
    assert N.model_edge_optimizer("alexnet+ref-optimizer", 7)["l2_decay"] == pytest.approx(5e-4)
    assert N.model_edge_optimizer("alexnet+ref-optimizer", 4)["weight_norm_constraint"] == 1.0
    # the plain models: constant momentum 0.9 (lenet 0.95)
    assert N.model_bn_layers("alexnet+bn")[3]["gamma_optimizer"] == _plain({"epsilon": f32(0.01), "final_momentum": f32(0.9)})
    assert N.model_bn_layers("lenet+bn")[1]["beta_optimizer"] == _plain({"epsilon": f32(0.01), "final_momentum": f32(0.95)})
    # the base model's own edge optimizers are untouched by +bn
    for e in range(19):
        assert N.model_edge_optimizer("alexnet+ref-optimizer+bn", e) == N.model_edge_optimizer("alexnet+ref-optimizer", e)


def test_parameter_layout_grows_by_exactly_the_padded_gamma_beta_slices():
    assert sum(N.model_edge_params("alexnet+bn")) == 104321000 == sum(N.model_edge_params("alexnet"))
    plain, bn = N.model_param_layout("alexnet"), N.model_param_layout("alexnet+bn")
    layers = N.model_bn_layers("alexnet+bn")
    assert len(layers) == 13
    assert plain["total"] == 104321024
    assert bn["total"] == plain["total"] + sum(pad(2 * l["channels"]) for l in layers)
    assert plain["bn_offsets"] == [None] * 20
    # [gamma | beta] of layer i directly follows the padded slice of edge i - 1, the edge that writes it
    sizes = N.model_edge_params("alexnet+bn")
    for l in layers:
        e = l["layer"] - 1
        assert bn["bn_offsets"][l["layer"]] == bn["edge_offsets"][e] + pad(sizes[e])
        if e + 1 < len(sizes):
            assert bn["edge_offsets"][e + 1] == bn["bn_offsets"][l["layer"]] + pad(2 * l["channels"])
    assert sum(o is not None for o in bn["bn_offsets"]) == 13


@pytest.mark.parametrize("model", ["alexnet", "lenet", "tiny", "gradcheck", "c3d", "alexnet+ref-optimizer"])
def test_plain_models_keep_their_layout(model):
    sizes = N.model_edge_params(model)
    offs, total = [], 0
    for s in sizes:
        offs.append(total)
        total += pad(s)
    lay = N.model_param_layout(model)
    assert lay["edge_offsets"] == offs and lay["total"] == total
    assert all(o is None for o in lay["bn_offsets"])
