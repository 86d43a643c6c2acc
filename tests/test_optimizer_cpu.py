"""CPU-only: the optimizer schedules (cnb_optimizer_schedule) against a restatement of the reference's
GetDecayedEpsilon / GetMomentum (src/optimizer.cc:83-104,158-165), and the optimizer blocks of the "+ref-optimizer" models
against the reference's pbtxt files (values hard-coded here with their line numbers)."""
import math

import numpy as np
import pytest

from convnet_b200 import net as N

f32 = np.float32


def ref_schedule(c, step):
    """optimizer.cc:83-104 (epsilon) and :158-165 (momentum) in float32, as the reference computes them"""
    full = dict(N.OptimizerConfig.from_dict(c).to_dict())
    eps0, ts = f32(full["epsilon"]), full["epsilon_decay_timescale"]
    mn, rule = f32(full["minimum_epsilon"]), full["epsilon_decay"]
    eps = eps0
    if ts > 0:
        f = f32(step) / f32(ts)
        if rule == 2:
            eps = eps0 * f32(math.exp(-f))
        elif rule == 1:
            eps = eps0 / (f32(1) + f)
        elif rule == 3:
            eps = eps0 * (f32(1) - f) + mn * f if f < 1 else mn
        elif rule == 4:
            eps = f32(float(eps0) * math.pow(float(f32(full["decay_factor"])), step // ts))   # integer quotient
    if eps < mn:
        eps = mn
    mts = full["momentum_transition_timescale"]
    m0, m1 = f32(full["initial_momentum"]), f32(full["final_momentum"])
    mom = m0 + (m1 - m0) * (f32(1) - f32(math.exp(-f32(step) / f32(mts)))) if mts > 0 else m1
    return float(eps), float(mom)


@pytest.mark.parametrize("rule", ["NONE", "INVERSE_T", "EXPONENTIAL", "LINEAR", "EXPONENTIAL_STEP"])
@pytest.mark.parametrize("minimum", [0.0, 0.004])
def test_schedule_matches_the_reference_formulas(rule, minimum):
    ts = 0 if rule == "NONE" else 100
    c = {"epsilon": 0.01, "epsilon_decay": rule, "epsilon_decay_timescale": ts, "minimum_epsilon": minimum,
         "decay_factor": 0.5, "initial_momentum": 0.5, "final_momentum": 0.9, "momentum_transition_timescale": 300}
    for step in (0, 1, 99, 100, 1000, 1050):
        got, want = N.optimizer_schedule(c, step), ref_schedule(c, step)
        np.testing.assert_allclose(got, want, rtol=1e-6, err_msg="%s step %d" % (rule, step))
        assert got[0] >= f32(minimum)                                    # the floor always applies
    if rule == "LINEAR":
        assert N.optimizer_schedule(c, 1000)[0] == f32(minimum)
    if rule == "EXPONENTIAL_STEP":                                       # piecewise constant between multiples of ts
        assert N.optimizer_schedule(c, 99)[0] == N.optimizer_schedule(c, 0)[0]
        assert N.optimizer_schedule(c, 100)[0] == pytest.approx(max(0.005, minimum), rel=1e-6)


def test_momentum_without_timescale_is_final_momentum():
    c = {"epsilon": 0.02, "initial_momentum": 0.5, "final_momentum": 0.95}
    for step in (0, 1, 5000):
        assert N.optimizer_schedule(c, step) == (f32(0.02), f32(0.95))
    ramp = dict(c, momentum_transition_timescale=2000)
    assert N.optimizer_schedule(ramp, 0)[1] == f32(0.5)
    np.testing.assert_allclose(N.optimizer_schedule(ramp, 2000)[1], 0.5 + 0.45 * (1 - math.exp(-1)), rtol=1e-6)


def test_invalid_configs_are_refused():
    with pytest.raises(KeyError):
        N.OptimizerConfig.from_dict({"nesterov_momentum": True})            # outside the SGD path
    with pytest.raises(ValueError):
        N.optimizer_schedule({"epsilon": 0.01, "epsilon_decay_timescale": 10}, 0)   # a timescale without a rule


# examples/imagenet/CLS_net_20140801232522.pbtxt: every weight / bias optimizer has epsilon 0.01 and momentum 0.5 -> 0.9
# over 2000 steps (e.g. :148-158); the extra weight settings by edge index of the alexnet chain
RAMP = {"epsilon": f32(0.01), "initial_momentum": f32(0.5), "final_momentum": f32(0.9), "momentum_transition_timescale": 2000}
ALEX_WEIGHTS = {
    0: {},                                             # input -> hidden1_conv, :148-153
    3: {},                                             # hidden1_rnorm -> hidden2_conv, :192-197
    4: {"weight_norm_constraint": 1.0},                # hidden2_conv_nin1, :213-219
    7: {"l2_decay": f32(0.0005)},                      # hidden3_conv, :257-263
    8: {"weight_norm_constraint": 1.0},                # hidden3_conv_nin1, :279-285
    9: {"l2_decay": f32(0.0005)},                      # hidden4_conv, :305-311
    10: {"weight_norm_constraint": 1.0},               # hidden4_conv_nin1, :327-333
    11: {"weight_norm_constraint": 1.0},               # hidden4_conv_nin2, :348-354
    12: {"l2_decay": f32(0.0005)},                     # hidden5_conv, :374-380
    13: {"weight_norm_constraint": 1.0},               # hidden5_conv_nin1, :396-402
    14: {"weight_norm_constraint": 1.0},               # hidden5_conv_nin2, :417-423
    16: {"weight_norm_limit": 4.0, "l2_decay": f32(0.0005)},   # hidden6, :447-454
    17: {"weight_norm_limit": 4.0, "l2_decay": f32(0.0005)},   # hidden7, :469-476
    18: {"weight_norm_limit": 4.0, "l2_decay": f32(0.0005)},   # output, :491-498
}
# examples/mnist-conv/net.pbtxt: weights epsilon 0.01, initial 0.5 / final 0.95 momentum (no timescale), l2 0.0005
# (:60-65, :90-95, :117-123, the FC edge also weight_norm_limit 4 at :121); biases epsilon 0.01, final 0.95 (:66-69)
LENET_W = {"epsilon": f32(0.01), "initial_momentum": f32(0.5), "final_momentum": f32(0.95), "l2_decay": f32(0.0005)}
LENET_WEIGHTS = {0: {}, 2: {}, 4: {"weight_norm_limit": 4.0}}
LENET_BIAS = {"epsilon": f32(0.01), "final_momentum": f32(0.95)}


def _expect(base, extra):
    d = N.OptimizerConfig.from_dict({}).to_dict()
    d.update(base)
    d.update(extra)
    return {k: float(v) for k, v in d.items()}


def test_alexnet_ref_optimizer_carries_the_pbtxt_blocks():
    n_edges = len(N.model_edge_params("alexnet"))
    assert n_edges == 19
    for e in range(n_edges):
        w = N.model_edge_optimizer("alexnet+ref-optimizer", e, "weights")
        if e not in ALEX_WEIGHTS:
            assert w is None, e                        # pooling / response-norm edges have no parameters
            continue
        assert w == _expect(RAMP, ALEX_WEIGHTS[e]), e
        assert N.model_edge_optimizer("alexnet+ref-optimizer", e, "bias") == _expect(RAMP, {}), e


def test_lenet_ref_optimizer_carries_the_pbtxt_blocks():
    for e in range(5):
        w = N.model_edge_optimizer("lenet+ref-optimizer", e, "weights")
        if e not in LENET_WEIGHTS:
            assert w is None
            continue
        assert w == _expect(LENET_W, LENET_WEIGHTS[e]), e
        assert N.model_edge_optimizer("lenet+ref-optimizer", e, "bias") == _expect(LENET_BIAS, {}), e


def test_plain_models_keep_their_constant_momentum_update():
    for e, l2 in ((0, 0.0), (7, f32(0.0005)), (16, 0.0)):
        assert N.model_edge_optimizer("alexnet", e) == _expect({"epsilon": f32(0.01), "final_momentum": f32(0.9)},
                                                               {"l2_decay": l2})
    assert N.model_edge_optimizer("lenet", 4)["final_momentum"] == float(f32(0.95))


def test_ref_optimizer_is_only_defined_for_alexnet_and_lenet(capfd):
    with pytest.raises(ValueError):
        N.model_edge_optimizer("tiny+ref-optimizer", 0)
    err = capfd.readouterr().err
    assert "alexnet" in err and "lenet" in err
    with pytest.raises(ValueError):
        N.model_edge_params("nosuchnet")
