"""CPU-only: the Adagrad and RMSProp optimizers (ADAGRAD_SGD / RMSPROP_SGD, src/optimizer.cc:202-279).  The config fields
and their refusals, the "+adagrad" / "+rmsprop" model blocks, and the float32 restatement of the kernel's state updates
(tests/opt_rules.py) against the reference's own CPU results (tests/golden/ref_opt.npz)."""
import os

import numpy as np
import pytest

import opt_rules as R
from convnet_b200 import net as N

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "ref_opt.npz")


def test_config_fields_carry_the_proto_defaults_and_names():
    d = N.OptimizerConfig.from_dict({}).to_dict()
    assert d["optimizer_type"] == 0 and d["adagrad_delta"] == 1.0 and d["rms_prop_factor"] == 0.0
    for name, v in N.OptimizerConfig.TYPE.items():
        assert N.OptimizerConfig.from_dict({"optimizer_type": name}).optimizer_type == v
    c = N.OptimizerConfig.from_dict({"optimizer_type": "RMSPROP_SGD", "rms_prop_factor": 0.9, "epsilon": 0.001})
    back = N.OptimizerConfig.from_dict(c.to_dict()).to_dict()
    assert back == c.to_dict() and back["optimizer_type"] == 3
    with pytest.raises(KeyError):
        N.OptimizerConfig.from_dict({"nesterov_momentum": True})


@pytest.mark.parametrize("bad", [{"optimizer_type": "LBFGS"}, {"optimizer_type": 7},
                                 {"optimizer_type": "RMSPROP_SGD", "rms_prop_factor": 1.5},
                                 {"optimizer_type": "RMSPROP_SGD", "rms_prop_factor": -0.1}])
def test_unsupported_configs_are_refused(bad, capfd):
    with pytest.raises(ValueError):
        N.optimizer_schedule(dict(bad, epsilon=0.01), 0)
    with pytest.raises(ValueError):
        N.check_bn_optimizer(dict(bad, epsilon=0.01))
    err = capfd.readouterr().err
    assert ("LBFGS" in err) if bad["optimizer_type"] == "LBFGS" else ("rms_prop_factor" in err or "optimizer_type" in err)


def test_adaptive_configs_keep_the_sgd_schedules():
    base = {"epsilon": 0.01, "epsilon_decay": "INVERSE_T", "epsilon_decay_timescale": 10, "initial_momentum": 0.5,
            "final_momentum": 0.9, "momentum_transition_timescale": 20}
    for t in ("ADAGRAD_SGD", "RMSPROP_SGD"):
        for step in (0, 7, 100):
            assert N.optimizer_schedule(dict(base, optimizer_type=t), step) == N.optimizer_schedule(base, step)
    N.check_bn_optimizer(dict(base, optimizer_type="RMSPROP_SGD", rms_prop_factor=1.0))


@pytest.mark.parametrize("model,base", [("alexnet", "alexnet"), ("lenet+ref-optimizer", "lenet+ref-optimizer"),
                                        ("alexnet+ref-optimizer", "alexnet+ref-optimizer"), ("tiny+bn", "tiny+bn")])
def test_adaptive_models_switch_every_optimizer(model, base):
    n_edges = len(N.model_edge_params(base))
    for suffix, t, scale, extra in (("+adagrad", 2, 0.1, {"adagrad_delta": 1.0}),
                                    ("+rmsprop", 3, 0.01, {"rms_prop_factor": float(np.float32(0.9))})):
        for e in range(n_edges):
            for which in ("weights", "bias"):
                plain = N.model_edge_optimizer(base, e, which)
                got = N.model_edge_optimizer(model + suffix, e, which)
                if plain is None:
                    assert got is None
                    continue
                want = dict(plain, optimizer_type=t, epsilon=float(np.float32(plain["epsilon"]) * np.float32(scale)),
                            minimum_epsilon=float(np.float32(plain["minimum_epsilon"]) * np.float32(scale)), **extra)
                assert got == want, (model + suffix, e, which)
        layers = N.model_bn_layers(model + suffix)
        assert len(layers) == len(N.model_bn_layers(base))
        for entry in layers:
            for k in ("gamma_optimizer", "beta_optimizer"):
                assert entry[k]["optimizer_type"] == t and entry[k]["l2_decay"] == 0.0


def test_adaptive_suffixes_compose_with_bn_either_way():
    a, b = N.model_bn_layers("tiny+bn+rmsprop"), N.model_bn_layers("tiny+rmsprop+bn")
    assert a == b and a and all(x["gamma_optimizer"]["optimizer_type"] == 3 for x in a)
    assert N.model_param_layout("lenet+adagrad") == N.model_param_layout("lenet")


def test_two_adaptive_rules_are_refused(capfd):
    with pytest.raises(ValueError):
        N.model_edge_optimizer("tiny+adagrad+rmsprop", 0)
    assert "one adaptive rule" in capfd.readouterr().err


def _golden_cases(z):
    for k in sorted(z.files):
        if k.endswith("_out"):
            b = k[:-4]
            yield b, z[b + "_s"], z[b + "_g"], float(z[b + "_param"]), z[k]


def test_state_restatement_matches_the_reference_bit_for_bit():
    """bit-identical: the reference's CPU library is compiled for plain x86-64 (no FMA instructions), so it contracts
    nothing and rounds every operation to float32, in the order the restatement (and the kernel) uses"""
    z = np.load(GOLDEN)
    cases = list(_golden_cases(z))
    assert len(cases) == 8
    for name, s, g, p, out in cases:
        mine = R.adagrad_state(s, g, p) if name.startswith("adagrad") else R.rms_prop_state(s, g, p)
        assert np.array_equal(mine.view(np.uint32), out.view(np.uint32)), name
        assert not np.isnan(out).any(), name
    # the 0 / 0 the reference meets (delta 0 on a fresh state, factor 0): the update's gradient term is 0 here
    _, s, g, p, out = [c for c in cases if c[0] == "rmsprop_0_fresh"][0]
    zero = (g == 0)
    assert zero.any() and (out[zero] == 0).all()
    w, h, s1 = R.opt_update(np.ones_like(g), np.zeros_like(g), s, g, R.RMSPROP, lr=0.1, mom=0.9, param=p)
    assert (w[zero] == 1).all() and (h[zero] == 0).all()


def test_adagrad_scale_is_the_double_square_root():
    assert R.adagrad_scale(0) == 1.0 and R.adagrad_scale(3) == 2.0
    assert R.adagrad_scale(1) == float(np.float32(np.sqrt(2.0)))


def test_goldens_regenerate_from_the_reference():
    import importlib.util
    from oracle_lib import RefLib
    if not RefLib.available():
        pytest.skip("oracle/_ref/libeigenmat_ref.so not built (needs the reference sources)")
    spec = importlib.util.spec_from_file_location("gen_opt_golden", os.path.join(ROOT, "tools", "gen_opt_golden.py"))
    gen = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(gen)
    fresh, z = gen.generate(RefLib.PATH), np.load(GOLDEN)
    assert sorted(fresh) == sorted(z.files)
    for k, v in fresh.items():
        assert np.array_equal(np.asarray(v).view(np.uint32), z[k].view(np.uint32)), k
