"""CPU-only: every built-in model name, with and without suffixes, describes the same model as the snapshot in
tests/golden/builtin_models.json (tools/gen_builtin_models_golden.py): its text, schedule, Polyak settings, data sets,
ties, frozen part, output layer, batch-normalised layers, edge optimizers and the initial weights of every edge with
weights of its own.  An unknown name is refused.
"""
import importlib.util
import json
import os

import pytest

from convnet_b200 import net as N

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_spec = importlib.util.spec_from_file_location("gen_builtin", os.path.join(ROOT, "tools", "gen_builtin_models_golden.py"))
gen = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(gen)
WANT = json.load(open(os.path.join(ROOT, "tests", "golden", "builtin_models.json")))


def test_snapshot_covers_every_base_model_and_suffix_combination():
    plans = json.load(open(os.path.join(ROOT, "tests", "golden", "model_plans.json")))
    assert set(plans) <= set(WANT)
    assert set(gen.BASES) <= set(WANT)
    for model in set(gen.names()) - set(WANT):              # the "+finetune" of a model without an FC edge
        with pytest.raises(ValueError, match="has none"):
            N.model_text(model)


@pytest.mark.parametrize("model", sorted(WANT))
def test_builtin_model_matches_its_snapshot(model):
    got = gen.record(model)
    for field, want in WANT[model].items():
        assert got[field] == want, (model, field)


def test_unknown_model_is_refused():
    with pytest.raises(ValueError, match="unknown model 'nosuchnet'"):
        N.model_text("nosuchnet")
    with pytest.raises(ValueError, match="unknown model 'nosuchnet'"):
        N.model_text("nosuchnet+bn")
