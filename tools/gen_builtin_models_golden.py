"""Write tests/golden/builtin_models.json: per built-in model and suffix combination, what the host-only queries report
about it: its Polyak settings, data sets, ties, frozen part and output layer as they are, and digests of its model_text,
its schedule, every edge's optimizers, its batch-normalised layers and the initial weights (seed 42) of every edge with
weights of its own.  The names are those of tests/golden/model_plans.json, plus each base model with "+finetune" where
that builds.  tests/test_builtin_models_cpu.py checks that every name still reports exactly this.

    python tools/gen_builtin_models_golden.py [out.json]
"""
import ctypes as ct
import hashlib
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

BASES = ["alexnet", "lenet", "c3d", "tiny", "lcnet", "gradcheck", "logcheck", "localcheck", "tiednet", "tiedcheck",
         "updown", "updowncheck"]


def names():
    """the model names the file covers (main() leaves out the "+finetune" names that do not build)"""
    plans = json.load(open(os.path.join(ROOT, "tests", "golden", "model_plans.json")))
    return sorted(plans) + [b + "+finetune" for b in BASES]


def digest(value):
    """the first 32 hex digits of the sha256 of a string, or of a JSON value with sorted keys"""
    text = value if isinstance(value, str) else json.dumps(value, sort_keys=True)
    return hashlib.sha256(text.encode()).hexdigest()[:32]


def initial_weights(model, seed=42):
    """per edge: the digest of model_initial_weights(model, edge, seed) as float32 bytes, or None for an edge without
    weights of its own (one call per edge into a buffer of the edge's parameter count, which holds its weights)"""
    from convnet_b200 import net as N
    out = []
    with N.Model(model) as m:
        for e, (_, _, _, params) in enumerate(m.edges()):
            buf = np.empty(max(params, 1), np.float32)
            n = N._check(m.H.cnb_net_initial_weights(m.h, e, seed, buf.ctypes.data_as(ct.POINTER(ct.c_float)), params))
            assert n <= params, (model, e)
            out.append(hashlib.sha256(buf[:n]).hexdigest()[:32] if n else None)
    return out


def record(model):
    """what the host-only queries report about `model`; ValueError for a name the package refuses"""
    from convnet_b200 import net as N
    edges = len(N.model_edge_params(model))
    optimizers = [[N.model_edge_optimizer(model, e, w) for w in ("weights", "bias")] for e in range(edges)]
    return {"text": digest(N.model_text(model)), "schedule": digest(N.model_schedule(model)),
            "polyak": N.model_polyak(model), "train_dataset": N.model_dataset(model, "train_dataset"),
            "valid_dataset": N.model_dataset(model, "valid_dataset"), "ties": N.model_ties(model),
            "frozen": N.model_frozen(model), "output_layer": N.model_output_layer(model),
            "bn_layers": digest(N.model_bn_layers(model)), "optimizers": digest(optimizers),
            "initial_weights": initial_weights(model)}


def main():
    out = {}
    for model in names():
        try:
            out[model] = record(model)
        except ValueError:
            assert model.endswith("+finetune"), model
    path = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "tests", "golden", "builtin_models.json")
    with open(path, "w") as f:                               # one model per line
        f.write("{\n" + ",\n".join("%s: %s" % (json.dumps(m), json.dumps(out[m], sort_keys=True)) for m in sorted(out)) +
                "\n}\n")
    print("%d models -> %s" % (len(out), path))


if __name__ == "__main__":
    main()
