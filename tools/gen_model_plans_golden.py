"""Write tests/golden/model_plans.json: per built-in model and suffix combination that builds, digests of its
model_text, its parameter layout, its fusion plan and its flops_train at batch 128 (float.hex), as this build computes
them.  The committed file holds the values of the build before block_backprop existed; tests/test_finetune_cpu.py checks
that every model without block_backprop keeps all of them exactly.

    python tools/gen_model_plans_golden.py [out.json]
"""
import hashlib
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

BASES = ["alexnet", "lenet", "c3d", "tiny", "lcnet", "gradcheck", "logcheck", "localcheck", "tiednet", "tiedcheck",
         "updown", "updowncheck"]
SUFFIXES = ["", "+bn", "+adagrad", "+rmsprop", "+gradcheck", "+logistic", "+squared-error", "+binary-ce", "+soft-targets",
            "+ref-optimizer", "+ref-optimizer+bn", "+ref-optimizer+rmsprop", "+bn+rmsprop", "+bn+gradcheck", "+bn+logistic"]


def digest(value):
    """the first 32 hex digits of the sha256 of a string, or of a JSON value with sorted keys"""
    text = value if isinstance(value, str) else json.dumps(value, sort_keys=True)
    return hashlib.sha256(text.encode()).hexdigest()[:32]


def plans(model):
    """the record of one model; ValueError for a combination the package refuses"""
    from convnet_b200 import net as N
    return {"text": digest(N.model_text(model)), "layout": digest(N.model_param_layout(model)),
            "fusion": digest(N.model_fusion(model)), "flops_train": N.model_flops(model, 128)["train"].hex()}


def main():
    out = {}
    for base in BASES:
        for suffix in SUFFIXES:
            try:
                out[base + suffix] = plans(base + suffix)
            except ValueError:
                pass
    path = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "tests", "golden", "model_plans.json")
    with open(path, "w") as f:
        json.dump(out, f, indent=0, sort_keys=True)
    print("%d models -> %s" % (len(out), path))


if __name__ == "__main__":
    main()
