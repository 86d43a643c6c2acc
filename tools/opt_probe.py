"""CUDA-event time and achieved bandwidth of the multi-tensor optimizer update (cnb_opt_update_multi) per rule, on the
tensors of a model's gradient buckets.

    python tools/opt_probe.py [--model alexnet] [--reps 20] [--bucket-floats 8388608]

Every bucket of the model's all-reduce plan (the unit of the eager update) is timed as one call with all its tensors on
one rule: SGD, Adagrad, RMSProp.  No norm rules and no staged bf16 copies (the plain model's update).  Bytes counted per
element: SGD reads w, h, g and writes w, h (20 B); the adaptive rules also read and write the state (28 B).  One JSON
line per bucket and rule, after a line with the GPU's name and power limit as nvidia-smi reports them."""
import argparse
import ctypes as ct
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
from convnet_b200 import lib  # noqa: E402
from convnet_b200.net import Net, plan_buckets  # noqa: E402
from test_gpu_adaptive_optimizer import CnbOptTensor, CnbOptTensorEx  # noqa: E402

RULES = {"sgd": (0, 0.0, 20), "adagrad": (1, 1.0, 28), "rmsprop": (2, 0.9, 28)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="alexnet")
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--bucket-floats", type=int, default=8 << 20)
    a = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True).stdout.strip()
    L = lib.load()
    net = Net(a.model, 1, seed=1)
    edges = net.edges()
    couts = [net.H.cnb_net_layer_channels(net.h, i + 1) for i in range(len(edges))]
    net.close()
    buckets, _ = plan_buckets([e[3] for e in edges], a.bucket_floats)
    offsets = [e[2] for e in edges]
    print(json.dumps({"gpu": gpu, "model": a.model, "reps": a.reps}))
    for lo, hi, _ in buckets:
        members = [i for i, e in enumerate(edges) if e[3] and lo <= offsets[i] < hi]
        sizes = []
        for i in members:
            sizes += [edges[i][3] - couts[i], couts[i]]          # weights, bias (every weighted edge of the model has one)
        n_total = sum(sizes)
        bufs = [[torch.randn(n, device="cuda") * 0.01 for _ in range(4)] for n in sizes]
        for b in bufs:
            b[3].abs_().add_(1.0)                                # a positive state
        row = {"edges": [edges[i][0] for i in members], "tensors": len(sizes), "Mfloats": round(n_total / 1e6, 2)}
        for name, (rule, param, bytes_per_el) in RULES.items():
            arr = (CnbOptTensorEx * len(sizes))(*[
                CnbOptTensorEx(CnbOptTensor(w.data_ptr(), h.data_ptr(), g.data_ptr(), w.numel(), 1e-6, 0.9, 0.0, 0.0, 1, 0, 0.0),
                               rule, 0, s.data_ptr(), param, 1.0) for w, h, g, s in bufs])
            call = (lambda arr=arr: L.cnb_opt_update_multi(arr, len(sizes)))
            for _ in range(3):
                call()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.reps):
                call()
            e1.record()
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / a.reps
            row[name + "_us"] = round(ms * 1e3, 1)
            row[name + "_TBs"] = round(bytes_per_el * n_total / (ms * 1e-3) / 1e12, 2)
        print(json.dumps(row), flush=True)
        del bufs
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
