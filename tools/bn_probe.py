"""CUDA-event time and achieved bandwidth of the batch-norm kernels at the layer shapes of a "+bn" model.

    python tools/bn_probe.py [--model alexnet+bn] [--batch 128] [--reps 20]

Bytes counted per call (fp32, the per-channel vectors ignored): statistics 2 reads of x (mean, then the variance about
it); apply 1 read of x + 1 write of y; backward 2 reads of (d, x) + 1 write of d.  One JSON line per layer, and the GPU's
name and power limit as nvidia-smi reports them."""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from convnet_b200 import lib  # noqa: E402
from convnet_b200.net import Net  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="alexnet+bn")
    ap.add_argument("--batch", type=int, default=128)
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True).stdout.strip()
    L = lib.load()
    net = Net(a.model, a.batch, seed=1)
    shapes = [(name, net.H.cnb_net_layer_floats(net.h, i) // c, c) for i, name, c, _ in net.bn_layers()]
    net.close()
    print(json.dumps({"gpu": gpu, "model": a.model, "batch": a.batch}))
    for name, n, C in shapes:
        x = torch.randn(C * n, device="cuda")
        y, d = torch.empty_like(x), torch.randn_like(x)
        v = torch.rand(6 * C, device="cuda") + 0.5
        gamma, beta, mu, sg, gg, gb = (v[k * C:(k + 1) * C] for k in range(6))
        calls = {
            "stats": (lambda: L.cnb_bn_stats(x.data_ptr(), n, C, 1e-5, 0.98, mu.data_ptr(), sg.data_ptr(), None, None), 8),
            "apply": (lambda: L.cnb_bn_apply(x.data_ptr(), y.data_ptr(), n, C, gamma.data_ptr(), beta.data_ptr(), mu.data_ptr(),
                                             sg.data_ptr(), 1), 8),
            "backward": (lambda: L.cnb_bn_backward(d.data_ptr(), x.data_ptr(), n, C, gamma.data_ptr(), mu.data_ptr(),
                                                   sg.data_ptr(), 1, gg.data_ptr(), gb.data_ptr()), 20),
        }
        row = {"layer": name, "n": n, "channels": C, "MB": round(4.0 * n * C / 1e6, 1)}
        for k, (fn, bytes_per_el) in calls.items():
            for _ in range(3):
                fn()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.reps):
                fn()
            e1.record()
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / a.reps
            row[k + "_us"] = round(ms * 1e3, 1)
            row[k + "_TBs"] = round(bytes_per_el * n * C / (ms * 1e-3) / 1e12, 2)
        print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
