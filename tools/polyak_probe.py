#!/usr/bin/env python3
"""Kernel time and achieved (algorithmic) TB/s of cnb_polyak_average at AlexNet's parameter count (104 M floats) for
k = 2, 4 and 8 queue slots, and the wall time of Net.save / Net.load for alexnet and alexnet+rmsprop.

The kernel reads k slots and writes one buffer: (k + 1) * 4 bytes per float.  Each time is the median of 20 calls timed
with CUDA events.  save / load are host- and disk-bound (a device-to-host copy and a write of ~0.8 GB, or a read and a
host-to-device copy): their times are wall-clock around the call, on the machine's temporary directory.  The card's name
and power limit are read in the same run.

    python tools/polyak_probe.py [--out results.json]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from convnet_b200 import lib  # noqa: E402
from convnet_b200.net import Net  # noqa: E402

ALEXNET_FLOATS = 104 * 1000 * 1000


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name(0)


def kernel(k, n=ALEXNET_FLOATS, iters=20):
    L = lib.load()
    queue = torch.randn(k * n, device="cuda")
    out = torch.empty(n, device="cuda")
    call = lambda: L.cnb_polyak_average(out.data_ptr(), queue.data_ptr(), n, n, k)   # noqa: E731
    call()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); call(); b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b) * 1e-3)
    t = statistics.median(ts)
    del queue, out
    torch.cuda.empty_cache()
    return {"k": k, "floats": n, "us": round(t * 1e6, 1), "TB/s": round((k + 1) * 4.0 * n / t / 1e12, 3)}


def save_load(model, batch=128):
    lib.set_precision("bf16")
    net = Net(model, batch, seed=1)
    net.input_tensor().normal_()
    net.labels_tensor().zero_()
    net.train_step(False)
    torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "net.ckpt")
        t0 = time.perf_counter(); net.save(path); t1 = time.perf_counter()
        size = os.path.getsize(path)
        net.load(path); torch.cuda.synchronize(); t2 = time.perf_counter()
    net.close()
    return {"model": model, "MB": round(size / 1e6, 1), "save_s": round(t1 - t0, 3), "load_s": round(t2 - t1, 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "the probe needs a GPU"
    res = {"card": card(), "polyak_average": [kernel(k) for k in (2, 4, 8)],
           "checkpoint": [save_load(m) for m in ("alexnet", "alexnet+rmsprop")]}
    print(json.dumps(res, indent=1))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
