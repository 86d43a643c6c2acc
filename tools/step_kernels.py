"""The kernels of the first training steps of a net, per step and per stream in issue order, recorded with torch.profiler:
the host's launch sequence, for comparing two versions of the host code.  Kernels on one stream run in the order they
were issued; the interleaving of different streams in time is not deterministic and is not recorded.

The input is filled as bench.py fills it (N(0,1) pixels and uniform labels from generator seed 1234, parameters from
seed 1234).  Steps 0-2 are recorded because the first step learns which conv calls run in bf16 and emits differently
from the later ones.  --eval adds one test-mode pass, fprop(False) then bprop(), after them (the grad check's path).
Writes {"model", "precision", "steps": [{"name", "launches", "streams": {stream: ["kernel <<<grid, block>>>", ...]}}]}.
One profiler session per process: a second session in the same process can miss kernel records.

    python tools/step_kernels.py --model alexnet [--batch 128] [--precision bf16] [--eval] --out kernels.json
"""
import argparse
import json
import os
import sys
import tempfile

import torch
from torch.profiler import ProfilerActivity, profile, record_function

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from convnet_b200 import lib  # noqa: E402
from convnet_b200.net import Net  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="alexnet")
    ap.add_argument("--batch", type=int, default=128)
    ap.add_argument("--precision", default="bf16", choices=["fp32", "tf32", "bf16"])
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--eval", action="store_true", help="then one fprop(False); bprop() pass")
    ap.add_argument("--out", required=True)
    args = ap.parse_args()

    L = lib.load()
    lib.set_precision(args.precision)
    net = Net(args.model, args.batch, seed=1234)
    g = torch.Generator(device="cuda").manual_seed(1234)
    net.input_tensor().normal_(generator=g)
    net.labels_tensor().copy_(torch.randint(0, net.num_classes, (args.batch,), device="cuda", generator=g, dtype=torch.int32))
    torch.cuda.synchronize()

    passes = [("step%d" % k, lambda: net.train_step(want_loss=False)) for k in range(args.steps)]
    if args.eval:
        passes.append(("eval", lambda: (net.fprop(False), net.bprop())))
    launches = []
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        for name, run in passes:
            L.convnet_b200_reset_launch_count()
            with record_function(name):
                run()
                torch.cuda.synchronize()
            launches.append(int(L.convnet_b200_launch_count()))
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "trace.json")
        prof.export_chrome_trace(path)
        with open(path) as f:
            events = json.load(f)["traceEvents"]
    net.close()

    # a kernel belongs to the pass whose range holds its launch call (matched through the correlation id)
    ranges = [(e["ts"], e["ts"] + e["dur"], e["name"]) for e in events if e.get("cat") == "user_annotation"]
    launch_ts = {e["args"]["correlation"]: e["ts"] for e in events
                 if e.get("cat") in ("cuda_runtime", "cuda_driver") and "correlation" in e.get("args", {})}
    steps = {name: {"name": name, "launches": n, "streams": {}} for (name, _), n in zip(passes, launches)}
    for e in sorted((e for e in events if e.get("cat") == "kernel"), key=lambda e: e["ts"]):
        t = launch_ts.get(e["args"].get("correlation"), e["ts"])
        owner = [name for lo, hi, name in ranges if lo <= t <= hi and name in steps]
        if not owner:
            continue
        a = e["args"]
        desc = "%s <<<%s, %s>>>" % (e["name"], a.get("grid"), a.get("block"))
        steps[owner[0]]["streams"].setdefault(str(a.get("stream")), []).append(desc)
    out = {"model": args.model, "precision": args.precision, "batch": args.batch,
           "steps": [steps[name] for name, _ in passes]}
    with open(args.out, "w") as f:
        json.dump(out, f, indent=1)
    print("%s %s: %s" % (args.model, args.precision, ", ".join(
        "%s %d launches / %d kernels on %d streams" % (s["name"], s["launches"], sum(map(len, s["streams"].values())),
                                                         len(s["streams"])) for s in out["steps"])))


if __name__ == "__main__":
    main()
