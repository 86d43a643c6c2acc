"""Time the untied conv ops of lcnet's local3 / local4 at batch 128: fprop (localUp), dgrad (localDown), wgrad (localOutp).

Paths: bf16 tensor cores with staged operands (as in training), tf32 tensor cores, fp32 CUDA cores.  CUDA events around
each call, after warm-up, with a 256 MiB write between launches so that no operand is served from L2 (the weights alone
are 42 / 29 MB in bf16).  Prints one line per (layer, op, path): microseconds (median), algorithmic bytes (weights at the
operand width, input and output / dW in fp32, plus the bf16 copy of the operands the call reads in bf16 mode), TB/s and
TFLOP/s, and the share of the HBM (3.35 TB/s) and dense tensor peak (bf16 989, tf32 494, fp32 67 TFLOP/s) reached.

    python tools/local_probe.py [--calls 20]
"""
import argparse
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from convnet_b200 import conv_gemm as cg  # noqa: E402
from convnet_b200 import lib  # noqa: E402
from convnet_b200.abi import GetConvDesc  # noqa: E402
from convnet_b200.matrix import CUDAMatrix  # noqa: E402

PEAK = {"bf16": 989e12, "tf32": 494e12, "fp32": 67e12}
HBM = 3.35e12
LAYERS = {"local3": (12, 1, 144), "local4": (12, 0, 100)}      # input side, padding, modules; 3x3, 128 -> 128 channels


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    args = ap.parse_args()
    L = lib.load()
    N, C, k = 128, 128, 3
    flush = torch.empty(64 << 20, dtype=torch.float32, device="cuda")
    # the card and its power limit, read in the same process as the timings (a capped card clocks lower)
    props = torch.cuda.get_device_properties(0)
    try:
        smi = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=power.limit,clocks.max.sm",
                              "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        smi = "nvidia-smi unavailable (%s)" % e
    print("device: %s, %d SMs; power limit, max SM clock: %s" % (props.name, props.multi_processor_count, smi))
    for name, (W, p, M) in LAYERS.items():
        m = int(M ** 0.5)
        K = k * k * C
        d = GetConvDesc(C, C, k, k, 1, 1, p, p)
        img = CUDAMatrix(N, W * W * C, (N, W, W, C)); img.storage.normal_()
        flt = CUDAMatrix(C, K * M, (C, k, k, C * M)); flt.storage.normal_(std=0.02)
        out = CUDAMatrix(N, M * C, (N, m, m, C)); out.storage.normal_()
        dimg = CUDAMatrix(N, W * W * C, (N, W, W, C))
        dw = CUDAMatrix(C, K * M, (C, k, k, C * M))
        flops = 2.0 * N * M * C * K
        for mode in ("bf16", "tf32", "fp32"):
            lib.set_precision(mode)
            wsz = 2 if mode == "bf16" else 4
            ops = {
                "fprop": (lambda: cg.localUp(img, flt, out, d, 0), (img, flt),
                          C * K * M * wsz + img.storage.numel() * 4 + out.storage.numel() * 4),
                "dgrad": (lambda: cg.localDown(out, flt, dimg, d, 0), (out, flt),
                          C * K * M * wsz + out.storage.numel() * 4 + dimg.storage.numel() * 4),
                "wgrad": (lambda: cg.localOutp(img, out, dw, d, 0, 1.0), (img, out),
                          img.storage.numel() * 4 + out.storage.numel() * 4 + C * K * M * 4),
            }
            for op, (fn, operands, nbytes) in ops.items():
                if mode == "bf16":                       # operands staged, as the training host keeps them
                    for t in operands:
                        L.convnet_b200_bf16_stage(t.ptr, t.storage.numel())
                    if op != "wgrad":                    # fprop / dgrad read the activation operand as bf16, not fp32
                        nbytes -= operands[0].storage.numel() * 2
                    else:
                        nbytes -= (img.storage.numel() + out.storage.numel()) * 2
                for _ in range(3):
                    fn()
                path = lib.last_conv_path()
                times = []
                for _ in range(args.calls):
                    flush.zero_()
                    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    a.record(); fn(); b.record()
                    torch.cuda.synchronize()
                    times.append(a.elapsed_time(b) * 1e3)
                    if mode == "bf16":                   # re-stage: the flush did not touch them, but keep it exact
                        for t in operands:
                            L.convnet_b200_bf16_ensure(t.ptr, t.storage.numel())
                us = sorted(times)[len(times) // 2]
                tbs, tfl = nbytes / us / 1e6, flops / us / 1e6
                print("%-6s %-5s %-4s path=%-14s %8.1f us  %6.1f MB  %5.2f TB/s (%3.0f%% HBM)  %6.1f TFLOP/s (%3.0f%% peak)"
                      % (name, op, mode, path, us, nbytes / 1e6, tbs, 100 * tbs * 1e12 / HBM, tfl,
                         100 * tfl * 1e12 / PEAK[mode if path != "cuda-core-fp32" else "fp32"]))
                L.convnet_b200_bf16_invalidate(None)


if __name__ == "__main__":
    main()
