"""Time the fused activation epilogues of AlexNet's conv2-conv5 and fc6 in bf16: fprop with bias + ReLU against bias + logistic
in the epilogue, dgrad with the ReLU' mask against sigma', at batch 128 and 256 (convnet_b200_fuse_next_act); and the
stand-alone cnb_logistic / cnb_logistic_deriv passes as achieved HBM bandwidth.

CUDA events around each call, after warm-up, operands staged in bf16 as in training, with a 256 MiB write between launches
so that no operand is served from L2.  Prints the card, its power limit and max SM clock first; then one line per (layer,
batch, op, activation): microseconds (median), and per pass: bytes moved (read + write, 4 bytes each), GB/s.

    python tools/act_probe.py [--calls 20]
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

# AlexNet (the alexnet text in models.cc): input side, Cin, Cout, kernel, stride, padding -> output side
LAYERS = {"conv2": (55, 96, 256, 5, 2, 1), "conv3": (14, 256, 384, 3, 1, 1), "conv4": (14, 768, 384, 3, 1, 1),
          "conv5": (14, 384, 512, 3, 1, 0), "fc6": (1, 512 * 36, 4096, 1, 1, 0)}
ACT = {"relu": 1, "logistic": 2}


def timed(fn, calls, flush, before=None):
    for _ in range(3):
        if before:
            before()
        fn()
    times = []
    for _ in range(calls):
        flush.zero_()
        if before:
            before()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); fn(); b.record()
        torch.cuda.synchronize()
        times.append(a.elapsed_time(b) * 1e3)
    return sorted(times)[len(times) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    args = ap.parse_args()
    L = lib.load()
    flush = torch.empty(64 << 20, dtype=torch.float32, device="cuda")
    props = torch.cuda.get_device_properties(0)
    try:
        smi = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=power.limit,clocks.max.sm",
                              "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        smi = "nvidia-smi unavailable (%s)" % e
    print("device: %s, %d SMs; power limit, max SM clock: %s" % (props.name, props.multi_processor_count, smi))
    lib.set_precision("bf16")
    for name, (S, cin, cout, k, s, p) in LAYERS.items():
        m = (S + 2 * p - k) // s + 1
        d = GetConvDesc(cin, cout, k, k, s, s, p, p)
        for N in (128, 256):
            img = CUDAMatrix(N, S * S * cin, (N, S, S, cin)); img.storage.normal_()
            flt = CUDAMatrix(cout, k * k * cin, (cout, k, k, cin)); flt.storage.normal_(std=0.02)
            out = CUDAMatrix(N, m * m * cout, (N, m, m, cout)); out.storage.normal_()
            dimg = CUDAMatrix(N, S * S * cin, (N, S, S, cin))
            state = torch.rand(dimg.storage.numel(), device="cuda")
            bias = torch.randn(cout, device="cuda")
            for t in (img, flt, out):
                L.convnet_b200_bf16_stage(t.ptr, t.storage.numel())
            for act, code in ACT.items():
                up = timed(lambda: cg.convUp(img, flt, out, d, 0), args.calls, flush,
                           lambda: (L.convnet_b200_fuse_next_act(bias.data_ptr(), code, None),
                                    L.convnet_b200_bf16_ensure(img.ptr, img.storage.numel())))
                path_up = lib.last_conv_path()
                down = timed(lambda: cg.convDown(out, flt, dimg, d, 0), args.calls, flush,
                             lambda: (L.convnet_b200_fuse_next_act(None, code, state.data_ptr()),
                                      L.convnet_b200_bf16_ensure(out.ptr, out.storage.numel())))
                print("%-5s N=%-3d %-8s fprop %8.1f us (%s)   dgrad %8.1f us (%s)"
                      % (name, N, act, up, path_up, down, lib.last_conv_path()))
            L.convnet_b200_bf16_invalidate(None)
    for n in (128 * 55 * 55 * 96, 128 * 13 * 13 * 768):
        x = torch.randn(n, device="cuda")
        y = torch.rand(n, device="cuda")
        us = timed(lambda: L.cnb_logistic(x.data_ptr(), n), args.calls, flush)
        print("cnb_logistic       n=%-10d %8.1f us  %7.1f GB/s (8 bytes per element)" % (n, us, 8.0 * n / us / 1e3))
        us = timed(lambda: L.cnb_logistic_deriv(x.data_ptr(), y.data_ptr(), n), args.calls, flush)
        print("cnb_logistic_deriv n=%-10d %8.1f us  %7.1f GB/s (12 bytes per element)" % (n, us, 12.0 * n / us / 1e3))


if __name__ == "__main__":
    main()
