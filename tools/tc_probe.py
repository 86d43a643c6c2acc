#!/usr/bin/env python3
"""Debug aid: run conv fprop/dgrad/wgrad in TF32 (tensor-core) mode and compare with the FP32 CUDA-core
path of the same library on the GPU (fast; the oracle-based parity lives in tests/)."""
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from convnet_b200 import conv_gemm as cg  # noqa: E402
from convnet_b200 import lib  # noqa: E402
from convnet_b200.abi import GetConvDesc, num_modules  # noqa: E402
from convnet_b200.matrix import CUDAMatrix  # noqa: E402

SHAPES = {
    "tiny": (32, 4, 4, 32, 32, 1, 1, 1, 1, 0, 0),
    "tiny3x3": (32, 6, 6, 32, 32, 3, 3, 1, 1, 1, 1),
    "n128": (128, 6, 6, 64, 64, 3, 3, 1, 1, 1, 1),
    "c40": (64, 5, 5, 40, 24, 3, 3, 1, 1, 1, 1),
    "stride2": (64, 12, 12, 32, 64, 3, 3, 2, 2, 1, 1),
    "conv3_b32": (32, 14, 14, 256, 384, 3, 3, 1, 1, 1, 1),
    "conv3": (256, 14, 14, 256, 384, 3, 3, 1, 1, 1, 1),
    "conv4": (256, 14, 14, 768, 384, 3, 3, 1, 1, 1, 1),
    "conv5": (256, 14, 14, 384, 512, 3, 3, 1, 1, 0, 0),
    "conv2": (256, 55, 55, 96, 256, 5, 5, 2, 2, 1, 1),
    "fc7": (256, 1, 1, 4096, 4096, 1, 1, 1, 1, 0, 0),
    "fc6": (128, 1, 1, 18432, 4096, 1, 1, 1, 1, 0, 0),
    "conv1_small": (32, 21, 21, 3, 16, 7, 7, 2, 2, 1, 1),
    "conv1": (128, 224, 224, 3, 96, 7, 7, 2, 2, 1, 1),
    "mnist1": (100, 28, 28, 1, 48, 4, 4, 1, 1, 0, 0),
}


def diff(a, b):
    a, b = a.double(), b.double()
    return ((a - b).abs().max() / (a + b).abs().mean().clamp_min(1e-30)).item()


def timed(fn, iters):
    fn(); torch.cuda.synchronize()
    if iters > 1:                       # warm the clocks up: ~30 ms of the same kernel before the timed loop
        t0 = time.time()
        while time.time() - t0 < 0.03:
            for _ in range(5):
                fn()
            torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def main():
    names = sys.argv[1:] or list(SHAPES)
    iters = int(os.environ.get("ITERS", "20"))
    for name in names:
        N, W, H, Cin, Cout, ky, kx, sy, sx, py, px = SHAPES[name]
        modY, modX = num_modules(H, ky, sy, py), num_modules(W, kx, sx, px)
        d = GetConvDesc(Cin, Cout, ky, kx, sy, sx, py, px)
        ish, fsh, tsh = (N, W, H, Cin), (Cout, kx, ky, Cin), (N, modX, modY, Cout)
        g = torch.Generator(device="cuda").manual_seed(0)
        x = CUDAMatrix(N, W * H * Cin, ish); x.storage.normal_(generator=g)
        w = CUDAMatrix(Cout, kx * ky * Cin, fsh); w.storage.normal_(generator=g).mul_(1 / np.sqrt(kx * ky * Cin))
        dv = CUDAMatrix(N, modX * modY * Cout, tsh); dv.storage.normal_(generator=g)
        flops = 2.0 * N * modX * modY * Cout * kx * ky * Cin
        res = {}
        fast = os.environ.get("MODE", "tf32")
        ref_iters = 1 if os.environ.get("FAST_REF") else iters
        for mode in ("fp32", fast):
            lib.set_precision(mode)
            up = CUDAMatrix(N, modX * modY * Cout, tsh); dn = CUDAMatrix(N, W * H * Cin, ish); dw = CUDAMatrix(Cout, kx * ky * Cin, fsh)
            up.fill_(float("nan")); dn.fill_(float("nan")); dw.fill_(float("nan"))
            it = ref_iters if mode == "fp32" else iters
            t_up = timed(lambda: cg.convUp(x, w, up, d), it); p_up = lib.last_conv_path()
            t_dn = timed(lambda: cg.convDown(dv, w, dn, d), it); p_dn = lib.last_conv_path()
            t_dw = timed(lambda: cg.convOutp(x, dv, dw, d, 0, 1.0 / N), it); p_dw = lib.last_conv_path()
            res[mode] = (up, dn, dw, (t_up, t_dn, t_dw), (p_up, p_dn, p_dw))
        a, b = res["fp32"], res[fast]
        for i, op in enumerate(("fprop", "dgrad", "wgrad")):
            print("%-10s %-5s %-14s Diff=%.2e  fp32 %8.3f ms (%6.1f TF/s)   fast %8.3f ms (%7.1f TF/s)" % (
                name, op, b[4][i], diff(a[i].storage, b[i].storage), a[3][i], flops / a[3][i] / 1e9,
                b[3][i], flops / b[3][i] / 1e9), flush=True)


def cublas_reference():
    """cuBLAS through torch.matmul on the same box, same warm-up: the practical tensor ceiling next to our numbers."""
    n = 8192
    for dt, name in ((torch.bfloat16, "bf16"), (torch.float32, "tf32")):
        torch.backends.cuda.matmul.allow_tf32 = True
        a = torch.randn(n, n, device="cuda", dtype=dt); b = torch.randn(n, n, device="cuda", dtype=dt)
        t = timed(lambda: torch.matmul(a, b), 10)
        print("cublas %s %d^3: %.3f ms (%.1f TF/s)" % (name, n, t, 2.0 * n ** 3 / t / 1e9), flush=True)


if __name__ == "__main__":
    if os.environ.get("CUBLAS_REF"):
        cublas_reference()
    main()
