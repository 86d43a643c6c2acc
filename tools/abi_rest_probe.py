#!/usr/bin/env python3
"""Kernel time and achieved (algorithmic) GB/s of the R-operators, within-map normalisation, RGB -> YUV and convInnerpGemm
at AlexNet's hidden1 shapes (hidden1_maxpool: 110 x 110 x 96 -> 55 x 55, 3 x 3 stride 2 pad 1; hidden1_rnorm: 55 x 55 x
96), batch 128 and 256, beside the reference's own CUDA kernels on the same inputs (oracle/_ref, when built).

Each time is the median of 20 single calls timed with CUDA events, the L2 cache flushed before each.  Bytes are what the
algorithm must move (every operand read once, every output written once), computed from the shape; GB/s is set against
the H100 SXM data-sheet 3.35 TB/s.  The card's name and power limit are read in the same run.

    python tools/abi_rest_probe.py
"""
import ctypes as ct
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from convnet_b200 import conv_gemm as cg, lib                    # noqa: E402
from convnet_b200.abi import GetConvDesc                          # noqa: E402
from convnet_b200.conv_gemm import Binding                        # noqa: E402
from convnet_b200.lib import SIGNATURES                           # noqa: E402
from convnet_b200.matrix import CUDAMatrix                        # noqa: E402

PEAK = 3.35e12
flush = None


def timed(fn, iters=20):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        flush.zero_()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); fn(); b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b) * 1e-3)
    return statistics.median(ts)


def ref_binding():
    gemm = os.path.join(ROOT, "oracle", "_ref", "libcudamat_conv_gemm_ref.so")
    conv = os.path.join(ROOT, "oracle", "_ref", "libcudamat_conv_ref.so")
    if not (os.path.exists(gemm) and os.path.exists(conv)):
        return None
    libs = {}
    for path, names in ((gemm, ["MaxPoolRpropGemm", "ResponseNormCrossMapRpropGemm", "convInnerpGemm"]),
                        (conv, ["ResponseNorm", "ResponseNormUndo", "ContrastNorm", "ContrastNormUndo", "RGBToYUV"])):
        h = ct.CDLL(path, mode=ct.RTLD_LOCAL)
        for n in names:
            getattr(h, n).argtypes = SIGNATURES[n]
            getattr(h, n).restype = None
            libs[n] = getattr(h, n)
        if path == gemm:
            h.cublasInit.restype = ct.c_int
            assert h.cublasInit() == 0

    class Lib:
        def __getattr__(self, n):
            return libs[n]
    return Binding(lambda: Lib(), "gemm")


def rnd(r, c, s4):
    m = CUDAMatrix(r, c, s4)
    m.storage.normal_()
    return m


def main():
    global flush
    assert torch.cuda.is_available(), "needs a GPU"
    lib.load()
    lib.set_precision("fp32")
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    print("device: %s | nvidia-smi: %s" % (torch.cuda.get_device_name(0), q[0] if q else "n/a"))
    ref = ref_binding()
    print("%-26s %5s %10s %9s %8s %7s %10s" % ("op", "batch", "time us", "MB", "GB/s", "of peak", "ref us"))
    for N in (128, 256):
        W, C, S = 110, 96, 55
        pd = GetConvDesc(C, C, 3, 3, 2, 2, 1, 1)
        ish, psh = (N, W, W, C), (N, S, S, C)
        im, rim = rnd(N, W * W * C, ish), rnd(N, W * W * C, ish)
        mx, pt, pt2 = CUDAMatrix(N, S * S * C, psh), CUDAMatrix(N, S * S * C, psh), CUDAMatrix(N, S * S * C, psh)
        cg.MaxPool(im, mx, pd)
        x, r, y, y2 = rnd(N, S * S * C, psh), rnd(N, S * S * C, psh), CUDAMatrix(N, S * S * C, psh), CUDAMatrix(N, S * S * C, psh)
        dn, tg, og, du = CUDAMatrix(N, S * S * C, psh), CUDAMatrix(N, S * S * C, psh), rnd(N, S * S * C, psh), CUDAMatrix(N, S * S * C, psh)
        acts = CUDAMatrix(N, S * S * C, psh)
        rgb, yuv = rnd(N, 224 * 224 * 3, (N, 224, 224, 3)), CUDAMatrix(N, 224 * 224 * 3, (N, 224, 224, 3))
        ip, ip2 = CUDAMatrix(1, 9, (1, 3, 3, 1)), CUDAMatrix(1, 9, (1, 3, 3, 1))
        cg.ResponseNorm(x, dn, tg, C, 5, 1e-4, 0.75)
        n_in, n_out, n_map = N * W * W * C, N * S * S * C, N * S * S * C
        ops = [
            ("MaxPoolRprop", lambda b: b.MaxPoolRprop(im, rim, mx, pt if b is cg else pt2, pd), 4 * (2 * n_in + 2 * n_out)),
            ("ResponseNormCrossMapRprop", lambda b: b.ResponseNormCrossMapRprop(x, r, y if b is cg else y2, 5, 1e-4, 0.75, False),
             4 * 3 * n_map),
            ("convInnerp", lambda b: b.convInnerp(im, mx, ip if b is cg else ip2, pd), 4 * (n_in + n_out)),
            ("ResponseNorm", lambda b: b.ResponseNorm(x, dn, tg if b is cg else y2, C, 5, 1e-4, 0.75), 4 * 3 * n_map),
            ("ContrastNorm", lambda b: b.ContrastNorm(x, r, dn, tg if b is cg else y2, C, 5, 1e-4, 0.75), 4 * 4 * n_map),
            ("ResponseNormUndo", lambda b: b.ResponseNormUndo(og, dn, x, tg if b is cg else acts, du if b is cg else y2, C, 5,
                                                              1e-4, 0.75), 4 * 5 * n_map),
            ("RGBToYUV", lambda b: b.RGBToYUV(rgb, yuv), 4 * 2 * N * 224 * 224 * 3),
        ]
        for name, call, nbytes in ops:
            t = timed(lambda: call(cg))
            if ref is not None:
                if name == "ResponseNormUndo":      # the reference overwrites acts: give it a fresh copy every call
                    tr = timed(lambda: (acts.storage.copy_(tg.storage), call(ref))) - timed(lambda: acts.storage.copy_(tg.storage))
                else:
                    tr = timed(lambda: call(ref))
                rs = "%10.1f" % (tr * 1e6)
            else:
                rs = "%10s" % "n/a"
            print("%-26s %5d %10.1f %9.1f %8.0f %6.1f%% %s" % (name, N, t * 1e6, nbytes / 1e6, nbytes / t / 1e9,
                                                           100 * nbytes / t / PEAK, rs))
        del im, rim, mx, pt, pt2, x, r, y, y2, dn, tg, og, du, acts, rgb, yuv
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
