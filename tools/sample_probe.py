"""Times the sampling calls of the updown model's edges at batch 128 on the GPU, fused and unfused, with CUDA events.

Per call: the fused call (its requests armed as ConvNet arms them) and the unfused call followed by the stand-alone
passes it replaces.  Besides the calls updown makes, the up-sampling with a ReLU + dropout destination (the forward
fusion a model file with such a layer gets) is timed at updown's shapes.  Bytes are the algorithm's (every tensor read
and written once per pass, fp32); the rate is set against the H100 SXM's 3.35 TB/s.  The card's name and power limit are read in the same run.  One JSON line per call.

  python tools/sample_probe.py [--batch 128] [--iters 50]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from convnet_b200 import lib  # noqa: E402
from convnet_b200.abi import GetConvDesc  # noqa: E402
from convnet_b200.matrix import CUDAMatrix  # noqa: E402

PEAK = 3.35e12


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def timed(fn, iters):
    for _ in range(3):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters * 1e-3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=128)
    ap.add_argument("--iters", type=int, default=50)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("sample_probe: no GPU")
    L = lib.load()
    lib.set_precision("bf16")
    N, who = args.batch, card()
    # (edge, small side, channels): updown's two DOWNSAMPLE and two UPSAMPLE edges, factor 2.  `in_updown`: updown makes
    # this call (its sampled layers are LINEAR; the ReLU + dropout rows are those of a ReLU layer with dropout after an
    # UPSAMPLE); `new`: the fused form is new with the sampling edges (the ReLU' mask and the bf16 twin of the average
    # undo were already fused)
    cases = [("down1", 64, 64), ("down2", 32, 128), ("up3", 32, 256), ("up4", 64, 128)]
    for name, s, C in cases:
        small = CUDAMatrix(N, s * s * C, (N, s, s, C)); big = CUDAMatrix(N, 4 * s * s * C, (N, 2 * s, 2 * s, C))
        small.storage.normal_(); big.storage.normal_()
        state_small = torch.relu(torch.randn_like(small.storage)); state_big = torch.relu(torch.randn_like(big.storage))
        gb = torch.zeros(C, device="cuda")
        d = GetConvDesc(C, C, 2, 2, 2, 2, 0, 0)
        ns, nb = small.storage.numel(), big.storage.numel()
        out = []
        if name.startswith("down"):
            def fprop_fused():
                L.convnet_b200_emit_bf16_next()
                L.DownSampleGemm(big.p_mat, small.p_mat, big.p_shape4d, small.p_shape4d, 2)

            def fprop_plain():
                L.DownSampleGemm(big.p_mat, small.p_mat, big.p_shape4d, small.p_shape4d, 2)
                L.convnet_b200_bf16_stage(small.storage.data_ptr(), ns)
            out.append(("fprop DownSampleGemm + bf16 twin", True, False, fprop_fused, fprop_plain, 4 * (nb + ns) + 2 * ns))

            def dgrad_fused():
                L.convnet_b200_fuse_next_act(None, 1, state_big.data_ptr())
                L.convnet_b200_emit_bf16_next()
                L.AvgPoolUndoGemm(small.p_mat, big.p_mat, small.p_shape4d, big.p_shape4d, d, 0.0)

            def dgrad_plain():
                L.AvgPoolUndoGemm(small.p_mat, big.p_mat, small.p_shape4d, big.p_shape4d, d, 0.0)
                L.cnb_relu_deriv(big.storage.data_ptr(), state_big.data_ptr(), nb)
                L.convnet_b200_bf16_stage(big.storage.data_ptr(), nb)
            out.append(("dgrad AvgPoolUndoGemm + ReLU' + bf16 twin", True, False, dgrad_fused, dgrad_plain,
                        4 * (ns + 2 * nb) + 2 * nb))
        else:
            def fprop_fused():
                L.convnet_b200_emit_bf16_next()
                L.UpSampleGemm(small.p_mat, big.p_mat, small.p_shape4d, big.p_shape4d, 2, 0.0)

            def fprop_plain():
                L.UpSampleGemm(small.p_mat, big.p_mat, small.p_shape4d, big.p_shape4d, 2, 0.0)
                L.convnet_b200_bf16_stage(big.storage.data_ptr(), nb)
            out.append(("fprop UpSampleGemm + bf16 twin", True, False, fprop_fused, fprop_plain, 4 * (ns + nb) + 2 * nb))

            def relu_fused():
                L.convnet_b200_fuse_next_act(None, 1, None)
                L.convnet_b200_fuse_next_dropout(0.5, 2.0, 17)
                L.convnet_b200_emit_bf16_next()
                L.UpSampleGemm(small.p_mat, big.p_mat, small.p_shape4d, big.p_shape4d, 2, 0.0)

            def relu_plain():
                L.UpSampleGemm(small.p_mat, big.p_mat, small.p_shape4d, big.p_shape4d, 2, 0.0)
                L.cnb_relu(big.storage.data_ptr(), nb)
                L.cnb_dropout(big.storage.data_ptr(), state_big.data_ptr(), nb, 0.5, 2.0, 17)
                L.convnet_b200_bf16_stage(big.storage.data_ptr(), nb)
            out.append(("fprop UpSampleGemm + ReLU + dropout + bf16 twin", False, True, relu_fused, relu_plain,
                        4 * (ns + nb) + 2 * nb))

            def dgrad_fused():
                L.convnet_b200_fuse_next_act(None, 1, state_small.data_ptr())
                L.convnet_b200_fuse_next_bias_grad(gb.data_ptr(), 0.0, 1.0 / N)
                L.convnet_b200_emit_bf16_next()
                L.AvgPoolGemm(big.p_mat, small.p_mat, big.p_shape4d, small.p_shape4d, d, 0.0, 4.0)

            def dgrad_plain():
                L.AvgPoolGemm(big.p_mat, small.p_mat, big.p_shape4d, small.p_shape4d, d, 0.0, 4.0)
                L.cnb_relu_deriv(small.storage.data_ptr(), state_small.data_ptr(), ns)
                L.cnb_channel_bias_grad(small.storage.data_ptr(), gb.data_ptr(), ns // C, C, 0.0, 1.0 / N)
                L.convnet_b200_bf16_stage(small.storage.data_ptr(), ns)
            out.append(("dgrad AvgPoolGemm(f^2) + ReLU' + bias grad + bf16 twin", True, True, dgrad_fused, dgrad_plain,
                        4 * (nb + 2 * ns) + 2 * ns))
        for what, in_updown, new, fused, plain, algo in out:
            tf, tp = timed(fused, args.iters), timed(plain, args.iters)
            print(json.dumps({"edge": name, "call": what, "in_updown": in_updown, "new": new, "batch": N, "card": who,
                              "algo_MB": round(algo / 1e6, 1),
                              "fused_us": round(tf * 1e6, 1), "unfused_us": round(tp * 1e6, 1),
                              "fused_TBps": round(algo / tf / 1e12, 3), "fused_share_of_3.35TBps": round(algo / tf / PEAK, 3),
                              "speedup": round(tp / tf, 2)}), flush=True)


if __name__ == "__main__":
    main()
