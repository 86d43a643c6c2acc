"""Cost of feeding training from an in-memory data set (net.DataHandler), measured on the GPU with CUDA events.

1. The crop kernel: cnb_extract_patches_indexed (crop through a permutation, labels gathered in the same launch) against
   convnet_b200_extract_patches, at AlexNet's 256 -> 224 crop of 3-colour images, batch 128 and 256.  Bytes moved are the
   crop's reads and writes (2 x N x 3 x 224 x 224 floats, plus the index and labels of the indexed kernel).
2. The AlexNet training step at batch 128 (bf16 tensor cores, as bench.py runs it) fed three ways, in alternating
   rounds: by a batch already on the device (the bench's resident arm), by a DataHandler whose chunk holds the whole
   data set, and by a DataHandler with pipeline_loads streaming a pinned data set four times its chunk.

    python tools/dataset_probe.py [--out results.json] [--steps 30] [--rounds 3]

The results are printed as JSON, and also written to --out when it is given.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def gpu_identity():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.TimeoutExpired):
        q = ""
    return q


def time_ms(torch, fn, iters):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def kernel_arms(torch, lib, batch, chunk_images=1024, iters=200, rounds=5):
    from convnet_b200.matrix import CUDAMatrix
    L = lib.load()
    C, S, G = 3, 256, 224
    g = torch.Generator(device="cuda").manual_seed(batch)
    chunk = torch.randn(chunk_images, C, S, S, device="cuda", generator=g)
    labels = torch.randint(0, 1000, (chunk_images,), device="cuda", dtype=torch.int32, generator=g)
    index = torch.randperm(chunk_images, device="cuda", generator=g)[:batch].to(torch.int32)
    wo = torch.randint(0, S - G + 1, (batch,), device="cuda", generator=g).float()
    ho = torch.randint(0, S - G + 1, (batch,), device="cuda", generator=g).float()
    fl = torch.rand(batch, device="cuda", generator=g)
    out_a, out_b = torch.empty(batch * C * G * G, device="cuda"), torch.empty(batch * C * G * G, device="cuda")
    lab = torch.empty(batch, dtype=torch.int32, device="cuda")
    first = chunk[:batch]                                     # extract_patches reads images [0, batch) of the chunk
    m = lambda t, r, c: CUDAMatrix(r, c, storage=t.reshape(-1))
    img, o, mw, mh, mf = m(first, C * S * S, batch), m(out_a, batch, C * G * G), m(wo, 1, batch), m(ho, 1, batch), m(fl, 1, batch)
    plain = lambda: L.convnet_b200_extract_patches(img.p_mat, o.p_mat, mw.p_mat, mh.p_mat, mf.p_mat, S, S, G, G)
    indexed = lambda: L.cnb_extract_patches_indexed(chunk.data_ptr(), out_b.data_ptr(), index.data_ptr(), wo.data_ptr(),
                                                    ho.data_ptr(), fl.data_ptr(), batch, C, S, S, G, G, labels.data_ptr(),
                                                    lab.data_ptr(), None, None, 0)
    assert plain() == 0 and indexed() == 0
    torch.cuda.synchronize()
    want = chunk[index.long()].contiguous()                   # the indexed crop is extract_patches on the permuted chunk
    img2 = m(want, C * S * S, batch)
    assert L.convnet_b200_extract_patches(img2.p_mat, o.p_mat, mw.p_mat, mh.p_mat, mf.p_mat, S, S, G, G) == 0
    torch.cuda.synchronize()
    assert torch.equal(out_a, out_b) and torch.equal(lab, labels[index.long()])
    for _ in range(20):
        plain(); indexed()
    t = {"extract_patches": [], "indexed": []}
    for _ in range(rounds):                                   # alternate the two kernels
        t["extract_patches"].append(time_ms(torch, plain, iters))
        t["indexed"].append(time_ms(torch, indexed, iters))
    crop_bytes = 2 * batch * C * G * G * 4
    res = {}
    for k, v in t.items():
        ms = statistics.median(v)
        extra = 3 * batch * 4 + (2 * batch * 4 if k == "indexed" else 0)   # offsets, mirror bits; index and labels
        res[k] = {"median_us": round(ms * 1e3, 2), "spread_us": round((max(v) - min(v)) * 1e3, 2),
                  "GB_per_s": round((crop_bytes + extra) / (ms * 1e-3) / 1e9, 1)}
    return res


def step_arms(torch, net, steps, rounds, batch=128):
    C, S, G = 3, 256, 224
    chunk = 256
    n = net.Net("alexnet", batch, seed=1)
    g = torch.Generator().manual_seed(7)
    images = torch.empty(4 * chunk, C, S, S).pin_memory()
    images.normal_(generator=g)
    labels = torch.randint(0, 1000, (4 * chunk,), generator=g, dtype=torch.int32)
    resident = net.DataHandler(images[:chunk], labels[:chunk], batch_size=batch, gpu_image_size=G, translate=True, flip=True,
                               randomize_gpu=True, seed=1)
    streamed = net.DataHandler(images, labels, batch_size=batch, chunk_size=chunk, gpu_image_size=G, translate=True,
                               flip=True, randomize_gpu=True, pipeline_loads=True, seed=1)
    x = n.input_tensor()
    x.copy_(torch.randn(x.numel(), device="cuda"))
    n.labels_tensor().copy_(torch.randint(0, 1000, (batch,), device="cuda", dtype=torch.int32))
    arms = {"device_tensor": lambda: n.train_step(want_loss=False),
            "handler_resident": lambda: (resident.get_batch(n), n.train_step(want_loss=False)),
            "handler_pipelined_4x": lambda: (streamed.get_batch(n), n.train_step(want_loss=False))}
    for fn in arms.values():                                  # warm every path, and let the stream cycle its chunks
        for _ in range(10):
            fn()
    t = {k: [] for k in arms}
    for _ in range(rounds):
        for k, fn in arms.items():
            t[k].append(time_ms(torch, fn, steps))
    resident.close(); streamed.close(); n.close()
    return {k: {"median_ms": round(statistics.median(v), 3), "spread_ms": round(max(v) - min(v), 3)} for k, v in t.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="also write the JSON results to this file")
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("dataset_probe: no GPU (a CPU run measures nothing)")
    from convnet_b200 import lib, net
    lib.set_precision("bf16")                                 # the bench's default arithmetic
    res = {"gpu": gpu_identity() or torch.cuda.get_device_name(),
           "kernel_256_to_224": {str(b): kernel_arms(torch, lib, b) for b in (128, 256)},
           "alexnet_step_batch128": step_arms(torch, net, args.steps, args.rounds)}
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
