"""What the training loop (Net.train) costs per step, measured on the GPU.

AlexNet at batch 128 (bf16 tensor cores, as bench.py runs it), fed by a DataHandler whose chunk holds a seeded data set of
3 x 256 x 256 images in pinned host memory, cropped to 224.  Two arms alternate in rounds, each on a fresh net:

- loop: Net.train with print_after 100 and no validation set.  Its train log gives the host time between consecutive
  prints: 100 steps, each with the loop's metric and cnb_sum launches, ending in the print's copy of the slots.
- bare: get_batch + train_step(want_loss=False), with a torch.cuda.synchronize() after every 100 steps.

The first 100-step window of each arm is warm-up and is left out.  Then Validate's rate on a held-out set of the same
images.  The card's name and power limit are read in the same run.

    python tools/train_loop_probe.py [--rounds 3] [--windows 4] [--out results.json]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def gpu_identity():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.TimeoutExpired):
        return ""


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--windows", type=int, default=4, help="100-step windows per arm and round, the first one warm-up")
    ap.add_argument("--images", type=int, default=1024)
    ap.add_argument("--out")
    a = ap.parse_args()
    import torch
    from convnet_b200 import lib
    from convnet_b200 import net as N
    assert torch.cuda.is_available(), "the probe measures on a GPU"
    lib.set_precision("bf16")
    batch, S, G, P = 128, 256, 224, 100
    g = torch.Generator().manual_seed(7)
    images = torch.randn(a.images, 3, S, S, generator=g).pin_memory()
    labels = torch.randint(0, 1000, (a.images,), generator=g, dtype=torch.int32)
    rates = {"loop": [], "bare": []}
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "alexnet.pbtxt")
        steps = P * a.windows
        with open(path, "w") as f:      # one checkpoint, after the last step (outside every timed window)
            f.write("max_iter: %d print_after: %d save_after: %d\n" % (steps, P, steps) + N.model_text("alexnet"))

        def handler():
            return N.DataHandler(images, labels, batch_size=batch, gpu_image_size=G, translate=True, flip=True,
                                 randomize_gpu=True, seed=3)

        for r in range(a.rounds):
            for arm in (("loop", "bare") if r % 2 == 0 else ("bare", "loop")):
                n, h = N.Net(path, batch, seed=1), handler()
                if arm == "loop":
                    n.train(h, checkpoint_dir=tmp, run_name="r%d" % r)
                    with open(os.path.join(tmp, "r%d_train.log" % r)) as f:
                        secs = [float(line.split()[1]) for line in f]
                else:
                    secs = []
                    torch.cuda.synchronize()
                    for _ in range(a.windows):
                        t0 = time.perf_counter()
                        for _ in range(P):
                            h.get_batch(n)
                            n.train_step(want_loss=False)
                        torch.cuda.synchronize()
                        secs.append(time.perf_counter() - t0)
                rates[arm] += [P * batch / s for s in secs[1:]]
                h.close()
                n.close()
        # Validate over the same data set as a held-out set: images // batch test-mode batches per call
        n, v = N.Net(path, batch, seed=1), N.DataHandler(images, labels, batch_size=batch, gpu_image_size=G)
        n.validate(v)
        torch.cuda.synchronize()
        vr = []
        for _ in range(5):
            t0 = time.perf_counter()
            n.validate(v)
            vr.append((a.images // batch) * batch / (time.perf_counter() - t0))
        v.close()
        n.close()
    summary = lambda x: {"median": round(statistics.median(x), 1), "min": round(min(x), 1), "max": round(max(x), 1),
                         "n": len(x)}
    out = {"gpu": gpu_identity(), "model": "alexnet", "batch": batch, "precision": "bf16", "window_steps": P,
           "loop_images_per_s": summary(rates["loop"]), "bare_images_per_s": summary(rates["bare"]),
           "loop_over_bare": round(statistics.median(rates["loop"]) / statistics.median(rates["bare"]), 4),
           "validate_images_per_s": summary(vr)}
    print(json.dumps(out))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
