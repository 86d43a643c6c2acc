#!/usr/bin/env python3
"""Run ONE AlexNet training step (batch 128) between cudaProfilerStart/Stop, after two warm-up steps.
For `ncu --profile-from-start off ...` launch lists and full captures."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from convnet_b200 import lib  # noqa: E402
from convnet_b200.net import Net  # noqa: E402

batch = int(os.environ.get("BATCH", "128"))
lib.load(); lib.set_precision(os.environ.get("PRECISION", "tf32"))
n = Net(os.environ.get("MODEL", "alexnet"), batch, seed=1)
n.input_tensor().normal_()
n.labels_tensor().copy_(torch.randint(0, n.num_classes, (batch,), device="cuda", dtype=torch.int32))
for _ in range(2):
    n.train_step(False)
torch.cuda.synchronize()
torch.cuda.profiler.start()
n.train_step(False)
torch.cuda.synchronize()
torch.cuda.profiler.stop()
print("done")
