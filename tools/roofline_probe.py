#!/usr/bin/env python3
"""Run bench.py's conv roofline leg alone (conv4 fprop, batch 256, operands staged in bf16 mode) — the target of the
`ncu --set full -k regex:tc_conv_kernel --launch-skip 19 --launch-count 1` capture."""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from convnet_b200 import lib  # noqa: E402

lib.load(); lib.set_precision(os.environ.get("PRECISION", "bf16"))
peaks, kind = bench.measured_peaks()
print(json.dumps(bench.conv_roofline(torch, lib, peaks, kind)))
