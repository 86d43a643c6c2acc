#!/usr/bin/env python3
"""Write rate of the two ways a conv epilogue can drain its output tiles on an H100 (tools/store_probe.cu).

    python tools/store_probe.py            ITERS=20

One CTA per SM with 227 KiB of shared memory, tiles of 128 rows x BN fp32 columns (512 bytes per column), laid out over a
buffer of conv1's output size (595 MB at batch 128: 96 planes of 128 x 110 x 110 floats; at BN 128, 128 planes of the
same total).  Rates, GB/s of output written, median of ITERS launches, each after a 256 MiB write that evicts L2:
  (a) 1, 3 and 7 warps writing 16-byte st.global, as the conv kernel's store warps do;
  (a') the same 3 or 7 warps fed through one staging tile by eight more warps and an mbarrier hand-off, as the conv
       kernel's consumers feed them, without the MMAs;
  (b) one 2-D tensor store per tile (box {128, BN}, no swizzle) from 1 or 2 staging slots, each slot rewritten in
      place by 3 or 7 warps before its store;
  (c) torch's zero_ of the same buffer.
The kernel is compiled into a temporary directory.
"""
import ctypes
import os
import subprocess
import sys
import tempfile

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
BYTES = 128 * 110 * 110 * 96 * 4


def build(tmp):
    so = os.path.join(tmp, "store_probe.so")
    subprocess.run([NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-shared",
                    "-Xcompiler", "-fPIC", "-o", so, os.path.join(HERE, "store_probe.cu")], check=True)
    return ctypes.CDLL(so)


def timed(fn, iters, flush):
    fn(); torch.cuda.synchronize()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(iters)]
    for a, b in ev:
        flush.zero_()
        a.record(); fn(); b.record()
    torch.cuda.synchronize()
    ts = sorted(a.elapsed_time(b) for a, b in ev)
    return ts[len(ts) // 2]


def main():
    if not torch.cuda.is_available():
        sys.exit("store_probe: no CUDA device")
    iters = int(os.environ.get("ITERS", "20"))
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print("device: %s (%d SMs) | nvidia-smi name, power limit, max SM clock, SM clock: %s" % (
        torch.cuda.get_device_name(), torch.cuda.get_device_properties(0).multi_processor_count, smi), flush=True)
    with tempfile.TemporaryDirectory() as tmp:
        lib = build(tmp)
        lib.store_probe_run.argtypes = [ctypes.c_void_p, ctypes.c_longlong, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                        ctypes.c_int, ctypes.c_int, ctypes.c_void_p]
        flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
        buf = torch.empty(BYTES // 4, dtype=torch.float32, device="cuda")
        stream = torch.cuda.current_stream().cuda_stream
        for bn in (96, 128):
            plane = BYTES // 4 // bn
            plane -= plane % 128
            nbytes = plane * bn * 4

            def run(mode, warps, slots):
                def fn():
                    r = lib.store_probe_run(buf.data_ptr(), plane, bn, bn, mode, warps, slots, stream)
                    if r:
                        raise RuntimeError("store_probe_run failed (%d)" % r)
                return fn

            rows = [("(a) st.global, %d warp%s" % (w, "s" if w > 1 else ""), run(0, w, 1)) for w in (1, 3, 7)]
            rows += [("(a') st.global behind hand-off, %d warps" % w, run(2, w, 1)) for w in (3, 7)]
            for slots in (1, 2):
                for warps in (3, 7):
                    rows.append(("(b) tensor store, %d slot%s, %d warps" % (slots, "s" if slots > 1 else "", warps),
                                 run(1, warps, slots)))
            view = buf[:nbytes // 4]
            rows.append(("(c) torch zero_", lambda: view.zero_()))
            res = {}
            for name, fn in rows:
                ms = timed(fn, iters, flush)
                res[name] = nbytes / ms / 1e6
                print("BN %3d  %-38s %8.1f us  %6.0f GB/s" % (bn, name, ms * 1e3, res[name]), flush=True)
            best_b2 = max(v for k, v in res.items() if k.startswith("(b)") and "2 slots" in k)
            print("BN %3d  (b) 2 slots / (a) 7 warps: %.2fx" % (bn, best_b2 / res["(a) st.global, 7 warps"]), flush=True)
    smi = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    print("SM clock after the runs: %s" % smi, flush=True)


if __name__ == "__main__":
    main()
