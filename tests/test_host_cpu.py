"""CPU-only tests of the host-side logic of the data-parallel path: the gradient-bucket plan computed by the native
host code, and (world_size 2, gloo) that averaging the flat gradient buffer bucket by bucket in plan order
reproduces the reference's Accumulate + Broadcast semantics (mean of the per-rank gradients, src/convnet.cc:407-450)."""
import os
import socket
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def host():
    from convnet_b200 import build, net
    build.build_host()
    net.load_host()
    return net


def test_alexnet_parameter_layout_matches_reference(host):
    sizes = host.model_edge_params("alexnet")
    assert len(sizes) == 19
    # SURVEY.md Appendix B: weights + one shared bias per output channel
    assert sizes[0] == 96 * (147 + 1) and sizes[3] == 256 * (2400 + 1) and sizes[16] == 4096 * (18432 + 1)
    assert sizes[1] == sizes[2] == 0                      # pool / rnorm edges have no parameters
    assert sum(sizes) == 104321000                        # "104.3 M parameters"
    assert host.model_edge_params("lenet") == [48 * 17, 0, 128 * (16 * 48 + 1), 0, 10 * (1152 + 1)]


@pytest.mark.parametrize("model", ["alexnet", "lenet", "c3d", "tiny"])
@pytest.mark.parametrize("bucket", [1, 1 << 16, 8 << 20, 1 << 30])
def test_bucket_plan_partitions_the_flat_buffer(host, model, bucket):
    sizes = host.model_edge_params(model)
    plan, total = host.plan_buckets(sizes, bucket)
    assert total % 128 == 0
    # back-to-front, contiguous, exact cover
    assert plan[0][1] == total and plan[-1][0] == 0
    for (lo, hi, trig), (lo2, hi2, trig2) in zip(plan, plan[1:]):
        assert lo == hi2 and trig > trig2
    for lo, hi, trig in plan:
        assert hi > lo and sizes[trig] > 0
        # a bucket may only be sent once its LOWEST edge (the trigger) has produced its gradient
        off = sum((s + 127) // 128 * 128 for s in sizes[:trig])
        assert off == lo
    weighted = [i for i, s in enumerate(sizes) if s > 0]
    # the FIRST weighted edge always travels alone: its gradient appears last, so only that small exchange is exposed
    if len(weighted) > 1:
        assert plan[-1][2] == weighted[0] and plan[-1][1] == (sizes[weighted[0]] + 127) // 128 * 128
    if bucket == 1 << 30:
        assert len(plan) == min(2, len(weighted))
    if bucket == 1:
        assert len(plan) == sum(1 for s in sizes if s > 0)


def test_default_bucket_plan_of_the_bench(host):
    """bench.py's default (--bucket-mb 128) on AlexNet: three exchanges per step — {fc8, fc7, fc6} as soon as fc6's
    gradient exists, {conv5 ... conv2}, and conv1 alone (DESIGN.md §5)."""
    sizes = host.model_edge_params("alexnet")
    plan, total = host.plan_buckets(sizes, int(128 * (1 << 20) / 4))
    assert [trig for _, _, trig in plan] == [16, 3, 0]         # lowest edge of each bucket: fc6, conv2, conv1
    mb = [round((hi - lo) * 4 / 1e6, 1) for lo, hi, _ in plan]
    assert mb == [385.5, 31.7, 0.1] and total == 104321024


WORKER = r'''
import os, sys, numpy as np, torch, torch.distributed as dist
sys.path.insert(0, sys.argv[1])
from convnet_b200 import net
rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
dist.init_process_group("gloo", rank=rank, world_size=world)
sizes = net.model_edge_params("lenet")
plan, total = net.plan_buckets(sizes, 4096)
g = torch.from_numpy(np.random.RandomState(100 + rank).randn(total).astype(np.float32))
ref = [torch.from_numpy(np.random.RandomState(100 + r).randn(total).astype(np.float32)) for r in range(world)]
for lo, hi, trig in plan:                  # what DataParallelSync::AllReduceAverageAsync does per bucket (ncclAvg)
    dist.all_reduce(g[lo:hi], op=dist.ReduceOp.SUM); g[lo:hi] /= world
want = sum(ref) / world
assert torch.allclose(g, want, atol=1e-6), (g - want).abs().max()
out = [torch.zeros_like(g) for _ in range(world)]
dist.all_gather(out, g)
assert all(torch.equal(o, out[0]) for o in out)      # bit-identical on every rank -> replicas stay in lock-step
dist.barrier(); dist.destroy_process_group()
print("OK", rank)
'''


def test_bucketed_average_world2_gloo(host, tmp_path):
    script = tmp_path / "w.py"
    script.write_text(WORKER)
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    procs = []
    for r in range(2):
        env = dict(os.environ, RANK=str(r), WORLD_SIZE="2", MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
        procs.append(subprocess.Popen([sys.executable, str(script), ROOT], env=env, stdout=subprocess.PIPE,
                                      stderr=subprocess.STDOUT, text=True))
    outs = [p.communicate(timeout=180)[0] for p in procs]
    assert all(p.returncode == 0 for p in procs), outs
    assert all("OK" in o for o in outs)


def test_bench_reference_arm_non_root_ranks_exit_quietly():
    env = dict(os.environ, RANK="1", WORLD_SIZE="2", LOCAL_RANK="1")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--gpus", "2"],
                       env=env, capture_output=True, text=True, timeout=120)
    assert r.returncode == 0 and r.stdout.strip() == ""


def test_cpu_reference_sample_is_fixed_by_the_budget_not_by_the_box(monkeypatch):
    """bench.py's CPU arm times a bounded sample of the step.  Which layers it times follows from the per-step budget (the
    command line) at a NOMINAL cost, never from a calibration of the box: the same command always times the same layers
    (round 1 chose per box and the result moved 5x between runs)."""
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import cpu_reference as cr

    class FakePool(cr.Pool):
        def __init__(self, sec_per_gflop):              # no worker processes
            self.cores, self.kind, self.rate, self.ran = 8, "port", sec_per_gflop, []

        def _run(self, layers, images_per_core=1):
            self.ran.append(layers)
            t = self.rate * cr.flops_per_image(layers) / 1e9 * images_per_core
            return t, t

    full = cr.flops_per_image(None)
    assert abs(full / 1e9 - 11.87) < 0.01                                   # BASELINE.md 2c
    for rate in (1.3, 23.0):                                                # an idle 8-core box / a loaded 128-core one
        big = FakePool(rate)
        v, desc = big.step(budget_s=40.0)                                   # 40 s >= 2.3 s/GFLOP * 11.87 GFLOP: the full step
        assert big.ran == [None] and "all 14 weighted edges" in desc
        assert abs(v - 8 / (rate * full / 1e9)) < 1e-9
        mid = FakePool(rate)
        v, desc = mid.step(budget_s=5.0)
        assert mid.ran == [cr.SAMPLES[1]] and "extrapolated by FLOPs" in desc and "not by box load" in desc
        assert abs(v - 8 / (rate * full / 1e9)) / v < 1e-6                 # extrapolation by FLOPs
        small = FakePool(rate)
        small.step(budget_s=0.5)
        assert small.ran == [cr.SAMPLES[0]]
