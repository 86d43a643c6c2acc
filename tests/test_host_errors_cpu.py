"""CPU-only: the host library has one way to fail.  Its code throws (nothing exits or aborts), one CUDA_CHECK and one
NCCL_CHECK turn a failed call into a DeviceError, and the C API reports every exception through Guard alone; Python
raises ValueError with the host's reason for a refusal and RuntimeError for a failed device call."""
import os
import re
import subprocess
import sys
import textwrap

import pytest

from convnet_b200 import net as N

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOST = os.path.join(ROOT, "convnet_b200", "host")


def _sources():
    return {f: open(os.path.join(HOST, f)).read() for f in sorted(os.listdir(HOST)) if f.endswith((".cc", ".h"))}


def test_nothing_in_the_host_library_ends_the_process():
    hits = ["%s:%d" % (f, text[:m.start()].count("\n") + 1) for f, text in _sources().items()
            for m in re.finditer(r"\b(exit|abort)\(", text)]
    assert hits == []


def test_one_definition_of_each_check_macro():
    defined = sorted(m.group(1) for text in _sources().values()
                     for m in re.finditer(r"#define\s+(\w*(?:CUDA|NCCL)_CHECK)\b", text))
    assert defined == ["CUDA_CHECK", "NCCL_CHECK"]


def test_guard_is_the_only_try_in_the_c_api():
    text = _sources()["capi.cc"]
    guard = re.search(r"static int Guard\(F f\) \{\n(.*?)\n\}\n", text, re.S)
    assert guard
    tries = [m.start() for m in re.finditer(r"\btry\b", text)]
    assert len(tries) == 1 and guard.start(1) <= tries[0] < guard.end(1)


def run(code):
    """`code` in a fresh interpreter with the package importable; its stdout (a regression to exit() fails the test
    instead of ending pytest)"""
    r = subprocess.run([sys.executable, "-c", "import sys; sys.path.insert(0, %r)\n" % ROOT + textwrap.dedent(code)],
                       capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, (r.returncode, r.stdout[-2000:], r.stderr[-2000:])
    return r.stdout


def test_optimizer_refusals_carry_their_reason():
    with pytest.raises(ValueError, match="LBFGS"):
        N.optimizer_schedule({"optimizer_type": "LBFGS", "epsilon": 0.01}, 0)
    with pytest.raises(ValueError, match="weight_norm_limit"):
        N.check_bn_optimizer({"epsilon": 0.01, "weight_norm_limit": 4.0})


def test_a_crop_larger_than_the_image_is_refused():
    out = run("""
        from convnet_b200 import net
        try:
            net.DataIterator(8, 3, 16, 20)
        except ValueError as e:
            print("REFUSED", e)
    """)
    assert "REFUSED" in out and "gpu_image_size" in out and "image_size" in out


def test_no_gpu_is_not_fatal():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    out = run("""
        from convnet_b200 import net
        try:
            net.Net("tiny", 4)
        except RuntimeError as e:
            print("DEVICE", e)
    """)
    assert "DEVICE" in out and "CUDA error" in out and "cudaMalloc" in out
