"""Worker of tests/test_gpu_elementwise_exact.py::test_kernel_names: the elementwise cases once more under
torch.profiler, in a process of their own, and the kernel names CUPTI recorded against the dispatch mirror's.  Prints
NAMES-OK <calls> when they match in order, NAMES-NONE when the profiler recorded no kernel of the library; a mismatch
fails an assertion (exit code 1)."""
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
import test_gpu_elementwise_exact as T  # noqa: E402
from convnet_b200 import conv_gemm as cg  # noqa: E402
from convnet_b200 import lib  # noqa: E402


class Env:
    pass


env = Env()
env.cg, env.lib, env.L = cg, lib, lib.load()
env.sms = torch.cuda.get_device_properties(0).multi_processor_count
env.L.convnet_b200_set_conv_precision(2)            # bf16: the mode in which twins are emitted, as in the test file
env.L.convnet_b200_bf16_invalidate(None)
got, want = T.profile_kernel_names(env)
if not got:
    print("NAMES-NONE")
    sys.exit(0)
assert len(got) == len(want), (len(got), len(want))
for i, (g, w) in enumerate(zip(got, want)):
    assert w in g, (i, w, g)
print("NAMES-OK %d" % len(got))
