"""The store warps' two compilations of the fprop / dgrad epilogue (conv_tc.cu: store_tiles).  A call that reads no
old target, no ReLU' mask and draws no dropout, into 16-byte-aligned outputs, takes the lean batches; any other call
takes the general ones.  A target 4 bytes off 16-byte alignment sends the same call down the general path, and the two
outputs must agree bit for bit; each is also checked against float64 by run().  The cases cover x-mode fprop with two
y-blocks (conv1's shape, scaled down), bias + ReLU, the bf16 twin, a ragged last n-tile, dgrad without a mask, and
grids with all but 1 or 3 SMs reserved (the library keeps at least 8), where each CTA walks many tiles.
"""
import pytest
import torch

from conv_exact import Geo
from test_gpu_conv_exact import TC, Case, env, hygiene, run  # noqa: F401

pytestmark = pytest.mark.gpu

CASES = [
    Case("lean_x_conv1", "fprop", Geo(128, 29, 29, 3, 96, 7, 7, 2, 2, 1, 1),
         "x-mode Cin 3, ky 7, bias + ReLU", ("tf32",), fuse={"bias": 1, "relu": 1}),
    Case("lean_1x1_relu", "fprop", Geo(128, 7, 7, 64, 200, 1, 1),
         "1x1, Cout 200 (a ragged last n-tile), bias + ReLU", TC, fuse={"bias": 1, "relu": 1}),
    Case("lean_3x3_twin", "fprop", Geo(128, 8, 8, 32, 64, 3, 3, 1, 1, 1, 1),
         "3x3, bias + ReLU + bf16 twin", TC, fuse={"bias": 1, "relu": 1, "emit": 1}),
    Case("lean_dgrad", "dgrad", Geo(128, 8, 8, 32, 64, 3, 3, 1, 1, 1, 1),
         "dgrad with no ReLU' mask", TC),
]


PARAMS = [(c, m) for c in CASES for m in c.modes]


@pytest.mark.parametrize("case,mode", PARAMS, ids=["%s-%s" % (c.name, m) for c, m in PARAMS])
def test_lean_store_matches_general(env, case, mode):
    for reserve in (0, env.sms - 1, env.sms - 3):
        # same grid and plan: only the store path differs between the two targets
        general, _, p_general, _ = run(env, case, mode, offset=33, reserve=reserve, controls=False)
        lean, _, p_lean, _ = run(env, case, mode, offset=32, reserve=reserve, controls=False)
        assert p_general == p_lean == case.expected_path(mode)
        assert torch.equal(lean.view(torch.int32), general.view(torch.int32)), (case.name, mode, reserve)
