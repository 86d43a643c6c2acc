"""wgrad's dW write in the tensor-core conv kernel.  Where four consecutive output features are one 16-byte-aligned
float4 (not x-mode), each consumer warp writes its 16 dW rows 32 columns at a time through a shared-memory transpose
area, 16 bytes per lane (conv_tc.cu: wgrad_stage_off).  A target 4 bytes off 16-byte alignment keeps the scalar stores
from the accumulators.  The two paths must agree bit for bit, and each output is checked against float64 by run().  The
cases cover ragged Cout (an o-tile of 4 rows) and ragged Cin (BN < 128, a last pass partly or wholly past the tile's
columns), scaleTargets != 0, a reduction split, and grids of 1 and 3 SMs, where each CTA walks many tiles.
"""
import pytest
import torch

from conv_exact import Geo
from test_gpu_conv_exact import TC, Case, env, hygiene, run  # noqa: F401

pytestmark = pytest.mark.gpu

CASES = [
    Case("wgs_fc_ragged", "wgrad", Geo(128, 1, 1, 200, 132, 1, 1),
         "FC: Cout 132, Cin 200 (BN 112, last tile 88 columns; tf32 in either mode), scaleTargets 0.5, "
         "scaleOutput 0.25", TC, path={"bf16": "tc-tf32"}, st=0.5, so=0.25),
    Case("wgs_fc_bf16", "wgrad", Geo(128, 1, 1, 224, 132, 1, 1),
         "FC: Cout 132, Cin 224 (BN 112: a fourth pass of 16 valid columns)", TC),
    Case("wgs_1x1_bn80", "wgrad", Geo(128, 6, 3, 72, 256, 1, 1),
         "1x1, Cin 72 (BN 80: a third pass of 8 valid columns)", TC),
    Case("wgs_3x3_split", "wgrad", Geo(32, 8, 8, 48, 68, 3, 3, 1, 1, 1, 1),
         "3x3, Cout 68, reduction split, scaleTargets 0.5", TC, st=0.5),
]


@pytest.mark.parametrize("mode", TC)
@pytest.mark.parametrize("case", CASES, ids=lambda c: c.name)
def test_wgrad_transposed_store_matches_scalar(env, case, mode):
    for reserve in (0, env.sms - 1, env.sms - 3):
        # same grid, same split count: only the store path differs between the two targets
        scalar, _, p_scalar, _ = run(env, case, mode, offset=33, reserve=reserve, controls=False)
        wide, _, p_wide, _ = run(env, case, mode, offset=32, reserve=reserve, controls=False)
        assert p_scalar == p_wide == case.expected_path(mode)
        assert torch.equal(wide.view(torch.int32), scalar.view(torch.int32)), (case.name, mode, reserve)
