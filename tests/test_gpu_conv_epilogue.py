"""The fprop / dgrad epilogue of the tensor-core conv kernel: the consumer warps hand each finished tile to the store warps
through one shared-memory staging tile, and the store warps write it with 16-byte accesses where the target allows.

- A fully fused fprop (bias, ReLU, dropout, bf16 twin, scaleTargets != 0) on grids of a few SMs, so that every CTA
  walks many tiles and the staging handoff wraps its phases many times: checked against float64 and bit for bit
  against the full-grid run.
- An fprop and a fused dgrad whose target is 4-byte but not 16-byte aligned: the store warps move one element at a time.
"""
import pytest
import torch

from conv_exact import Geo
from test_gpu_conv_exact import DROP, TC, Case, _check_twin, env, hygiene, run  # noqa: F401  (fixtures)

pytestmark = pytest.mark.gpu

FUSED = Case("epi_fused_st", "fprop", Geo(128, 12, 12, 32, 96, 3, 3, 1, 1, 1, 1),
             "bias + ReLU + dropout + bf16 twin, scaleTargets 0.5", TC, launches={"tf32": 1, "bf16": 1},
             st=0.5, fuse={"bias": 1, "relu": 1, "drop": DROP, "emit": 1})


@pytest.mark.parametrize("mode", TC)
def test_fused_fprop_small_grid(env, mode):
    full, l_full, p_full, out = run(env, FUSED, mode, controls=False)
    assert l_full == 1
    if mode == "bf16":
        _check_twin(env, FUSED, out)
    for usable in (1, 3):
        y, launches, path, out = run(env, FUSED, mode, reserve=env.sms - usable, controls=False)
        assert (path, launches) == (p_full, l_full)
        assert torch.equal(y.view(torch.int32), full.view(torch.int32)), (mode, usable)
        if mode == "bf16":
            _check_twin(env, FUSED, out)


UNALIGNED = [
    Case("epi_unaligned_fprop", "fprop", Geo(128, 8, 8, 32, 64, 3, 3, 1, 1, 1, 1),
         "target 4 bytes off 16-byte alignment: scalar stores", TC, launches={"tf32": 1, "bf16": 1},
         st=0.5, fuse={"bias": 1, "relu": 1}),
    Case("epi_unaligned_dgrad", "dgrad", Geo(128, 8, 8, 32, 64, 3, 3, 1, 1, 1, 1),
         "target 4 bytes off 16-byte alignment, ReLU' mask: scalar stores", TC, launches={"tf32": 1, "bf16": 2},
         fuse={"mask": 1}),
]


@pytest.mark.parametrize("mode", TC)
@pytest.mark.parametrize("case", UNALIGNED, ids=lambda c: c.name)
def test_unaligned_target(env, case, mode):
    _, launches, path, _ = run(env, case, mode, offset=33, controls=True)
    assert path == case.expected_path(mode)
    assert launches == case.launches[mode]
