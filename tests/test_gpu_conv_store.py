"""How the tensor-core conv kernel writes a tile, in the layouts the older epilogue tests leave out.  fprop / dgrad tiles
leave through the store warps: 16 bytes per lane where the target allows it (a column of 128 images at once when
N % 128 == 0, one image chunk at a time otherwise), one element at a time elsewhere, and in fprop the tile's bias
loaded once per tile.  wgrad tiles leave from the MMA warps' registers.

- wgrad with scaleTargets != 0 on grids of 1 and 3 SMs, so that every CTA walks many tiles: checked against float64 and
  bit for bit against the full-grid run.  One module row keeps the reduction unsplit whatever the grid, so the sums are
  the same.
- wgrad with scaleTargets != 0 in each layout: reduction splits (raw partial sums into scratch), FC-shaped, x-mode
  (Cin 3, its columns scattered over the filter's taps), and Cout 42 (not a multiple of 4).
- wgrad whose target is 4-byte but not 16-byte aligned.
- fprop (bias, ReLU, scaleTargets) and fused dgrad with a batch that is not a multiple of 128: a tile's rows are
  several image chunks on different pixels.
"""
import pytest
import torch

from conv_exact import Geo
from test_gpu_conv_exact import TC, Case, env, hygiene, run, wgrad_splits  # noqa: F401  (fixtures)

pytestmark = pytest.mark.gpu

WG_SMALL_GRID = Case("store_wg_small_grid", "wgrad", Geo(128, 16, 3, 64, 256, 3, 3, 1, 1, 0, 0),
                     "one module row, scaleTargets 0.5, scaleOutput 0.25", TC, st=0.5, so=0.25, split=False)


@pytest.mark.parametrize("mode", TC)
def test_wgrad_small_grid(env, mode):
    full, l_full, p_full, _ = run(env, WG_SMALL_GRID, mode, controls=False)
    assert l_full == 1
    for usable in (1, 3):
        y, launches, path, _ = run(env, WG_SMALL_GRID, mode, reserve=env.sms - usable, controls=False)
        assert (path, launches) == (p_full, l_full)
        assert torch.equal(y.view(torch.int32), full.view(torch.int32)), (mode, usable)


WGRAD = [
    Case("store_wg_split", "wgrad", Geo(32, 14, 14, 64, 64, 3, 3, 1, 1, 1, 1),
         "reduction splits, scaleTargets 0.5", TC, st=0.5, so=0.5, split=True),
    Case("store_wg_fc", "wgrad", Geo(128, 1, 1, 512, 256, 1, 1),
         "FC, scaleTargets 1", TC, st=1.0, so=0.25, split=False),
    Case("store_wg_x", "wgrad", Geo(128, 29, 29, 3, 96, 7, 7, 2, 2, 1, 1),
         "x-mode Cin 3, ky 7, scaleTargets 0.5", TC, path={"bf16": "tc-tf32"}, st=0.5),
    Case("store_wg_cout42", "wgrad", Geo(32, 8, 8, 32, 42, 3, 3, 1, 1, 1, 1),
         "Cout 42: the o-tile ends inside a group of four rows", TC, st=0.5),
]


@pytest.mark.parametrize("mode", TC)
@pytest.mark.parametrize("case", WGRAD, ids=lambda c: c.name)
def test_wgrad_layouts(env, case, mode):
    _, launches, path, _ = run(env, case, mode, controls=True)
    assert path == case.expected_path(mode)
    splits = wgrad_splits(case.g, path == "tc-bf16", env.sms)
    if case.split is not None:
        assert (splits > 1) == case.split, (case.name, mode, splits)
    assert launches == 1 + (splits > 1)


@pytest.mark.parametrize("mode", TC)
def test_wgrad_unaligned_target(env, mode):
    c = Case("store_wg_unaligned", "wgrad", Geo(32, 8, 8, 32, 64, 3, 3, 1, 1, 1, 1),
             "target 4 bytes off 16-byte alignment", TC, st=0.5)
    _, _, path, _ = run(env, c, mode, offset=33, controls=True)
    assert path == c.expected_path(mode)


RAGGED_BATCH = [
    Case("store_fp_n96", "fprop", Geo(96, 8, 8, 32, 64, 3, 3, 1, 1, 1, 1),
         "N 96: chunks on different pixels, bias + ReLU, scaleTargets 0.5", TC, launches={"tf32": 1, "bf16": 1},
         st=0.5, fuse={"bias": 1, "relu": 1}),
    Case("store_dg_n96_mask", "dgrad", Geo(96, 8, 8, 32, 64, 3, 3, 1, 1, 1, 1),
         "N 96: chunks on different pixels, ReLU' mask", TC, launches={"tf32": 1, "bf16": 1}, fuse={"mask": 1}),
]


@pytest.mark.parametrize("mode", TC)
@pytest.mark.parametrize("case", RAGGED_BATCH, ids=lambda c: c.name)
def test_batch_not_a_multiple_of_128(env, case, mode):
    _, launches, path, _ = run(env, case, mode, controls=True)
    assert path == case.expected_path(mode)
    assert launches == case.launches[mode]
