"""The fprop / dgrad store role of the tensor-core conv kernel at seven store warps, the plan of launches whose tiles are
bound by their epilogue (conv_tc.cu: pick_store_warps), as every case here is (one or two k-blocks per tile): store
warp w writes the tile's channels w, w + 7, ... in batches of 4, and holds the bias of its (at most 19) channels one
per lane.

Each case runs on grids of 1 and 3 SMs with 18 tiles, so that every CTA walks many tiles through the one staging tile
and its phase wraps an odd number of times on both grids.  Each output is checked against float64 and bit for bit
against the full-grid run:
- fprop with bias + ReLU + dropout + bf16 twin;
- a fused dgrad with the ReLU' mask and scaleTargets != 0;
- the tf32 x-mode fprop (96 channels: 13 or 14 per warp, the last batch partly empty);
- a target 4 bytes off 16-byte alignment (one element per store);
- 4 output channels: store warps 4-6 have no channel and only release the staging tile;
- the logistic (SIG) instances: bias + logistic in fprop, the logistic derivative in a dgrad with scaleTargets != 0
  (bit for bit against the full grid).
"""
import math

import pytest
import torch

from conv_exact import Geo
from test_gpu_conv_exact import DROP, TC, Case, _check_twin, _matrix, _randn, env, hygiene, run  # noqa: F401

pytestmark = pytest.mark.gpu

# 1x1 convs on a 6 x 3 grid at batch 128: 18 m-tiles of one pixel each and one n-tile
CASES = [
    Case("drain_fp_fused", "fprop", Geo(128, 6, 3, 64, 128, 1, 1),
         "bias + ReLU + dropout + bf16 twin", TC, launches={"tf32": 1, "bf16": 1},
         fuse={"bias": 1, "relu": 1, "drop": DROP, "emit": 1}),
    Case("drain_dg_mask_st", "dgrad", Geo(128, 6, 3, 128, 64, 1, 1),
         "ReLU' mask, scaleTargets 0.5 (gather form)", TC, launches={"tf32": 1, "bf16": 1},
         st=0.5, fuse={"mask": 1}),
    Case("drain_fp_x", "fprop", Geo(128, 21, 7, 3, 96, 7, 7, 2, 2, 1, 1),
         "x-mode Cin 3, ky 7 (tf32 in either mode), bias + ReLU", TC, path={"bf16": "tc-tf32"},
         launches={"tf32": 1, "bf16": 1}, fuse={"bias": 1, "relu": 1}),
    Case("drain_fp_cout4", "fprop", Geo(128, 6, 3, 64, 4, 1, 1),
         "4 channels: three store warps without a channel (tf32 in either mode)", TC, path={"bf16": "tc-tf32"},
         launches={"tf32": 1, "bf16": 1}, st=0.5, fuse={"bias": 1, "relu": 1}),
]
OFFSET = {"drain_fp_fused": 32, "drain_dg_mask_st": 32, "drain_fp_x": 32, "drain_fp_cout4": 36}
UNALIGNED = Case("drain_fp_unaligned", "fprop", Geo(128, 6, 3, 64, 128, 1, 1),
                 "target 4 bytes off 16-byte alignment", TC, launches={"tf32": 1, "bf16": 1},
                 st=0.5, fuse={"bias": 1, "relu": 1})


def _small_grids(env, case, mode, offset):
    full, l_full, p_full, _ = run(env, case, mode, offset=offset, controls=False)
    assert (p_full, l_full) == (case.expected_path(mode), case.launches[mode])
    for usable in (1, 3):
        y, launches, path, out = run(env, case, mode, offset=offset, reserve=env.sms - usable, controls=False)
        assert (path, launches) == (p_full, l_full)
        assert torch.equal(y.view(torch.int32), full.view(torch.int32)), (case.name, mode, usable)
        if case.fuse and "emit" in case.fuse and mode == "bf16":
            _check_twin(env, case, out)


@pytest.mark.parametrize("mode", TC)
@pytest.mark.parametrize("case", CASES, ids=lambda c: c.name)
def test_store_warps_small_grid(env, case, mode):
    _small_grids(env, case, mode, OFFSET[case.name])


@pytest.mark.parametrize("mode", TC)
def test_store_warps_unaligned_target(env, mode):
    _small_grids(env, UNALIGNED, mode, offset=33)


@pytest.mark.parametrize("mode", TC)
def test_store_warps_logistic(env, mode):
    """the SIG instances: bias + logistic in fprop, the logistic derivative in a dgrad with scaleTargets != 0"""
    g = Geo(128, 6, 3, 64, 64, 1, 1)
    gen = torch.Generator(device="cuda").manual_seed(7)
    img = _randn(*g.img_dims(), g.img_shape(), gen)
    flt = _randn(*g.flt_dims(), g.flt_shape(), gen, scale=1.0 / math.sqrt(g.K))
    der = _randn(*g.out_dims(), g.out_shape(), gen)
    bias = torch.randn(g.Cout, generator=gen, device="cuda")
    state = torch.sigmoid(torch.randn(img.storage.numel(), generator=gen, device="cuda"))
    t0 = torch.randn(img.storage.numel(), generator=gen, device="cuda")
    L, cg, d = env.L, env.cg, g.desc()
    env.lib.set_precision(mode)
    ups, downs, paths = [], [], []
    for usable in (env.sms, 1, 3):
        L.convnet_b200_reserve_sms(env.sms - usable)
        up, _ = _matrix(*g.out_dims(), g.out_shape())
        L.convnet_b200_fuse_next_act(bias.data_ptr(), 2, None)
        cg.convUp(img, flt, up, d, 0)
        paths.append(env.lib.last_conv_path())
        dn, _ = _matrix(*g.img_dims(), g.img_shape())
        dn.storage.copy_(t0)
        L.convnet_b200_fuse_next_act(None, 2, state.data_ptr())
        cg.convDown(der, flt, dn, d, 0.5)
        paths.append(env.lib.last_conv_path())
        L.convnet_b200_reserve_sms(0)
        torch.cuda.synchronize()
        assert torch.isfinite(up.storage).all() and torch.isfinite(dn.storage).all()
        ups.append(up.storage.clone())
        downs.append(dn.storage.clone())
    assert set(paths) == {"tc-" + mode}, paths
    for i in (1, 2):
        assert torch.equal(ups[i].view(torch.int32), ups[0].view(torch.int32)), (mode, "fprop", i)
        assert torch.equal(downs[i].view(torch.int32), downs[0].view(torch.int32)), (mode, "dgrad", i)
