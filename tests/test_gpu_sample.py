"""The sampling calls' fused epilogues on the GPU: UpSampleGemm (forward ReLU, mask-free dropout), AvgPoolGemm /
DownSampleGemm (ReLU' mask, dropout fold, bias gradient) and AvgPoolUndoGemm (dropout fold), each against the unfused call
followed by the stand-alone passes it replaces, for factors 2, 3 and 4 (4: the forward pool misses the row kernels and
runs the passes inside the call), N % 4 == 0 and != 0, scaleTargets 0 and 1, and a 3-D layer (frames folded into the
planes); the results against pool_exact's float64 restatement; the true gradients against the reference's convention."""
import pytest
import torch

import pool_exact as px
from pool_exact import PG

pytestmark = pytest.mark.gpu

P, SCALE, SEED = 0.3, 1.0 / 0.7, 0x1234ABCD


class Env:
    pass


@pytest.fixture(scope="module")
def env():
    from convnet_b200 import conv_gemm as cg
    from convnet_b200 import lib
    e = Env()
    e.L, e.cg = lib.load(), cg
    lib.set_precision("fp32")
    return e


def _mat(shape, data=None):
    from convnet_b200.matrix import CUDAMatrix
    N, W, H, C = shape
    m = CUDAMatrix(N, W * H * C, shape)
    if data is not None:
        m.storage.copy_(data)
    return m


def _rand(n, seed):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return torch.randn(n, generator=g).cuda()


# (N, small side, channels x frames, factor)
CASES = [(8, 6, 3, 2), (6, 5, 4, 2), (8, 4, 2, 3), (5, 3, 3, 3), (8, 3, 2, 4), (7, 2, 3, 4), (4, 4, 2 * 3, 2)]


def _geoms(N, S, C, f):
    small, big = (N, S, S, C), (N, S * f, S * f, C)
    return small, big, PG(N, S * f, S * f, C, f, f, f, f)


def _up(env, x, small, big, f, st, t0):
    a, y = _mat(small, x), _mat(big, t0)
    env.L.UpSampleGemm(a.p_mat, y.p_mat, a.p_shape4d, y.p_shape4d, f, st)
    return y.storage


def _pool(env, x, small, big, f, so):
    from convnet_b200.abi import GetConvDesc
    a, y = _mat(big, x), _mat(small)
    d = GetConvDesc(big[3], big[3], f, f, f, f, 0, 0)
    env.L.AvgPoolGemm(a.p_mat, y.p_mat, a.p_shape4d, y.p_shape4d, d, 0.0, so)
    return y.storage


@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("st", [0.0, 1.0])
def test_upsample_forward_epilogue(env, case, st):
    N, S, C, f = case
    small, big, g = _geoms(*case)
    x, t0 = _rand(N * S * S * C, 1), _rand(N * S * S * C * f * f, 2)
    plain = _up(env, x, small, big, f, st, t0)
    assert px.check(plain, px.upsample(g, x, st=st, t0=t0, factor=f)).ok
    env.L.cnb_relu(plain.data_ptr(), plain.numel())
    mask = torch.empty_like(plain)
    env.L.cnb_dropout(plain.data_ptr(), mask.data_ptr(), plain.numel(), P, SCALE, SEED)
    env.L.convnet_b200_fuse_next_act(None, 1, None)
    env.L.convnet_b200_fuse_next_dropout(P, SCALE, SEED)
    fused = _up(env, x, small, big, f, st, t0)
    torch.cuda.synchronize()
    assert torch.equal(fused, plain)


@pytest.mark.parametrize("case", CASES)
def test_block_sum_dgrad_epilogue(env, case):
    """AvgPoolGemm with scaleOutput f^2 (UPSAMPLE's derivative): dropout fold, ReLU' mask and bias gradient"""
    N, S, C, f = case
    small, big, g = _geoms(*case)
    d, state = _rand(N * S * S * C * f * f, 3), torch.relu(_rand(N * S * S * C, 4))
    plain = _pool(env, d, small, big, f, float(f * f))
    assert px.check(plain, px.pool_fwd(g, d, False, so=float(f * f))).ok
    env.L.cnb_mult(plain.data_ptr(), torch.full_like(plain, SCALE).data_ptr(), plain.numel())
    env.L.cnb_relu_deriv(plain.data_ptr(), state.data_ptr(), plain.numel())
    gb_plain, gb_fused = torch.full((C,), 0.5, device="cuda"), torch.full((C,), 0.5, device="cuda")
    env.L.cnb_channel_bias_grad(plain.data_ptr(), gb_plain.data_ptr(), N * S * S, C, 1.0, 0.25)
    env.L.convnet_b200_fuse_next_act(None, 1, state.data_ptr())
    env.L.convnet_b200_fuse_next_scale(SCALE)
    env.L.convnet_b200_fuse_next_bias_grad(gb_fused.data_ptr(), 1.0, 0.25)
    fused = _pool(env, d, small, big, f, float(f * f))
    torch.cuda.synchronize()
    assert torch.equal(fused, plain)
    # the kernel sums per row slice, the pass per column: the same sum in another order
    ref = 0.5 + 0.25 * plain.double().view(C, -1).sum(1)
    bar = 1e-6 * (1 + 0.25 * plain.double().abs().view(C, -1).sum(1))
    assert ((gb_fused.double() - ref).abs() <= bar).all() and ((gb_plain.double() - ref).abs() <= bar).all()


@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("st", [0.0, 1.0])
def test_avg_undo_scale(env, case, st):
    """AvgPoolUndoGemm (DOWNSAMPLE's derivative) with the dropout fold and the ReLU' mask"""
    N, S, C, f = case
    small, big, g = _geoms(*case)
    from convnet_b200.abi import GetConvDesc
    dsc = GetConvDesc(C, C, f, f, f, f, 0, 0)
    d, t0, state = _rand(N * S * S * C, 5), _rand(N * S * S * C * f * f, 6), torch.relu(_rand(N * S * S * C * f * f, 7))

    def undo():
        a, y = _mat(small, d), _mat(big, t0)
        env.L.AvgPoolUndoGemm(a.p_mat, y.p_mat, a.p_shape4d, y.p_shape4d, dsc, st)
        return y.storage
    plain = undo()
    assert px.check(plain, px.avg_undo(g, d, st=st, t0=t0)).ok
    env.L.cnb_mult(plain.data_ptr(), torch.full_like(plain, SCALE).data_ptr(), plain.numel())
    env.L.cnb_relu_deriv(plain.data_ptr(), state.data_ptr(), plain.numel())
    env.L.convnet_b200_fuse_next_act(None, 1, state.data_ptr())
    env.L.convnet_b200_fuse_next_scale(SCALE)
    fused = undo()
    torch.cuda.synchronize()
    assert torch.equal(fused, plain)


@pytest.mark.parametrize("case", CASES[:4])
def test_downsample_forward_epilogue_and_logistic(env, case):
    """DownSampleGemm with a forward ReLU + dropout, and with sigma (a pass inside the call) + dropout"""
    N, S, C, f = case
    small, big, g = _geoms(*case)
    x = _rand(N * S * S * C * f * f, 8)

    def down():
        a, y = _mat(big, x), _mat(small)
        env.L.DownSampleGemm(a.p_mat, y.p_mat, a.p_shape4d, y.p_shape4d, f)
        return y.storage
    for act, pass_ in ((1, env.L.cnb_relu), (2, env.L.cnb_logistic)):
        plain = down()
        pass_(plain.data_ptr(), plain.numel())
        env.L.cnb_dropout(plain.data_ptr(), torch.empty_like(plain).data_ptr(), plain.numel(), P, SCALE, SEED)
        env.L.convnet_b200_fuse_next_act(None, act, None)
        env.L.convnet_b200_fuse_next_dropout(P, SCALE, SEED)
        fused = down()
        torch.cuda.synchronize()
        assert torch.equal(fused, plain), act


@pytest.mark.parametrize("case", CASES[:3])
def test_no_request_is_the_plain_call(env, case):
    """no request: the plain kernels (EPI off), whose results pool_exact restates"""
    N, S, C, f = case
    small, big, g = _geoms(*case)
    x = _rand(N * S * S * C, 9)
    a = _up(env, x, small, big, f, 0.0, torch.zeros(N * S * S * C * f * f, device="cuda"))
    assert px.check(a, px.upsample(g, x, factor=f)).ok
    b = _pool(env, a, small, big, f, 1.0)
    assert px.check(b, px.pool_fwd(g, a, False)).ok


@pytest.mark.parametrize("f", [2, 4])
def test_true_gradients_against_the_reference_convention(env, f):
    """UPSAMPLE's derivative (block sum) is f^2 x DownSample (block mean), DOWNSAMPLE's (d / f^2) is UpSample / f^2:
    bit for bit, f being a power of two"""
    N, S, C = 8, 4, 3
    small, big, g = _geoms(N, S, C, f)
    from convnet_b200.abi import GetConvDesc
    d_big, d_small = _rand(N * S * S * C * f * f, 10), _rand(N * S * S * C, 11)
    block_sum = _pool(env, d_big, small, big, f, float(f * f))
    ref_mean = _pool(env, d_big, small, big, f, 1.0)
    torch.cuda.synchronize()
    assert torch.equal(block_sum, ref_mean * (f * f))
    a, y = _mat(small, d_small), _mat(big)
    env.L.AvgPoolUndoGemm(a.p_mat, y.p_mat, a.p_shape4d, y.p_shape4d, GetConvDesc(C, C, f, f, f, f, 0, 0), 0.0)
    rep = _up(env, d_small, small, big, f, 0.0, torch.zeros(N * S * S * C * f * f, device="cuda"))
    torch.cuda.synchronize()
    assert torch.equal(y.storage, rep / (f * f))
