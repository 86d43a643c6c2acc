"""Buffers and call bookkeeping shared by the element-by-element GPU tests (test_gpu_pool_exact.py,
test_gpu_elementwise_exact.py): NaN-sentinel targets with guard zones, launch counting and the exact read-back of a
staged bf16 twin."""
import torch

import pool_exact as px

SENTINEL = 0x7FC0DEAD
GUARD = 64


def matrix(rows, cols, s4, offset=0, guard=GUARD):
    """a CUDAMatrix whose storage starts `offset` floats into a NaN-sentinel buffer with `guard` floats after it"""
    from convnet_b200.matrix import CUDAMatrix
    n = rows * cols
    buf = torch.empty(offset + n + guard, dtype=torch.float32, device="cuda")
    buf.view(torch.int32).fill_(SENTINEL)
    return CUDAMatrix(rows, cols, s4, storage=buf[offset:offset + n]), buf


def guards_ok(buf, offset, n):
    s = buf.view(torch.int32)
    return bool((s[:offset] == SENTINEL).all()) and bool((s[offset + n:] == SENTINEL).all())


def launched(env, fn):
    env.L.convnet_b200_reset_launch_count()
    fn()
    n = int(env.L.convnet_b200_launch_count())
    torch.cuda.synchronize()
    return n


def check_twin(env, m, shape):
    """the staged bf16 copy of m, read exactly by a bf16 1x1 conv with identity filters (no conversion launch), must be
    the round-to-nearest-even bf16 of m's fp32 values"""
    from conv_exact import Geo
    L = env.L
    N, W, H, C = shape
    n = N * W * H * C
    assert L.convnet_b200_bf16_is_staged(m.ptr, n) == 1, "no staged twin"
    g2 = Geo(N, W, H, C, C, 1, 1)
    flt, _ = matrix(*g2.flt_dims(), g2.flt_shape(), guard=0)
    flt.storage.copy_(torch.eye(C, device="cuda").reshape(-1))
    L.convnet_b200_bf16_stage(flt.ptr, C * C)
    res, _ = matrix(*g2.out_dims(), g2.out_shape(), guard=0)
    launches = launched(env, lambda: env.cg.convUp(m, flt, res, g2.desc()))
    assert env.lib.last_conv_path() == "tc-bf16", env.lib.last_conv_path()
    want = px.bf16_rne(m.storage[:n]) + 0.0             # the conv's sum gives +0 for a -0 input
    assert torch.equal(res.storage[:n].view(torch.int32), want.view(torch.int32)), "bf16 twin is not RNE of the output"
    # the same conv on an explicitly staged copy launches as many kernels: the twin saved the conversion
    L.convnet_b200_bf16_stage(m.ptr, n)
    assert launched(env, lambda: env.cg.convUp(m, flt, res, g2.desc())) == launches
