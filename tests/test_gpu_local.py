"""Locally connected (untied) convolution on the GPU: localUp / localDown / localOutp on the tensor cores, element by element
against float64 on the kernel's own rounded operands (the bar of tests/conv_exact.py), the SIMT fallback, the fused
per-feature-bias epilogue, and the LOCAL edge of the host (grad check, `lcnet` training, bf16 staging coherence).

Untied layout: filter bank of module m = mx + modX*my at w[o + Cout*(k + K*m)], k = tx + kx*(ty + ky*c); the output
column of (module m, channel o) is m + modules*o, which is also the index of its bias."""
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import conv_exact as cx
from conv_exact import Geo

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAN = 0x7FC0DEAD
PATH_MODEL = {"cuda-core-fp32": "fp32", "tc-tf32": "tf32", "tc-bf16": "bf16"}


@pytest.fixture(scope="module")
def env():
    assert torch.cuda.is_available()
    from convnet_b200 import conv_gemm as cg
    from convnet_b200 import lib, net
    L = lib.load()
    net.load_host()
    yield cg, lib, L, net
    lib.set_precision("tf32")


@pytest.fixture(autouse=True)
def hygiene(env):
    _, _, L, _ = env
    prec = L.convnet_b200_get_conv_precision()
    try:
        yield
    finally:
        L.convnet_b200_set_conv_precision(prec)
        L.convnet_b200_bf16_invalidate(None)
        L.cnb_relu_deriv(None, None, 0)


# ---------------------------------------------------------------------------------------------------------------------
# untied float64 reference
# ---------------------------------------------------------------------------------------------------------------------
def _banks(b, g):
    """flat filters -> (modules, Cout, K)"""
    M = g.modX * g.modY
    return b[: g.Cout * g.K * M].view(M, g.K, g.Cout).transpose(1, 2)


def local_raw(op, g, a, b):
    """the un-scaled untied op on float64 flat operands -> flat result (fprop: a images, b filters; dgrad: a derivs,
    b filters; wgrad: a images, b derivs)"""
    M = g.modX * g.modY
    if op == "fprop":
        cols = cx._cols(cx._act(a, g.N, g.W, g.H, g.Cin), g)                       # (N, K, M)
        out = torch.einsum("mok,nkm->nom", _banks(b, g), cols)
        return cx._unact(out.reshape(g.N, g.Cout, g.modY, g.modX))
    if op == "dgrad":
        der = cx._act(a, g.N, g.modX, g.modY, g.Cout).reshape(g.N, g.Cout, M)
        cols = torch.einsum("mok,nom->nkm", _banks(b, g), der)
        img = torch.nn.functional.fold(cols, (g.H, g.W), (g.ky, g.kx), padding=(g.py, g.px), stride=(g.sy, g.sx))
        return cx._unact(img)
    cols = cx._cols(cx._act(a, g.N, g.W, g.H, g.Cin), g)
    der = cx._act(b, g.N, g.modX, g.modY, g.Cout).reshape(g.N, g.Cout, M)
    dw = torch.einsum("nom,nkm->mko", der, cols)                                    # element (o, k, m) at o + Cout*(k + K*m)
    return dw.reshape(-1)


def local_expect(op, g, a, b, kind, t0=None, st=0.0, so=1.0, bias=None, relu=False):
    A, B = cx.model(a, kind), cx.model(b, kind)
    ref = so * local_raw(op, g, A, B)
    S = abs(so) * local_raw(op, g, A.abs(), B.abs())
    if st != 0.0:
        t = t0.to(torch.float64)
        ref, S = ref + st * t, S + (st * t).abs()
    if bias is not None:                                # bias[column], column = m + modules*o; flat = n + N*column
        bb = bias.to(torch.float64).repeat_interleave(g.N)
        ref, S = ref + bb, S + bb.abs()
    if relu:
        ref = ref.clamp_min(0.0)
    return ref, S


def verdict(y, ref, S):
    err = (y.to(torch.float64) - ref).abs()
    pos = S > 0
    ratio = torch.where(pos, err / torch.where(pos, S, torch.ones_like(S)), torch.zeros_like(err))
    ratio = torch.where(torch.isnan(ratio), torch.full_like(ratio, float("inf")), ratio)
    exact_bad = int(((~pos) & (err != 0)).sum().item()) + int(torch.isnan(y).sum().item())
    worst = float(ratio.max().item())
    return worst <= cx.BAR and exact_bad == 0, worst, exact_bad


# ---------------------------------------------------------------------------------------------------------------------
# one call
# ---------------------------------------------------------------------------------------------------------------------
def _mat(rows, cols, s4, fill=None, gen=None):
    from convnet_b200.matrix import CUDAMatrix
    t = torch.empty(rows * cols, dtype=torch.float32, device="cuda")
    if gen is not None:
        t.normal_(generator=gen)
    else:
        t.view(torch.int32).fill_(NAN)
    return CUDAMatrix(rows, cols, s4, storage=t)


def operands(g, seed):
    gen = torch.Generator(device="cuda").manual_seed(seed)
    M = g.modX * g.modY
    img = _mat(g.N, g.W * g.H * g.Cin, (g.N, g.W, g.H, g.Cin), gen=gen)
    flt = _mat(g.Cout, g.K * M, (g.Cout, g.kx, g.ky, g.Cin * M), gen=gen)
    der = _mat(g.N, M * g.Cout, (g.N, g.modX, g.modY, g.Cout), gen=gen)
    return img, flt, der


def run_op(env, op, g, mode, seed=1, st=0.0, so=1.0, stage=True):
    cg, lib, L, _ = env
    lib.set_precision(mode)
    img, flt, der = operands(g, seed)
    M = g.modX * g.modY
    d = g.desc()
    if op == "fprop":
        out = _mat(g.N, M * g.Cout, (g.N, g.modX, g.modY, g.Cout), gen=torch.Generator(device="cuda").manual_seed(99)) \
            if st else _mat(g.N, M * g.Cout, (g.N, g.modX, g.modY, g.Cout))
        a, b = img, flt
    elif op == "dgrad":
        out = _mat(g.N, g.W * g.H * g.Cin, (g.N, g.W, g.H, g.Cin), gen=torch.Generator(device="cuda").manual_seed(99)) \
            if st else _mat(g.N, g.W * g.H * g.Cin, (g.N, g.W, g.H, g.Cin))
        a, b = der, flt
    else:
        out = _mat(g.Cout, g.K * M, (g.Cout, g.kx, g.ky, g.Cin * M), gen=torch.Generator(device="cuda").manual_seed(99)) \
            if st else _mat(g.Cout, g.K * M, (g.Cout, g.kx, g.ky, g.Cin * M))
        a, b = img, der
    t0 = out.storage.clone()
    if stage and mode == "bf16":
        for m in (a, b):
            L.convnet_b200_bf16_stage(m.ptr, m.storage.numel())
    if op == "fprop":
        cg.localUp(img, flt, out, d, st)
    elif op == "dgrad":
        cg.localDown(der, flt, out, d, st)
    else:
        cg.localOutp(img, der, out, d, st, so)
    torch.cuda.synchronize()
    assert op == "wgrad" or so == 1.0
    return lib.last_conv_path(), out.storage, a.storage, b.storage, t0


LC3 = dict(W=12, H=12, Cin=128, Cout=128, ky=3, kx=3, py=1, px=1)       # lcnet local3: 144 modules, K 1152
LC4 = dict(W=12, H=12, Cin=128, Cout=128, ky=3, kx=3)                   # lcnet local4: 100 modules
RAGGED = {
    "cout40": dict(W=8, H=8, Cin=64, Cout=40, ky=3, kx=3, py=1, px=1),
    "cin72": dict(W=7, H=7, Cin=72, Cout=64, ky=3, kx=3, py=1, px=1),
    "stride2": dict(W=9, H=9, Cin=64, Cout=64, ky=3, kx=3, sy=2, sx=2),
    "asym_pad": dict(W=8, H=6, Cin=64, Cout=64, ky=3, kx=5, py=0, px=2),
}
CASES = [("local3", LC3, 128), ("local3", LC3, 256), ("local4", LC4, 128), ("local4", LC4, 256)] + \
        [(k, v, 128) for k, v in RAGGED.items()]


@pytest.mark.parametrize("mode", ["tf32", "bf16"])
@pytest.mark.parametrize("op", ["fprop", "dgrad", "wgrad"])
@pytest.mark.parametrize("name,geo,N", CASES, ids=["%s-N%d" % (c[0], c[2]) for c in CASES])
def test_untied_tensor_core_per_element(env, name, geo, N, op, mode):
    g = Geo(N=N, **geo)
    for st, so in ((0.0, 1.0), (1.0, 0.75 if op == "wgrad" else 1.0)):
        path, y, a, b, t0 = run_op(env, op, g, mode, seed=3, st=st, so=so)
        assert path == "tc-" + mode, (name, op, path)
        ref, S = local_expect(op, g, a, b, mode, t0=t0, st=st, so=so)
        ok, worst, bad = verdict(y, ref, S)
        assert ok, (name, op, mode, st, so, worst, bad)
        if st == 0.0:                                   # controls: the wrong operand models must fail the bar
            for wrong in cx.CONTROLS[mode]:
                r2, S2 = local_expect(op, g, a, b, wrong, t0=t0, st=st, so=so)
                assert not verdict(y, r2, S2)[0], (name, op, mode, wrong)


@pytest.mark.parametrize("N", [8, 100])
@pytest.mark.parametrize("op", ["fprop", "dgrad", "wgrad"])
def test_untied_ineligible_batches_stay_on_cuda_cores(env, N, op):
    g = Geo(N=N, **RAGGED["cout40"])
    path, y, a, b, t0 = run_op(env, op, g, "bf16", seed=5)
    assert path == "cuda-core-fp32"
    ref, S = local_expect(op, g, a, b, "fp32", t0=t0)
    ok, worst, bad = verdict(y, ref, S)
    assert ok, (worst, bad)


@pytest.mark.parametrize("mode,N,path", [("bf16", 128, "tc-bf16"), ("tf32", 128, "tc-tf32"), ("bf16", 8, "cuda-core-fp32")])
def test_fused_local_epilogue_is_bit_identical_to_the_passes(env, mode, N, path):
    """per-feature bias + ReLU + dropout (+ bf16 twin) on localUp, and ReLU' mask + scale on localDown: the fused call
    equals the unfused call followed by the separate passes, bit for bit"""
    cg, lib, L, _ = env
    g = Geo(N=N, **LC4)
    M, n_out = g.modX * g.modY, None
    img, flt, der = operands(g, 7)
    bias = torch.randn(M * g.Cout, device="cuda")
    lib.set_precision(mode)
    d = g.desc()
    outs = []
    for fused in (True, False):
        out = _mat(N, M * g.Cout, (N, g.modX, g.modY, g.Cout))
        n_out = out.storage.numel()
        if fused:
            L.convnet_b200_fuse_next(bias.data_ptr(), 1, None)
            L.convnet_b200_fuse_next_dropout(0.5, 2.0, 1234)
            L.convnet_b200_emit_bf16_next()
            cg.localUp(img, flt, out, d, 0)
            assert lib.last_conv_path() == path
            assert L.convnet_b200_bf16_is_staged(out.ptr, n_out) == (1 if mode == "bf16" else 0)
        else:
            cg.localUp(img, flt, out, d, 0)
            L.cnb_add_channel_bias(out.ptr, bias.data_ptr(), N, M * g.Cout)
            L.cnb_relu(out.ptr, n_out)
            mask = torch.empty(n_out, device="cuda")
            L.cnb_dropout(out.ptr, mask.data_ptr(), n_out, 0.5, 2.0, 1234)
        torch.cuda.synchronize()
        outs.append(out.storage.clone())
    assert torch.equal(outs[0].view(torch.int32), outs[1].view(torch.int32))
    # localDown with the ReLU' mask of its target and the dropout scale.  For untied calls conv_down (abi.cu) always
    # applies the mask as a trailing cnb_relu_deriv pass, so today both branches run the same passes: this half pins the
    # request semantics (scale, then mask) and would start to compare two different code paths only if the mask ever
    # moved into the untied dgrad epilogue (DESIGN.md §4.1 states it is a trailing pass)
    state = torch.randn(N * g.W * g.H * g.Cin, device="cuda").clamp_min(0)
    res = []
    for fused in (True, False):
        t = _mat(N, g.W * g.H * g.Cin, (N, g.W, g.H, g.Cin))
        if fused:
            L.convnet_b200_fuse_next(None, 0, state.data_ptr())
            L.convnet_b200_fuse_next_scale(2.0)
            cg.localDown(der, flt, t, d, 0)
            assert lib.last_conv_path() == path
        else:
            L.convnet_b200_fuse_next_scale(2.0)
            cg.localDown(der, flt, t, d, 0)
            L.cnb_relu_deriv(t.ptr, state.data_ptr(), t.storage.numel())
        torch.cuda.synchronize()
        res.append(t.storage.clone())
    assert torch.equal(res[0].view(torch.int32), res[1].view(torch.int32))


# ---------------------------------------------------------------------------------------------------------------------
# the host's LOCAL edge
# ---------------------------------------------------------------------------------------------------------------------
def test_lcnet_size_flops_and_initial_scale(env):
    _, lib, _, net = env
    lib.set_precision("tf32")
    n = net.Net("lcnet", 128, seed=1)
    try:
        assert abs(n.flops_fprop / 128 - 207273984) < 1
        assert abs(n.flops_train / 128 / 1e9 - 0.59970) < 5e-5
        names = [e[0] for e in n.edges()]
        p = n.params_tensor()
        for idx, modules, init_wt in ((names.index("pool2:local3"), 144, 12.0), (names.index("local3:local4"), 100, 10.0)):
            _, _, off, size = n.edges()[idx]
            w = p[off: off + 128 * 1152 * modules]
            bound = init_wt / math.sqrt(1152 * modules / 3.0)       # uniform(-0.5, 0.5) * 2 * init_wt / sqrt(fan_in / 3)
            assert float(w.abs().max()) <= bound * (1 + 1e-6)
            assert float(w.abs().max()) > 0.99 * bound
            assert float(p[off + 128 * 1152 * modules: off + size].abs().max()) == 0.0   # biases start at 0
    finally:
        n.close()


def test_local_grad_check(env):
    _, lib, _, net = env
    lib.set_precision("fp32")
    for seed in (1, 5, 9):
        n = net.Net("localcheck", 8, seed=3, grad_checker=True)
        res = n.grad_check(seed=seed)
        n.close()
        assert len(res) == 3
        for name, eps, dw, db in res:
            assert dw < 0.01 and db < 0.01, (seed, res)


@pytest.mark.parametrize("mode", ["tf32", "bf16"])
def test_lcnet_training_reduces_the_loss_deterministically(env, mode):
    _, lib, L, net = env
    lib.set_precision(mode)
    runs = []
    for _ in range(2):
        n = net.Net("lcnet", 128, seed=1)
        g = torch.Generator(device="cuda").manual_seed(0)
        n.input_tensor().normal_(generator=g)
        n.labels_tensor().copy_(torch.randint(0, 1000, (128,), device="cuda", generator=g, dtype=torch.int32))
        losses = [n.train_step(True) / 128 for _ in range(60 if not runs else 20)]
        runs.append((losses, n.params_tensor().clone()))
        n.close()
    losses = runs[0][0]
    assert all(math.isfinite(v) for v in losses)
    assert min(losses[30:]) < 0.8 * losses[0], losses[::6]
    assert runs[0][0][:20] == runs[1][0]                         # no atomics: the same losses step for step


def test_lcnet_params_bit_identical_across_runs():
    def run():
        r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "staging_worker.py"), "params", "lcnet", "128", "3"],
                           capture_output=True, text=True, timeout=900,
                           env={k: v for k, v in os.environ.items() if k != "CONVNET_B200_STAGE_VERIFY"})
        lines = [ln for ln in r.stdout.splitlines() if ln.startswith("PARAMS")]
        assert r.returncode == 0 and lines, (r.returncode, r.stdout[-1000:], r.stderr[-1500:])
        return lines[-1]
    assert run() == run()


def test_lcnet_bf16_copies_verify():
    """CONVNET_B200_STAGE_VERIFY=1: every staged bf16 copy used across lcnet steps equals a fresh conversion of its fp32
    source (the untied filter banks are staged at their full Cout x K x modules size)"""
    env = dict(os.environ, CONVNET_B200_STAGE_VERIFY="1")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "staging_worker.py"), "train", "lcnet", "128", "3"],
                       capture_output=True, text=True, timeout=900, env=env)
    assert r.returncode == 0 and "VERIFY-TRAIN-OK" in r.stdout, (r.returncode, r.stdout[-1500:], r.stderr[-1500:])
