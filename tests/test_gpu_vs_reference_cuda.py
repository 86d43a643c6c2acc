"""BASELINE-size parity on the GPU against the REFERENCE'S OWN CUDA KERNELS.

The reference outputs are cudamat/cudamat_conv_gemm.cu + cudamat_conv3d_gemm.cu compiled unmodified for sm_90
(oracle/Makefile), run on an H100 on the same seeded inputs these tests generate.  Every layer of net A
(examples/imagenet/CLS_net_20140801232522.pbtxt, SURVEY.md Appendix B) at batch 128 (BASELINE config 2) and 256
(config 3), and the cfg4 C3D conv1a / conv2a shapes at batch 32: fprop / dgrad / wgrad, pool1/2/5 (+undo),
rnorm1/2 (+undo).  The tensors are hundreds of MB, so tests/golden/ref_cuda_samples.npz keeps, of each reference output,
its element count and its values at a fixed set of elements: the first and last EDGE (the first and last images of the
first and last columns, i.e. the corner tiles) and SAMPLES seeded random ones.  The product's output is compared with the
reference on those elements; its WHOLE output (pre-filled with NaN) must be finite, so no element may be left unwritten.  To re-record
it where oracle/_ref/libcudamat_conv_gemm_ref.so exists: CONVNET_B200_RECORD_REF=<file.npz> python -m pytest -m gpu
tests/test_gpu_vs_reference_cuda.py (the reference runs, every comparison is made against its live output, and the
samples are written to <file.npz>).

Metric and tolerances are the ones of tests/test_gpu_parity.py: Diff = max|a-b| / mean|a+b| (py/test_conv.py:382-385);
fp32 mode 1e-4 (the reference's own bar), tf32 5e-3, bf16 2.5e-2; max-pool values bit-exact; pool-undo / rnorm 1e-4, rnorm
undo 2e-4.
"""
import os
import zlib

import numpy as np
import pytest

import ref_cuda_lib
from convnet_b200.abi import GetConvDesc, num_modules

pytestmark = pytest.mark.gpu

TOL = {"fp32": 1e-4, "tf32": 5e-3, "bf16": 2.5e-2}
TOL_MEM = 1e-4
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "ref_cuda_samples.npz")
SAMPLES = 384
EDGE = 64


@pytest.fixture(scope="module")
def env():
    import torch
    assert torch.cuda.is_available(), "these tests need a CUDA device"
    record = os.environ.get("CONVNET_B200_RECORD_REF")
    if record and not ref_cuda_lib.available():
        pytest.fail("recording needs oracle/_ref/libcudamat_conv_gemm_ref.so: run `make -C oracle` where the reference exists")
    from convnet_b200 import conv_gemm as cg
    from convnet_b200 import lib
    from convnet_b200.matrix import CUDAMatrix
    lib.load()

    class E:
        pass
    e = E()
    e.torch, e.lib, e.ours, e.M = torch, lib, cg.gemm, CUDAMatrix
    e.ref = ref_cuda_lib.binding() if record else None
    stored = {} if record else dict(np.load(GOLDEN))
    recorded = {}

    def rand(rows, cols, s4, gen, scale=1.0, uniform=False):
        m = CUDAMatrix(rows, cols, s4)
        if uniform:
            m.storage.uniform_(generator=gen)
        else:
            m.storage.normal_(generator=gen)
        if scale != 1.0:
            m.storage.mul_(scale)
        return m

    def nan(rows, cols, s4):
        m = CUDAMatrix(rows, cols, s4)
        m.fill_(float("nan"))
        return m
    e.rand, e.nan = rand, nan
    e.zeros = lambda rows, cols, s4: CUDAMatrix(rows, cols, s4)      # reference targets (not the object under test)

    def sample_index(key, numel):
        rand = np.random.RandomState(zlib.crc32(key.encode())).randint(0, numel, SAMPLES)
        edge = np.concatenate([np.arange(min(EDGE, numel)), np.arange(max(numel - EDGE, 0), numel)])
        return torch.from_numpy(np.concatenate([edge, rand])).cuda()

    def reference(key, names, compute):
        """the reference's outputs `names` of case `key` as (sampled indices, reference values there, element count):
        computed live while recording, else the stored samples"""
        outs = compute() if record else None
        res = []
        for i, name in enumerate(names):
            k = key + "/" + name
            if record:
                torch.cuda.synchronize()
                numel = outs[i].rows * outs[i].cols
                idx = sample_index(k, numel)
                vals = outs[i].storage[idx].clone()
                recorded[k], recorded[k + "#numel"] = vals.cpu().numpy(), np.int64(numel)
            else:
                numel = int(stored[k + "#numel"])
                idx = sample_index(k, numel)
                vals = torch.from_numpy(stored[k]).cuda()
            res.append((idx, vals, numel))
        return res
    e.reference = reference

    def whole(a, ref):
        """the product's output `a` has the reference output's size and every element of it is finite"""
        numel = ref[2]
        assert a.rows * a.cols == numel, (a.rows * a.cols, numel)
        assert torch.isfinite(a.storage[:numel]).all(), "non-finite (or unwritten) elements in the output"

    def diff(a, ref):
        """Diff of the product's output `a` against a reference output, over the reference's sampled elements"""
        whole(a, ref)
        idx, b, _ = ref
        a = a.storage[idx]
        assert torch.isfinite(b).all()
        num = (a - b).abs().max().item()
        den = (a + b).abs().mean(dtype=torch.float64).item()
        return num / den if den > 0 else num
    e.diff = diff

    def same(a, ref):
        whole(a, ref)
        return torch.equal(a.storage[ref[0]], ref[1])
    e.same = same
    yield e
    lib.set_precision("tf32")
    if record:
        np.savez_compressed(record, **recorded)


# name: W, H, Cin, Cout, ky, kx, sy, sx, py, px        (net A, SURVEY.md Appendix B)
ALEX_CONV = {
    "conv1": (224, 224, 3, 96, 7, 7, 2, 2, 1, 1),
    "conv2": (55, 55, 96, 256, 5, 5, 2, 2, 1, 1),
    "nin2_1": (27, 27, 256, 256, 1, 1, 1, 1, 0, 0),
    "conv3": (14, 14, 256, 384, 3, 3, 1, 1, 1, 1),
    "nin3_1": (14, 14, 384, 768, 1, 1, 1, 1, 0, 0),
    "conv4": (14, 14, 768, 384, 3, 3, 1, 1, 1, 1),
    "nin4_1": (14, 14, 384, 768, 1, 1, 1, 1, 0, 0),
    "nin4_2": (14, 14, 768, 384, 1, 1, 1, 1, 0, 0),
    "conv5": (14, 14, 384, 512, 3, 3, 1, 1, 0, 0),
    "nin5_1": (12, 12, 512, 1024, 1, 1, 1, 1, 0, 0),
    "nin5_2": (12, 12, 1024, 512, 1, 1, 1, 1, 0, 0),
    "fc6": (1, 1, 18432, 4096, 1, 1, 1, 1, 0, 0),         # FC as a 1x1 conv on a 1x1 image (host/edge.cc FCEdge)
    "fc7": (1, 1, 4096, 4096, 1, 1, 1, 1, 0, 0),
    "fc8": (1, 1, 4096, 1000, 1, 1, 1, 1, 0, 0),
}


@pytest.mark.parametrize("N", [128, 256])
@pytest.mark.parametrize("layer", list(ALEX_CONV))
def test_alexnet_conv_layers(env, layer, N):
    torch = env.torch
    W, H, Cin, Cout, ky, kx, sy, sx, py, px = ALEX_CONV[layer]
    modY, modX = num_modules(H, ky, sy, py), num_modules(W, kx, sx, px)
    d = GetConvDesc(Cin, Cout, ky, kx, sy, sx, py, px)
    ish, fsh, tsh = (N, W, H, Cin), (Cout, kx, ky, Cin), (N, modX, modY, Cout)
    K = kx * ky * Cin
    g = torch.Generator(device="cuda").manual_seed(zlib.crc32(("%s_%d" % (layer, N)).encode()) & 0xFFFF)
    x = env.rand(N, W * H * Cin, ish, g)
    w = env.rand(Cout, K, fsh, g, scale=1.0 / np.sqrt(K))
    dv = env.rand(N, modX * modY * Cout, tsh, g)

    def ref_outputs():
        r_up = env.zeros(N, modX * modY * Cout, tsh); env.ref.convUp(x, w, r_up, d, 0)
        r_dn = env.zeros(N, W * H * Cin, ish); env.ref.convDown(dv, w, r_dn, d, 0)
        r_dw = env.zeros(Cout, K, fsh); env.ref.convOutp(x, dv, r_dw, d, 0, 1.0 / N)
        return r_up, r_dn, r_dw
    r_up, r_dn, r_dw = env.reference("%s_b%d" % (layer, N), ("fprop", "dgrad", "wgrad"), ref_outputs)
    for mode in ("fp32", "tf32", "bf16"):
        env.lib.set_precision(mode)
        out = env.nan(N, modX * modY * Cout, tsh); env.ours.convUp(x, w, out, d, 0); p_up = env.lib.last_conv_path()
        d_up = env.diff(out, r_up)
        out = env.nan(N, W * H * Cin, ish); env.ours.convDown(dv, w, out, d, 0); p_dn = env.lib.last_conv_path()
        d_dn = env.diff(out, r_dn)
        out = env.nan(Cout, K, fsh); env.ours.convOutp(x, dv, out, d, 0, 1.0 / N); p_dw = env.lib.last_conv_path()
        d_dw = env.diff(out, r_dw)
        # a call that the tensor path declines runs on the fp32 CUDA-core kernels and must then meet the fp32 bar
        for name, dd, path in (("fprop", d_up, p_up), ("dgrad", d_dn, p_dn), ("wgrad", d_dw, p_dw)):
            tol = TOL["fp32"] if path == "cuda-core-fp32" else TOL[mode]
            assert dd < tol, (layer, N, mode, name, path, dd)


@pytest.mark.parametrize("N", [128, 256])
def test_alexnet_conv_accumulate(env, N):
    """scaleTargets = 1 at BASELINE size (conv3, all three ops) against the reference's kWriteRowsMult / Sgemm beta path."""
    torch = env.torch
    W, H, Cin, Cout, ky, kx, sy, sx, py, px = ALEX_CONV["conv3"]
    d = GetConvDesc(Cin, Cout, ky, kx, sy, sx, py, px)
    ish, fsh, tsh = (N, W, H, Cin), (Cout, kx, ky, Cin), (N, 14, 14, Cout)
    K = kx * ky * Cin
    g = torch.Generator(device="cuda").manual_seed(77 + N)
    x, w, dv = env.rand(N, W * H * Cin, ish, g), env.rand(Cout, K, fsh, g, 1.0 / np.sqrt(K)), env.rand(N, 196 * Cout, tsh, g)
    i_up, i_dn, i_dw = env.rand(N, 196 * Cout, tsh, g), env.rand(N, W * H * Cin, ish, g), env.rand(Cout, K, fsh, g)

    def run(api):
        a = env.M(N, 196 * Cout, tsh); a.storage.copy_(i_up.storage); api.convUp(x, w, a, d, 1)
        b = env.M(N, W * H * Cin, ish); b.storage.copy_(i_dn.storage); api.convDown(dv, w, b, d, 1)
        c = env.M(Cout, K, fsh); c.storage.copy_(i_dw.storage); api.convOutp(x, dv, c, d, 1, 0.5)
        return a, b, c
    ref = env.reference("conv3_accum_b%d" % N, ("fprop", "dgrad", "wgrad"), lambda: run(env.ref))
    for mode in ("fp32", "tf32", "bf16"):
        env.lib.set_precision(mode)
        for name, a, b in zip(("fprop", "dgrad", "wgrad"), run(env.ours), ref):
            dd = env.diff(a, b)
            assert dd < TOL[mode], (mode, name, dd)


ALEX_POOL = {"pool1": (110, 96), "pool2": (27, 256), "pool5": (12, 512)}      # image size, channels; 3x3 stride 2 pad 1


@pytest.mark.parametrize("N", [128, 256])
@pytest.mark.parametrize("layer", list(ALEX_POOL))
def test_alexnet_pool_layers(env, layer, N):
    torch = env.torch
    W, C = ALEX_POOL[layer]
    mod = num_modules(W, 3, 2, 1)
    d = GetConvDesc(C, C, 3, 3, 2, 2, 1, 1)
    ish, psh = (N, W, W, C), (N, mod, mod, C)
    g = torch.Generator(device="cuda").manual_seed(5 + N)
    x = env.rand(N, W * W * C, ish, g)
    gr = env.rand(N, mod * mod * C, psh, g)
    inits = [env.rand(N, W * W * C, ish, g) for _ in (0, 1)]

    def ref_outputs():
        r_mx = env.zeros(N, mod * mod * C, psh); env.ref.MaxPool(x, r_mx, d)
        r_av = env.zeros(N, mod * mod * C, psh); env.ref.AvgPool(x, r_av, d)
        outs = [r_mx, r_av]
        for st in (0, 1):
            r = env.M(N, W * W * C, ish); r.storage.copy_(inits[st].storage); env.ref.MaxPoolUndo(x, gr, r_mx, r, d, st)
            outs.append(r)
            r = env.M(N, W * W * C, ish); r.storage.copy_(inits[st].storage); env.ref.AvgPoolUndo(gr, r, d, st)
            outs.append(r)
        return outs
    names = ("max", "avg", "max_undo_st0", "avg_undo_st0", "max_undo_st1", "avg_undo_st1")
    ref = dict(zip(names, env.reference("%s_b%d" % (layer, N), names, ref_outputs)))
    o_mx = env.nan(N, mod * mod * C, psh); env.ours.MaxPool(x, o_mx, d)
    assert env.same(o_mx, ref["max"]), "max-pool values must be bit-exact"
    o_av = env.nan(N, mod * mod * C, psh); env.ours.AvgPool(x, o_av, d)
    res = {"avg": env.diff(o_av, ref["avg"])}
    for st in (0, 1):
        init = inits[st]
        o = env.M(N, W * W * C, ish); o.storage.copy_(init.storage if st else torch.full_like(init.storage, float("nan")))
        env.ours.MaxPoolUndo(x, gr, o_mx, o, d, st)
        res["max_undo_st%d" % st] = env.diff(o, ref["max_undo_st%d" % st])
        o = env.M(N, W * W * C, ish); o.storage.copy_(init.storage if st else torch.full_like(init.storage, float("nan")))
        env.ours.AvgPoolUndo(gr, o, d, st)
        res["avg_undo_st%d" % st] = env.diff(o, ref["avg_undo_st%d" % st])
    for k, v in res.items():
        assert v < TOL_MEM, (layer, N, k, v)


ALEX_RNORM = {"rnorm1": (55, 96, 24), "rnorm2": (14, 256, 64)}      # image size, channels, window (frac 0.25)


@pytest.mark.parametrize("N", [128, 256])
@pytest.mark.parametrize("layer", list(ALEX_RNORM))
def test_alexnet_rnorm_layers(env, layer, N):
    torch = env.torch
    W, C, k = ALEX_RNORM[layer]
    ish = (N, W, W, C)
    g = torch.Generator(device="cuda").manual_seed(9 + N)
    x, dy = env.rand(N, W * W * C, ish, g), env.rand(N, W * W * C, ish, g)

    def ref_outputs():
        outs = []
        for blocked in (False, True):
            r = env.zeros(N, W * W * C, ish); env.ref.ResponseNormCrossMap(x, r, k, 5e-4, 0.75, blocked); outs.append(r)
            r = env.zeros(N, W * W * C, ish); env.ref.ResponseNormCrossMapUndo(dy, x, r, k, 5e-4, 0.75, blocked); outs.append(r)
        return outs
    names = ("fwd_blocked0", "undo_blocked0", "fwd_blocked1", "undo_blocked1")
    ref = dict(zip(names, env.reference("%s_b%d" % (layer, N), names, ref_outputs)))
    res = {}
    for blocked in (False, True):
        o = env.nan(N, W * W * C, ish); env.ours.ResponseNormCrossMap(x, o, k, 5e-4, 0.75, blocked)
        res["fwd_blocked%d" % blocked] = env.diff(o, ref["fwd_blocked%d" % blocked])
        o = env.nan(N, W * W * C, ish); env.ours.ResponseNormCrossMapUndo(dy, x, o, k, 5e-4, 0.75, blocked)
        res["undo_blocked%d" % blocked] = env.diff(o, ref["undo_blocked%d" % blocked])
    for kk, v in res.items():
        assert v < (2 * TOL_MEM if kk.startswith("undo") else TOL_MEM), (layer, N, kk, v)


# BASELINE config 4 (SURVEY.md 8(d)): clips of 16 frames 112x112x3, batch 32, 3x3x3 kernels, pad y/x 1, pad t 0
C3D_CONV = {
    # name: W, Cin, T, Cout
    "conv1a": (112, 3, 16, 64),
    "conv2a": (56, 64, 14, 128),
}


@pytest.mark.parametrize("layer", list(C3D_CONV))
def test_c3d_conv_layers(env, layer):
    torch = env.torch
    N = 32
    W, Cin, T, Cout = C3D_CONV[layer]
    kt, To = 3, T - 2
    d = GetConvDesc(Cin, Cout, 3, 3, 1, 1, 1, 1, kernel_size_t=kt, stride_t=1, padding_t=0)
    ish, fsh, tsh = (N, W, W, Cin * T), (Cout, 3, 3, Cin * kt), (N, W, W, Cout * To)
    K = 9 * Cin * kt
    g = torch.Generator(device="cuda").manual_seed(31)
    x = env.rand(N, W * W * Cin * T, ish, g)
    w = env.rand(Cout, K, fsh, g, scale=1.0 / np.sqrt(K))
    dv = env.rand(N, W * W * Cout * To, tsh, g)

    def ref_outputs():
        r_up = env.zeros(N, W * W * Cout * To, tsh); env.ref.convUp3D(x, w, r_up, d, 0)
        r_dn = env.zeros(N, W * W * Cin * T, ish); env.ref.convDown3D(dv, w, r_dn, d, 0)
        r_dw = env.zeros(Cout, K, fsh); env.ref.convOutp3D(x, dv, r_dw, d, 0, 1.0 / N)
        return r_up, r_dn, r_dw
    r_up, r_dn, r_dw = env.reference("c3d_%s_b%d" % (layer, N), ("fprop", "dgrad", "wgrad"), ref_outputs)
    for mode in ("fp32", "tf32", "bf16"):
        env.lib.set_precision(mode)
        out = env.nan(N, W * W * Cout * To, tsh); env.ours.convUp3D(x, w, out, d, 0); p_up = env.lib.last_conv_path()
        d_up = env.diff(out, r_up)
        out = env.nan(N, W * W * Cin * T, ish); env.ours.convDown3D(dv, w, out, d, 0); p_dn = env.lib.last_conv_path()
        d_dn = env.diff(out, r_dn)
        out = env.nan(Cout, K, fsh); env.ours.convOutp3D(x, dv, out, d, 0, 1.0 / N); p_dw = env.lib.last_conv_path()
        d_dw = env.diff(out, r_dw)
        for name, dd, path in (("fprop", d_up, p_up), ("dgrad", d_dn, p_dn), ("wgrad", d_dw, p_dw)):
            tol = TOL["fp32"] if path == "cuda-core-fp32" else TOL[mode]
            assert dd < tol, (layer, mode, name, path, dd)


def test_c3d_pool_layer(env):
    """cfg4's 2x2x2 max-pool (kernel_size_t / stride_t through kPool, cudamat_conv_gemm.cu:153-200) at batch 32."""
    torch = env.torch
    N, W, C, T = 32, 56, 128, 12
    d = GetConvDesc(C, C, 2, 2, 2, 2, 0, 0, kernel_size_t=2, stride_t=2, padding_t=0)
    ish, psh = (N, W, W, C * T), (N, W // 2, W // 2, C * (T // 2))
    g = torch.Generator(device="cuda").manual_seed(3)
    x = env.rand(N, W * W * C * T, ish, g)
    gr = env.rand(N, (W // 2) ** 2 * C * (T // 2), psh, g)

    def ref_outputs():
        r_mx = env.zeros(gr.rows, gr.cols, psh); env.ref.MaxPool(x, r_mx, d)
        r = env.zeros(x.rows, x.cols, ish); env.ref.MaxPoolUndo(x, gr, r_mx, r, d, 0)
        return r_mx, r
    ref_mx, ref_undo = env.reference("c3d_pool2_b32", ("max", "max_undo"), ref_outputs)
    o_mx = env.nan(gr.rows, gr.cols, psh); env.ours.MaxPool(x, o_mx, d)
    assert env.same(o_mx, ref_mx)
    o = env.nan(x.rows, x.cols, ish); env.ours.MaxPoolUndo(x, gr, o_mx, o, d, 0)
    dd = env.diff(o, ref_undo)
    assert dd < TOL_MEM
