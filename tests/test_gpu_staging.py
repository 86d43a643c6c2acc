"""bf16 staging coherence (csrc/stage.cu): copies written by the producing kernels, invalidation by library writes,
and the CONVNET_B200_STAGE_VERIFY debug mode that catches a stale copy."""
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu


def _run(*args, **extra_env):
    env = dict(os.environ, CONVNET_B200_STAGE_VERIFY="1", **extra_env)
    return subprocess.run([sys.executable, os.path.join(ROOT, "tests", "staging_worker.py"), *args],
                          capture_output=True, text=True, timeout=900, env=env)


@pytest.mark.parametrize("model,batch,steps", [("tiny", 32, 3), ("alexnet", 32, 2), ("alexnet", 128, 2)])
def test_emitted_copies_equal_a_fresh_conversion(model, batch, steps):
    r = _run("train", model, str(batch), str(steps))
    assert r.returncode == 0 and "VERIFY-TRAIN-OK" in r.stdout, (r.returncode, r.stdout[-1500:], r.stderr[-1500:])


def test_fused_dropout_and_prestaged_banks_do_not_change_the_training_step():
    """AlexNet, batch 128, bf16: the step with dropout fused into the 1x1 / fc epilogues (no mask tensor), its derivative
    folded into the dgrad above, and the dgrad filter banks rebuilt behind the optimizer step, leaves bit-identical
    parameters and losses to the step with separate dropout / mask passes and banks built on first use."""
    def run(**env):
        e = dict(os.environ, **env)
        e.pop("CONVNET_B200_STAGE_VERIFY", None)
        r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "staging_worker.py"), "params", "alexnet", "128", "3"],
                           capture_output=True, text=True, timeout=900, env=e)
        lines = [ln for ln in r.stdout.splitlines() if ln.startswith("PARAMS")]
        assert r.returncode == 0 and lines, (r.returncode, r.stdout[-1000:], r.stderr[-1500:])
        return lines[-1]
    fused = run()
    plain = run(CONVNET_B200_NO_FUSED_DROPOUT="1", CONVNET_B200_NO_DROPOUT_FOLD="1", CONVNET_B200_NO_PRESTAGE="1")
    assert fused == plain


def test_stale_copy_is_detected_in_verify_mode():
    r = _run("stale")
    assert "FIRST-USE-OK" in r.stdout and "NOT-DETECTED" not in r.stdout
    assert r.returncode != 0 and "STAGE_VERIFY" in r.stderr, (r.returncode, r.stdout, r.stderr[-1500:])


def test_library_writes_keep_copies_coherent():
    import torch
    from convnet_b200 import conv_gemm as cg
    from convnet_b200 import lib
    from convnet_b200.abi import GetConvDesc
    from convnet_b200.matrix import CUDAMatrix
    L = lib.load()
    lib.set_precision("bf16")
    try:
        N, W, Cin, Cout = 128, 8, 64, 64
        d = GetConvDesc(Cin, Cout, 3, 3, 1, 1, 1, 1)
        x = CUDAMatrix(N, W * W * Cin, (N, W, W, Cin)); x.storage.normal_()
        w = CUDAMatrix(Cout, 9 * Cin, (Cout, 3, 3, Cin)); w.storage.normal_().mul_(0.05)
        y = CUDAMatrix(N, W * W * Cout, (N, W, W, Cout))
        n = x.storage.numel()
        staged = lambda m: L.convnet_b200_bf16_is_staged(m.ptr, m.storage.numel())
        L.convnet_b200_bf16_stage(x.ptr, n)
        assert staged(x) == 1
        L.cnb_relu(x.ptr, n)                                   # a library write without an emit request: the copy is dropped
        assert staged(x) == 0
        L.convnet_b200_emit_bf16_next(); L.cnb_relu(x.ptr, n)  # with the request: a fresh copy from the same kernel
        assert staged(x) == 1
        # conv output: requested -> staged, and the copy equals a conversion of the fp32 output
        L.convnet_b200_emit_bf16_next(); cg.convUp(x, w, y, d)
        assert lib.last_conv_path() == "tc-bf16" and staged(y) == 1
        y2 = CUDAMatrix(N, W * W * Cout, (N, W, W, Cout)); cg.convUp(x, w, y2, d)
        assert staged(y2) == 0
        # consumer results with the emitted copy == results with an explicit conversion
        w2 = CUDAMatrix(Cout, 9 * Cout, (Cout, 3, 3, Cout)); w2.storage.normal_().mul_(0.05)
        z1 = CUDAMatrix(N, W * W * Cout, (N, W, W, Cout)); cg.convUp(y, w2, z1, d)
        z2 = CUDAMatrix(N, W * W * Cout, (N, W, W, Cout)); cg.convUp(y2, w2, z2, d)
        assert torch.equal(z1.storage, z2.storage)
        # the SGD kernel refreshes the staged copy of the weights it updates
        L.convnet_b200_bf16_stage(w.ptr, w.storage.numel())
        h, g_ = torch.zeros_like(w.storage), torch.randn_like(w.storage)
        L.cnb_sgd_momentum(w.ptr, h.data_ptr(), g_.data_ptr(), w.storage.numel(), 0.01, 0.9, 5e-4)
        assert staged(w) == 1
        z3 = CUDAMatrix(N, W * W * Cout, (N, W, W, Cout)); cg.convUp(x, w, z3, d)          # refreshed copy
        L.convnet_b200_bf16_invalidate(w.ptr)
        z4 = CUDAMatrix(N, W * W * Cout, (N, W, W, Cout)); cg.convUp(x, w, z4, d)          # converted inside the call
        assert torch.equal(z3.storage, z4.storage)
    finally:
        L.convnet_b200_bf16_invalidate(None)
        lib.set_precision("fp32")


@pytest.mark.parametrize("pad", [1, 0, 3])
@pytest.mark.parametrize("shape", [(128, 27, 27, 64), (32, 110, 110, 8), (7, 9, 9, 5), (4, 8, 8, 3)])
def test_max_pool_undo_from_tie_masks_is_bit_identical(shape, pad):
    """convnet_b200_pool_cache_next: the undo fed by the forward pass's tie masks equals the compare-based undo bit for bit —
    with ties (quantised inputs), with scaleTargets, with the fused ReLU' mask that is the pool input (that mask together
    with scaleTargets != 0 stays on the compare path), odd and even widths, with and without padding (padding 3 records no
    masks: both undos compare) — and it falls back as soon as the library writes one of the two tensors."""
    import torch
    from convnet_b200 import conv_gemm as cg
    from convnet_b200 import lib
    from convnet_b200.abi import GetConvDesc, num_modules
    from convnet_b200.matrix import CUDAMatrix
    L = lib.load()
    N, W, H, C = shape
    mod = num_modules(W, 3, 2, pad)
    d = GetConvDesc(C, C, 3, 3, 2, 2, pad, pad)
    ish, psh = (N, W, H, C), (N, mod, mod, C)
    g = torch.Generator(device="cuda").manual_seed(4)
    x = CUDAMatrix(N, W * H * C, ish)
    x.storage.copy_(torch.round(torch.randn(x.storage.numel(), device="cuda", generator=g) * 2) / 2)      # many ties, both signs
    gr = CUDAMatrix(N, mod * mod * C, psh); gr.storage.normal_(generator=g)
    init = torch.randn(x.storage.numel(), device="cuda", generator=g)
    try:
        for with_mask in (False, True):
            for st in (0.0, 1.0):
                # compare-based reference path
                acts = CUDAMatrix(N, mod * mod * C, psh); cg.MaxPool(x, acts, d)
                ref = CUDAMatrix(N, W * H * C, ish); ref.storage.copy_(init)
                if with_mask:
                    L.convnet_b200_fuse_next(None, 0, x.ptr)
                cg.MaxPoolUndo(x, gr, acts, ref, d, st)
                # mask-based path
                acts2 = CUDAMatrix(N, mod * mod * C, psh)
                L.convnet_b200_pool_cache_next(); cg.MaxPool(x, acts2, d)
                assert torch.equal(acts.storage, acts2.storage)
                out = CUDAMatrix(N, W * H * C, ish); out.storage.copy_(init)
                if with_mask:
                    L.convnet_b200_fuse_next(None, 0, x.ptr)
                cg.MaxPoolUndo(x, gr, acts2, out, d, st)
                assert torch.equal(out.storage, ref.storage), (with_mask, st)
        # a library write to the pool input drops the masks: the undo must follow the CURRENT tensors (compare path)
        acts2 = CUDAMatrix(N, mod * mod * C, psh)
        L.convnet_b200_pool_cache_next(); cg.MaxPool(x, acts2, d)
        L.cnb_relu(x.ptr, x.storage.numel())
        ref = CUDAMatrix(N, W * H * C, ish); out = CUDAMatrix(N, W * H * C, ish)
        cg.MaxPoolUndo(x, gr, acts2, out, d, 0)
        x2 = CUDAMatrix(N, W * H * C, ish); x2.storage.copy_(x.storage)
        acts3 = CUDAMatrix(N, mod * mod * C, psh); acts3.storage.copy_(acts2.storage)
        cg.MaxPoolUndo(x2, gr, acts3, ref, d, 0)
        assert torch.equal(out.storage, ref.storage)
    finally:
        L.convnet_b200_bf16_invalidate(None)


@pytest.mark.parametrize("precision", ["bf16", "fp32"])
@pytest.mark.parametrize("k,pad", [(1, 0), (3, 1)])
def test_fused_dropout_equals_the_separate_pass(precision, k, pad):
    """convnet_b200_fuse_next_dropout: bias + ReLU + dropout in the conv call == the same call followed by cnb_dropout with
    the same seed, bit for bit — in the lean bf16 kernel's epilogue and on the trailing-pass fallback (fp32) — and the
    bf16 twin requested with it holds the values AFTER the dropout."""
    import torch
    from convnet_b200 import conv_gemm as cg
    from convnet_b200 import lib
    from convnet_b200.abi import GetConvDesc
    from convnet_b200.matrix import CUDAMatrix
    L = lib.load()
    lib.set_precision(precision)
    try:
        N, W, Cin, Cout = 128, 14, 64, 128
        d = GetConvDesc(Cin, Cout, k, k, 1, 1, pad, pad)
        g = torch.Generator(device="cuda").manual_seed(11)
        x = CUDAMatrix(N, W * W * Cin, (N, W, W, Cin)); x.storage.normal_(generator=g)
        w = CUDAMatrix(Cout, k * k * Cin, (Cout, k, k, Cin)); w.storage.normal_(generator=g).mul_(0.05)
        b = torch.randn(Cout, device="cuda", generator=g)
        n_out = N * W * W * Cout
        seed, prob = 0x1234567890ABCDEF, 0.3
        scale = 1.0 / (1.0 - prob)
        # reference: conv (+bias, ReLU) then the stand-alone dropout pass
        ref = CUDAMatrix(N, W * W * Cout, (N, W, W, Cout)); mask = torch.empty(n_out, device="cuda")
        L.convnet_b200_fuse_next(b.data_ptr(), 1, None); cg.convUp(x, w, ref, d)
        L.cnb_dropout(ref.ptr, mask.data_ptr(), n_out, prob, scale, seed)
        # fused
        out = CUDAMatrix(N, W * W * Cout, (N, W, W, Cout))
        if precision == "bf16":                                   # operands staged: the call is the conv kernel alone
            L.convnet_b200_bf16_stage(x.ptr, x.storage.numel()); L.convnet_b200_bf16_stage(w.ptr, w.storage.numel())
        L.convnet_b200_reset_launch_count()
        L.convnet_b200_fuse_next(b.data_ptr(), 1, None); L.convnet_b200_fuse_next_dropout(prob, scale, seed)
        L.convnet_b200_emit_bf16_next(); cg.convUp(x, w, out, d)
        if precision == "bf16":
            assert lib.last_conv_path() == "tc-bf16"
            assert L.convnet_b200_launch_count() == 1             # bias, ReLU, dropout and the bf16 twin all in its epilogue
        assert torch.equal(out.storage, ref.storage)
        kept = (out.storage != 0).float().mean().item()
        assert 0.2 < kept < 0.5                                   # ~ half pass the ReLU, 70 % of those are kept
        if precision == "bf16":                                   # the twin the next edge would read == a conversion of the result
            assert L.convnet_b200_bf16_is_staged(out.ptr, n_out) == 1
            w2 = CUDAMatrix(Cout, Cout, (Cout, 1, 1, Cout)); w2.storage.normal_(generator=g).mul_(0.05)
            d2 = GetConvDesc(Cout, Cout, 1, 1, 1, 1, 0, 0)
            z1 = CUDAMatrix(N, W * W * Cout, (N, W, W, Cout)); cg.convUp(out, w2, z1, d2)
            L.convnet_b200_bf16_invalidate(out.ptr)
            z2 = CUDAMatrix(N, W * W * Cout, (N, W, W, Cout)); cg.convUp(out, w2, z2, d2)
            assert torch.equal(z1.storage, z2.storage)
        # the request is one-shot
        out2 = CUDAMatrix(N, W * W * Cout, (N, W, W, Cout))
        L.convnet_b200_fuse_next(b.data_ptr(), 1, None); cg.convUp(x, w, out2, d)
        assert (out2.storage != 0).float().mean().item() > kept + 0.1
    finally:
        L.convnet_b200_bf16_invalidate(None)
        lib.set_precision("fp32")


def test_prestaged_dgrad_banks_are_used_and_dropped_on_weight_writes():
    """convnet_b200_prestage_next: the convDown that follows builds nothing and returns the same derivative; touching the
    weights through the library drops the banks again."""
    import torch
    from convnet_b200 import conv_gemm as cg
    from convnet_b200 import lib
    from convnet_b200.abi import GetConvDesc, num_modules
    from convnet_b200.matrix import CUDAMatrix
    L = lib.load()
    lib.set_precision("bf16")
    try:
        N, W, Cin, Cout, k, s, pad = 128, 27, 64, 96, 5, 2, 1
        mod = num_modules(W, k, s, pad)
        d = GetConvDesc(Cin, Cout, k, k, s, s, pad, pad)
        g = torch.Generator(device="cuda").manual_seed(5)
        w = CUDAMatrix(Cout, k * k * Cin, (Cout, k, k, Cin)); w.storage.normal_(generator=g).mul_(0.05)
        dy = CUDAMatrix(N, mod * mod * Cout, (N, mod, mod, Cout)); dy.storage.normal_(generator=g)
        dx0 = CUDAMatrix(N, W * W * Cin, (N, W, W, Cin)); dx1 = CUDAMatrix(N, W * W * Cin, (N, W, W, Cin))
        dx1.storage.fill_(7.0)
        cg.convDown(dy, w, dx0, d)                                 # builds the banks on first use
        assert lib.last_conv_path() == "tc-bf16"
        L.convnet_b200_bf16_invalidate(None)
        L.convnet_b200_reset_launch_count()
        L.convnet_b200_prestage_next(); cg.convDown(dy, w, dx1, d)
        assert L.convnet_b200_launch_count() == 1                  # the bank kernel only
        assert torch.all(dx1.storage == 7.0)                       # the target was not touched
        L.convnet_b200_reset_launch_count()
        cg.convDown(dy, w, dx1, d)
        with_banks = L.convnet_b200_launch_count()
        assert torch.equal(dx1.storage, dx0.storage)
        L.cnb_relu(w.ptr, w.storage.numel())                       # a library write to the weights: banks stale
        L.convnet_b200_reset_launch_count()
        cg.convDown(dy, w, dx1, d)
        assert L.convnet_b200_launch_count() == with_banks + 1     # rebuilt
    finally:
        L.convnet_b200_bf16_invalidate(None)
        lib.set_precision("fp32")


def test_describing_a_model_keeps_a_live_nets_copies():
    """a host-only Model (here through model_flops) touches no library state: the bf16 copies of the weights that a
    training step staged for the next forward pass stay staged."""
    from convnet_b200 import lib
    from convnet_b200 import net as N
    L = lib.load()
    lib.set_precision("bf16")
    net = N.Net("alexnet", 32, seed=3)
    try:
        base = net.params_tensor().data_ptr()                   # (taking the pointer drops the copies: before the step)
        net.input_tensor().normal_()
        net.labels_tensor().zero_()
        net.train_step(False)
        staged = lambda: [name for name, _, off, size in net.edges() if size and L.convnet_b200_bf16_is_staged(base + 4 * off, 1)]
        before = staged()
        assert before
        N.model_flops("alexnet", 32)
        assert staged() == before
    finally:
        net.close()
        L.convnet_b200_bf16_invalidate(None)
        lib.set_precision("fp32")
