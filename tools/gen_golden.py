#!/usr/bin/env python3
"""Generate tests/golden/*.npz by RUNNING the reference's own numpy oracle.

The reference's only executable spec of the hot path is py/conv_cpu.py (Python 2).
This script loads that file from /root/reference AT GENERATION TIME (nothing is
copied into the repo), applies the two mechanical Python-2 -> 3 fixes it needs
in memory (`xrange` -> `range`, `/` -> Python-2 division semantics, `print`
statements dropped), executes its functions on small seeded inputs and stores
inputs + outputs.  The committed .npz files are what travels to the GPU box;
tests/test_oracle_vs_reference.py pins oracle/conv_oracle.c against them and
tests/test_gpu_parity.py pins the CUDA path against them.

Run (here, where /root/reference exists):  python tools/gen_golden.py
"""
import ast
import os
import re
import sys

import numpy as np

REF = os.environ.get("CONVNET_REFERENCE", "/root/reference")
OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")


def _py2_div(a, b):
    if isinstance(a, (int, np.integer)) and isinstance(b, (int, np.integer)):
        return a // b
    return a / b


class _Div(ast.NodeTransformer):
    def visit_BinOp(self, node):
        self.generic_visit(node)
        if isinstance(node.op, ast.Div):
            return ast.copy_location(
                ast.Call(func=ast.Name(id="_py2_div", ctx=ast.Load()), args=[node.left, node.right], keywords=[]),
                node)
        return node


def load_reference_numpy_oracle():
    src = open(os.path.join(REF, "py", "conv_cpu.py")).read()
    src = re.sub(r"^(\s*)print .*$", r"\1pass", src, flags=re.M)
    src = src.replace("xrange", "range")
    tree = ast.fix_missing_locations(_Div().visit(ast.parse(src)))
    ns = {"_py2_div": _py2_div}
    exec(compile(tree, "conv_cpu.py(py3)", "exec"), ns)
    return ns


def mods(sz, k, s, p):
    return (sz + 2 * p - k) // s + 1


def case2d(ref, name, seed, N, W, H, Cin, Cout, ky, kx, sy, sx, py, px, sizeF, add_scale, pow_scale, ps=(0, 0)):
    r = np.random.RandomState(seed)
    modY, modX = mods(H, ky, sy, py), mods(W, kx, sx, px)
    ishape = (N, W, H, Cin)
    spec = (Cout, ky, kx, sy, sx, py, px)
    pspec = (Cin, ky, kx, sy, sx, py, px)
    images = r.randn(N, W * H * Cin).astype(np.float32)
    filters = r.randn(Cout, kx * ky * Cin).astype(np.float32)
    derivs = r.randn(N, modX * modY * Cout).astype(np.float32)
    g = dict(kind="2d", N=N, W=W, H=H, Cin=Cin, Cout=Cout, ky=ky, kx=kx, sy=sy, sx=sx, py=py, px=px,
             modY=modY, modX=modX, sizeF=sizeF, add_scale=add_scale, pow_scale=pow_scale,
             psy=ps[0], psx=ps[1], images=images, filters=filters, derivs=derivs)
    g["convUp"] = ref["ConvUp"](images, filters, ishape, spec)
    g["convDown"] = ref["ConvDown"](derivs, filters, ishape, spec)
    outp, psums = ref["ConvOutp"](images, derivs, ishape, spec, partial_sum_y=ps[0], partial_sum_x=ps[1])
    g["convOutp"], g["convOutpPartial"] = outp, psums
    # pooling (channels preserved)
    pimages = r.rand(N, W * H * Cin).astype(np.float32)         # uniform, test_conv.py:114
    pderivs = r.randn(N, modX * modY * Cin).astype(np.float32)
    g["pool_images"], g["pool_derivs"] = pimages, pderivs
    g["maxPool"] = ref["MaxPool"](pimages, ishape, pspec)
    g["avgPool"] = ref["AvgPool"](pimages, ishape, pspec)
    g["maxPoolUndo"] = ref["MaxPoolUndo"](pimages, g["maxPool"], pderivs, ishape, (N, modX, modY, Cin), pspec)
    g["avgPoolUndo"] = ref["AvgPoolUndo"](pderivs, ishape, pspec)
    # response norm over Cin channels
    rderivs = r.randn(N, W * H * Cin).astype(np.float32)
    g["rnorm_derivs"] = rderivs
    for blocked in (False, True):
        tag = "_blocked" if blocked else ""
        g["rnorm" + tag] = ref["ResponseNormCrossMap"](images, ishape, sizeF, add_scale, pow_scale, blocked)
        g["rnormUndo" + tag] = ref["ResponseNormCrossMapUndo"](rderivs, images, ishape, sizeF, add_scale,
                                                               pow_scale, blocked)
    np.savez_compressed(os.path.join(OUT, name + ".npz"), **g)
    print("wrote", name, {k: v.shape for k, v in g.items() if hasattr(v, "shape") and v.ndim})


def case3d(ref, name, seed, N, W, H, T, Cin, Cout, ky, kx, kt, sy, sx, st, py, px):
    r = np.random.RandomState(seed)
    pt = 0
    modY, modX, modT = mods(H, ky, sy, py), mods(W, kx, sx, px), mods(T, kt, st, pt)
    ishape = (N, W, H, Cin, T)
    spec = (Cout, ky, kx, kt, sy, sx, st, py, px, pt)
    pspec = (Cin, ky, kx, kt, sy, sx, st, py, px, pt)
    images = r.randn(N, W * H * Cin * T).astype(np.float32)
    filters = r.randn(Cout, kx * ky * Cin * kt).astype(np.float32)
    derivs = r.randn(N, modX * modY * Cout * modT).astype(np.float32)
    g = dict(kind="3d", N=N, W=W, H=H, T=T, Cin=Cin, Cout=Cout, ky=ky, kx=kx, kt=kt, sy=sy, sx=sx, st=st,
             py=py, px=px, pt=pt, modY=modY, modX=modX, modT=modT, images=images, filters=filters, derivs=derivs)
    g["convUp3D"] = ref["ConvUp3D"](images, filters, ishape, spec)
    g["convDown3D"] = ref["ConvDown3D"](derivs, filters, ishape, spec)
    g["convOutp3D"] = ref["ConvOutp3D"](images, derivs, ishape, spec)
    pimages = r.rand(N, W * H * Cin * T).astype(np.float32)
    pderivs = r.randn(N, modX * modY * Cin * modT).astype(np.float32)
    g["pool_images"], g["pool_derivs"] = pimages, pderivs
    g["maxPool3D"] = ref["MaxPool3D"](pimages, ishape, pspec)
    g["avgPool3D"] = ref["AvgPool3D"](pimages, ishape, pspec)
    g["maxPool3DUndo"] = ref["MaxPool3DUndo"](pimages, g["maxPool3D"], pderivs, ishape,
                                              (N, modX, modY, Cin, modT), pspec)
    g["avgPool3DUndo"] = ref["AvgPool3DUndo"](pderivs, ishape, pspec)
    np.savez_compressed(os.path.join(OUT, name + ".npz"), **g)
    print("wrote", name, {k: v.shape for k, v in g.items() if hasattr(v, "shape") and v.ndim})


def main():
    if not os.path.isdir(REF):
        sys.exit("reference tree not found at %s (golden files are generated in the build container only)" % REF)
    os.makedirs(OUT, exist_ok=True)
    ref = load_reference_numpy_oracle()
    # the py/test_conv.py:394-441 2-D geometry (12x12x32 -> 64, 3x3 s2 p1, rnorm 8 / 0.005 / 0.75), batch cut to 2
    # (keeps the file under 1 MB)
    case2d(ref, "ref2d_testconv", 1, 2, 12, 12, 32, 64, 3, 3, 2, 2, 1, 1, 8, 0.005, 0.75, ps=(3, 3))
    # rectangular everything, odd channel counts, ragged batch
    case2d(ref, "ref2d_rect", 2, 5, 9, 7, 3, 10, 3, 2, 1, 2, 1, 0, 2, 0.01, 0.5)
    # AlexNet conv1-like: 7x7 s2 p1 on Cin=3 (small image), rnorm window > half the channels
    case2d(ref, "ref2d_conv1", 3, 4, 21, 21, 3, 16, 7, 7, 2, 2, 1, 1, 3, 5e-4, 0.75)
    # the py/test_conv.py:443-482 3-D geometry (7x7x3, s 2/2/2, p 1/1/0, Cin 3), image/batch cut down
    case3d(ref, "ref3d_testconv", 4, 4, 16, 12, 8, 3, 8, 7, 7, 3, 2, 2, 2, 1, 1)
    # C3D-like 3x3x3 s1 p1/1/0
    case3d(ref, "ref3d_c3d", 5, 4, 8, 8, 5, 4, 8, 3, 3, 3, 1, 1, 1, 1, 1)


if __name__ == "__main__":
    main()
