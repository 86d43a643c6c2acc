#!/usr/bin/env python3
"""Write tests/golden/ref_opt.npz: the state updates of the reference's Adagrad and RMSProp optimizers, computed by the
reference's own CPU library on seeded inputs: eigenmat's adagrad / rms_prop (eigenmat/eigenmat.cc:2139-2178), which
oracle/_ref/libeigenmat_ref.so exports under their C++ names and which are called here through a ctypes mirror of the
reference's `struct eigenmat` (eigenmat/eigenmat.h:18-24).

Each case <name> stores <name>_s (the state before), <name>_g (the gradient), <name>_param (delta or factor) and
<name>_out (the state after).  The inputs hold exact zeros, and magnitudes from 1e-25 (whose squares underflow) to 1e15.

    python tools/gen_opt_golden.py          (needs oracle/_ref/libeigenmat_ref.so: __graft_entry__.build() next to the
                                              reference sources)"""
import ctypes as ct
import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_LIB = os.path.join(ROOT, "oracle", "_ref", "libeigenmat_ref.so")
OUT = os.path.join(ROOT, "tests", "golden", "ref_opt.npz")
N = 1024


def _inputs(rng, fresh, base):
    """(state, gradient): a gradient of mixed magnitudes with exact zeros; a fresh state (the optimizer's start) or a
    state some updates in"""
    g = (rng.standard_normal(N) * 10.0 ** rng.integers(-6, 2, N)).astype(np.float32)
    g[rng.random(N) < 0.1] = 0
    g[:16] = [0, -0.0, 1e-25, -3e-25, 1e-19, 2e-20, 1e15, -7e14, 1e-38, 3e-45, 1, -1, 0.5, 65504, 1e-3, -1e-30]
    if fresh:
        s = np.full(N, base, np.float32)
    else:
        s = (base + np.abs(rng.standard_normal(N)) * 10.0 ** rng.integers(-4, 3, N)).astype(np.float32)
        s[16:32] = base
    return s, g


# int adagrad(eigenmat* history, eigenmat* grad, float delta) / int rms_prop(eigenmat*, eigenmat*, float factor)
SYMBOLS = {"adagrad": "_Z7adagradP8eigenmatS0_f", "rmsprop": "_Z8rms_propP8eigenmatS0_f"}


class EigenMat(ct.Structure):
    _fields_ = [("data", ct.POINTER(ct.c_float)), ("size", ct.c_int * 2), ("is_trans", ct.c_int), ("owns_data", ct.c_int)]


def _mat(a):
    m = EigenMat()
    m.data = a.ctypes.data_as(ct.POINTER(ct.c_float))
    m.size[0], m.size[1], m.is_trans, m.owns_data = 1, a.size, 0, 0
    return m


def reference_functions(lib_path=REF_LIB):
    """{"adagrad": f, "rmsprop": f}, f(history, grad, param) updating the float32 array `history` in place"""
    L = ct.CDLL(lib_path)
    out = {}
    for rule, sym in SYMBOLS.items():
        fn = getattr(L, sym)
        fn.argtypes, fn.restype = [ct.POINTER(EigenMat), ct.POINTER(EigenMat), ct.c_float], ct.c_int

        def call(history, grad, param, fn=fn):
            g = grad.copy()
            h, gm = _mat(history), _mat(g)
            assert fn(ct.byref(h), ct.byref(gm), param) == 0
        out[rule] = call
    return out


def generate(lib_path=REF_LIB):
    ref = reference_functions(lib_path)
    rng = np.random.default_rng(20140801)
    out = {}
    for rule, fn, params in (("adagrad", ref["adagrad"], (0.0, 1.0)), ("rmsprop", ref["rmsprop"], (0.0, 0.9))):
        for p in params:
            for fresh in (True, False):
                # the start: adagrad_delta for Adagrad, 1 for RMSProp (a delta-0 Adagrad state also starts at 0)
                s, g = _inputs(rng, fresh, p if rule == "adagrad" else 1.0)
                res = s.copy()
                fn(res, g, p)
                name = "%s_%g_%s" % (rule, p, "fresh" if fresh else "later")
                out.update({name + "_s": s, name + "_g": g, name + "_param": np.float32(p), name + "_out": res})
    return out


if __name__ == "__main__":
    np.savez(OUT, **generate())
    print("wrote", OUT)
