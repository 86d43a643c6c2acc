#!/usr/bin/env python3
"""Write tests/golden/ref_loss.npz: the logistic unit and the output-layer rules of the reference, computed by the
reference's own CPU library on seeded inputs: eigenmat's apply_sigmoid, apply_logistic_deriv, apply_logistic_grad,
compute_cross_entropy, compute_cross_entropy_bernoulli, get_softmax_correct_row_major and get_logistic_correct_normalized
(eigenmat/eigenmat.cc), which oracle/_ref/libeigenmat_ref.so exports under their C++ names, called through a ctypes
mirror of `struct eigenmat` (eigenmat/eigenmat.h:18-24).

Matrices are column-major [ROWS images x COLS features], images fastest, like a layer state.  Keys:
  x, sigmoid                   apply_sigmoid(x)
  d, s, logistic_deriv         apply_logistic_deriv(d, s) = d * s * (1 - s)
  y, t, logistic_grad          apply_logistic_grad(y, t) = (t < 0) ? 0 : y - t      (t holds don't-care entries < 0)
  p, q, cross_entropy          compute_cross_entropy(q, p, 1e-10) = -q * log(p + 1e-10)       (q: soft targets)
  cross_entropy_bernoulli      compute_cross_entropy_bernoulli(tb, y, 1e-10), tb = t with the don't-cares set to 0
  labels, softmax_correct      get_softmax_correct_row_major(p, labels)              (per image)
  logistic_correct             get_logistic_correct_normalized(y, t)                 (per image)

    python tools/gen_loss_golden.py          (needs oracle/_ref/libeigenmat_ref.so: __graft_entry__.build() next to the
                                              reference sources)"""
import ctypes as ct
import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_LIB = os.path.join(ROOT, "oracle", "_ref", "libeigenmat_ref.so")
OUT = os.path.join(ROOT, "tests", "golden", "ref_loss.npz")
ROWS, COLS = 37, 21                                  # ragged on purpose

SYMBOLS = {
    "apply_sigmoid": "_Z13apply_sigmoidP8eigenmatS0_",
    "apply_logistic_deriv": "_Z20apply_logistic_derivP8eigenmatS0_S0_",
    "apply_logistic_grad": "_Z19apply_logistic_gradP8eigenmatS0_S0_",
    "compute_cross_entropy": "_Z21compute_cross_entropyP8eigenmatS0_S0_f",
    "compute_cross_entropy_bernoulli": "_Z31compute_cross_entropy_bernoulliP8eigenmatS0_S0_f",
    "get_softmax_correct_row_major": "_Z29get_softmax_correct_row_majorP8eigenmatS0_S0_",
    "get_logistic_correct_normalized": "_Z31get_logistic_correct_normalizedP8eigenmatS0_S0_",
}


class EigenMat(ct.Structure):
    _fields_ = [("data", ct.POINTER(ct.c_float)), ("size", ct.c_int * 2), ("is_trans", ct.c_int), ("owns_data", ct.c_int)]


def _mat(a):
    """an eigenmat view of the Fortran-ordered float32 array a (rows x cols)"""
    assert a.dtype == np.float32 and a.flags.f_contiguous
    m = EigenMat()
    m.data = a.ctypes.data_as(ct.POINTER(ct.c_float))
    m.size[0], m.size[1] = a.shape if a.ndim == 2 else (a.shape[0], 1)
    m.is_trans, m.owns_data = 0, 0
    return m


def reference_functions(lib_path=REF_LIB):
    """{name: f(*arrays[, tiny]) -> result array}, each f calling the eigenmat function of that name"""
    L = ct.CDLL(lib_path)
    P = ct.POINTER(EigenMat)

    def fn(name, nmat, tiny=False):
        f = getattr(L, SYMBOLS[name])
        f.argtypes, f.restype = [P] * nmat + ([ct.c_float] if tiny else []), ct.c_int
        return f

    def call(name, args, out_shape, tiny=None):
        out = np.zeros(out_shape, np.float32, order="F")
        keep = [np.asfortranarray(a, dtype=np.float32) for a in args]
        mats = [_mat(a) for a in keep] + [_mat(out)]
        f = fn(name, len(mats), tiny is not None)
        rc = f(*[ct.byref(m) for m in mats], *([tiny] if tiny is not None else []))
        assert rc == 0, (name, rc)
        return out

    return {
        "sigmoid": lambda x: call("apply_sigmoid", [x], x.shape),
        "logistic_deriv": lambda d, s: call("apply_logistic_deriv", [d, s], d.shape),
        "logistic_grad": lambda y, t: call("apply_logistic_grad", [y, t], y.shape),
        "cross_entropy": lambda q, p: call("compute_cross_entropy", [q, p], q.shape, 1e-10),
        "cross_entropy_bernoulli": lambda t, y: call("compute_cross_entropy_bernoulli", [t, y], t.shape, 1e-10),
        "softmax_correct": lambda p, lab: call("get_softmax_correct_row_major", [p, lab.reshape(-1, 1)], (p.shape[0], 1)),
        "logistic_correct": lambda y, t: call("get_logistic_correct_normalized", [y, t], (y.shape[0], 1)),
    }


def inputs(seed=20141015):
    rng = np.random.default_rng(seed)
    f = lambda a: np.asfortranarray(np.asarray(a, np.float32))
    x = rng.standard_normal((ROWS, COLS)) * 6
    x.flat[:8] = [0, -0.0, 30, -30, 90, -90, 1e-6, -1e-6]
    y = rng.uniform(0, 1, (ROWS, COLS))
    t = (rng.uniform(0, 1, (ROWS, COLS)) < 0.5).astype(np.float64)
    t[rng.uniform(0, 1, (ROWS, COLS)) < 0.2] = -1          # don't care
    t[3, :] = -1                                            # an image with no target at all
    t[:, 0] = rng.uniform(0, 1, ROWS)                       # soft binary targets too
    logits = rng.standard_normal((ROWS, COLS)) * 3
    p = np.exp(logits - logits.max(1, keepdims=True)); p /= p.sum(1, keepdims=True)
    q = rng.uniform(0, 1, (ROWS, COLS)); q /= q.sum(1, keepdims=True)
    labels = rng.integers(0, COLS, ROWS)
    labels[:ROWS // 2] = p[:ROWS // 2].argmax(1)            # half of them right
    return {"x": f(x), "d": f(rng.standard_normal((ROWS, COLS))), "s": f(y), "y": f(y), "t": f(t), "p": f(p), "q": f(q),
            "labels": f(labels)}


def generate(lib_path=REF_LIB):
    ref = reference_functions(lib_path)
    a = inputs()
    tb = np.asfortranarray(np.maximum(a["t"], 0).astype(np.float32))
    out = dict(a)
    out.update(sigmoid=ref["sigmoid"](a["x"]), logistic_deriv=ref["logistic_deriv"](a["d"], a["s"]),
               logistic_grad=ref["logistic_grad"](a["y"], a["t"]), cross_entropy=ref["cross_entropy"](a["q"], a["p"]),
               cross_entropy_bernoulli=ref["cross_entropy_bernoulli"](tb, a["y"]),
               softmax_correct=ref["softmax_correct"](a["p"], a["labels"]).ravel(),
               logistic_correct=ref["logistic_correct"](a["y"], a["t"]).ravel())
    return out


if __name__ == "__main__":
    np.savez(OUT, **generate())
    print("wrote", OUT)
