#!/usr/bin/env python3
"""Write tests/golden/ref_elementwise.npz: softmax, ReLU and the batch-norm sequence of the reference, computed by the
reference's own CPU library (eigenmat/eigenmat.cc, oracle/_ref/libeigenmat_ref.so) on seeded inputs, called through
the ctypes mirror of tools/gen_loss_golden.py.

Matrices are column-major, images (softmax) or the n values of a channel (batch norm) fastest.  Keys:
  sm_x, sm_p        softmax_row_major_multi(x, cols) on [SM_ROWS x SM_COLS] (the layout Matrix::ApplySoftmax uses)
  relu_x, relu_y    lower_bound_scalar(x, 0)
  bn_x [n x C], bn_gamma, bn_beta, bn_d, bn_eps, and the sequence of Layer::ApplyBatchNormalization (train) and
  ApplyDerivativeofBatchNormalization (src/layer.cc:452-510):
    bn_mu      sum_by_axis(x, axis 0, 1/n)
    bn_sigma   sqsum_by_axis(x - mu, axis 0, 1/n), add_scalar(eps), apply_sqrt
    bn_y       add_row_vec(div_by_row_vec(x - mu, sigma) * gamma (mult_by_row_vec), beta)
    bn_grad_beta   sum_by_axis(d, axis 0, 1/n)
    bn_grad_gamma, bn_dx   bn_bprop_inplace(d, xhat) (restated, see below), mult_by_row_vec(gamma), div_by_row_vec(sigma)
  Channel 0 of bn_x sits at mean 1e3 with sd 1e-2 (the large-offset channel); n is ragged.

    python tools/gen_elementwise_golden.py      (needs oracle/_ref/libeigenmat_ref.so)"""
import ctypes as ct
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from gen_loss_golden import REF_LIB, ROOT, EigenMat, _mat  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "ref_elementwise.npz")
SM_ROWS, SM_COLS = 37, 1001
BN_N, BN_C = 3001, 5

SYMBOLS = {
    "softmax_row_major_multi": "_Z23softmax_row_major_multiP8eigenmati",
    "lower_bound_scalar": "_Z18lower_bound_scalarP8eigenmatfS0_",
    "sum_by_axis": "_Z11sum_by_axisP8eigenmatS0_iff",
    "sqsum_by_axis": "_Z13sqsum_by_axisP8eigenmatS0_iff",
    "add_row_vec": "_Z11add_row_vecP8eigenmatS0_S0_",
    "add_scalar": "_Z10add_scalarP8eigenmatfS0_",
    "apply_sqrt": "_Z10apply_sqrtP8eigenmatS0_",
    "div_by_row_vec": "_Z14div_by_row_vecP8eigenmatS0_S0_",
    "mult_by_row_vec": "_Z15mult_by_row_vecP8eigenmatS0_S0_",
}


def _f(a):
    return np.asfortranarray(np.asarray(a, np.float32))


def bn_bprop_inplace(d, xh):
    """eigenmat's bn_bprop_inplace restated in float32 with its sequential sums: stat = sum(d * xh) / n is dgamma,
    d -= stat * xh, then d -= sum(d) / n.  The library's own symbol cannot be called: the function has no return
    statement, and the optimised build runs off its end."""
    n = d.shape[0]
    d = d.copy(order="F")
    gg = np.zeros((1, d.shape[1]), np.float32)
    for c in range(d.shape[1]):
        stat = np.cumsum(d[:, c] * xh[:, c], dtype=np.float32)[-1] / np.float32(n)
        gg[0, c] = stat
        d[:, c] = d[:, c] - stat * xh[:, c]
        d[:, c] = d[:, c] - np.cumsum(d[:, c], dtype=np.float32)[-1] / np.float32(n)
    return d, gg


def generate(lib_path=REF_LIB):
    L = ct.CDLL(lib_path)
    P = ct.POINTER(EigenMat)

    def fn(name, *args):
        f = getattr(L, SYMBOLS[name])
        f.argtypes, f.restype = list(args), ct.c_int
        return f

    def row(v):                                          # a 1 x C row vector
        return _f(np.asarray(v, np.float32).reshape(1, -1))

    def call(name, argtypes, *args, check=True):
        rc = fn(name, *argtypes)(*args)
        assert not check or rc == 0, (name, rc)

    rng = np.random.default_rng(20141016)
    out = {}
    # softmax
    x = _f(rng.standard_normal((SM_ROWS, SM_COLS)) * 3)
    x[1, :] = 2.5                                        # an image of equal logits
    x[2, 7] = x[2].max() + 200                           # a one-hot image
    p = x.copy(order="F")
    m = _mat(p)
    call("softmax_row_major_multi", [P, ct.c_int], ct.byref(m), SM_COLS)
    out.update(sm_x=x, sm_p=p)
    # ReLU
    rx = _f(rng.standard_normal((SM_ROWS, 21)))
    rx.flat[:4] = [0.0, -0.0, 1e-45, -1e-45]
    ry = np.zeros_like(rx, order="F")
    a, b = _mat(rx), _mat(ry)
    call("lower_bound_scalar", [P, ct.c_float, P], ct.byref(a), 0.0, ct.byref(b))
    out.update(relu_x=rx, relu_y=ry)
    # batch norm
    bx = rng.standard_normal((BN_N, BN_C)) * rng.uniform(0.5, 3, BN_C) + rng.uniform(-2, 2, BN_C)
    bx[:, 0] = 1e3 + 1e-2 * rng.standard_normal(BN_N)
    bx = _f(bx)
    gamma, beta = row(rng.uniform(0.5, 1.5, BN_C)), row(rng.standard_normal(BN_C))
    d = _f(rng.standard_normal((BN_N, BN_C)))
    eps = np.float32(1e-5)
    V = [P, P, ct.c_int, ct.c_float, ct.c_float]
    mu = row(np.zeros(BN_C))
    xm, mx = _mat(bx), _mat(mu)
    call("sum_by_axis", V, ct.byref(xm), ct.byref(mx), 0, np.float32(1.0 / BN_N), 0.0)
    xc = np.zeros_like(bx, order="F")
    neg = row(-mu)
    call("add_row_vec", [P, P, P], ct.byref(_mat(bx)), ct.byref(_mat(neg)), ct.byref(_mat(xc)))
    sigma = row(np.zeros(BN_C))
    call("sqsum_by_axis", V, ct.byref(_mat(xc)), ct.byref(_mat(sigma)), 0, np.float32(1.0 / BN_N), 0.0)
    call("add_scalar", [P, ct.c_float, P], ct.byref(_mat(sigma)), eps, ct.byref(_mat(sigma)))
    call("apply_sqrt", [P, P], ct.byref(_mat(sigma)), ct.byref(_mat(sigma)))
    xh = np.zeros_like(bx, order="F")
    call("div_by_row_vec", [P, P, P], ct.byref(_mat(xc)), ct.byref(_mat(sigma)), ct.byref(_mat(xh)))
    y = np.zeros_like(bx, order="F")
    call("mult_by_row_vec", [P, P, P], ct.byref(_mat(xh)), ct.byref(_mat(gamma)), ct.byref(_mat(y)))
    call("add_row_vec", [P, P, P], ct.byref(_mat(y)), ct.byref(_mat(beta)), ct.byref(_mat(y)))
    gb = row(np.zeros(BN_C))
    call("sum_by_axis", V, ct.byref(_mat(d)), ct.byref(_mat(gb)), 0, np.float32(1.0 / BN_N), 0.0)
    dx, gg = bn_bprop_inplace(d, xh)
    call("mult_by_row_vec", [P, P, P], ct.byref(_mat(dx)), ct.byref(_mat(gamma)), ct.byref(_mat(dx)))
    call("div_by_row_vec", [P, P, P], ct.byref(_mat(dx)), ct.byref(_mat(sigma)), ct.byref(_mat(dx)))
    out.update(bn_x=bx, bn_gamma=gamma.ravel(), bn_beta=beta.ravel(), bn_d=d, bn_eps=np.float32(eps),
               bn_mu=mu.ravel(), bn_sigma=sigma.ravel(), bn_y=y, bn_grad_beta=gb.ravel(), bn_grad_gamma=gg.ravel(),
               bn_dx=dx)
    return out


if __name__ == "__main__":
    np.savez(OUT, **generate())
    print("wrote", OUT)
