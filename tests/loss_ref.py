"""float64 restatements of the logistic unit and the output-layer rules (include/convnet_b200_ext.h: cnb_logistic,
cnb_logistic_deriv, cnb_loss_deriv, cnb_metric), and the per-element bars their documented float32 arithmetic implies.

Arrays are [images x columns] (numpy row = image).  Bars (u = 2^-24, the unit roundoff of float32):
  sigma        |y - sigma(x)| <= 6u * sigma(x) + 2^-126        expf within 2 ulp, then one rounded add and divide
  sigma'       |r - d s (1 - s)| <= 3u * |d s (1 - s)| + 2^-148 three rounded operations
  derivative   y - t and (y - onehot) are one rounded subtraction, times w one more: <= 2u * |(y - t) w| (exact for w = 1)
  per image    a left-to-right float sum of `cols` terms c * log(a) (or (y - t)^2 / 2, y - t).  The argument a = y + 1e-10
               (or 1 - y + 1e-10) carries <= 2u relative error, which log turns into <= 2u ABSOLUTE error, logf adds
               <= 1 ulp and the product one rounding: |term error| <= 4u * |c| * (|log a| + 1) =: 4u * m.  With the
               sum's rounding: |v - ref| <= (cols + 8) * 2u * sum m  (+ 1e-30 absolute)
"""
import numpy as np

U = 2.0 ** -24
TINY = 1e-10


def sigmoid(x):
    return 1.0 / (1.0 + np.exp(-np.asarray(x, np.float64)))


def sigmoid_bar(x):
    return 6 * U * sigmoid(x) + 2.0 ** -126


def logistic_deriv(d, s):
    d, s = np.asarray(d, np.float64), np.asarray(s, np.float64)
    return d * s * (1 - s)


def logistic_deriv_bar(d, s):
    return 3 * U * np.abs(logistic_deriv(d, s)) + 2.0 ** -148


def onehot(labels, cols):
    o = np.zeros((len(labels), cols))
    o[np.arange(len(labels)), np.asarray(labels, np.int64)] = 1
    return o


# loss / metric codes (proto LossFunction numbers)
SQUARED_ERROR, LINEAR_ERROR, CE_MULTINOMIAL, CE_BINARY, CE_DISTRIBUTED, CLASS_MULTINOMIAL, CLASS_BINARY = range(7)


def loss_terms(loss, y, t=None, labels=None):
    """(derivative before the weight, per-element terms of the per-image value, their error magnitudes m) in float64"""
    y = np.asarray(y, np.float64)
    if loss == CE_MULTINOMIAL:
        oh = onehot(labels, y.shape[1])
        terms, mags = np.zeros_like(y), np.zeros_like(y)
        idx = (np.arange(len(y)), np.asarray(labels, np.int64))
        terms[idx] = -np.log(np.maximum(y[idx], 1e-30))
        mags[idx] = np.abs(terms[idx]) + 1
        return y - oh, terms, mags
    t = np.asarray(t, np.float64)
    if loss == SQUARED_ERROR:
        return y - t, 0.5 * (y - t) ** 2, (y - t) ** 2
    if loss == LINEAR_ERROR:
        return np.ones_like(y), y - t, np.abs(y - t)
    if loss == CE_BINARY:
        care = t >= 0
        l1, l0 = np.log(y + TINY), np.log(1 - y + TINY)
        terms = np.where(care, -t * l1 - (1 - t) * l0, 0.0)
        mags = np.where(care, np.abs(t) * (np.abs(l1) + 1) + np.abs(1 - t) * (np.abs(l0) + 1), 0.0)
        return np.where(care, y - t, 0.0), terms, mags
    if loss == CE_DISTRIBUTED:
        l1 = np.log(y + TINY)
        return y - t, -t * l1, np.abs(t) * (np.abs(l1) + 1)
    raise ValueError(loss)


def loss_ref(loss, y, t=None, labels=None, weight=1.0):
    """(derivative, its bar, per-image loss, its bar)"""
    g, terms, mags = loss_terms(loss, y, t, labels)
    d = g * weight
    d_bar = 2 * U * np.abs(d)
    v = terms.sum(1)
    v_bar = (terms.shape[1] + 8) * 2 * U * mags.sum(1) + 1e-30
    return d, d_bar, v, v_bar


def classification_multinomial(y, labels):
    """kSoftMaxCorrectRowMajor's decision (32 threads): per lane the first strict maximum of its columns, then the lanes in
    order, strictly; starting values -FLT_MAX"""
    y = np.asarray(y, np.float32)
    out = np.zeros(len(y))
    fmax = np.float32(-3.402823466e38)
    for n in range(len(y)):
        lane_m, lane_a = [], []
        for j in range(32):
            m, a = fmax, 0
            for c in range(j, y.shape[1], 32):
                if y[n, c] > m:
                    m, a = y[n, c], c
            lane_m.append(m); lane_a.append(a)
        bm, ba = fmax, 0
        for m, a in zip(lane_m, lane_a):
            if m > bm:
                bm, ba = m, a
        out[n] = 1.0 if ba == int(labels[n]) else 0.0
    return out


def classification_binary(y, t):
    y, t = np.asarray(y, np.float32), np.asarray(t, np.float32)
    care = t >= 0
    correct = (care & (((t >= 0.5) & (y >= 0.5)) | ((t < 0.5) & (y < 0.5)))).sum(1)
    total = care.sum(1)
    return np.where(total > 0, correct / np.maximum(total, 1), 0.0)
