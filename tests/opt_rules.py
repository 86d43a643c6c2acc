"""float32 numpy restatement of the update of cnb_opt_update_multi (include/convnet_b200_ext.h), in the kernel's operation
order: every operation rounded to nearest in float32, fma the one fused operation.  Bit-for-bit the kernel's result,
except for rows a norm rule rescales (their scale comes from a fixed-order sum of squares on the device)."""
import numpy as np

f32 = np.float32
SGD, ADAGRAD, RMSPROP = 0, 1, 2
NONE, LIMIT, CONSTRAINT = 0, 1, 2


def fma32(a, b, c):
    """float32 fma(a, b, c) rounded once: a*b is exact in float64; the float64 sum is rounded to odd (TwoSum gives its
    error), and rounding that to float32 is the correctly rounded result (53 >= 24 + 2 bits)"""
    a, b, c = (np.asarray(x, np.float32).astype(np.float64) for x in (a, b, c))
    with np.errstate(invalid="ignore", over="ignore"):
        p = a * b
        s = p + c
        bb = s - p
        err = (p - (s - bb)) + (c - bb)
        even = (s.view(np.int64) & 1) == 0
        fix = (err != 0) & even & np.isfinite(s)
        s = np.where(fix, np.nextafter(s, np.where(err > 0, np.inf, -np.inf)), s)
    return s.astype(np.float32)


def safe_div(x, s):
    """x / s, and 0 where x is 0"""
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.where(x == 0, f32(0), x / s).astype(np.float32)


def adagrad_state(s, g, delta):
    """kAdagrad: delta + sqrt((s - delta)^2 + g^2)"""
    delta = f32(delta)
    e = s - delta
    return (delta + np.sqrt(e * e + g * g)).astype(np.float32)


def rms_prop_state(s, g, factor):
    """kRMSProp: sqrt((f*s)*s + ((1-f)*g)*g)"""
    f = f32(factor)
    return np.sqrt((f * s) * s + ((f32(1) - f) * g) * g).astype(np.float32)


def opt_update(w, h, s, g, rule=SGD, lr=0.0, mom=0.0, l2=0.0, clip=0.0, param=0.0, scale=1.0, state_only=False):
    """one update of a tensor without a norm rule (or before its rescale); returns new (w, h, s) as float32 arrays"""
    w, h, g = (np.array(x, np.float32) for x in (w, h, g))
    s = None if s is None else np.array(s, np.float32)
    if rule == ADAGRAD:
        s = adagrad_state(s, g, param)
        if state_only:
            return w, h, s
        g = safe_div(g, s) * f32(scale)
    d = fma32(f32(l2), w, g)
    if clip > 0:
        c = f32(clip)
        d = np.where(d > c, c, np.where(d < -c, -c, d)).astype(np.float32)
    if rule == RMSPROP:
        s = rms_prop_state(s, d, param)
        d = safe_div(d, s)
    h = fma32(f32(mom), h, f32(lr) * d)
    w = (w - h).astype(np.float32)
    return w, h, s


def apply_norm(w, rows, mode, value):
    """the row-norm rule on updated weights (rows fastest), norms in float64: the rescaled rows agree with the kernel's to
    a few ulp; returns (w, mask of the rescaled rows)"""
    m = w.astype(np.float64).reshape(-1, rows)
    if mode == NONE:
        return w, np.zeros(rows, bool)
    nrm = np.sqrt((m * m).sum(axis=0))
    bite = (nrm > 0) & ((nrm > value) if mode == LIMIT else True)
    out = m.copy()
    out[:, bite] *= value / nrm[bite]
    return np.where(np.broadcast_to(bite, m.shape), out, m).astype(np.float32).reshape(-1), bite


def adagrad_scale(step):
    """gradient.Mult(sqrt(step_ + 1)): the square root of an int in double, used as a float"""
    return float(f32(np.sqrt(float(step + 1))))
