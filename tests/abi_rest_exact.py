"""Float64 restatements, per-element bars and a dispatch mirror of the max-pool and cross-map R-operators, within-map
normalisation and its undo, the RGB -> YUV transform and the filter-tap inner products of convInnerpGemm
(csrc/pool.cu, rnorm.cu, mapnorm.cu, conv_simt.cu).

Conventions as in tests/pool_exact.py: layout a[n + N*(x + W*(y + H*c))], torch float64 on the device of the inputs,
u = 2^-24, positive paddings (GetConvDesc).  Every restatement is the exact expression on the kernel's own fp32 operands
(where a kernel output feeds a second output, e.g. the stored denoms of ResponseNorm, the second is restated on the
stored value), and the bar charges each fp32 rounding of the kernel once, times a safety factor of 2.

* max-pool R-op: st * t0 + the sum of R over the window elements equal to the stored maximum.  m terms summed in order:
  |y - ref| <= (m + 2) u (|st t0| + sum|terms|).  Dyadic inputs make every partial sum exact: bar 0.
* cross-map R-op t_j = R_j base^-b - 2ab x_j base^(-b-1) sum_{window(j)} x_i R_i: the bars of pool_exact.rnorm_undo,
  with both window sums (of x^2 and of x R) charged on their prefix mass.
* within-map forward: denoms = 1 + a * sum_{sizeX x sizeX window} md^2 as row sums then column sums (at most 2 sizeX
  terms deep): |d - ref| <= (2 sizeX + 3) u (1 + a sum md^2); targets = images * d^-b on the stored d: e_pow + 2u.
* within-map undo: inputs * (-2ab) * sum_{inverse window} acts * og / denoms + og * denoms^-b; each term two roundings,
  the sum 2 sizeX deep, then three products and one addition.
* RGB -> YUV: three products of fp32 coefficients, two additions (or fused): 4 u sum|c x|.
* convInnerp: st * t0 + so * sum over (n, module, channel): per-thread sums of `per_thread` terms, a 5-level warp tree,
  8 warp sums, then `splits` partial sums: (per_thread + 13 + splits + 3) u (|st t0| + |so| sum|terms|).
"""
import torch

import pool_exact as px
from pool_exact import PG, U, Expect, e_pow

SAFETY = 2.0
SMS = 132


def _zeros_bool(n, dev):
    return torch.zeros(n, dtype=torch.bool, device=dev)


# ---------------------------------------------------------------------------------------------------------------------
# max-pool R-operator
# ---------------------------------------------------------------------------------------------------------------------
def max_rprop(g, x, R, maxes, st=0.0, t0=None, exact_arm=False):
    X = px._vol(x.to(torch.float64), g, False)
    RR = px._vol(R.to(torch.float64), g, False)
    M = px._vol(maxes.to(torch.float64), g, True)
    acc = torch.zeros_like(M)
    mag = torch.zeros_like(M)
    terms = torch.zeros_like(M)
    for dt, dy, dx in px._offsets(g):
        v, valid, *_ = px._gather(X, g, dt, dy, dx)
        r, *_ = px._gather(RR, g, dt, dy, dx)
        tie = valid & (v == M)
        c = torch.where(tie, r, torch.zeros_like(r))
        acc, mag, terms = acc + c, mag + c.abs(), terms + tie.to(torch.float64)
    if st != 0.0:
        old = st * px._vol(t0.to(torch.float64), g, True)
        acc, mag = acc + old, mag + old.abs()
    bar = torch.zeros_like(acc) if exact_arm else SAFETY * (terms + 2) * U * mag
    return Expect(acc.reshape(-1), bar.reshape(-1), _zeros_bool(acc.numel(), acc.device))


# ---------------------------------------------------------------------------------------------------------------------
# cross-map R-operator
# ---------------------------------------------------------------------------------------------------------------------
def rnorm_rprop(x, R, F, k, alpha, beta, blocked):
    X, S, base, dS = px._rn_parts(x, F, k, alpha, beta, blocked, 1, None)
    RR = R.to(torch.float64).reshape(1, F, -1)
    xr = X * RR
    Sxr = px._window_sum(xr, k, blocked, False)
    lo, hi = px._windows(F, k, blocked, False, X.device)
    cS = (2 * hi + k + 10).to(torch.float64).view(1, -1, 1)
    dSxr = cS * U * px._prefix(xr.abs()).index_select(1, hi)
    c2 = 2.0 * alpha * beta
    den = base ** (-beta - 1)
    p = RR * base ** -beta
    q = c2 * X * den * Sxr
    ref = p - q
    ep = e_pow(beta + 1, base) + (2 * beta + 5) * U
    bar = SAFETY * (p.abs() * ep + RR.abs() * beta * alpha * den * dS
                    + q.abs() * (ep + 4 * U) + (c2 * X).abs() * (beta + 1) * alpha * base ** (-beta - 2) * dS * Sxr.abs()
                    + (c2 * X * den).abs() * dSxr + 2 * U * (p.abs() + q.abs()))
    return Expect(ref.reshape(-1), bar.reshape(-1), _zeros_bool(ref.numel(), ref.device))


# ---------------------------------------------------------------------------------------------------------------------
# within-map normalisation
# ---------------------------------------------------------------------------------------------------------------------
def map_window(S, sizeX, inverse, dev):
    """[lo, hi) of every pixel along one axis: window (kCNorm_*) or inverse window (kRNormUndo), clipped"""
    p = torch.arange(S, device=dev)
    off = sizeX // 2 - sizeX + 1 if inverse else -(sizeX // 2)
    return (p + off).clamp(0, S), (p + off + sizeX).clamp(0, S)


def _box(v, S, sizeX, inverse):
    """float64 sums of v (F, S_y, S_x, N) over the window of every pixel (direct, via 2-D prefix sums in float64)"""
    dev = v.device
    lo, hi = map_window(S, sizeX, inverse, dev)
    c = torch.nn.functional.pad(v.cumsum(1).cumsum(2), (0, 0, 1, 0, 1, 0))     # exclusive 2-D prefix, exact enough in f64
    def at(yi, xi):
        return c[:, yi][:, :, xi]
    return at(hi, hi) - at(lo, hi) - at(hi, lo) + at(lo, lo)


def _maps(t, N, S, F):
    return t.to(torch.float64).reshape(F, S, S, N)


def mapnorm_denoms(md, N, S, F, sizeX, alpha):
    M = _maps(md, N, S, F)
    s = _box(M * M, S, sizeX, False)
    ref = 1.0 + alpha * s
    bar = SAFETY * (2 * sizeX + 3) * U * ref.abs()
    return Expect(ref.reshape(-1), bar.reshape(-1), _zeros_bool(ref.numel(), ref.device))


def mapnorm_targets(images, denoms_stored, beta):
    d = denoms_stored.to(torch.float64)
    ref = images.to(torch.float64) * d ** -beta
    bar = SAFETY * ref.abs() * (e_pow(beta, d) + 2 * U)
    return Expect(ref.reshape(-1), bar.reshape(-1), _zeros_bool(ref.numel(), ref.device))


def mapnorm_undo(outGrads, denoms, inputs, acts, N, S, F, sizeX, alpha, beta):
    og, dn, inp, ac = (_maps(t, N, S, F) for t in (outGrads, denoms, inputs, acts))
    v = ac * og / dn
    s = _box(v, S, sizeX, True)
    mag = _box(v.abs(), S, sizeX, True)
    c2 = -2.0 * alpha * beta
    q = inp * c2 * s
    p = og * dn ** -beta
    ref = q + p
    bar = SAFETY * ((c2 * inp).abs() * (2 * sizeX + 7) * U * mag + p.abs() * (e_pow(beta, dn) + 2 * U) + U * ref.abs())
    return Expect(ref.reshape(-1), bar.reshape(-1), _zeros_bool(ref.numel(), ref.device))


# ---------------------------------------------------------------------------------------------------------------------
# RGB -> YUV
# ---------------------------------------------------------------------------------------------------------------------
YUV = [[0.2126, 0.7152, 0.0722], [-0.09991, -0.33609, 0.436], [0.615, -0.55861, -0.05639]]


def rgb_to_yuv(images):
    """images: flat (3, pixels * N) planes"""
    x = images.to(torch.float64).reshape(3, -1)
    c = torch.tensor(YUV, dtype=torch.float32).to(torch.float64).to(x.device)     # the kernel's fp32 coefficients
    ref = c @ x
    bar = SAFETY * 4 * U * (c.abs() @ x.abs())
    return Expect(ref.reshape(-1), bar.reshape(-1), _zeros_bool(ref.numel(), ref.device))


# ---------------------------------------------------------------------------------------------------------------------
# convInnerp
# ---------------------------------------------------------------------------------------------------------------------
def innerp_splits(N, pairs, sms=SMS):
    """the split count conv_innerp picks (about 16K image values per CTA, at most 2 x SMs CTAs)"""
    splits = min(max(1, -(-pairs * N // 16384)), 2 * sms)
    per = -(-pairs // splits)
    return -(-pairs // per), per


def innerp(g, images, derivs, st=0.0, t0=None, so=1.0, sms=SMS):
    """g: PG of the image -> module geometry (C = channels of both tensors); derivs (modY, modX) maps"""
    X = px._vol(images.to(torch.float64), g, False)
    D = px._vol(derivs.to(torch.float64), g, True)
    ref = torch.zeros(g.ky, g.kx, dtype=torch.float64, device=X.device)
    mag = torch.zeros_like(ref)
    for dt, dy, dx in px._offsets(g):
        v, valid, *_ = px._gather(X, g, dt, dy, dx)
        prod = torch.where(valid, v * D, torch.zeros_like(v))
        ref[dy, dx] = prod.sum()
        mag[dy, dx] = prod.abs().sum()
    splits, per = innerp_splits(g.N, g.C * g.modX * g.modY, sms)
    depth = -(-per * g.N // 256) + 13 + splits + 3
    ref, mag = so * ref, abs(so) * mag
    if st != 0.0:
        old = st * t0.to(torch.float64).reshape(g.ky, g.kx)
        ref, mag = ref + old, mag + old.abs()
    bar = SAFETY * depth * U * mag
    return Expect(ref.reshape(-1), bar.reshape(-1), _zeros_bool(ref.numel(), ref.device))


# ---------------------------------------------------------------------------------------------------------------------
# dispatch mirror
# ---------------------------------------------------------------------------------------------------------------------
def max_rprop_branch(N, aligned=True):
    return "pool_rprop_kernel<%d>" % (4 if N % 4 == 0 and aligned else 1)


def rnorm_rprop_branch(L, F, blocked, aligned=True):
    tl = px.pick_tile(F, 4)
    if tl:
        return "rnorm_tile_kernel<%d, (cnb::RnPass)2>" % tl, ("vec" if L % 4 == 0 and aligned else "scalar")
    return "rnorm_rprop_kernel<%s>" % ("true" if blocked else "false"), "ring"


def mapnorm_branch(N, undo, aligned=True):
    return "mapnorm_kernel<%s, %d>" % ("true" if undo else "false", 4 if N % 4 == 0 and aligned else 1)


def mapnorm_width(S, sizeX, vec):
    R = min(sizeX, S) + 1
    ti = 16 if vec else 8
    while ti > (4 if vec else 1) and 4 * (R + 1) * S * ti > 200 * 1024:
        ti //= 2
    return ti


def innerp_launches(N, pairs, sms=SMS):
    splits, _ = innerp_splits(N, pairs, sms)
    return 1 if splits == 1 else 2


def yuv_branch(n_per_plane, aligned=True):
    return "rgb_to_yuv_kernel<%d>" % (4 if n_per_plane % 4 == 0 and aligned else 1)


def alexnet_shapes(N):
    """AlexNet's hidden1_maxpool (110 x 110 x 96 -> 55 x 55, 3 x 3 stride 2 pad 1) and hidden1_rnorm (55 x 55 x 96)"""
    return PG(N, 110, 110, 96, 3, 3, 2, 2, 1, 1), (N, 55, 55, 96)
