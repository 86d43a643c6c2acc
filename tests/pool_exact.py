"""Float64 references of pooling and cross-map response normalisation, the per-element bar of each op, and a mirror
of the kernel dispatch of csrc/pool.cu and csrc/rnorm.cu.

Layout (DESIGN.md §3): a[n + N*(x + W*(y + H*c))], 3-D tensors stack frames as channel blocks (channel c + C*t).  Every
reference is torch float64 on the device of its inputs.  Paddings are POSITIVE here (GetConvDesc convention); the
kernels see them negated.  u = 2^-24 is the unit roundoff of fp32; a sum of m fp32 terms in any order is within
gamma_{m-1} * sum|terms| of the exact sum (gamma_n = n*u / (1 - n*u) <= (n + 1)*u for the n here), and every other fp32
operation adds one relative u.

Bars, per output element:

* max forward: BIT-EXACT.  The maximum of fp32 values is one of them, and so * max is one rounding of an exact float64
  product (24 + 24 bits fit in 53), so ref rounded to fp32 is the kernel's value.  The tie decision of the max undo
  compares the same fp32 values (the pool input and the kernel's own max output) in float64: also exact.
* empty windows (padding >= kernel): the reference's kPool divides by (end - start) products of the CLIPPED bounds,
  which are <= 0 there: the average is so * (0 / region), i.e. NaN when a factor is 0 and a signed zero otherwise, and
  the maximum is so * -2e38 (gemm.cu:71, :185).  Pinned bit for bit.
* avg forward: m window terms summed (m - 1 roundings), one division, one scaling:
      |y - ref| <= (m + 2) u |so| sum|x| / region.
* max / avg undo: the m covering windows each contribute a term (max: so*g where the element ties the window's
  maximum; avg: so*g/region, two roundings), then st * old is added and the ReLU' mask applied:
      |y - ref| <= (m + 4) u (sum|terms| + |st * old|),
  and elements the mask drops are exactly 0.  EXACT ARM: with dyadic inputs (multiples of 2^-4 of size <= 8, st and so
  powers of two, max pooling) every product and partial sum is an fp32 number, so the bar is 0: y must EQUAL float64.
  A dropped, duplicated or misplaced term fails it however small it is.
* bias gradient (st_b * b + so_b * sum over images and pixels of the STORED target): compared with the float64 sum of
  the kernel's own fp32 target, so only the summation is charged.  The depth of the sum is the values one thread adds
  (`per_thread`), the 5-level warp tree, the 8 warps of a CTA and the `slices` partial sums colsum_finish adds (per
  slice sums of the row kernels; up to 64 slices of cnb_channel_bias_grad), plus st*b, so*s and their sum:
      |y - ref| <= (per_thread + 13 + slices + 3) u (|st_b * b| + |so_b| sum|target|).
  Exact arm as above.
* response norm, forward y_j = x_j * base_j^-beta, base_j = 1 + alpha * S_j, S_j the sum of x_i^2 over the window
  [j - a, j + b] (a = k/2, b = k - a - 1) or the block of k channels holding j:
  - __powf.  The CUDA C++ Programming Guide (Intrinsic Functions, single precision) gives the error of __powf(x, y) as
    "derived from its implementation as exp2f(y * __log2f(x))", with __log2f: "for x in [0.5, 2], the maximum absolute
    error is 2^-22, otherwise, the maximum ulp error is 2", and exp2f: "the maximum ulp error is 2".  So for base >= 1
      e_pow(y, base) = ln2 |y| (2^-22 + 2^-22 |log2 base| + u |log2 base|) + 2^-22     (relative),
    and forming base (two roundings, scaled by beta) and x * pw add (2 beta + 1) u.
  - the window sum.  Both the reference's running add / subtract sum (kCrossMapRNorm) and this library's kernels take
    S from sums that run over EARLIER channels too: the tile kernel as Q[hi] - Q[lo] of an fp32 exclusive prefix over
    all channels (<= hi + 4 terms each, the 4 for the segment totals of rn_prefix), the ring kernels as a running sum
    that adds x_q^2 and subtracts the square leaving the window (every square sits in at most k running sums).  Either
    way the error of S is charged on the PREFIX MASS P_hi = sum_{i < hi} x_i^2, hi the end of the window:
      |dS| <= c_S u P_hi,   c_S = 2 hi + k + 10,
    and moves y by |x| beta alpha base^(-beta-1) |dS|.  A bar charged on the window's own mass is wrong: a channel
    whose window is cold but whose prefix holds hot channels (tests/test_pool_exact_cpu.py emulates the tile kernel on
    such an input) has an error far above it.
  - undo dx_j = p_j - 2 alpha beta x_j R_j, p_j = dy_j base_j^-beta, t_i = dy_i x_i base_i^(-beta-1), R_j the sum of t
    over the inverse window [j - b, j + a] (or the block): p and every t carry e_pow(-beta-1, base) + (2 beta + 5) u
    and the effect of their dS; R is a prefix difference / running sum of t, charged on the prefix mass of |t| with
    the same c_S.
  The bar is twice the first-order sum of these terms (the factor 2 covers the dropped second-order products, gamma_n
  against n u, and base^(-beta-1) taken at the reference's base instead of the kernel's).
* bf16 twins: bit-equal to the round-to-nearest-even bf16 of the fp32 output the kernel stored.
"""
import dataclasses
import math

import torch

from convnet_b200.abi import GetConvDesc, num_modules

U = 2.0 ** -24
MAX_BASE = -1.9999999360571348e+38        # float32(-2e38): the max-pool base value (gemm.cu:71)
RN_SAFETY = 2.0
SMS = 132                                  # H100 SXM; the mirror takes the live count where a GPU is present


# ---------------------------------------------------------------------------------------------------------------------
# geometry
# ---------------------------------------------------------------------------------------------------------------------
@dataclasses.dataclass
class PG:
    N: int
    W: int
    H: int
    C: int                   # channels per frame
    ky: int
    kx: int
    sy: int = 1
    sx: int = 1
    py: int = 0              # positive paddings
    px: int = 0
    T: int = 1               # frames
    kt: int = 1
    st_t: int = 1
    pt: int = 0

    @property
    def modX(self):
        return num_modules(self.W, self.kx, self.sx, self.px)

    @property
    def modY(self):
        return num_modules(self.H, self.ky, self.sy, self.py)

    @property
    def modT(self):
        return num_modules(self.T, self.kt, self.st_t, self.pt)

    @property
    def two_d(self):
        return self.kt == 1 and self.T == 1 and self.modT == 1

    def desc(self):
        return GetConvDesc(self.C, self.C, self.ky, self.kx, self.sy, self.sx, self.py, self.px,
                           kernel_size_t=self.kt, stride_t=self.st_t, padding_t=self.pt)

    def in_shape(self):
        return (self.N, self.W, self.H, self.C * self.T)

    def out_shape(self):
        return (self.N, self.modX, self.modY, self.C * self.modT)

    def in_dims(self):
        return self.N, self.W * self.H * self.C * self.T

    def out_dims(self):
        return self.N, self.modX * self.modY * self.C * self.modT


def _vol(a, g, out):
    """flat buffer -> (frames, C, H, W, N) view"""
    T, W, H = (g.modT, g.modX, g.modY) if out else (g.T, g.W, g.H)
    return a[: g.N * W * H * g.C * T].view(T, g.C, H, W, g.N)


def _axis(n, mods, k, s, p, d, dev):
    """input index of window offset d of every module along one axis, and whether it is inside the image"""
    i = torch.arange(mods, device=dev) * s - p + d
    return i.clamp(0, n - 1), (i >= 0) & (i < n)


def _count(n, mods, k, s, p, dev):
    """the reference's clipped extent per module: min(start + k, n) - max(start, 0) (<= 0 for an empty window)"""
    s0 = torch.arange(mods, device=dev) * s - p
    return (torch.clamp(s0 + k, max=n) - torch.clamp(s0, min=0)).to(torch.float64)


def _offsets(g):
    for dt in range(g.kt):
        for dy in range(g.ky):
            for dx in range(g.kx):
                yield dt, dy, dx


def _gather(X, g, dt, dy, dx):
    dev = X.device
    it, vt = _axis(g.T, g.modT, g.kt, g.st_t, g.pt, dt, dev)
    iy, vy = _axis(g.H, g.modY, g.ky, g.sy, g.py, dy, dev)
    ix, vx = _axis(g.W, g.modX, g.kx, g.sx, g.px, dx, dev)
    v = X.index_select(0, it).index_select(2, iy).index_select(3, ix)
    valid = vt.view(-1, 1, 1, 1, 1) & vy.view(1, 1, -1, 1, 1) & vx.view(1, 1, 1, -1, 1)
    return v, valid, (it, vt), (iy, vy), (ix, vx)


def _scatter(acc, contrib, ax):
    """add contrib (module-shaped) into acc (input-shaped) at the input positions of one window offset: for a fixed
    offset the module -> input map is injective along every axis, so index_add_ axis by axis is exact"""
    (it, vt), (iy, vy), (ix, vx) = ax
    c = contrib[:, :, :, vx]
    a1 = torch.zeros(c.shape[0], c.shape[1], c.shape[2], acc.shape[3], c.shape[4], dtype=acc.dtype, device=acc.device)
    a1.index_add_(3, ix[vx], c)
    c = a1[:, :, vy]
    a2 = torch.zeros(c.shape[0], c.shape[1], acc.shape[2], c.shape[3], c.shape[4], dtype=acc.dtype, device=acc.device)
    a2.index_add_(2, iy[vy], c)
    acc.index_add_(0, it[vt], a2[vt])


def region(g, dev):
    """(modT, 1, modY, modX, 1) clipped region sizes (gemm.cu:185), float64"""
    ct = _count(g.T, g.modT, g.kt, g.st_t, g.pt, dev).view(-1, 1, 1, 1, 1)
    cy = _count(g.H, g.modY, g.ky, g.sy, g.py, dev).view(1, 1, -1, 1, 1)
    cx = _count(g.W, g.modX, g.kx, g.sx, g.px, dev).view(1, 1, 1, -1, 1)
    return ct * cy * cx


@dataclasses.dataclass
class Expect:
    ref: torch.Tensor         # float64 flat, the whole target
    bar: torch.Tensor         # float64 flat absolute bound
    exact: torch.Tensor       # bool flat: must equal float32(ref) bit for bit (NaN: any NaN)


def _flat(t):
    return t.reshape(-1)


# ---------------------------------------------------------------------------------------------------------------------
# pooling
# ---------------------------------------------------------------------------------------------------------------------
def pool_fwd(g, x, is_max, so=1.0, fault=None):
    """max / avg pooling of flat fp32 x; fault (controls): 'shift' moves every window one pixel right, 'unclipped'
    divides by kx*ky*kt"""
    X = _vol(x.to(torch.float64), g, False)
    dev = X.device
    shape = (g.modT, g.C, g.modY, g.modX, g.N)
    acc = torch.full(shape, MAX_BASE if is_max else 0.0, dtype=torch.float64, device=dev)
    mag = torch.zeros(shape, dtype=torch.float64, device=dev)
    for dt, dy, dx in _offsets(g):
        v, valid, *_ = _gather(X, g, dt, dy, dx + (1 if fault == "shift" else 0))
        if is_max:
            acc = torch.where(valid, torch.maximum(acc, v), acc)
        else:
            acc = acc + torch.where(valid, v, torch.zeros_like(v))
            mag = mag + torch.where(valid, v.abs(), torch.zeros_like(v))
    if is_max:
        ref = so * acc
        bar = torch.zeros_like(ref)
        exact = torch.ones_like(ref, dtype=torch.bool)
    else:
        reg = region(g, dev).expand(shape)
        if fault == "unclipped":
            reg = torch.full_like(reg, float(g.kx * g.ky * g.kt))
        ref = so * (acc / reg)
        empty = ~(reg > 0)
        bar = torch.where(empty, torch.zeros_like(ref), (reg + 2) * U * abs(so) * mag / reg.clamp(min=1))
        exact = empty.clone()
    return Expect(_flat(ref), _flat(bar), _flat(exact))


def _finish_undo(g, acc, mag, terms, t0, st, mask, exact_arm):
    if st != 0.0:
        old = _vol(t0.to(torch.float64), g, False)
        acc = acc + st * old
        mag = mag + (st * old).abs()
    bar = (terms + 4) * U * mag
    if mask is not None:
        drop = ~(_vol(mask, g, False) > 0)
        acc = torch.where(drop, torch.zeros_like(acc), acc)
        bar = torch.where(drop, torch.zeros_like(bar), bar)
    if exact_arm:
        bar = torch.zeros_like(bar)
    return Expect(_flat(acc), _flat(bar), torch.zeros(acc.numel(), dtype=torch.bool, device=acc.device))


def max_undo(g, x, grads, acts, st=0.0, t0=None, so=1.0, mask=None, exact_arm=False, fault=None):
    """fault (controls): 'no_dup' gives a tied gradient to the first tying element of the window only;
    'drop_bit' drops window element (dx, dy) = (2, 2) (bit 8 of a 3 x 3 tie mask); 'mask_first' applies the ReLU'
    mask before adding st * old"""
    X = _vol(x.to(torch.float64), g, False)
    G = _vol(grads.to(torch.float64), g, True)
    A = _vol(acts.to(torch.float64), g, True)
    dev = X.device
    acc, mag, terms = torch.zeros_like(X), torch.zeros_like(X), torch.zeros_like(X)
    taken = torch.zeros(A.shape, dtype=torch.bool, device=dev)
    for dt, dy, dx in _offsets(g):
        v, valid, *ax = _gather(X, g, dt, dy, dx)
        tie = valid & (v == A)
        if fault == "no_dup":
            tie, taken = tie & ~taken, taken | tie
        if fault == "drop_bit" and (dx, dy) == (2, 2):
            tie = torch.zeros_like(tie)
        c = torch.where(tie, so * G, torch.zeros_like(G))
        _scatter(acc, c, ax)
        _scatter(mag, c.abs(), ax)
        _scatter(terms, tie.to(torch.float64), ax)
    if fault == "mask_first" and mask is not None:
        drop = ~(_vol(mask, g, False) > 0)
        acc = torch.where(drop, torch.zeros_like(acc), acc)
        e = _finish_undo(g, acc, mag, terms, t0, st, None, exact_arm)
        return e
    return _finish_undo(g, acc, mag, terms, t0, st, mask, exact_arm)


def avg_undo(g, grads, st=0.0, t0=None, so=1.0, mask=None, exact_arm=False, fault=None):
    """fault (controls): 'unclipped' divides by kx*ky*kt at the border"""
    G = _vol(grads.to(torch.float64), g, True)
    dev = G.device
    shape = (g.T, g.C, g.H, g.W, g.N)
    acc = torch.zeros(shape, dtype=torch.float64, device=dev)
    mag, terms = torch.zeros_like(acc), torch.zeros_like(acc)
    reg = region(g, dev)
    if fault == "unclipped":
        reg = torch.full_like(reg, float(g.kx * g.ky * g.kt))
    val = so * G / reg.clamp(min=1)
    for dt, dy, dx in _offsets(g):
        _, valid, *ax = _gather(acc, g, dt, dy, dx)
        c = torch.where(valid, val, torch.zeros_like(val))
        _scatter(acc, c, ax)
        _scatter(mag, c.abs(), ax)
        _scatter(terms, valid.to(torch.float64).expand(c.shape).contiguous(), ax)
    return _finish_undo(g, acc, mag, terms, t0, st, mask, exact_arm)


def bias_grad(y, rows_per_channel, C, frames, b0, st, so, per_thread, slices, exact_arm=False, fault=None):
    """y: the kernel's stored target (flat fp32, (frames, C, rows) blocks); fault 'drop_row' leaves out row 0"""
    Y = y[: frames * C * rows_per_channel].to(torch.float64).view(frames, C, rows_per_channel)
    if fault == "drop_row":
        Y = Y[:, :, 1:]
    s = Y.sum(dim=(0, 2))
    mag = Y.abs().sum(dim=(0, 2))
    b = b0.to(torch.float64)
    ref = st * b + so * s
    bar = (per_thread + 13 + slices + 3) * U * ((st * b).abs() + abs(so) * mag)
    if exact_arm:
        bar = torch.zeros_like(bar)
    return Expect(ref, bar, torch.zeros(C, dtype=torch.bool, device=ref.device))


def upsample(g_small_to_big, grads, st=0.0, t0=None, factor=2):
    """UpSample == avg-pool undo of a factor x factor, stride factor pool, scaled by factor^2 (gemm.cu:1503-1521);
    the geometry is the big image's"""
    return avg_undo(g_small_to_big, grads, st=st, t0=t0, so=float(factor * factor))


# ---------------------------------------------------------------------------------------------------------------------
# response normalisation
# ---------------------------------------------------------------------------------------------------------------------
def _windows(F, k, blocked, inverse, dev):
    j = torch.arange(F, device=dev)
    if blocked:
        lo = (j // k) * k
        return lo, torch.clamp(lo + k, max=F)
    a = k // 2
    b = k - a - 1
    if inverse:
        a, b = b, a
    return torch.clamp(j - a, min=0), torch.clamp(j + b + 1, max=F)


def _window_sum(v, k, blocked, inverse):
    """direct float64 window sums along dim 1 of (frames, F, L)"""
    fr, F, L = v.shape
    if blocked:
        nb = -(-F // k)
        pad = torch.zeros(fr, nb * k - F, L, dtype=v.dtype, device=v.device)
        s = torch.cat([v, pad], 1).view(fr, nb, k, L).sum(2)
        return s.repeat_interleave(k, dim=1)[:, :F]
    a = k // 2
    b = k - a - 1
    if inverse:
        a, b = b, a
    z = torch.zeros(fr, k, L, dtype=v.dtype, device=v.device)
    p = torch.cat([z, v, z], 1)
    s = torch.zeros_like(v)
    for d in range(-a, b + 1):
        s += p[:, k + d: k + d + F]
    return s


def _prefix(v):
    fr, F, L = v.shape
    return torch.cat([torch.zeros(fr, 1, L, dtype=v.dtype, device=v.device), torch.cumsum(v, 1)], 1)


def e_pow(y, base):
    lb = torch.log2(base).abs()
    return math.log(2.0) * abs(y) * (2.0 ** -22 + 2.0 ** -22 * lb + U * lb) + 2.0 ** -22


def _rn_parts(x, F, k, alpha, beta, blocked, frames, fault):
    X = x.to(torch.float64).reshape(frames, F, -1)
    dev = X.device
    sq = X * X
    fb = (not blocked) if fault == "blocked_swap" else blocked
    S = _window_sum(sq, k, fb, inverse=(fault == "window_swap"))
    lo, hi = _windows(F, k, blocked, False, dev)
    P = _prefix(sq).index_select(1, hi)
    cS = (2 * hi + k + 10).to(torch.float64).view(1, -1, 1)
    return X, S, 1.0 + alpha * S, cS * U * P


def rnorm_fwd(x, F, k, alpha, beta, blocked, frames=1, relu=False, fault=None, local_bar=False):
    """fault (controls): 'window_swap' uses the inverse window, 'blocked_swap' the other windowing; local_bar charges
    the window sum on the window's own mass (a wrong bar)"""
    X, S, base, dS = _rn_parts(x, F, k, alpha, beta, blocked, frames, fault)
    if local_bar:
        dS = (2 * k + 10) * U * _window_sum(X * X, k, blocked, False)
    pw = base ** -beta
    ref = X * pw
    bar = RN_SAFETY * (ref.abs() * (e_pow(beta, base) + (2 * beta + 1) * U)
                       + X.abs() * beta * alpha * base ** (-beta - 1) * dS)
    if relu:
        ref = ref.clamp_min(0.0)
    return Expect(_flat(ref), _flat(bar), torch.zeros(ref.numel(), dtype=torch.bool, device=ref.device))


def rnorm_undo(dy, x, F, k, alpha, beta, blocked, frames=1, fault=None):
    X, S, base, dS = _rn_parts(x, F, k, alpha, beta, blocked, frames, fault)
    D = dy.to(torch.float64).reshape(frames, F, -1)
    den = base ** (-beta - 1)
    t = D * X * den
    p = D * base ** -beta
    fb = (not blocked) if fault == "blocked_swap" else blocked
    R = _window_sum(t, k, fb, inverse=(fault != "window_swap"))
    c2 = 2.0 * alpha * beta
    ref = p - c2 * X * R
    ep = e_pow(beta + 1, base) + (2 * beta + 5) * U
    et = t.abs() * ep + (D * X).abs() * (beta + 1) * alpha * base ** (-beta - 2) * dS
    lo, hi = _windows(F, k, blocked, True, X.device)
    PT = _prefix(t.abs()).index_select(1, hi)
    cT = (2 * hi + k + 10).to(torch.float64).view(1, -1, 1)
    dR = _window_sum(et, k, blocked, True) + cT * U * PT
    bar = RN_SAFETY * (p.abs() * ep + D.abs() * beta * alpha * den * dS
                       + (c2 * X).abs() * (dR + 2 * U * R.abs()) + 2 * U * (p.abs() + (c2 * X * R).abs()))
    return Expect(_flat(ref), _flat(bar), torch.zeros(ref.numel(), dtype=torch.bool, device=ref.device))


def round_mantissa(v, bits):
    m, e = torch.frexp(v)
    return torch.ldexp(torch.round(m * 2.0 ** bits) / 2.0 ** bits, e)


# ---------------------------------------------------------------------------------------------------------------------
# bf16 twins
# ---------------------------------------------------------------------------------------------------------------------
def bf16_rne(y):
    return y.to(torch.float32).to(torch.bfloat16).to(torch.float32)


def bf16_trunc(y):
    b = y.to(torch.float32).contiguous().view(torch.int32) & ~0xFFFF
    return b.view(torch.float32)


# ---------------------------------------------------------------------------------------------------------------------
# the check
# ---------------------------------------------------------------------------------------------------------------------
@dataclasses.dataclass
class Verdict:
    ok: bool
    worst: float              # max |y - ref| / bar over elements with bar > 0
    bad: int
    where: str

    def __str__(self):
        return "ok=%s worst |err|/bar=%.3e bad=%d %s" % (self.ok, self.worst, self.bad, self.where)


def check(y, e):
    """kernel output y (flat fp32, at least as long as e.ref) against an Expect"""
    n = e.ref.numel()
    y = y[:n]
    yd = y.to(torch.float64)
    r32 = e.ref.to(torch.float32)
    same_bits = (y.view(torch.int32) == r32.view(torch.int32)) | (torch.isnan(y) & torch.isnan(r32))
    err = (yd - e.ref).abs()
    pos = (e.bar > 0) & ~e.exact
    ratio = torch.where(pos, err / torch.where(pos, e.bar, torch.ones_like(e.bar)), torch.zeros_like(err))
    ratio = torch.where(torch.isnan(ratio), torch.full_like(ratio, float("inf")), ratio)
    bad = torch.where(e.exact, ~same_bits, torch.where(pos, ~(ratio <= 1.0), ~(yd == e.ref)))
    nbad = int(bad.sum())
    worst = float(ratio.max()) if n else 0.0
    where = ""
    if nbad:
        i = int(torch.nonzero(bad)[0])
        where = "first bad element %d: y=%r ref=%r bar=%.3e" % (i, float(y[i]), float(e.ref[i]), float(e.bar[i]))
    return Verdict(nbad == 0, worst, nbad, where)


# ---------------------------------------------------------------------------------------------------------------------
# dispatch mirror
# ---------------------------------------------------------------------------------------------------------------------
@dataclasses.dataclass
class Branch:
    name: str                 # template-level name, e.g. rows<4,max,K3,S2>
    kernel: str               # what the demangled kernel name contains
    in_kernel_twin: bool = False
    slices: int = 0           # per-slice bias sums the kernel leaves for colsum_finish (0: a column-sum pass)
    masks: bool = False       # the forward pass records tie masks
    fused: bool = True        # the kernel applies the request's steps and ReLU' mask (else: passes after it)


def patch_geometry(g):
    return (g.two_d and max(g.kx, g.ky) == 3 and g.sx == 2 and g.sy == 2 and 0 <= g.px <= 2 and 0 <= g.py <= 2
            and g.N * g.W * g.H < 2 ** 31)


def _vec(g, aligned):
    return 4 if g.N % 4 == 0 and aligned else 1


def _rows_kernel(name, v, is_max, A, S, epi):
    """the row-kernel instance: EPI (a request's epilogue) is an average-pooling instance"""
    return "%s<%d, %s, %d, %d, %s>" % (name, v, "true" if is_max else "false", A, S, "true" if epi else "false")


def pool_fwd_branch(g, is_max, aligned=True, cache=False, so=1.0, epi=False):
    """epi: the average call has a request to fuse (steps, ReLU' mask or bias gradient)"""
    v = _vec(g, aligned)
    mx = "true" if is_max else "false"
    k = max(g.kx, g.ky) if g.two_d else 99
    masks = bool(cache and is_max and so == 1.0 and patch_geometry(g))
    epi = epi and not is_max
    if k <= 3 and g.N * g.W * g.H < 2 ** 31:
        K = 2 if k <= 2 else 3
        S = g.sx if g.sx == g.sy and g.sx <= 2 else 0
        return Branch("rows<%d,%s,K%d,S%d>%s" % (v, "max" if is_max else "avg", K, S, "+epi" if epi else ""),
                      _rows_kernel("pool_fwd_rows_kernel", v, is_max, K, S, epi), True,
                      g.modY if epi else 0, masks=masks)
    K = 2 if k <= 2 else 3 if k == 3 else 4 if k == 4 else 0
    return Branch("generic<%d,%s,K%d>" % (v, "max" if is_max else "avg", K),
                  "pool_fwd_kernel<%d, %s, %d>" % (v, mx, K), False, masks=masks, fused=not epi)


def pool_undo_branch(g, is_max, aligned=True, mask=None, st=0.0, cached=False, epi=False):
    """mask: None, 'input' (the ReLU' mask is the pool input) or 'other'; cached: the forward pass recorded tie masks
    for this (input, output) pair; epi: the average undo has steps to fuse (ReLU, dropout or scale)"""
    v = _vec(g, aligned)
    mx = "true" if is_max else "false"
    kind = "max" if is_max else "avg"
    epi = epi and not is_max
    q = max(-(-g.kx // g.sx), -(-g.ky // g.sy)) if g.two_d else 99
    if q <= 2 and (g.N // v) * g.W * g.H * v < 2 ** 31:
        if is_max and patch_geometry(g):
            PY = (g.H - 1 + g.py) // 2 + 1
            if cached and (mask is None or (mask == "input" and st == 0.0)):
                return Branch("masked_patch<%d>" % v, "pool_undo_masked_patch_kernel<%d>" % v, True, PY)
            return Branch("patch<%d>" % v, "pool_undo_patch_kernel<%d>" % v, True, PY)
        S = g.sx if g.sx == g.sy and g.sx <= 2 else 0
        Q = 1 if q <= 1 else 2
        return Branch("undo_rows<%d,%s,Q%d,S%d>%s" % (v, kind, Q, S, "+epi" if epi else ""),
                      _rows_kernel("pool_undo_rows_kernel", v, is_max, Q, S, epi), True, g.H)
    Q = 1 if q <= 1 else 2 if q == 2 else 0
    return Branch("undo_generic<%d,%s,Q%d>" % (v, kind, Q), "pool_undo_kernel<%d, %s, %d>" % (v, mx, Q), False, 0,
                  fused=not epi)


def bias_depth(branch, g):
    """(values one thread adds, slices colsum_finish adds) of the bias-gradient sum of a branch"""
    v = 4 if branch.name.split("<")[1].startswith("4") else 1
    NV = g.N // v
    fwd = branch.kernel.startswith("pool_fwd")        # (the bias gradient of a forward call sums its output)
    if branch.slices and "patch" in branch.name:
        PX = (g.W - 1 + g.px) // 2 + 1
        return -(-NV * PX // 256) * 4 * v, branch.slices
    if branch.slices:
        return -(-NV * (g.modX if fwd else g.W) // 256) * v, branch.slices
    rows = g.N * (g.modX * g.modY * g.modT if fwd else g.W * g.H * g.T)
    slices = max(1, min(64, (4 * SMS) // g.C))
    slices = min(slices, max(1, rows // 1024))
    return -(-(-(-rows // slices)) // 256), slices


def pick_tile(F, arrays):
    sm = 224 * 1024
    for per_sm in (3, 2, 1):
        for tl in (64, 32):
            if 4 * (arrays * (F + 1) * tl + 128) + 1024 <= sm // per_sm:
                return tl
    return 0


def pick_segments(owners, F, k, sms=SMS):
    blocks = -(-owners // 128)
    want = -(-2 * sms // blocks)
    return max(1, min(want, max(1, F // max(k, 1))))


def _segments(owners, F, k, blocked, sms):
    segs = pick_segments(owners, F, k, sms)
    seg = -(-F // segs)
    if blocked:
        seg = -(-seg // k) * k
    return -(-F // seg)


def rnorm_can_fuse(F):
    """rnorm_forward's result: its kernel applied the ReLU and wrote the twin (the tile kernel) or neither (the ring)"""
    return pick_tile(F, 2) != 0


def rnorm_fwd_branch(L, F, k, blocked, aligned=True, sms=SMS):
    """L = locations per frame.  Names: the kernel template and its data path (tile: 16-byte or scalar loads; ring:
    shared-memory or global ring); after '|' the partial last tile / channel segments, which are not branches of their
    own but must each be reached by a case."""
    bl = "true" if blocked else "false"
    tl = pick_tile(F, 2)
    if tl:
        vec = L % 4 == 0 and aligned
        return Branch("tile_fwd<%d,%s>%s" % (tl, "vec" if vec else "scalar", "|partial" if L % tl else ""),
                      "rnorm_tile_kernel<%d, (cnb::RnPass)0>" % tl, True)
    wide = L % 4 == 0 and aligned and L // 4 // 128 >= 4 * sms
    v = 4 if wide else 1
    segs = _segments(L // v, F, k, blocked, sms)
    ring = "gring" if 4 * k * 128 * v > 160 * 1024 else "smem"
    return Branch("ring_fwd<%s,%d,%s>%s" % (bl, v, ring, "|seg" if segs > 1 else ""),
                  "rnorm_fwd_kernel<%s, %d>" % (bl, v), False)


def rnorm_undo_branch(L, F, k, blocked, aligned=True, sms=SMS):
    tl = pick_tile(F, 4)
    if tl:
        vec = L % 4 == 0 and aligned
        return Branch("tile_undo<%d,%s>%s" % (tl, "vec" if vec else "scalar", "|partial" if L % tl else ""),
                      "rnorm_tile_kernel<%d, (cnb::RnPass)1>" % tl, False)
    segs = _segments(L, F, k, blocked, sms)
    ring = "gring" if 4 * 3 * k * 128 > 160 * 1024 else "smem"
    bl = "true" if blocked else "false"
    return Branch("ring_undo<%s,%s>%s" % (bl, ring, "|seg" if segs > 1 else ""), "rnorm_undo_kernel<%s>" % bl, False)
