"""Float64 references of the elementwise kernels of csrc/elementwise.cu (bias add, bias gradient, ReLU, ReLU', dropout,
the mask multiply, the three batch-norm passes, softmax and the loss sum), the per-element bar of each op, and a mirror
of their dispatch.

Layout (DESIGN.md §3): a [rows x cols] matrix is column-major, a column is one channel (bias: channel c holds the
elements [c*rows, (c+1)*rows); batch norm: [c*n, (c+1)*n)).  Every reference is torch on the device of its inputs.
u = 2^-24 is the unit roundoff of fp32.  One fp32 operation computed in float64 and rounded to fp32 is the correctly
rounded fp32 result (53 >= 2*24 + 2: double rounding is harmless for + - * / sqrt), which is how the bit-exact
restatements below are written; fma32 emulates a fused multiply-add (the float64 product of two fp32 numbers is exact,
a TwoSum with the addend keeps the error, and a float64 value that is exactly halfway between two fp32 numbers is
rounded by the sign of that error).

Three kinds of expectation.

* BIT-EXACT, one rounding or none (compiled code: FADD / FMUL / FMNMX / ISETP, checked in `cuobjdump -sass`):
  - bias add fl(x + b[c]) and bias + ReLU fmaxf(fl(x + b[c]), 0);
  - ReLU fmaxf(x, 0): fmaxf(NaN, 0) = 0.  The sign fmaxf gives for x = -0 is not assumed: a -0 input may come back as
    either zero (compared by value), and the GPU test records which one it saw;
  - ReLU' y > 0 ? d : +0: NaN and +-0 states give +0, a positive subnormal state passes d (the build has no FTZ);
  - dropout: element i draws u = float32(hash(seed + i)) * 2^-32 (rounded to nearest, so u can be 1.0), keeps it when
    u >= p; the value is fl(x * scale) or x * 0, the mask scale or 0;
  - the mask multiply fl(a * b);
  - every bf16 twin: the round-to-nearest-even bf16 of the fp32 value the kernel stored.
* BIT-EXACT GIVEN THE KERNEL'S OWN INPUTS.  The SASS of bn_channel_kernel<BnApplyOp> is FADD (x - mu), an IEEE division
  for gamma / sigma (MUFU.RCP and its FFMA fix-up), one FFMA, FMNMX; <BnBackOp> is FADD (x - mu), the IEEE
  reciprocal of sigma, FMUL (gamma * inv), FMUL ((x - mu) * inv), FADD (d - E[d]), FFMA with the product negated,
  FMUL.  So, with mu and sigma the ones the call was given (or the kernel wrote) and the kernel's own grad_gamma /
  grad_beta:
  - bn_apply:    fma(fl(x - mu), fl(gamma / sigma), beta), then fmaxf(., 0);
  - bn_backward: fl(a * fma(-fl(fl(x - mu) * inv), E[d*xhat], fl(d - E[d]))), inv = fl(1 / sigma), a = fl(gamma * inv);
                 with train = 0 the two means are 0 (the running statistics are constants);
  - the running averages fma(fl(1 - f), mu, fl(f * run)) (written with __fmaf_rn).
* BARS, with exact arms, for the reductions.  A sum of m fp32 terms in any order is within gamma_{D} sum|terms| of the
  exact sum, D the depth of the summation tree (gamma_D = D u / (1 - D u) <= (D + 1) u for the D here).
  - colsum_partial_kernel (the bias gradient with SumOp, the batch-norm sums with SumOp, SqDevOp and BnGradOp): one
    block of 256 threads per (column, slice).  A thread adds `per_thread` values in order (VEC: float4 groups, each a
    pair tree of depth 2 first), then a 5-level warp shuffle, then the 8 warp sums in a second 5-level shuffle, then
    the per-column kernel adds the `slices` partial sums in order:
        D = per_thread (+ 2 VEC) + 10 + slices.
  - bias gradient st * b + so * sum(target): pool_exact.bias_grad, whose depth (per_thread + 13 + slices + 3) is this
    one plus st * b, so * s and their sum.
  - batch-norm mean mu = fl(s * fl(1/n)): |mu - sum(x)/n| <= (D + 2) u sum|x| / n.
  - sigma = sqrtf(fl(s * fl(1/n)) + eps) with s = sum fl(x - mu)^2 about the KERNEL'S mu (so the reference's variance
    V = sum (x - mu)^2 / n is taken about that mu too).  Each square carries 3u (2u from fl(x - mu), one rounding), the
    sum D u, 1/n and the product 2u, + eps u (the compiler may contract s * (1/n) + eps into one FFMA: one rounding
    fewer), sqrtf (IEEE) halves the relative error of its argument and adds u:
        |sigma - sqrt(V + eps)| <= ((D + 6) / 2 + 1) u sigma.
  - grad_beta = fl(fl(sum d) * fl(1/n)): (D + 2) u sum|d| / n.  grad_gamma = fl(fl(sum d * xhat) * fl(1/n)) with the
    kernel's xhat = fl(fl(x - mu) * fl(1/sigma)) (3u) and the fma or product (1u): (D + 6) u sum|d (x - mu) / sigma| / n.
  - cnb_sum: one block of 256 threads, thread t adds elements t, t + 256, ... in order, then the two 5-level shuffles:
        D = ceil(n / 256) + 10,  |s - sum| <= (D + 1) u sum|a|.
  - softmax p_j = fl(e_j * fl(1 / s)), e_j = expf(fl(x_j - m)), m the exact column maximum (fmaxf), s the sum of the
    e_j: each warp adds its ceil(cols / 8) columns in order, then the 8 warp sums are added in order, depth
    ceil(cols / 8) + 8.  expf is within 2 ulp (CUDA C++ Programming Guide, Mathematical Functions), i.e. 4u relative;
    the subtraction moves the argument by |x_j - m| u, so e_j carries d_j = 4u + |x_j - m| u.  s inherits the largest
    d_k and adds its depth; the reciprocal and the product add 2u:
        |p_j - ref_j| <= (1 + 2^-10) (d_j + max_k d_k + (ceil(cols/8) + 10) u) ref_j + 2^-146,
    the factor covering the dropped second-order terms and the absolute floor the subnormal e_j (2 ulp of 2^-149 each,
    with s >= 1).
  EXACT ARMS: dyadic inputs small enough that every partial sum is an fp32 number make every one of these sums exact,
  so the result must EQUAL float64; one dropped or doubled term at n ~ 1.5 M fails them.  Cases: the bias gradient and
  cnb_sum on multiples of 2^-4; the batch-norm mean with n a power of two; the variance of +-1 data of zero mean
  (sigma = fl(sqrt(fl(1 + eps)))); the backward sums with a caller-supplied dyadic mu and sigma = 2 (xhat is exact);
  softmax with equal logits (every p is fl(1 / cols)) and with one logit 200 above the rest (an exact one-hot).
"""
import dataclasses
import math

import numpy as np
import torch

import conv_exact as cx
import pool_exact as px
from pool_exact import Expect, Verdict, bf16_rne, check  # noqa: F401  (re-exported for the test files)

U = 2.0 ** -24
SMS = 132                                  # H100 SXM; the mirror takes the live count where a GPU is present
BLOCK = 256


# ---------------------------------------------------------------------------------------------------------------------
# fp32 arithmetic, restated
# ---------------------------------------------------------------------------------------------------------------------
def _d(t):
    return t.to(torch.float64)


def r32(t):
    """one rounding to fp32 of a float64 tensor"""
    return t.to(torch.float32)


def fma32(a, b, c):
    """fp32 fma(a, b, c), rounded once"""
    a, b, c = torch.broadcast_tensors(*(torch.as_tensor(v, dtype=torch.float32) for v in (a, b, c)))
    p = _d(a) * _d(b)
    c64 = _d(c)
    s = p + c64
    bb = s - p
    e = (p - (s - bb)) + (c64 - bb)                        # TwoSum: p + c == s + e exactly
    r = s.to(torch.float32)
    dlt = s - _d(r)
    nb = torch.nextafter(r, torch.where(dlt > 0, torch.full_like(r, math.inf), torch.full_like(r, -math.inf)))
    mid = (dlt != 0) & ((_d(nb) - _d(r)) == 2 * dlt)
    fix = mid & (e != 0) & ((e > 0) == (dlt > 0))
    return torch.where(fix, nb, r)


def _exp(ref, exact):
    """an Expect from float64 ref: exact elements bit for bit, the others by value with a zero bar"""
    return Expect(ref, torch.zeros_like(ref), exact)


def _bits(y, signless_zero=None):
    """Expect of a bit-exact fp32 result y; signless_zero: elements whose zero may carry either sign"""
    y = y.to(torch.float32)
    exact = torch.ones(y.shape, dtype=torch.bool, device=y.device)
    if signless_zero is not None:
        exact &= ~(signless_zero & (y == 0))
    return _exp(_d(y).reshape(-1), exact.reshape(-1))


# ---------------------------------------------------------------------------------------------------------------------
# bit-exact ops
# ---------------------------------------------------------------------------------------------------------------------
def bias_add(x, bias, rows, cols, relu=False, fault=None):
    """fl(x + b[i // rows]) [, fmaxf(., 0)]; fault 'mod_cols' indexes the bias by i % cols, 'relu_first' clamps x
    before the add"""
    i = torch.arange(rows * cols, device=x.device)
    c = i % cols if fault == "mod_cols" else i // rows
    xv = torch.clamp_min(x, 0.0) if fault == "relu_first" else x
    y = r32(_d(xv) + _d(bias[c]))
    if relu and fault != "relu_first":
        y = torch.fmax(y, torch.zeros_like(y))
    return _bits(y, signless_zero=torch.ones_like(y, dtype=torch.bool) if relu else None)


def relu(x):
    y = torch.fmax(x, torch.zeros_like(x))
    return _bits(y, signless_zero=(x == 0))


def relu_deriv(d, y, fault=None):
    """y > 0 ? d : +0; fault 'ge' tests y >= 0, 'ftz' flushes subnormal states to zero first"""
    if fault == "ge":
        keep = y >= 0
    elif fault == "ftz":
        keep = y >= 2.0 ** -126
    else:
        keep = y > 0
    return _bits(torch.where(keep, d, torch.zeros_like(d)))


def dropout(x, p, scale, seed, idx=None, n4=None, fault=None):
    """(value, mask) Expects of cnb_dropout on x (fp32, the elements idx of the target; default all of them).
    n4: float4 groups of the vector body (faults only).  fault 'gt' keeps u > p, 'tail0' draws the scalar tail from
    hash(seed + i - 4 n4), 'lanes' swaps lanes 0 and 1 of every float4, 'mask1' writes a mask of 1"""
    dev = x.device
    n = x.numel()
    if idx is None:
        idx = np.arange(n, dtype=np.int64)
    idx = np.asarray(idx, dtype=np.int64)
    j = idx.copy()
    if fault == "tail0":
        j = np.where(idx >= 4 * n4, idx - 4 * n4, idx)
    if fault == "lanes":
        j = np.where((idx < 4 * n4) & (idx % 4 < 2), idx ^ 1, idx)
    u = cx.dropout_u(seed, j.astype(np.uint64))
    keep = u > np.float32(p) if fault == "gt" else u >= np.float32(p)
    keep = torch.from_numpy(keep).to(dev)
    m = torch.where(keep, torch.full_like(x, scale), torch.zeros_like(x))
    v = r32(_d(x) * _d(m))
    if fault == "mask1":
        m = torch.where(keep, torch.ones_like(x), torch.zeros_like(x))
    return _bits(v), _bits(m)


def mult(a, b):
    return _bits(r32(_d(a) * _d(b)))


# ---------------------------------------------------------------------------------------------------------------------
# reductions: depths, references, bars
# ---------------------------------------------------------------------------------------------------------------------
def cdiv(a, b):
    return -(-a // b)


def colsum_depth(rows, slices, vec):
    """(values one thread adds in order, tree depth D) of colsum_partial_kernel + its per-column finish"""
    per = cdiv(rows // 4 if vec else rows, slices)
    t = cdiv(per, BLOCK)
    return t, t + (2 if vec else 0) + 10 + slices


def bias_grad_slices(rows, cols, sms=SMS):
    s = max(1, min(64, (4 * sms) // cols))
    return min(s, max(1, rows // 1024))


def bias_grad(target, rows, cols, b0, st, so, sms=SMS, exact_arm=False, fault=None):
    """cnb_channel_bias_grad: st * b + so * (column sums), pool_exact.bias_grad with this kernel's depth.
    fault 'read_target' reads b0 even when st == 0 (the NaN prefill leaks), 'drop_row' leaves out row 0 of
    every column"""
    slices = bias_grad_slices(rows, cols, sms)
    per_thread, _ = colsum_depth(rows, slices, False)
    b = b0 if st != 0.0 else torch.zeros_like(b0)      # the prefill of a st == 0 target is not read
    e = px.bias_grad(target, rows, cols, 1, b, st, so, per_thread, slices, exact_arm=exact_arm,
                     fault="drop_row" if fault == "drop_row" else None)
    if fault == "read_target" and st == 0.0:
        e = Expect(e.ref + _d(b0), e.bar, e.exact)
    return e


def sum_ref(a, exact_arm=False, fault=None):
    """cnb_sum; fault 'first256' sums the first 256 elements only"""
    n = a.numel()
    v = _d(a[:256] if fault == "first256" else a)
    D = cdiv(n, BLOCK) + 10
    ref = v.sum().reshape(1)
    bar = torch.zeros_like(ref) if exact_arm else (D + 1) * U * _d(a).abs().sum().reshape(1)
    return Expect(ref, bar, torch.zeros(1, dtype=torch.bool, device=a.device))


def _cols(x, n, C):
    return _d(x[: n * C]).view(C, n)


def bn_mean(x, n, C, slices, vec, exact_arm=False, fault=None):
    """fault 'drop' leaves out the last element of every column"""
    X = _cols(x, n, C)
    if fault == "drop":
        X = X[:, :-1]
    _, D = colsum_depth(n, slices, vec)
    ref = X.sum(1) / n
    bar = torch.zeros_like(ref) if exact_arm else (D + 2) * U * X.abs().sum(1) / n
    return Expect(ref, bar, torch.zeros(C, dtype=torch.bool, device=x.device))


def bn_sigma(x, n, C, mu, eps, slices, vec, exact_arm=False, fault=None):
    """sigma about the kernel's mu.  faults: 'one_pass' E[x^2] - E[x]^2 evaluated in fp32 (returned as the value to
    test), 'n_minus_1' divides by n - 1, 'eps_outside' sqrt(V) + eps"""
    eps = float(np.float32(eps))
    X = _cols(x, n, C)
    m = _d(mu[:C]).view(C, 1)
    V = ((X - m) ** 2).sum(1) / (n - 1 if fault == "n_minus_1" else n)
    ref = torch.sqrt(V) + eps if fault == "eps_outside" else torch.sqrt(V + eps)
    _, D = colsum_depth(n, slices, vec)
    if exact_arm:
        one = r32(torch.tensor(1.0, dtype=torch.float64, device=x.device) + eps)
        ref = _d(r32(torch.sqrt(_d(one)))).expand(C).clone()
        return Expect(ref, torch.zeros_like(ref), torch.ones(C, dtype=torch.bool, device=x.device))
    bar = ((D + 6) / 2 + 1) * U * ref.abs()
    return Expect(ref, bar, torch.zeros(C, dtype=torch.bool, device=x.device))


def bn_sigma_one_pass(x, n, C, eps):
    """the fault: sigma from E[x^2] - E[x]^2, each mean an fp32 sum (what a one-pass kernel would compute)"""
    X = x[: n * C].view(C, n)
    ex = X.sum(1, dtype=torch.float32) / n
    ex2 = (X * X).sum(1, dtype=torch.float32) / n
    return torch.sqrt(torch.clamp_min(ex2 - ex * ex, 0) + eps)


def bn_running(run, val, f):
    """fma(fl(1 - f), val, fl(f * run)), bit-exact"""
    f = float(np.float32(f))
    omf = r32(torch.tensor(1.0, dtype=torch.float64, device=run.device) - f)
    return _bits(fma32(omf, val, r32(f * _d(run))))


def bn_apply(x, n, C, gamma, beta, mu, sigma, relu=False, fault=None):
    """fault 'bf16_a' rounds gamma / sigma to bf16"""
    X = x[: n * C].view(C, n)
    a = r32(_d(gamma[:C]) / _d(sigma[:C]))
    if fault == "bf16_a":
        a = bf16_rne(a)
    r = fma32(r32(_d(X) - _d(mu[:C]).view(C, 1)), a.view(C, 1), beta[:C].view(C, 1))
    if relu:
        z = r == 0
        r = torch.fmax(r, torch.zeros_like(r))
        return _bits(r.reshape(-1), signless_zero=z.reshape(-1))
    return _bits(r.reshape(-1))


def bn_grads(d, x, n, C, mu, sigma, slices, vec, exact_arm=False, fault=None):
    """(grad_gamma, grad_beta) Expects: mean(d * (x - mu) / sigma) and mean(d), with the caller's mu, sigma"""
    Dd, X = _cols(d, n, C), _cols(x, n, C)
    xh = (X - _d(mu[:C]).view(C, 1)) / _d(sigma[:C]).view(C, 1)
    _, D = colsum_depth(n, slices, vec)
    gg = (Dd * xh).sum(1) / n
    gb = Dd.sum(1) / n
    z = torch.zeros(C, dtype=torch.bool, device=d.device)
    if exact_arm:
        return Expect(gg, torch.zeros_like(gg), z), Expect(gb, torch.zeros_like(gb), z)
    return (Expect(gg, (D + 6) * U * (Dd * xh).abs().sum(1) / n, z),
            Expect(gb, (D + 2) * U * Dd.abs().sum(1) / n, z.clone()))


def bn_backward(d, x, n, C, gamma, mu, sigma, gg, gb, train, fault=None):
    """the elementwise pass, given the kernel's grad_gamma / grad_beta.  faults: 'no_xhat' drops the xhat * E[d xhat]
    term, 'train0_batch' applies the batch terms with train = 0"""
    Dd, X = d[: n * C].view(C, n), x[: n * C].view(C, n)
    inv = r32(1.0 / _d(sigma[:C])).view(C, 1)
    a = r32(_d(gamma[:C]).view(C, 1) * _d(inv))
    use = bool(train) or fault == "train0_batch"
    md = gb[:C].view(C, 1) if use else torch.zeros_like(inv)
    mdx = gg[:C].view(C, 1) if use else torch.zeros_like(inv)
    if fault == "no_xhat":
        mdx = torch.zeros_like(mdx)
    xm = r32(_d(X) - _d(mu[:C]).view(C, 1))
    t = -r32(_d(xm) * _d(inv))
    q = fma32(t, mdx.expand_as(t), r32(_d(Dd) - _d(md)))
    return _bits(r32(_d(a) * _d(q)).reshape(-1))


def softmax(x, rows, cols, exact=None, fault=None):
    """softmax over the classes of column-major [rows x cols] fp32 x.  exact: 'equal' (every p = fl(1/cols)) or
    'onehot'.  fault 'one_warp' takes the maximum over warp 0's columns only, 'drop_warp' leaves warp 7's partial sum
    out of s"""
    X = _d(x[: rows * cols]).view(cols, rows)
    if fault == "one_warp":
        m = X[0::8].max(0).values
    else:
        m = X.max(0).values
    e = torch.exp(X - m)
    s = e[[c for c in range(cols) if not (fault == "drop_warp" and c % 8 == 7)]].sum(0)
    ref = e / s
    z = torch.zeros(ref.numel(), dtype=torch.bool, device=x.device)
    if exact == "equal":
        return Expect(torch.full_like(ref, float(np.float32(1.0) / np.float32(cols))).reshape(-1),
                      torch.zeros(ref.numel(), dtype=torch.float64, device=x.device), ~z)
    if exact == "onehot":
        return Expect(ref.reshape(-1), torch.zeros(ref.numel(), dtype=torch.float64, device=x.device), ~z)
    dj = 4 * U + (X - m).abs() * U
    bar = (1 + 2.0 ** -10) * (dj + dj.max(0).values + (cdiv(cols, 8) + 10) * U) * ref + 2.0 ** -146
    return Expect(ref.reshape(-1), bar.reshape(-1), z)


# ---------------------------------------------------------------------------------------------------------------------
# fp32 emulations of the kernels' summation orders (CPU tests: the bars must accept them)
# ---------------------------------------------------------------------------------------------------------------------
def _shfl_tree(s):
    """xor-shuffle reduction over the last axis (32 lanes), fp32, as __shfl_xor_sync with offsets 16 .. 1"""
    lane = torch.arange(32)
    for o in (16, 8, 4, 2, 1):
        s = s + s[..., lane ^ o]
    return s[..., 0]


def colsum_emulate(step, rows, C, slices, vec):
    """fp32 colsum_partial_kernel + per-column finish.  step(acc, r0, r1) -> the fp32 [C, r1 - r0] accumulators of
    the threads that take rows (VEC: float4 groups) r0 .. r1 - 1 after they add them, the way Op::add / add4 does"""
    rv = rows // 4 if vec else rows
    per = cdiv(rv, slices)
    parts = []
    for sl in range(slices):
        r0, r1 = sl * per, min(rv, sl * per + per)
        acc = torch.zeros(C, BLOCK, dtype=torch.float32)
        r = r0
        while r < r1:
            k = min(BLOCK, r1 - r)
            acc[:, :k] = step(acc[:, :k], r, r + k)
            r += k
        w = _shfl_tree(acc.view(C, 8, 32))
        t = torch.zeros(C, 32, dtype=torch.float32)
        t[:, :8] = w
        parts.append(_shfl_tree(t))
    s = torch.zeros(C, dtype=torch.float32)
    for p in parts:
        s = s + p
    return s


def sum_emulate(a):
    """fp32 sum_kernel (one block of 256)"""
    n = a.numel()
    acc = torch.zeros(BLOCK, dtype=torch.float32)
    for r in range(0, n, BLOCK):
        k = min(BLOCK, n - r)
        acc[:k] = acc[:k] + a[r:r + k]
    w = _shfl_tree(acc.view(8, 32))
    t = torch.zeros(32, dtype=torch.float32)
    t[:8] = w
    return _shfl_tree(t)


def softmax_emulate(x, rows, cols, fault=None):
    """fp32 softmax_kernel: warp w takes columns w, w + 8, ...; fault 'one_warp' / 'drop_warp' as in softmax()"""
    X = x[: rows * cols].view(cols, rows).clone()
    wm = torch.full((8, rows), -math.inf)
    for c in range(cols):
        wm[c % 8] = torch.fmax(wm[c % 8], X[c])
    m = wm[0] if fault == "one_warp" else wm.max(0).values
    ws = torch.zeros(8, rows)
    for c in range(cols):
        e = torch.exp(X[c] - m)
        X[c] = e
        ws[c % 8] = ws[c % 8] + e
    s = torch.zeros(rows)
    for w in range(8):
        if not (fault == "drop_warp" and w == 7):
            s = s + ws[w]
    inv = r32(1.0 / _d(s))
    return (X * inv).reshape(-1)


# ---------------------------------------------------------------------------------------------------------------------
# dispatch mirror
# ---------------------------------------------------------------------------------------------------------------------
@dataclasses.dataclass
class Branch:
    name: str                 # what a case claims, e.g. relu<vec+tail>|gs
    kernels: list             # substrings of the demangled names of the library kernels launched, in order
    twin: str = "none"        # bf16 twin when requested: 'kernel' (written in the kernel), 'pass' (cvt pass), 'none'

    def launches(self, emit=False):
        return len(self.kernels) + (1 if emit and self.twin == "pass" else 0)


def blocks_for(work, sms=SMS):
    return max(1, min(cdiv(work, BLOCK), sms * 16))


def _gs(work, sms):
    return "|gs" if cdiv(work, BLOCK) > sms * 16 else ""


def bias_branch(rows, cols, aligned, relu, sms=SMS):
    vec = rows % 4 == 0 and aligned
    k = "stream_kernel<cnb::BiasOp<%d>" % (1 if relu else 0)
    work = rows // 4 * cols if vec else rows * cols
    return Branch("bias%s<%s>%s" % ("_relu" if relu else "", "vec" if vec else "scalar", _gs(work, sms)), [k],
                  "pass" if aligned else "none")


# the act template argument is the library's Act: 1 = ReLU (demanglers differ in writing the closing "> >")
_N4_KERNEL = {"relu": "stream_kernel<cnb::ActOp<1>", "relu_deriv": "stream_kernel<cnb::ActDerivOp<1>",
              "dropout": "stream_kernel<cnb::DropOp>", "mult": "stream_kernel<cnb::MultOp>"}


def n4_of(n, aligned_all):
    return n // 4 if aligned_all else 0


def n4_branch(op, n, aligned_target, aligned_other=True, sms=SMS):
    """relu (aligned_other ignored), relu_deriv (y), dropout (mask), mult (b)"""
    n4 = n4_of(n, aligned_target and (aligned_other or op == "relu"))
    kind = "scalar" if n4 == 0 else ("vec" if n == 4 * n4 else "vec+tail")
    twin = ("pass" if op == "relu_deriv" else "kernel") if aligned_target else "none"
    return Branch("%s<%s>%s" % (op, kind, _gs(max(n4, n - 4 * n4), sms)), [_N4_KERNEL[op]], twin)


def colsum_slices_name(slices, cap):
    return "1" if slices == 1 else ("%d" % slices if slices == cap else "k")


def bias_grad_branch(rows, cols, st, sms=SMS):
    s = bias_grad_slices(rows, cols, sms)
    return Branch("bias_grad<%s slices>%s" % (colsum_slices_name(s, 64), "|st" if st != 0 else ""),
                  ["colsum_partial_kernel<cnb::SumOp, false>", "colsum_final_kernel<cnb::BiasGradFin>"])


def bn_slices(n, C, sms=SMS):
    want, most = cdiv(8 * sms, C), max(1, n // 2048)
    return max(1, min(min(want, most), 1024))


def bn_grid_x(n, C, vec, sms=SMS):
    per, fill = cdiv(n // 4 if vec else n, BLOCK), cdiv(16 * sms, C)
    return max(1, min(per, fill))


def bn_stats_branch(n, C, aligned_x, run, sms=SMS):
    vec = n % 4 == 0 and aligned_x
    s = bn_slices(n, C, sms)
    v = "true" if vec else "false"
    return Branch("bn_stats<%s,%s slices>%s" % ("vec" if vec else "scalar", colsum_slices_name(s, 1024),
                                               "|run" if run else ""),
                  ["colsum_partial_kernel<cnb::SumOp, %s>" % v, "colsum_final_kernel<cnb::MeanFin>",
                   "colsum_partial_kernel<cnb::SqDevOp, %s>" % v, "colsum_final_kernel<cnb::SigmaFin>"])


def bn_apply_branch(n, C, aligned_x, aligned_y, relu, sms=SMS):
    vec = n % 4 == 0 and aligned_x and aligned_y
    gs = "|gs" if bn_grid_x(n, C, vec, sms) < cdiv(n // 4 if vec else n, BLOCK) else ""
    return Branch("bn_apply<%s,%s>%s" % ("vec" if vec else "scalar", "relu" if relu else "linear", gs),
                  ["bn_channel_kernel<cnb::BnApplyOp<%d>" % (1 if relu else 0)], "kernel" if aligned_y else "none")


def bn_backward_branch(n, C, aligned_x, aligned_d, train, sms=SMS):
    vec = n % 4 == 0 and aligned_x and aligned_d
    s = bn_slices(n, C, sms)
    return Branch("bn_backward<%s,%s slices>%s" % ("vec" if vec else "scalar", colsum_slices_name(s, 1024),
                                                  "" if train else "|test"),
                  ["colsum_partial_kernel<cnb::BnGradOp, %s>" % ("true" if vec else "false"),
                   "colsum_final_kernel<cnb::BnGradFin>", "bn_channel_kernel<cnb::BnBackOp>"], "kernel" if aligned_d else "none")


def softmax_branch(rows, cols):
    return Branch("softmax<%s>%s" % ("cols<8" if cols < 8 else ("cols%8" if cols % 8 else "cols=8k"),
                                     "|partial" if rows % 32 else ""), ["softmax_kernel"])


def sum_branch(n):
    return Branch("sum<%s>" % ("n<=256" if n <= BLOCK else "n>256"), ["sum_kernel"])


# every library kernel the mirror can name (the profiler test filters on these)
KERNEL_NAMES = ("stream_kernel", "colsum_partial_kernel", "colsum_final_kernel", "bn_channel_kernel", "softmax_kernel",
                "sum_kernel")
