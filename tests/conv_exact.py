"""Float64 reference of the three conv ops on the kernel's own rounded operands, and the per-element bar.

A tensor-core conv rounds its operands (bf16: round to nearest even in the staging pass, stage.cu; tf32: the tensor core
reads the fp32 bits with the low 13 mantissa bits ignored) and then multiplies and accumulates in fp32.  Computing the same
convolution in float64 from the SAME rounded operands leaves only the fp32 accumulation and epilogue error, which is
tiny next to the error of a kernel that rounds one thing wrongly (see tests/test_conv_exact_cpu.py for the simulated faults).
So every output element y is held to

    |y - ref| <= BAR * S,   S = |so| * sum|a*b| + |st * t0| + |bias|                (BAR = 2^-16)

with ref and sum|a*b| computed in float64 from the modelled operands; where S == 0 the output must equal ref exactly.
ReLU is applied to ref (it is 1-Lipschitz); elements the ReLU' mask or the dropout drops must be exactly 0, and elements
outside the call's output channel range must keep their bits.  A logistic unit's sigma (fprop) and sigma' (dgrad) move
the bar with them: sigma' <= 1/4 scales S by 1/4, the logistic derivative mask s(1 - s) scales it by s(1 - s), and each
adds the bar of its own float32 arithmetic (loss_ref.sigmoid_bar, loss_ref.logistic_deriv_bar) as (bar / BAR) to S.

Layouts are the library's (DESIGN.md §3): activations a[n + N*(x + W*(y + H*c))], filters f[o + Cout*(x + kx*(y + ky*c))];
3-D tensors stack frames as channel blocks (channel c + C*t).  Everything here is torch float64 on the device of the inputs,
in image chunks so the unfolded operand stays near CHUNK_BYTES.
"""
import dataclasses

import numpy as np
import torch
import torch.nn.functional as tF

from convnet_b200.abi import GetConvDesc, num_modules

BAR = 2.0 ** -16
U = 2.0 ** -24
CHUNK_BYTES = 512 << 20


# ---------------------------------------------------------------------------------------------------------------------
# operand models: float32 tensor -> float64 tensor of the values the kernel multiplies
# ---------------------------------------------------------------------------------------------------------------------
def _bits(x):
    return x.contiguous().view(torch.int32).to(torch.int64) & 0xFFFFFFFF


def _from_bits(b):
    b = torch.where(b >= 2 ** 31, b - 2 ** 32, b)
    return b.to(torch.int32).view(torch.float32)


def _round_bits(x, drop):
    """round to nearest even at `drop` low bits (NaN and Inf pass through, overflow rounds to Inf like the hardware)"""
    b = _bits(x)
    half = (1 << (drop - 1)) - 1
    r = (b + half + ((b >> drop) & 1)) & ~((1 << drop) - 1)
    finite = torch.isfinite(x)
    return torch.where(finite, _from_bits(r & 0xFFFFFFFF), x)


def _trunc_bits(x, drop):
    b = _bits(x)
    return torch.where(torch.isnan(x), x, _from_bits(b & ~((1 << drop) - 1) & 0xFFFFFFFF))


# tf32: mma.sync reads the raw fp32 bits and ignores the low 13 (truncation, established by the controls of
# tests/test_gpu_conv_exact.py: the round-to-nearest model fails there); bf16: __float2bfloat16_rn in stage.cu.
MODELS = {
    "fp32": lambda x: x,
    "bf16": lambda x: x.to(torch.bfloat16).to(torch.float32),
    "tf32": lambda x: _trunc_bits(x, 13),
    # wrong models, for the controls
    "bf16_trunc": lambda x: _trunc_bits(x, 16),
    "tf32_rn": lambda x: _round_bits(x, 13),
}
# operand model of each precision, and the wrong models its output must fail
MODEL_OF = {"fp32": "fp32", "tf32": "tf32", "bf16": "bf16"}
CONTROLS = {"fp32": ("bf16",), "tf32": ("fp32", "tf32_rn"), "bf16": ("fp32", "bf16_trunc")}


def model(x, kind):
    return MODELS[kind](x.to(torch.float32)).to(torch.float64)


# ---------------------------------------------------------------------------------------------------------------------
# dispatch mirror: the operand model of the path a call takes (conv_tc.cu tc_conv_*_impl and abi.cu), for whole,
# 16-byte-aligned 2-D operands whose filters have a staged bf16 copy (the training host keeps one for every edge that may
# take a bf16 path), which lets an FC-shaped fprop / dgrad take bf16.
# ---------------------------------------------------------------------------------------------------------------------
PATH_MODEL = {"cuda-core-fp32": "fp32", "tc-tf32": "tf32", "tc-bf16": "bf16"}


def conv_path(op, g, mode):
    """'cuda-core-fp32', 'tc-tf32' or 'tc-bf16': the path of a conv call in precision `mode`"""
    x_mode = g.Cin * g.kt < 8           # (a 3-D call folds its kt frames into Cin * kt channels)
    rows = g.N * g.modX * g.modY * g.modT
    if mode == "fp32" or (x_mode and (g.kx > 8 or g.ky > 8)):
        return "cuda-core-fp32"
    if op == "fprop":
        tc = g.N % 4 == 0 and g.Cout % 4 == 0
        bf = not x_mode and g.N % 8 == 0 and g.Cout % 8 == 0
    elif op == "dgrad":
        tc = g.N % 4 == 0 and g.Cout % 4 == 0 and g.Cout >= 8 and g.Cin * g.kt >= 8 and g.kx <= 32 and g.ky <= 32
        bf = g.N % 8 == 0 and g.Cout % 8 == 0
    else:
        tc = g.N % 4 == 0 and g.Cout >= 8
        bf = not x_mode and g.N % 8 == 0 and (rows >= 1024 or (g.modT == 1 and g.N % 128 == 0 and g.Cin * g.kt % 32 == 0))
    if not tc:
        return "cuda-core-fp32"
    return "tc-bf16" if mode == "bf16" and bf else "tc-tf32"


# ---------------------------------------------------------------------------------------------------------------------
# geometry of one call
# ---------------------------------------------------------------------------------------------------------------------
@dataclasses.dataclass
class Geo:
    N: int
    W: int
    H: int
    Cin: int                 # input channels the call uses (per frame)
    Cout: int                # output channels the call writes
    ky: int
    kx: int
    sy: int = 1
    sx: int = 1
    py: int = 0              # positive paddings (GetConvDesc convention)
    px: int = 0
    T: int = 1               # image frames
    kt: int = 1
    st_t: int = 1            # frame stride
    cin0: int = 0            # channel sub-ranges: [cin0, cin0+Cin) of CinT, [cout0, cout0+Cout) of CoutT
    CinT: int = 0
    cout0: int = 0
    CoutT: int = 0

    def __post_init__(self):
        self.CinT = self.CinT or self.cin0 + self.Cin
        self.CoutT = self.CoutT or self.cout0 + self.Cout
        assert self.kt == 1 and self.T == 1 or (self.cin0 == 0 and self.Cin == self.CinT)

    @property
    def modX(self):
        return num_modules(self.W, self.kx, self.sx, self.px)

    @property
    def modY(self):
        return num_modules(self.H, self.ky, self.sy, self.py)

    @property
    def modT(self):
        return (self.T - self.kt) // self.st_t + 1

    @property
    def K(self):
        return self.kx * self.ky * self.Cin * self.kt

    # the ABI's shapes and descriptor
    def desc(self):
        return GetConvDesc(self.CinT, self.CoutT, self.ky, self.kx, self.sy, self.sx, self.py, self.px,
                           kernel_size_t=self.kt, stride_t=self.st_t,
                           input_channel_begin=self.cin0, input_channel_end=self.cin0 + self.Cin,
                           output_channel_begin=self.cout0, output_channel_end=self.cout0 + self.Cout)

    def img_shape(self):
        return (self.N, self.W, self.H, self.CinT * self.T)

    def flt_shape(self):
        return (self.Cout, self.kx, self.ky, self.Cin * self.kt)

    def out_shape(self):
        return (self.N, self.modX, self.modY, self.CoutT * self.modT)

    def img_dims(self):      # (rows, cols) of the cudamat
        return self.N, self.W * self.H * self.CinT * self.T

    def flt_dims(self):
        return self.Cout, self.K

    def out_dims(self):
        return self.N, self.modX * self.modY * self.CoutT * self.modT


# ---------------------------------------------------------------------------------------------------------------------
# the three ops in float64 (one frame window: 2-D conv of Cin*kt channels)
# ---------------------------------------------------------------------------------------------------------------------
def _act(flat, N, W, H, C):
    """flat activation buffer -> (N, C, H, W) view"""
    return flat[: N * W * H * C].view(C, H, W, N).permute(3, 0, 1, 2)


def _unact(t):
    """(N, C, H, W) -> flat, image fastest"""
    return t.permute(1, 2, 3, 0).reshape(-1)


def _chunk(g, per_image):
    return max(1, min(g.N, CHUNK_BYTES // max(1, 8 * per_image)))


def _cols(x, g):
    """unfolded windows (n, K, L) of a (n, Cin*kt, H, W) float64 window, K index = tx + kx*(ty + ky*c)"""
    return tF.unfold(x, (g.ky, g.kx), padding=(g.py, g.px), stride=(g.sy, g.sx))


def _fprop_frame(img, wm, g):
    """img (N, Ck, H, W), wm (Cout, K) -> (N, Cout, modY, modX)"""
    out = torch.empty(g.N, g.Cout, g.modY * g.modX, dtype=torch.float64, device=img.device)
    step = _chunk(g, g.K * g.modX * g.modY)
    for n0 in range(0, g.N, step):
        out[n0:n0 + step] = torch.matmul(wm, _cols(img[n0:n0 + step], g))
    return out.view(g.N, g.Cout, g.modY, g.modX)


def _dgrad_frame(der, wm, g):
    """der (N, Cout, modY, modX), wm (Cout, K) -> (N, Ck, H, W)"""
    Ck = g.Cin * g.kt
    out = torch.empty(g.N, Ck, g.H, g.W, dtype=torch.float64, device=der.device)
    step = _chunk(g, g.K * g.modX * g.modY)
    wt = wm.t()
    for n0 in range(0, g.N, step):
        d = der[n0:n0 + step].reshape(-1, g.Cout, g.modY * g.modX)
        cols = torch.matmul(wt, d)
        out[n0:n0 + step] = tF.fold(cols, (g.H, g.W), (g.ky, g.kx), padding=(g.py, g.px), stride=(g.sy, g.sx))
    return out


def _wgrad_frame(img, der, g):
    """img (N, Ck, H, W), der (N, Cout, modY, modX) -> (Cout, K)"""
    acc = torch.zeros(g.Cout, g.K, dtype=torch.float64, device=img.device)
    step = _chunk(g, g.K * g.modX * g.modY)
    for n0 in range(0, g.N, step):
        cols = _cols(img[n0:n0 + step], g)
        d = der[n0:n0 + step].reshape(-1, g.Cout, g.modY * g.modX)
        acc += torch.einsum("nol,nkl->ok", d, cols)
    return acc


def _raw(op, g, a, b):
    """the un-scaled op on float64 flat operands -> float64 flat result over the whole target buffer (zeros outside
    the call's channel range).  fprop: a = images, b = filters; dgrad: a = derivs, b = filters; wgrad: a = images,
    b = derivs."""
    Ck = g.Cin * g.kt
    if op == "wgrad":
        img = _act(a, g.N, g.W, g.H, g.CinT * g.T)
        der = _act(b, g.N, g.modX, g.modY, g.CoutT * g.modT)
        acc = torch.zeros(g.Cout, g.K, dtype=torch.float64, device=a.device)
        for f in range(g.modT):
            c0 = g.cin0 + f * g.st_t * g.CinT
            o0 = g.cout0 + f * g.CoutT
            acc += _wgrad_frame(img[:, c0:c0 + Ck], der[:, o0:o0 + g.Cout], g)
        return acc.t().reshape(-1)                       # element (o, k) at o + Cout*k
    wm = b[: g.Cout * g.K].view(g.K, g.Cout).t()
    if op == "fprop":
        img = _act(a, g.N, g.W, g.H, g.CinT * g.T)
        out = torch.zeros(g.N, g.CoutT * g.modT, g.modY, g.modX, dtype=torch.float64, device=a.device)
        for f in range(g.modT):
            c0 = g.cin0 + f * g.st_t * g.CinT
            o0 = g.cout0 + f * g.CoutT
            out[:, o0:o0 + g.Cout] = _fprop_frame(img[:, c0:c0 + Ck], wm, g)
        return _unact(out)
    assert op == "dgrad"
    der = _act(a, g.N, g.modX, g.modY, g.CoutT * g.modT)
    out = torch.zeros(g.N, g.CinT * g.T, g.H, g.W, dtype=torch.float64, device=a.device)
    for f in range(g.modT):                            # overlapping frame windows are summed
        c0 = g.cin0 + f * g.st_t * g.CinT
        o0 = g.cout0 + f * g.CoutT
        out[:, c0:c0 + Ck] += _dgrad_frame(der[:, o0:o0 + g.Cout], wm, g)
    return _unact(out)


def written_mask(op, g, device):
    """bool flat mask of the target elements the call computes (the rest of an fprop / wgrad target keeps its bits)"""
    if op == "wgrad":
        return torch.ones(g.Cout * g.K, dtype=torch.bool, device=device)
    if op == "fprop":
        m = torch.zeros(g.N, g.CoutT * g.modT, g.modY, g.modX, dtype=torch.bool, device=device)
        for f in range(g.modT):
            m[:, g.cout0 + f * g.CoutT: g.cout0 + f * g.CoutT + g.Cout] = True
        return _unact(m)
    m = torch.zeros(g.N, g.CinT * g.T, g.H, g.W, dtype=torch.bool, device=device)
    m[:, g.cin0: g.cin0 + g.Cin * g.kt] = True
    if g.T > 1:
        m[:] = True
    return _unact(m)


# ---------------------------------------------------------------------------------------------------------------------
# dropout generator (common.cuh: hash_u32 / dropout_keep), restated in numpy uint64
# ---------------------------------------------------------------------------------------------------------------------
def hash_u32(x):
    x = np.asarray(x, dtype=np.uint64)
    with np.errstate(over="ignore"):
        x = x + np.uint64(0x9E3779B97F4A7C15)
        x = (x ^ (x >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        x = (x ^ (x >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        return ((x ^ (x >> np.uint64(31))) >> np.uint64(32)).astype(np.uint32)


def dropout_u(seed, idx):
    """float32 u of the elements idx: float32(hash(seed + i)) * 2^-32, the conversion rounded to nearest (so u can be
    1.0), the seed wrapping modulo 2^64"""
    with np.errstate(over="ignore"):
        x = np.asarray(idx, dtype=np.uint64) + np.uint64(seed)
    return hash_u32(x).astype(np.float32) * np.float32(2.0 ** -32)


def dropout_kept(n, prob, seed, return_u=False):
    """bool[n]: element i of the target is kept (hash(seed + i) * 2^-32 >= prob, in float32 as the kernel computes it);
    with return_u also the u of every element"""
    u = dropout_u(seed, np.arange(n, dtype=np.uint64))
    kept = u >= np.float32(prob)
    return (kept, u) if return_u else kept


# ---------------------------------------------------------------------------------------------------------------------
# reference + bar
# ---------------------------------------------------------------------------------------------------------------------
@dataclasses.dataclass
class Expect:
    ref: torch.Tensor         # float64, whole target buffer
    S: torch.Tensor           # float64 error scale per element
    zero: torch.Tensor        # bool: must be exactly 0 (ReLU' mask, dropout)
    keep: torch.Tensor        # bool: must keep the prefilled bits (outside the call's output channels)


def expect(op, g, a, b, kind, t0=None, st=0.0, so=1.0, bias=None, relu=False, mask=None, drop=None, logistic=False,
           lmask=None):
    """Expected result of one call.  a, b: the fp32 operands (flat tensors, see _raw); t0: the target's contents before
    the call; bias: fprop bias per output channel of the call; mask: dgrad ReLU' mask (flat, target-shaped);
    drop: (prob, scale, seed) of the fused fprop dropout; logistic: fprop applies sigma; lmask: the dgrad logistic
    derivative mask, the stored state s of the logistic layer below (flat, target-shaped): the result is times s(1 - s)."""
    A, B = model(a, kind), model(b, kind)
    ref = so * _raw(op, g, A, B)
    S = abs(so) * _raw(op, g, A.abs(), B.abs())
    n = ref.numel()
    dev = ref.device
    written = written_mask(op, g, dev)
    keep = ~written
    if st != 0.0:
        t = t0[:n].to(torch.float64)
        if op == "dgrad":            # the whole target is scaled first (the reference's convDown)
            ref = ref + st * t
            S = S + (st * t).abs()
            keep = torch.zeros_like(keep) if st != 1.0 else keep
        else:
            ref = torch.where(written, ref + st * t, ref)
            S = torch.where(written, S + (st * t).abs(), S)
    elif op == "dgrad":
        keep = torch.zeros_like(keep)  # scaleTargets 0 clears the whole target
    if bias is not None:             # one bias per output channel, added to every output frame
        assert op == "fprop"
        shape = (g.modT, g.CoutT, g.modY * g.modX, g.N)
        full = torch.zeros(g.CoutT, dtype=torch.float64, device=dev)
        full[g.cout0:g.cout0 + g.Cout] = bias.to(torch.float64).view(-1)
        fb = full.view(1, -1, 1, 1).expand(shape).reshape(-1)
        ref = torch.where(written, ref + fb, ref)
        S = torch.where(written, S + fb.abs(), S)
    if relu:
        ref = torch.where(written, ref.clamp_min(0.0), ref)
    if logistic:                     # sigma' <= 1/4; sigma itself: 6u sigma + 2^-126 (loss_ref.sigmoid_bar)
        sig = torch.sigmoid(ref)
        ref = torch.where(written, sig, ref)
        S = torch.where(written, S / 4 + (6 * U * sig + 2.0 ** -126) / BAR, S)
    if lmask is not None:            # d s (1 - s): three roundings, 3u |r| + 2^-148 (loss_ref.logistic_deriv_bar)
        sl = lmask[:n].to(torch.float64)
        ds = sl * (1 - sl)
        ref = ref * ds
        S = S * ds + (3 * U * ref.abs() + 2.0 ** -148) / BAR
    zero = torch.zeros(n, dtype=torch.bool, device=dev)
    if drop is not None:
        prob, scale, seed = drop
        kept = torch.from_numpy(dropout_kept(n, prob, seed)).to(dev)
        zero |= written & ~kept
        ref = torch.where(written, ref * scale, ref)
        S = torch.where(written, S * abs(scale), S)
    if mask is not None:
        zero |= ~(mask[:n] > 0)
    ref = torch.where(zero, torch.zeros_like(ref), ref)
    S = torch.where(zero | keep, torch.zeros_like(S), S)
    return Expect(ref, S, zero, keep)


@dataclasses.dataclass
class Verdict:
    ok: bool
    worst_ratio: float        # max |y - ref| / S over elements with S > 0
    share_over: float         # fraction of elements over the bar (or wrong where exactness is required)
    bad_exact: int            # elements that had to be exact (S == 0, zeroed, kept) and were not
    where: str                # the worst element

    def __str__(self):
        return "ok=%s worst |err|/S=%.3e share over=%.2e inexact=%d at %s" % (
            self.ok, self.worst_ratio, self.share_over, self.bad_exact, self.where)


def locate(op, g, i):
    """(n, x, y, c) of target element i (for wgrad: (o, tx, ty, c))"""
    if op == "wgrad":
        o, k = i % g.Cout, i // g.Cout
        return "o=%d tx=%d ty=%d c=%d" % (o, k % g.kx, (k // g.kx) % g.ky, k // (g.kx * g.ky))
    W, H = (g.modX, g.modY) if op == "fprop" else (g.W, g.H)
    n, r = i % g.N, i // g.N
    return "n=%d x=%d y=%d c=%d" % (n, r % W, (r // W) % H, r // (W * H))


def check(op, g, y, e, t0=None, bar=BAR):
    """compare the kernel's float32 output y (flat, the whole target) with an Expect"""
    n = e.ref.numel()
    y = y[:n]
    yd = y.to(torch.float64)
    err = (yd - e.ref).abs()
    pos = e.S > 0
    ratio = torch.where(pos, err / torch.where(pos, e.S, torch.ones_like(e.S)), torch.zeros_like(err))
    ratio = torch.where(torch.isnan(ratio), torch.full_like(ratio, float("inf")), ratio)
    over = pos & ~(ratio <= bar)
    exact = ~pos & ~e.keep & ~(yd == e.ref)
    if t0 is not None:
        exact |= e.keep & (y.view(torch.int32) != t0[:n].view(torch.int32))
    else:
        exact |= e.keep & ~(yd == e.ref)
    bad = over | exact
    nbad = int(bad.sum())
    worst = float(ratio[pos].max()) if bool(pos.any()) else 0.0
    if nbad:
        score = torch.where(exact, torch.full_like(ratio, float("inf")), ratio)
        i = int(torch.argmax(torch.where(bad, score, torch.full_like(score, -1.0))))
        kind = "inexact" if bool(exact[i]) else "ratio %.3e" % float(ratio[i])
        where = "%s (%s: y=%r ref=%r S=%.3e)" % (locate(op, g, i), kind, float(y[i]), float(e.ref[i]), float(e.S[i]))
    else:
        i = int(torch.argmax(ratio))
        where = locate(op, g, i)
    return Verdict(nbad == 0, worst, nbad / max(n, 1), int(exact.sum()), where)
