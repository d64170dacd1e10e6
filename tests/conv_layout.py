"""The shifted-row convolution layout of conv_gemm_f16 (include/vfeat.h: vf_conv_gemm_f16), restated in plain torch.

Activations are channels-last rows of a zero-bordered volume [n][Tp][Hp][Wp], `pitch` columns per row, optionally behind
`row0` guard rows.  A filter tap is a constant row shift; the A operand of tap j is the overlapping-row view
A_j[p] = X.flat[(p + tap_off[j]) * pitch : ... + k_per_tap], zero where p + tap_off[j] lies outside [0, P).

volume() builds X from an NC(T)HW tensor, merged_filter() / unmerged_filter() build Wt, tap_off and lo_mask the way the
I3D and RAFT engines do, gathered_volume() / engine_filter() the repacks and filters of the ResNet and R(2+1)D engines,
and emulate() computes in float64 what the kernel computes.  Test infrastructure only."""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np
import torch
import torch.nn.functional as F

ACT_NONE, ACT_QUICKGELU, ACT_RELU, ACT_SIGMOID, ACT_TANH = 0, 1, 2, 3, 4


@dataclass
class Vol:
    n: int
    Tp: int
    Hp: int
    Wp: int
    t0: int
    t1: int
    h0: int
    h1: int
    w0: int
    w1: int
    row0: int = 0

    @property
    def rows(self) -> int:
        return self.n * self.Tp * self.Hp * self.Wp

    @property
    def P(self) -> int:
        """GEMM rows: the guard rows and the volume."""
        return self.row0 + self.rows

    def region(self) -> list:
        return [self.Tp, self.Hp, self.Wp, self.t0, self.t1, self.h0, self.h1, self.w0, self.w1]

    def keep(self) -> torch.Tensor:
        """[P] bool: output rows inside the valid region (the rest are written as zeros)."""
        m = torch.arange(self.P) - self.row0
        mm = m.clamp_min(0)
        w, r = mm % self.Wp, mm // self.Wp
        h, r = r % self.Hp, r // self.Hp
        t = r % self.Tp
        return ((m >= 0) & (w >= self.w0) & (w < self.w1) & (h >= self.h0) & (h < self.h1)
                & (t >= self.t0) & (t < self.t1))

    def valid_rows(self, y: torch.Tensor) -> torch.Tensor:
        """[P, N] output rows -> [n, N, T, H, W], the valid region in NCTHW order."""
        v = y[self.row0:].reshape(self.n, self.Tp, self.Hp, self.Wp, -1)
        v = v[:, self.t0:self.t1, self.h0:self.h1, self.w0:self.w1]
        return v.permute(0, 4, 1, 2, 3)


def _as5d(t: torch.Tensor) -> torch.Tensor:
    return t if t.dim() == 5 else t.unsqueeze(2)


def split_f16(x: torch.Tensor):
    """x -> (hi, lo) fp16 with hi = fp16(x), lo = fp16(x - hi)."""
    hi = x.half()
    lo = (x - hi.double()).half()
    return hi, lo


def volume(x: torch.Tensor, border, pitch: int | None = None, chan=None, chan_lo=None, row0: int = 0,
           tail_rows: int = 0, junk: float = 0.0, generator: torch.Generator | None = None):
    """Channels-last, zero-bordered rows of x ([n, C, T, H, W] or [n, C, H, W], any float type).

    border: ((t_before, t_after), (h_before, h_after), (w_before, w_after)).  Channel c goes to column chan[c] (default
    c); with chan_lo the row carries a split-fp16 pair, hi at chan[c] and lo = fp16(x - hi) at chan_lo[c].  Columns no
    channel maps to hold uniform values in [-junk, junk] in every row (they meet zero weight columns).  `row0` guard rows
    of junk precede the volume and `tail_rows` rows of random values follow it (the overlapping-row view reads past the
    last row).  Returns (X fp16 [row0 + rows + tail_rows, pitch], Vol, x_eff float64 NC(T)HW: the values the kernel
    multiplies, hi or hi + lo)."""
    x5 = _as5d(x).double()
    n, C, T, H, W = x5.shape
    (tb, ta), (hb, ha), (wb, wa) = border
    chan = list(range(C)) if chan is None else list(chan)
    pitch = pitch if pitch is not None else C
    used = chan + (list(chan_lo) if chan_lo is not None else [])
    assert len(chan) == C and max(used) < pitch and len(set(used)) == len(used)
    v = Vol(n, T + tb + ta, H + hb + ha, W + wb + wa, tb, tb + T, hb, hb + H, wb, wb + W, row0)
    g = generator
    X = torch.zeros(v.P + tail_rows, pitch, dtype=torch.float64)
    if junk:
        X.uniform_(-junk, junk, generator=g)
    body = X[row0:row0 + v.rows].view(n, v.Tp, v.Hp, v.Wp, pitch)
    body[..., used] = 0.0                               # the zero border of the conv input
    hi, lo = split_f16(x5)
    inner = body[:, tb:tb + T, hb:hb + H, wb:wb + W]
    inner[..., chan] = hi.double().permute(0, 2, 3, 4, 1)
    x_eff = hi.double()
    if chan_lo is not None:
        inner[..., list(chan_lo)] = lo.double().permute(0, 2, 3, 4, 1)
        x_eff = x_eff + lo.double()
    if tail_rows:
        X[v.P:].uniform_(-1.0, 1.0, generator=g)
    if x.dim() == 4:
        x_eff = x_eff.squeeze(2)
    return X.half(), v, x_eff


def _weights(w: torch.Tensor, nsplit: int):
    hi, lo = split_f16(w.double())
    return hi, lo, (hi.double() + lo.double()) if nsplit == 2 else hi.double()


def _finish(cols, w5, n_out, ntaps, kpt, nsplit):
    """cols(a, b, d) -> [(hi columns, lo columns or None)]: the K columns of the ci input channels at filter position
    (a, b, d).  Builds Wt ([W_hi | W_lo] along K for nsplit = 2) and lo_mask."""
    co, ci, kt, kh, kw = w5.shape
    hi, lo, w_eff = _weights(w5, nsplit)
    Kb = ntaps * kpt
    Wt = torch.zeros(n_out, nsplit * Kb, dtype=torch.float16)
    has_hi = torch.zeros(Kb, dtype=torch.bool)
    for a in range(kt):
        for b in range(kh):
            for d in range(kw):
                for k_hi, k_lo in cols(a, b, d):
                    k_hi = torch.tensor(k_hi)
                    k_lo = None if k_lo is None else torch.tensor(k_lo)
                    Wt[:co, k_hi] = hi[:, :, a, b, d]
                    has_hi[k_hi] = True
                    if nsplit == 2:
                        Wt[:co, Kb + k_hi] = lo[:, :, a, b, d]
                    if k_lo is not None:
                        Wt[:co, k_lo] = hi[:, :, a, b, d]
                        if nsplit == 2:
                            Wt[:co, Kb + k_lo] = lo[:, :, a, b, d]
    # lo_mask as the engines compute it: a K block of a tap that no tap uses for a hi (or single) activation column
    # multiplies only lo halves, and a_lo . w_lo is below fp32 resolution: its W_lo pass is skipped
    lo_mask = 0
    kb = (kpt + 63) // 64
    if nsplit == 2 and kb <= 64:
        hh = has_hi.view(ntaps, kpt)
        for kk in range(kb):
            if not bool(hh[:, kk * 64:(kk + 1) * 64].any()):
                lo_mask |= 1 << kk
    return Wt, lo_mask, w_eff


def _tap_shift(vol: Vol, dt: int, dh: int, dw: int) -> int:
    return (dt * vol.Hp + dh) * vol.Wp + dw


def merged_filter(w: torch.Tensor, vol: Vol, pitch: int, chan=None, chan_lo=None, nsplit: int = 1,
                  n_out: int | None = None):
    """One tap per (dt, dh) whose kw positions are one run of kw * pitch elements (i3d.cu 3x3x3 / 1x1x1 units,
    raft.cu prep_same_conv).  Stride 1, kernel centred at k // 2.  Returns a dict with Wt (fp16 [n_out,
    nsplit * ntaps * k_per_tap]), ntaps, k_per_tap, tap_off, lo_mask, w_eff (float64, hi or hi + lo, filter layout)."""
    w5 = _as5d(w)
    co, ci, kt, kh, kw = w5.shape
    chan = list(range(ci)) if chan is None else list(chan)
    ntaps, kpt = kt * kh, kw * pitch

    def cols(a, b, d):
        base = (a * kh + b) * kpt + d * pitch
        return [([base + chan[c] for c in range(ci)], None if chan_lo is None else [base + k for k in chan_lo])]

    Wt, lo_mask, w_eff = _finish(cols, w5, n_out or co, ntaps, kpt, nsplit)
    tap_off = [_tap_shift(vol, a - kt // 2, b - kh // 2, -(kw // 2)) for a in range(kt) for b in range(kh)]
    return dict(Wt=Wt, ntaps=ntaps, k_per_tap=kpt, tap_off=tap_off, lo_mask=lo_mask, nsplit=nsplit,
                w_eff=w_eff if w.dim() == 5 else w_eff.squeeze(2))


def unmerged_filter(w: torch.Tensor, vol: Vol, k_per_tap: int, chan=None, chan_lo=None, nsplit: int = 1,
                    n_out: int | None = None):
    """One tap per (dt, dh, dw), each reading k_per_tap columns from the start of its row (raft.cu prep_unmerged_conv).
    Same return value as merged_filter."""
    w5 = _as5d(w)
    co, ci, kt, kh, kw = w5.shape
    chan = list(range(ci)) if chan is None else list(chan)
    ntaps = kt * kh * kw

    def cols(a, b, d):
        base = ((a * kh + b) * kw + d) * k_per_tap
        return [([base + chan[c] for c in range(ci)], None if chan_lo is None else [base + k for k in chan_lo])]

    Wt, lo_mask, w_eff = _finish(cols, w5, n_out or co, ntaps, k_per_tap, nsplit)
    tap_off = [_tap_shift(vol, a - kt // 2, b - kh // 2, d - kw // 2)
               for a in range(kt) for b in range(kh) for d in range(kw)]
    return dict(Wt=Wt, ntaps=ntaps, k_per_tap=k_per_tap, tap_off=tap_off, lo_mask=lo_mask, nsplit=nsplit,
                w_eff=w_eff if w.dim() == 5 else w_eff.squeeze(2))


def act64(y: torch.Tensor, act: int) -> torch.Tensor:
    if act == ACT_QUICKGELU:
        return y * torch.sigmoid(1.702 * y)
    if act == ACT_RELU:
        return torch.relu(y)
    if act == ACT_SIGMOID:
        return torch.sigmoid(y)
    if act == ACT_TANH:
        return torch.tanh(y)
    return y


def epilogue(y: torch.Tensor, bias=None, scale=None, act: int = ACT_NONE) -> torch.Tensor:
    if scale is not None:
        y = y * scale.double()
    if bias is not None:
        y = y + bias.double()
    return act64(y, act)


def emulate(X: torch.Tensor, pitch: int, vol: Vol, f: dict, bias=None, scale=None, act: int = ACT_NONE,
            mask: bool = True, lo_mask: bool = True) -> torch.Tensor:
    """float64 [P, n_out]: what the kernel computes.  lo_mask=False multiplies W_hi + W_lo on every K block, i.e. the
    convolution of the effective operands; lo_mask=True skips W_lo on the lo_mask blocks as the kernel does (the
    difference is a_lo . w_lo, below fp32 resolution for true lo halves, but not for arbitrary data in those columns)."""
    P, kpt, ntaps = vol.P, f["k_per_tap"], f["ntaps"]
    flat = X.reshape(-1).double()
    assert flat.numel() >= (P - 1) * pitch + kpt, "X must be readable for (P-1)*pitch + k_per_tap elements"
    Wt = f["Wt"].to(X.device).double()
    Kb = ntaps * kpt
    W = Wt
    if f["nsplit"] == 2:
        keep_lo = torch.ones(Kb, dtype=torch.float64, device=X.device)
        if lo_mask:
            # per K block in Python integers: bit 63 of a 64-block tap does not fit a signed int64 tensor
            skip = torch.tensor([float((f["lo_mask"] >> kk) & 1) for kk in range((kpt + 63) // 64)])
            keep_lo = (1.0 - skip[torch.arange(Kb) % kpt // 64]).double().to(X.device)
        W = Wt[:, :Kb] + Wt[:, Kb:] * keep_lo
    y = torch.zeros(P, Wt.shape[0], dtype=torch.float64, device=X.device)
    cols = torch.arange(kpt, device=X.device)
    for j in range(ntaps):
        r = torch.arange(P, device=X.device) + f["tap_off"][j]
        ok = (r >= 0) & (r < P)
        A = flat[r.clamp(0, P - 1)[:, None] * pitch + cols[None]] * ok[:, None]
        y += A @ W[:, j * kpt:(j + 1) * kpt].T
    y = epilogue(y, bias, scale, act)
    if mask:
        y = y * vol.keep().to(y.device)[:, None]
    return y


def reference_conv(x_eff: torch.Tensor, w_eff: torch.Tensor, bias=None, scale=None, act: int = ACT_NONE, stride=1,
                   padding=None):
    """F.conv3d / F.conv2d in float64, then the epilogue.  Without `padding`: stride 1, zero padding k // 2 before and
    k - 1 - k // 2 after (the output keeps the input's extent); with it: F.conv's own `stride` and symmetric `padding`.
    Returns NCTHW (or NCHW for 2-D input) with channels last moved to dim 1."""
    x, w = x_eff.double(), w_eff.double()
    conv = F.conv3d if w.dim() == 5 else F.conv2d
    if padding is not None:
        y = conv(x, w, stride=stride, padding=padding)
    else:
        pad = []
        for k in reversed(w.shape[2:]):
            pad += [k // 2, k - 1 - k // 2]
        y = conv(F.pad(x, pad), w)
    shape = [1, -1] + [1] * (y.dim() - 2)
    if scale is not None:
        y = y * scale.double().view(shape)
    if bias is not None:
        y = y + bias.double().view(shape)
    return act64(y, act)


# ----------------------------------------------------------------------------- the geometries the parity tests run
# HX rows of RAFT's GRU (csrc/raft_kernels.h): 384 conv input channels over 768 columns, hi and lo halves in alternate
# 128-column blocks
HX_CHAN = [c if c < 128 else (128 + c if c < 256 else 256 + c) for c in range(384)]
HX_CHAN_LO = [128 + c if c < 128 else (256 + c if c < 256 else 384 + c) for c in range(384)]


def _i3d3(C, N, n, T, HW, out):
    return dict(id=f"i3d3x3x3-c{C}-n{N}-{n}x{T}x{HW}", x=(n, C, T, HW, HW), k=(3, 3, 3), border=((1, 1),) * 3,
                layout="merged", pitch=C, N=N, act=ACT_RELU if out != "f32" else ACT_NONE, out=out, row0=0,
                c_off=8, ctot=8 + N + 8)


def _pair1(C, N, n, T, HW):
    # a 1x1x1 unit of a Mixed block: pair rows [hi C | lo C] in, the split output into a channel slice of the concat
    # row (mixed_block: out + c_off, ldo = 2 * ctot, split_off = ctot)
    return dict(id=f"i3d1x1x1-pair-c{C}-n{N}-{n}x{T}x{HW}", x=(n, C, T, HW, HW), k=(1, 1, 1), border=((1, 1),) * 3,
                layout="merged", pitch=2 * C, chan_lo=[C + c for c in range(C)], N=N, act=ACT_RELU, out="split",
                c_off=16, ctot=16 + N + 24, row0=0)


I3D_CASES = [
    _i3d3(16, 48, 1, 2, 7, "f32"),        # k_per_tap 48: one partial K block per tap
    _i3d3(24, 16, 2, 4, 14, "f16"),       # 72: a 64 + 8 tail; N = 16 in a 64-wide tile
    _i3d3(48, 64, 1, 8, 28, "split"),     # 144
    _i3d3(112, 96, 1, 4, 7, "f16"),       # 336; 128-wide tile, N tail
    _i3d3(96, 208, 3, 4, 14, "f32"),      # 288; 256-wide tile, N tail
    _i3d3(112, 288, 2, 2, 28, "f16"),     # 192-wide tiles
    _i3d3(144, 320, 1, 11, 14, "split"),  # 432; 192-wide, N tail
    _i3d3(192, 384, 3, 8, 28, "f32"),     # 576; 422 tiles: several per CTA
    _pair1(40, 24, 2, 4, 7),              # the hi / lo boundary (column 40) inside K block 0
    _pair1(192, 64, 1, 4, 28),
    _pair1(480, 192, 2, 4, 14),
    _pair1(528, 256, 1, 4, 14),
    _pair1(832, 384, 3, 2, 7),
]

RAFT_CASES = [
    # encoder 3x3 over pair rows, split output; `row0` guard rows in front
    dict(id="raft3x3-pair-c64", x=(2, 64, 12, 16), k=(3, 3), border=((0, 0), (1, 1), (1, 1)), layout="merged",
         pitch=128, chan_lo=[64 + c for c in range(64)], N=64, act=ACT_RELU, out="split", c_off=0, ctot=64, row0=21),
    dict(id="raft3x3-pair-c96", x=(2, 96, 10, 14), k=(3, 3), border=((0, 0), (1, 1), (1, 1)), layout="merged",
         pitch=192, chan_lo=[96 + c for c in range(96)], N=96, act=ACT_RELU, out="split", c_off=0, ctot=96, row0=5),
    # GRU gates on HX rows: 1x5 (one tap of 5 x 768 columns) and 5x1 (five taps of 768), fp32 sigmoid / tanh
    dict(id="raft1x5-hx-zr-sigmoid", x=(2, 384, 9, 13), k=(1, 5), border=((0, 0), (3, 3), (3, 3)), layout="merged",
         pitch=768, chan=HX_CHAN, chan_lo=HX_CHAN_LO, N=256, act=ACT_SIGMOID, out="f32", row0=3 * 19 + 3),
    dict(id="raft5x1-hx-q-tanh", x=(2, 384, 9, 13), k=(5, 1), border=((0, 0), (3, 3), (3, 3)), layout="merged",
         pitch=768, chan=HX_CHAN, chan_lo=HX_CHAN_LO, N=128, act=ACT_TANH, out="f32", row0=3 * 19 + 3),
    # 7x7 over a 2-channel pair (convf1: flow8 rows of 8 columns), 56 columns per tap
    dict(id="raft7x7-merged-flow", x=(2, 2, 12, 12), k=(7, 7), border=((0, 0), (3, 3), (3, 3)), layout="merged",
         pitch=8, chan_lo=[2, 3], N=128, act=ACT_RELU, out="f16", row0=3),
    # unmerged: one tap per filter position, each reading the first k_per_tap columns of a wider row
    dict(id="raft7x7-unmerged-49taps", x=(2, 24, 11, 9), k=(7, 7), border=((0, 0), (3, 3), (3, 3)), layout="unmerged",
         pitch=64, kpt=48, chan_lo=[24 + c for c in range(24)], N=64, act=ACT_NONE, out="f32", row0=9),
    dict(id="raft8x8-unmerged-64taps", x=(1, 8, 10, 12), k=(8, 8), border=((0, 0), (4, 3), (4, 3)), layout="unmerged",
         pitch=16, kpt=16, chan_lo=[8 + c for c in range(8)], N=32, act=ACT_NONE, out="f32", row0=0),
]

ALL_CASES = I3D_CASES + RAFT_CASES


def build_case(case: dict, nsplit: int, seed: int, n_out: int | None = None) -> dict:
    """Seeded operands of one case: X, the filter (merged_filter / unmerged_filter), bias, scale, and the float64
    operands x_eff / w_eff as the kernel sees them.  n_out < N keeps only the first output channels (the layout does
    not depend on them)."""
    if case["layout"] in ENGINE_FILTERS:
        return build_engine_case(case, nsplit, seed, n_out)
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(*case["x"], generator=g) * 0.5
    ci = case["x"][1]
    N = case["N"] if n_out is None else n_out
    w = torch.randn(N, ci, *case["k"], generator=g) * (ci * float(torch.tensor(case["k"]).prod())) ** -0.5
    bias = torch.randn(N, generator=g) * 0.1
    scale = 1 + 0.1 * torch.randn(N, generator=g)
    pitch = case["pitch"]
    kpt = case.get("kpt", pitch * case["k"][-1])
    tail = max(0, -(-(kpt - pitch) // pitch))           # the last row's view runs kpt - pitch elements past it
    X, vol, x_eff = volume(x, case["border"], pitch=pitch, chan=case.get("chan"), chan_lo=case.get("chan_lo"),
                           row0=case["row0"], tail_rows=tail, junk=1.0, generator=g)
    if case["layout"] == "merged":
        f = merged_filter(w, vol, pitch, chan=case.get("chan"), chan_lo=case.get("chan_lo"), nsplit=nsplit)
    else:
        f = unmerged_filter(w, vol, kpt, chan=case.get("chan"), chan_lo=case.get("chan_lo"), nsplit=nsplit)
    return dict(X=X, pitch=pitch, vol=vol, f=f, bias=bias, scale=scale, act=case["act"], x_eff=x_eff, w_eff=f["w_eff"])


# ----------------------------------------------------------------- the ResNet and R(2+1)D layouts (csrc/resnet.cu, r21d.cu)
# Every activation is a split pair row [hi C | lo C]; every filter a hi + lo pair over both halves (nsplit = 2).  The
# strided convs read repacks of their input, restated here by gathered_volume():
#   2-D phase repack (raft_phase_repack): phase row (qh, qw) holds x[2(qh - q0) + ph][2(qw - q0) + pw] for the 4 phases
#     (ph, pw), each a [hi C | lo C] run at column (2 ph + pw) * 2C; q0 = 1 (rows of a border-1 volume), q0 = 2 for the
#     stems' phase volumes (rows [16 hi | 16 lo], phase p's 3 channels at 4p .. 4p + 2, column 4p + 3 unused);
#   temporal phase repack (r21d_temporal_phase): frame row q holds [x[2(q - 1)] | x[2(q - 1) + 1]], each a pair run;
#   (2,2,2) subsample (r21d_subsample): row (t, h, w) holds x[2(t - 1)][2(h - 1)][2(w - 1)].
# ENGINE_FILTERS mirror the prep_* builders of resnet.cu / r21d.cu: (ntaps, k_per_tap, tap shifts (dt, dh, dw),
# K column of the hi half of channel c at filter position (kt, kh, kw), column offset of its lo half).

def pad8(c: int) -> int:
    return (c + 7) // 8 * 8


def _idx(n_pos: int, size: int, f) -> torch.Tensor:
    """Source index f(q) of each volume position q, or `size` (a zero slice) outside [0, size)."""
    i = torch.tensor([f(q) for q in range(n_pos)])
    return torch.where((i >= 0) & (i < size), i, size)


def gathered_volume(x: torch.Tensor, shape, placements, lo_off: int, pitch: int, chan_pad: int | None = None,
                    tail_rows: int = 0, junk: float = 1.0, generator: torch.Generator | None = None):
    """x [n, C, T, H, W] (or [n, C, H, W]) -> (X fp16 [rows + tail_rows, pitch], x_eff float64 hi + lo of x).

    Position (b, t, h, w) of the [n][Tp][Hp][Wp] volume `shape` holds, per placement (col, ft, fh, fw), the split pair
    of x[b, :, ft(t), fh(h), fw(w)] (zero where an index falls outside x): hi of channel c at column col + c, lo at
    col + lo_off + c.  The pad channels C .. chan_pad of a padded width hold zeros, as the engines write them; columns
    no channel maps to hold uniform values in [-junk, junk], and so do the tail rows."""
    x5 = _as5d(x).double()
    n, C, T, H, W = x5.shape
    Tp, Hp, Wp = shape
    X = torch.empty(n * Tp * Hp * Wp + tail_rows, pitch, dtype=torch.float64).uniform_(-junk, junk, generator=generator)
    body = X[:n * Tp * Hp * Wp].view(n, Tp, Hp, Wp, pitch)
    hi, lo = split_f16(x5)
    hp, lp = F.pad(hi.double(), (0, 1, 0, 1, 0, 1)), F.pad(lo.double(), (0, 1, 0, 1, 0, 1))
    width = chan_pad or C
    for col, ft, fh, fw in placements:
        it, ih, iw = _idx(Tp, T, ft), _idx(Hp, H, fh), _idx(Wp, W, fw)
        for src, off in ((hp, col), (lp, col + lo_off)):
            v = src[:, :, it][:, :, :, ih][:, :, :, :, iw].permute(0, 2, 3, 4, 1)
            body[..., off:off + width] = 0.0
            body[..., off:off + C] = v
    return X.half(), (hi.double() + lo.double()) if x.dim() == 5 else (hi.double() + lo.double()).squeeze(2)


def _stride2_col(kpt, cpp):
    def col(kt, kh, kw, c):
        a, ph, b, pw = (kh + 1) // 2, (kh + 1) % 2, (kw + 1) // 2, (kw + 1) % 2
        return (a * 2 + b) * kpt + (ph * 2 + pw) * cpp + c
    return col


def _stem_col(kt, kh, kw, c):
    a, ph, b, pw = (kh + 1) // 2, (kh + 1) % 2, (kw + 1) // 2, (kw + 1) % 2
    return a * 128 + b * 32 + (ph * 2 + pw) * 4 + c


ENGINE_FILTERS = {
    # prep_same: k kernel rows, each a run of k * 2ci_p; k = 1 is also the stride-2 downsample, which
    # reads phase (0, 0), the first 2ci columns of a phase row
    "same": lambda k, ci, ci_p: (k, 2 * k * ci_p, [(0, a - k // 2, -(k // 2)) for a in range(k)],
                                 lambda kt, kh, kw, c: kh * 2 * k * ci_p + kw * 2 * ci_p + c, ci_p),
    # prep_stride2: tap (a, b) reads phase row (q + a - 1, q' + b - 1); kh = 2a + ph - 1
    "stride2": lambda k, ci, ci_p: (4, 8 * ci, [(0, t // 2 - 1, t % 2 - 1) for t in range(4)],
                                    _stride2_col(8 * ci, 2 * ci), ci),
    # prep_stem (both engines): 4 taps of kernel row pairs, each 4 phase positions x 32 columns
    "stem": lambda k, ci, ci_p: (4, 128, [(0, a - 2, -2) for a in range(4)], _stem_col, 16),
    # prep_temporal: 3 taps one frame apart
    "temporal": lambda k, ci, ci_p: (3, 2 * ci_p, [(a - 1, 0, 0) for a in range(3)],
                                     lambda kt, kh, kw, c: kt * 2 * ci_p + c, ci_p),
    # prep_temporal2: frame 2t - 1 from the odd half of row t - 1, frames 2t and 2t + 1 from row t
    "temporal2": lambda k, ci, ci_p: (2, 4 * ci_p, [(-1, 0, 0), (0, 0, 0)],
                                      lambda kt, kh, kw, c: 2 * ci_p + c if kt == 0 else 4 * ci_p + (kt - 1) * 2 * ci_p + c,
                                      ci_p),
    # prep_same (k = 1): 1x1x1 over the subsampled block input
    "point": lambda k, ci, ci_p: (1, 2 * ci, [(0, 0, 0)], lambda kt, kh, kw, c: c, ci),
}


def engine_filter(kind: str, w: torch.Tensor, vol: Vol, ci_p: int | None = None, n_out: int | None = None,
                  nsplit: int = 2):
    """The filter of one engine conv: Wt (fp16 [n_out, nsplit * ntaps * k_per_tap], rows past co zero), tap_off,
    lo_mask (bit kk: K block kk of every tap meets only lo halves; a tap of exactly 64 blocks keeps bit 63), w_eff
    (float64, hi or hi + lo, zero filters for the pad rows up to n_out)."""
    w5 = _as5d(w)
    co, ci, kt, kh, kw = w5.shape
    ntaps, kpt, shifts, col, lo_off = ENGINE_FILTERS[kind](kh, ci, ci_p or ci)
    n_out = n_out or co

    def cols(a, b, d):
        k = [col(a, b, d, c) for c in range(ci)]
        return [(k, [j + lo_off for j in k])]

    Wt, lo_mask, w_eff = _finish(cols, w5, n_out, ntaps, kpt, nsplit)
    w_eff = torch.cat([w_eff, w_eff.new_zeros(n_out - co, *w_eff.shape[1:])])
    return dict(Wt=Wt, ntaps=ntaps, k_per_tap=kpt, shifts=shifts, tap_off=[_tap_shift(vol, *s) for s in shifts],
                lo_mask=lo_mask, nsplit=nsplit, w_eff=w_eff if w.dim() == 5 else w_eff.squeeze(2))


def _geometry(case):
    """(volume shape, Vol of the output, placements, lo_off, pitch, chan_pad) of a case: the output volume and the
    rows the conv reads on it."""
    n, C, T, H, W = case["x"] if len(case["x"]) == 5 else (case["x"][0], case["x"][1], 1) + tuple(case["x"][2:])
    src, Cp = case["src"], case.get("ci_p", C)
    b, tb = case["border"], case.get("t_border", 0)      # spatial / temporal border before the valid region
    if src == "rows":                   # the activation itself, [hi Cp | lo Cp]
        Tp, Hp, Wp = T + 2 * tb, H + b + 1, W + b + 1
        pl = [(0, lambda t: t - tb, lambda h: h - b, lambda w: w - b)]
        lo_off, pitch = Cp, 2 * Cp
        valid = (tb, tb + T, b, b + H, b, b + W)
    elif src in ("phase", "stem_phase"):
        q0 = 2 if src == "stem_phase" else 1
        S = H // 2
        Tp, Hp, Wp = T + 2 * tb, S + q0 + 1, S + q0 + 1
        cpp = 4 if src == "stem_phase" else 2 * C
        pl = [((2 * ph + pw) * cpp, lambda t: t - tb, lambda q, ph=ph: 2 * (q - q0) + ph,
               lambda q, pw=pw: 2 * (q - q0) + pw) for ph in (0, 1) for pw in (0, 1)]
        lo_off, pitch = (16, 32) if src == "stem_phase" else (C, 8 * C)
        valid = (tb, tb + T, q0, q0 + S, q0, q0 + S)
    elif src == "temporal_phase":       # on the output's frames (T' = (T - 1) // 2 + 1), spatial border 1
        To = (T - 1) // 2 + 1
        Tp, Hp, Wp = To + 2, H + 2, W + 2
        pl = [(p * 2 * Cp, lambda q, p=p: 2 * (q - 1) + p, lambda h: h - 1, lambda w: w - 1) for p in (0, 1)]
        lo_off, pitch = Cp, 4 * Cp
        valid = (1, To + 1, 1, H + 1, 1, W + 1)
    else:                               # "subsample": (2,2,2) subsample of the block input on the output volume
        To, S = (T - 1) // 2 + 1, H // 2
        Tp, Hp, Wp = To + 2, S + 2, S + 2
        pl = [(0, lambda q: 2 * (q - 1), lambda h: 2 * (h - 1), lambda w: 2 * (w - 1))]
        lo_off, pitch = C, 2 * C
        valid = (1, To + 1, 1, S + 1, 1, S + 1)
    return (Tp, Hp, Wp), Vol(n, Tp, Hp, Wp, *valid), pl, lo_off, pitch, (Cp if Cp != C else None)


def build_engine_case(case: dict, nsplit: int, seed: int, n_out: int | None = None) -> dict:
    """build_case() for the ResNet / R(2+1)D layouts.  N is the padded width; pad output channels have zero filters,
    scale and bias, as the engines upload them.  `conv` holds F.conv's stride and padding for reference_conv."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(*case["x"], generator=g) * 0.5
    ci = case["x"][1]
    co = case.get("co", case["N"]) if n_out is None else min(n_out, case.get("co", case["N"]))
    N = case["N"] if n_out is None else n_out
    k = case["k"]
    w = torch.randn(co, ci, *k, generator=g) * (ci * float(torch.tensor(k).prod())) ** -0.5
    bias = torch.zeros(N)
    scale = torch.zeros(N)
    bias[:co] = torch.randn(co, generator=g) * 0.1
    scale[:co] = 1 + 0.1 * torch.randn(co, generator=g)
    shape, vol, pl, lo_off, pitch, chan_pad = _geometry(case)
    f = engine_filter(case["layout"], w, vol, ci_p=case.get("ci_p"), n_out=N, nsplit=nsplit)
    tail = max(0, -(-(f["k_per_tap"] - pitch) // pitch))
    X, x_eff = gathered_volume(x, shape, pl, lo_off, pitch, chan_pad=chan_pad, tail_rows=tail, generator=g)
    return dict(X=X, pitch=pitch, vol=vol, f=f, bias=bias, scale=scale, act=case["act"], x_eff=x_eff, w_eff=f["w_eff"],
                conv=case["conv"], co=co)


def _res(id, layout, x, k, N, src, border, conv, act=ACT_RELU):
    return dict(id=id, layout=layout, x=x, k=k, N=N, src=src, border=border, conv=conv, act=act, out="split",
                c_off=0, ctot=N, row0=0)


def _r21(id, layout, x, k, N, src, conv, co=None, ci_p=None, border=1, act=ACT_RELU):
    c = dict(id=id, layout=layout, x=x, k=k, N=N, src=src, border=border, t_border=1, conv=conv, act=act, out="split",
             c_off=0, ctot=N, row0=0)
    if co is not None:
        c["co"] = co
    if ci_p is not None:
        c["ci_p"] = ci_p
    return c


S2 = dict(stride=2, padding=1)
RESNET_CASES = [
    # stem 7x7/2 pad 3 on the transform's phase volume: [n][115][115] rows of 32, 4 taps x 128
    _res("resnet-stem-115", "stem", (2, 3, 224, 224), (7, 7), 64, "stem_phase", 0, dict(stride=2, padding=3)),
    # stride-1 3x3 at 58^2 (layer1, basic block): 3 taps of 3 x 128
    _res("resnet-3x3-c64-58", "same", (2, 64, 56, 56), (3, 3), 64, "rows", 1, dict(stride=1, padding=1), ACT_NONE),
    # stride-2 3x3 on the phase repack: layer2.0 conv1 of a basic block (58^2 -> 30^2), 4 taps of 8 x 64
    _res("resnet-3x3s2-c64-30", "stride2", (2, 64, 56, 56), (3, 3), 128, "phase", 1, S2),
    # layer3.0 conv2 of a bottleneck (width 256, 30^2 -> 16^2)
    _res("resnet-3x3s2-c256-16", "stride2", (1, 256, 28, 28), (3, 3), 256, "phase", 1, S2),
    # layer4.0 conv2 of a bottleneck at width 512 (16^2 -> 9^2): k_per_tap 4096 = 64 K blocks, lo_mask bit 63 set
    _res("resnet-3x3s2-c512-9", "stride2", (2, 512, 14, 14), (3, 3), 512, "phase", 1, S2),
    # stride-2 1x1 downsample: phase (0, 0) of the same repack, the first 2C of an 8C row
    _res("resnet-down-c64-30", "same", (2, 64, 56, 56), (1, 1), 128, "phase", 1, dict(stride=2, padding=0), ACT_NONE),
    # ResNet-50 layer4.0 downsample: 2048 columns of an 8192-element phase row
    _res("resnet-down-c1024-9", "same", (2, 1024, 14, 14), (1, 1), 2048, "phase", 1, dict(stride=2, padding=0),
         ACT_NONE),
    # layer4 conv1 1x1 at cin 2048: 64 K blocks, the lo half in blocks 32 .. 63
    _res("resnet-1x1-c2048-9", "same", (2, 2048, 7, 7), (1, 1), 512, "rows", 1, dict(stride=1, padding=0)),
]

R21D_CASES = [
    # stem (1,7,7)/(1,2,2) on the per-frame phase volume [T+2][59][59], 45 outputs padded to 48
    _r21("r21d-stem-59-T5", "stem", (1, 3, 5, 112, 112), (1, 7, 7), 48, "stem_phase", dict(stride=(1, 2, 2),
         padding=(0, 3, 3)), co=45),
    # the stem's temporal conv 45 -> 64 over 48-wide pair rows: K 96, the lo half from column 48 inside block 0
    _r21("r21d-temporal-c45-59-T5", "temporal", (1, 45, 5, 56, 56), (3, 1, 1), 64, "rows",
         dict(stride=1, padding=(1, 0, 0)), ci_p=48, border=2),
    # layer2.0 conv1 spatial stride (1,2,2) on the phase repack of every frame: 64 -> 230 (232)
    _r21("r21d-spatial2-c64-30-T5", "stride2", (1, 64, 5, 56, 56), (1, 3, 3), 232, "phase",
         dict(stride=(1, 2, 2), padding=(0, 1, 1)), co=230),
    # layer2.0 conv1 temporal stride (2,1,1) on the temporal phase repack: 230 (232) -> 128, K 928 (a 32-column tail)
    _r21("r21d-temporal2-c230-30-T5", "temporal2", (1, 230, 5, 28, 28), (3, 1, 1), 128, "temporal_phase",
         dict(stride=(2, 1, 1), padding=(1, 0, 0)), ci_p=232),
    # layer2.0 downsample: 1x1x1 over the (2,2,2) subsample of the block input
    _r21("r21d-down-c64-30-T5", "point", (1, 64, 5, 56, 56), (1, 1, 1), 128, "subsample", dict(stride=2, padding=0),
         act=ACT_NONE),
    # layer3 conv2 spatial 256 -> 460 (464) at 16^2
    _r21("r21d-spatial-c256-16-T3", "same", (2, 256, 3, 14, 14), (1, 3, 3), 464, "rows",
         dict(stride=1, padding=(0, 1, 1)), co=460),
    # layer4.0 conv1 spatial stride (1,2,2): 256 -> 921 (928) at 9^2, k_per_tap 2048
    _r21("r21d-spatial2-c256-9-T3", "stride2", (1, 256, 3, 14, 14), (1, 3, 3), 928, "phase",
         dict(stride=(1, 2, 2), padding=(0, 1, 1)), co=921),
    # layer4 conv2 temporal 921 (928) -> 512 at 9^2, T' = 1 (a 32-column tail of a 1856-column tap)
    _r21("r21d-temporal-c921-9-T1", "temporal", (2, 921, 1, 7, 7), (3, 1, 1), 512, "rows",
         dict(stride=1, padding=(1, 0, 0)), ci_p=928, act=ACT_NONE),
]

ENGINE_CASES = RESNET_CASES + R21D_CASES


# ------------------------------------------------------------------ the I3D and RAFT filters as the engines upload them
# Restated from i3d.cu prepare_unit and raft.cu upload_conv / prep_* (vf_i3d_conv, vf_raft_conv read them back).  Each
# returns, per conv: Wt (fp16 [n_out, nsplit * ntaps * k_per_tap], W_hi | W_lo), ntaps, k_per_tap, nsplit, the tap
# shifts (dt, dh, dw), lo_mask, and the fp32 scale / bias of the epilogue (pad rows zero).

def _f32(t):
    return t.detach().float().numpy()


def _bn_fold(sd, p):
    """BatchNorm eval folded in fp32 the way the engines do it: s = g / sqrtf(v + 1e-5f), shift = b - m s.  In numpy
    float32 (one IEEE rounding per operation, as the host C code; torch's vectorised CPU kernels may differ by 1 ulp)."""
    g, v, b, m = (_f32(sd[p + k]) for k in (".weight", ".running_var", ".bias", ".running_mean"))
    s = g / np.sqrt(v + np.float32(1e-5))
    return torch.from_numpy(s), torch.from_numpy(b - m * s)


def _upload(w, cols, n_out, ntaps, kpt, nsplit, shifts, scale, bias, lo_mask=None):
    w5 = _as5d(w.float())
    Wt, mask, _ = _finish(cols, w5, n_out, ntaps, kpt, nsplit)
    co = w5.shape[0]
    sc, bi = torch.zeros(n_out), torch.zeros(n_out)
    sc[:co], bi[:co] = scale, bias
    return dict(Wt=Wt, ntaps=ntaps, k_per_tap=kpt, nsplit=nsplit, shifts=shifts,
                lo_mask=mask if lo_mask is None else lo_mask, scale=sc, bias=bi, n_out=n_out)


# i3d.cu prepare_unit's `chosen`: the stem and the 3x3x3 convs of mixed_3b / 3c keep single fp16 weights
I3D_SINGLE_UNITS = (0, 5, 7, 11, 13)


def i3d_engine_filter(sd, name: str, index: int, nsplit: int):
    """Unit `name` (index in unit_names() order) as i3d.cu uploads it with weight split nsplit:
    1x1x1: one tap over both halves of a pair row [hi ci | lo ci], lo_mask bit kk where K block kk starts in the lo half;
    3x3x3: 9 taps (kt, kh), each a run of the 3 kw positions x ci; the stem (7x7x7 stride 2 over the 8-phase volume):
    4 t-taps of 4 w-positions x (4 h-slots x 8 phases x ci), filter index 2a + p, the k = 7 positions left empty."""
    w = sd[name + ".conv3d.weight"].float()
    co, ci, k = w.shape[0], w.shape[1], w.shape[2]
    s, sh = _bn_fold(sd, name + ".batch3d")
    if k == 1:
        cols, ntaps, kpt, shifts = (lambda a, b, d: [(list(range(ci)), [ci + c for c in range(ci)])]), 1, 2 * ci, [(0, 0, 0)]
    elif k == 3:
        ntaps, kpt = 9, 3 * ci
        cols = lambda a, b, d: [([(a * 3 + b) * kpt + d * ci + c for c in range(ci)], None)]
        shifts = [(j // 3 - 1, j % 3 - 1, -1) for j in range(9)]
    else:
        pc = 8 * ci
        ntaps, kpt = 4, 16 * pc

        def cols(kt, kh, kw):
            a, pt, b, ph, cw, pw = kt // 2, kt % 2, kh // 2, kh % 2, kw // 2, kw % 2
            return [([a * kpt + cw * 4 * pc + b * pc + ((pt * 2 + ph) * 2 + pw) * ci + c for c in range(ci)], None)]
        shifts = [(a - 1, 0, -1) for a in range(4)]
    f = _upload(w, cols, co, ntaps, kpt, nsplit, shifts, s, sh)
    if k != 1:
        f["lo_mask"] = 0            # only the 1x1x1 units read pair rows
    return f


def i3d_engine_filters(sd, unit_names, single=I3D_SINGLE_UNITS, fast=False):
    """Every unit; `single`: the units with single fp16 weights (() for VF_I3D_SINGLE=none), fast: all of them."""
    return [i3d_engine_filter(sd, n, i, 1 if (fast or i in single) else 2) for i, n in enumerate(unit_names)]


RAFT_CF_LO = 384                     # csrc/raft_kernels.h: the correlation features' lo half
RAFT_CF, RAFT_HX = 768, 768


def _raft_same(w, b, n_out, pitch, chan=None, chan_lo=None, nsplit=2, scale=None, shift=None, extra=1.0):
    """prep_same_conv: taps = kernel rows (dh = a - kh/2), each a run of kw x pitch from kw/2 positions to the left."""
    co, ci, kh, kw = w.shape
    chan = list(range(ci)) if chan is None else list(chan)
    kpt = kw * pitch

    def cols(_, a, d):
        base = a * kpt + d * pitch
        return [([base + chan[c] for c in range(ci)], None if chan_lo is None else [base + k for k in chan_lo])]
    return _upload(w, cols, n_out, kh, kpt, nsplit, [(0, a - kh // 2, -(kw // 2)) for a in range(kh)],
                   *_raft_epilogue(b, scale, shift, extra))


def _raft_epilogue(b, scale, shift, extra):
    """upload_conv: scale s = bn_scale x extra, bias = b s + bn_shift x extra (fp32, no fused multiply-add)."""
    e = np.float32(extra)
    s = (_f32(scale) if scale is not None else np.ones(b.shape[0], np.float32)) * e
    sh = _f32(shift) if shift is not None else np.zeros(b.shape[0], np.float32)
    return torch.from_numpy(s), torch.from_numpy(_f32(b) * s + sh * e)


def _raft_unmerged(w, b, n_out, nsplit=2, extra=1.0):
    """prep_unmerged_conv with dup: one tap per (kh, kw) reading [x_hi ci | x_lo ci], the weight in both halves."""
    co, ci, kh, kw = w.shape
    kpt = 2 * ci

    def cols(_, a, d):
        base = (a * kw + d) * kpt
        return [([base + c for c in range(ci)], [base + ci + c for c in range(ci)])]
    shifts = [(0, a - kh // 2, d - kw // 2) for a in range(kh) for d in range(kw)]
    return _upload(w, cols, n_out, kh * kw, kpt, nsplit, shifts, *_raft_epilogue(b, None, None, extra))


def _raft_stride2(w, b, n_out, pitch, phase_stride, lo_off, scale, shift):
    """prep_stride2_conv: k x k stride 2 over the phase repack; tap a reads phase row q + a - B (B = 2 for k = 7, 1 for
    k = 3); filter index kh = 2a + ph - 1, kw = 2bq + pw - 1; lo half lo_off columns right of the hi half."""
    co, ci, k, _ = w.shape
    na, before = (4, 2) if k == 7 else (2, 1)
    kpt = na * pitch

    def col(kh, kw, c):
        a, ph, bq, pw = (kh + 1) // 2, (kh + 1) % 2, (kw + 1) // 2, (kw + 1) % 2
        return a * kpt + bq * pitch + (ph * 2 + pw) * phase_stride + c

    def cols(_, kh, kw):
        hi = [col(kh, kw, c) for c in range(ci)]
        return [(hi, [j + lo_off for j in hi])]
    return _upload(w, cols, n_out, na, kpt, 2, [(0, a - before, -before) for a in range(na)],
                   *_raft_epilogue(b, scale, shift, 1.0))


def raft_engine_filters(sd_in):
    """Every conv of raft.cu in vf_raft_conv's order (include/vfeat.h), with the names of their weights."""
    sd = {(k[7:] if k.startswith("module.") else k): v.float() for k, v in sd_in.items()}
    out = []

    def add(name, f):
        out.append((name, f))

    for p, batch in (("fnet", False), ("cnet", True)):
        def bn(n):
            return _bn_fold(sd, f"{p}.{n}") if batch else (None, None)

        def W(n):
            return sd[f"{p}.{n}.weight"], sd[f"{p}.{n}.bias"]

        def same3(n, norm, c):
            return _raft_same(*W(n), c, 2 * c, chan_lo=[c + i for i in range(c)], scale=bn(norm)[0], shift=bn(norm)[1])
        # stem: input phase rows [16 hi | 16 lo], 4 (3 used) channels per phase
        add(f"{p}.conv1", _raft_stride2(*W("conv1"), 64, 32, 4, 16, *bn("norm1")))
        for blk in range(2):
            for cv in (1, 2):
                add(f"{p}.layer1.{blk}.conv{cv}", same3(f"layer1.{blk}.conv{cv}", f"layer1.{blk}.norm{cv}", 64))
        for L, (ci, co) in ((2, (64, 96)), (3, (96, 128))):
            lp = f"layer{L}"
            add(f"{p}.{lp}.0.conv1", _raft_stride2(*W(f"{lp}.0.conv1"), co, 8 * ci, 2 * ci, ci, *bn(f"{lp}.0.norm1")))
            wd, bd = W(f"{lp}.0.downsample.0")
            # the 1x1 stride-2 downsample reads phase (0, 0) of the repacked row: [hi ci | lo ci]
            add(f"{p}.{lp}.0.downsample.0",
                _upload(wd, lambda a, b, d, ci=ci: [(list(range(ci)), [ci + c for c in range(ci)])], co, 1, 2 * ci, 2,
                        [(0, 0, 0)], *_raft_epilogue(bd, *bn(f"{lp}.0.downsample.1"), 1.0)))
            for n, norm in ((".0.conv2", ".0.norm2"), (".1.conv1", ".1.norm1"), (".1.conv2", ".1.norm2")):
                add(f"{p}.{lp}{n}", same3(lp + n, lp + norm, co))
        add(f"{p}.conv2", _raft_same(*W("conv2"), 256, 256, chan_lo=[128 + c for c in range(128)]))

    u = "update_block."

    def W(n):
        return sd[u + n + ".weight"], sd[u + n + ".bias"]
    lo256 = [256 + c for c in range(256)]
    add("encoder.convc1", _raft_same(*W("encoder.convc1"), 256, RAFT_CF, chan_lo=[RAFT_CF_LO + c for c in range(324)]))
    add("encoder.convc2", _raft_same(*W("encoder.convc2"), 192, 512, chan_lo=lo256))
    # flow8 rows = (fx_hi, fy_hi, fx_lo, fy_lo, 0 ...)
    add("encoder.convf1", _raft_same(*W("encoder.convf1"), 128, 8, chan_lo=[2, 3]))
    add("encoder.convf2", _raft_same(*W("encoder.convf2"), 64, 256, chan_lo=[128 + c for c in range(128)]))
    add("encoder.conv", _raft_same(*W("encoder.conv"), 128, 512, chan_lo=lo256))        # 126 rows padded to 128
    for sfx in ("1", "2"):
        wz, bz = W("gru.convz" + sfx)
        wr, br = W("gru.convr" + sfx)
        add("gru.convz|r" + sfx, _raft_same(torch.cat([wz, wr]), torch.cat([bz, br]), 256, RAFT_HX, chan=HX_CHAN,
                                            chan_lo=HX_CHAN_LO))
        add("gru.convq" + sfx, _raft_same(*W("gru.convq" + sfx), 128, RAFT_HX, chan=HX_CHAN, chan_lo=HX_CHAN_LO))
    add("flow_head.conv1", _raft_unmerged(*W("flow_head.conv1"), 256))
    add("flow_head.conv2", _raft_same(*W("flow_head.conv2"), 8, 512, chan_lo=lo256))      # 2 rows padded to 8
    add("mask.0", _raft_unmerged(*W("mask.0"), 256, nsplit=1))
    add("mask.2", _raft_same(*W("mask.2"), 576, 256, nsplit=1, extra=0.25))
    return out
