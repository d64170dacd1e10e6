"""The shifted-row convolution layout of conv_gemm_f16 (include/vfeat.h: vf_conv_gemm_f16), restated in plain torch.

Activations are channels-last rows of a zero-bordered volume [n][Tp][Hp][Wp], `pitch` columns per row, optionally behind
`row0` guard rows.  A filter tap is a constant row shift; the A operand of tap j is the overlapping-row view
A_j[p] = X.flat[(p + tap_off[j]) * pitch : ... + k_per_tap], zero where p + tap_off[j] lies outside [0, P).

volume() builds X from an NC(T)HW tensor, merged_filter() / unmerged_filter() build Wt, tap_off and lo_mask the way the
I3D and RAFT engines do, and emulate() computes in float64 what the kernel computes.  Test infrastructure only."""
from __future__ import annotations

from dataclasses import dataclass

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
            blk = torch.arange(Kb, device=X.device) % kpt // 64
            keep_lo = ((f["lo_mask"] >> blk.cpu()) & 1 == 0).double().to(X.device)
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


def reference_conv(x_eff: torch.Tensor, w_eff: torch.Tensor, bias=None, scale=None, act: int = ACT_NONE):
    """F.conv3d / F.conv2d in float64, stride 1, zero padding k // 2 before and k - 1 - k // 2 after (the output keeps
    the input's extent), then the epilogue.  Returns NCTHW (or NCHW for 2-D input) with channels last moved to dim 1."""
    x, w = x_eff.double(), w_eff.double()
    ks = w.shape[2:]
    pad = []
    for k in reversed(ks):
        pad += [k // 2, k - 1 - k // 2]
    xp = F.pad(x, pad)
    y = F.conv3d(xp, w) if w.dim() == 5 else F.conv2d(xp, w)
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
