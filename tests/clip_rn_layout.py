"""Restated layouts of the CLIP ResNet engine (csrc/clip_resnet.cu): the stem's phase volume and 3x3/2 filter, the
AvgPool2d(2) + 1x1 conv as one tap over the phase repack (the weight in all four phase slots, 1/4 in the scale), the
stride-1 filters, the attention-pool linears, and every conv as vf_clip_rn_conv reports it.  Written from the layout
comments, not from the driver's code; test_clip_rn_layout_cpu.py pins the layouts against float64 convolutions."""
import numpy as np
import torch


def split(x: torch.Tensor):
    """x -> (hi, lo) fp16 with hi = fp16(x), lo = fp16(x - hi) (the difference taken in fp32, as on the device)."""
    x = x.float()
    hi = x.half()
    return hi, (x - hi.float()).half()


def volume(x: torch.Tensor, dtype=torch.float64):
    """x (n, C, H, W) -> zero-bordered (border 1) channels-last split rows (n, H+2, W+2, 2C): [hi C | lo C]."""
    n, c, h, w = x.shape
    hi, lo = split(x)
    v = torch.zeros(n, h + 2, w + 2, 2 * c, dtype=dtype)
    v[:, 1:h + 1, 1:w + 1, :c] = hi.permute(0, 2, 3, 1).to(dtype)
    v[:, 1:h + 1, 1:w + 1, c:] = lo.permute(0, 2, 3, 1).to(dtype)
    return v


def phase_repack(v: torch.Tensor):
    """raft_phase_repack of a border-1 volume (n, 2S+2, 2S+2, C2) -> (n, S+2, S+2, 4 C2): phase row q holds
    x[2(q-1)+p] (valid-region coordinates), phase p = 2 ph + pw at columns p C2 ..; zero outside."""
    n, hp, wp, c2 = v.shape
    s = (hp - 2) // 2
    out = torch.zeros(n, s + 2, s + 2, 4 * c2, dtype=v.dtype)
    for ph in range(2):
        for pw in range(2):
            p = 2 * ph + pw
            out[:, 1:s + 1, 1:s + 1, p * c2:(p + 1) * c2] = v[:, 1 + ph:2 * s + 1:2, 1 + pw:2 * s + 1:2, :]
    return out


def stem_phase_volume(x: torch.Tensor, dtype=torch.float64):
    """normalised (n, 3, npx, npx) -> the transform's (n, npx/2 + 2, npx/2 + 2, 32): row (hq, wq) holds
    x[2(hq-1)+ph][2(wq-1)+pw][c] at column (2 ph + pw) 4 + c of [16 hi | 16 lo]."""
    n, _, npx, _ = x.shape
    s = npx // 2
    hi, lo = split(x)
    out = torch.zeros(n, s + 2, s + 2, 32, dtype=dtype)
    for ph in range(2):
        for pw in range(2):
            p = 2 * ph + pw
            for c in range(3):
                out[:, 1:s + 1, 1:s + 1, p * 4 + c] = hi[:, c, ph::2, pw::2].to(dtype)
                out[:, 1:s + 1, 1:s + 1, 16 + p * 4 + c] = lo[:, c, ph::2, pw::2].to(dtype)
    return out


def _fill(w: torch.Tensor, ntaps, kpt, lo_off, cols):
    """w [co][ci][k][k] -> Wt fp16 [co, 2 ntaps kpt] (W_hi | W_lo) and the has-hi mask [ntaps kpt]; cols(kh, kw, c)
    -> the hi columns that weight goes to (its lo half's column is lo_off further)."""
    co, ci, k, _ = w.shape
    ktot = ntaps * kpt
    wt = torch.zeros(co, 2 * ktot, dtype=torch.float16)
    has_hi = np.zeros(ktot, bool)
    wh, wl = split(w)
    for kh in range(k):
        for kw in range(k):
            for c in range(ci):
                for kc in cols(kh, kw, c):
                    for kk in (kc, kc + lo_off):
                        wt[:, kk] = wh[:, c, kh, kw]
                        wt[:, ktot + kk] = wl[:, c, kh, kw]
                    has_hi[kc] = True
    return wt, has_hi


def _lo_mask(has_hi, ntaps, kpt):
    """bit kk set: K block kk of no tap holds a hi column (taps of more than 64 blocks carry no mask)."""
    nb = (kpt + 63) // 64
    if nb > 64:
        return 0
    hh = has_hi.reshape(ntaps, kpt)
    return sum(1 << kk for kk in range(nb) if not hh[:, kk * 64:(kk + 1) * 64].any())


def stem_filter(w):
    """stem conv1 3x3/2: 2 taps (dh = a - 1, dw = -1) of 64: column a 64 + b 32 + (2 ph + pw) 4 + c, kh = 2a + ph - 1."""
    def cols(kh, kw, c):
        a, ph, b, pw = (kh + 1) // 2, (kh + 1) % 2, (kw + 1) // 2, (kw + 1) % 2
        return [a * 64 + b * 32 + (ph * 2 + pw) * 4 + c]
    wt, hh = _fill(w, 2, 64, 16, cols)
    return dict(Wt=wt, ntaps=2, k_per_tap=64, shifts=[(0, -1, -1), (0, 0, -1)], lo_mask=_lo_mask(hh, 2, 64))


def same_filter(w):
    """stride-1 k x k, pad k/2, on split rows of 2 ci: one tap per kernel row (dh = a - k/2, dw = -k/2) of k 2ci."""
    co, ci, k, _ = w.shape
    kpt = k * 2 * ci
    wt, hh = _fill(w, k, kpt, ci, lambda a, d, c: [a * kpt + d * 2 * ci + c])
    return dict(Wt=wt, ntaps=k, k_per_tap=kpt, shifts=[(0, a - k // 2, -(k // 2)) for a in range(k)],
                lo_mask=_lo_mask(hh, k, kpt))


def pooled_filter(w):
    """AvgPool2d(2) + 1x1 over the phase repack of split rows of 2 ci: one tap of 8 ci, the weight at p 2ci + c for
    each phase p (its lo half ci further)."""
    co, ci = w.shape[:2]
    wt, hh = _fill(w, 1, 8 * ci, ci, lambda a, d, c: [p * 2 * ci + c for p in range(4)])
    return dict(Wt=wt, ntaps=1, k_per_tap=8 * ci, shifts=[(0, 0, 0)], lo_mask=_lo_mask(hh, 1, 8 * ci))


def linear_filter(w):
    """nn.Linear weight [co][ci] on split rows [hi ci | lo ci]: one tap of 2 ci."""
    co, ci = w.shape
    wt, hh = _fill(w.reshape(co, ci, 1, 1), 1, 2 * ci, ci, lambda a, d, c: [c])
    return dict(Wt=wt, ntaps=1, k_per_tap=2 * ci, shifts=[(0, 0, 0)], lo_mask=_lo_mask(hh, 1, 2 * ci))


def bn_fold(sd, p, mul=1.0):
    """eval BatchNorm folded in float64, then rounded to fp32: scale = fp32(g / sqrt(v + 1e-5)) x mul (mul a power of
    two, applied in fp32), shift = fp32(b - m s)."""
    g, b, m, v = (sd[p + s].double().numpy() for s in (".weight", ".bias", ".running_mean", ".running_var"))
    s = g / np.sqrt(v + 1e-5)
    return (torch.from_numpy(s.astype(np.float32) * np.float32(mul)),
            torch.from_numpy((b - m * s).astype(np.float32)))


def engine_convs(sd, cfg):
    """Every conv in vf_clip_rn_conv's order, as the engine should upload it: dict(Wt, ntaps, k_per_tap, shifts,
    lo_mask, scale, bias, name)."""
    out = []

    def add(f, name, scale, bias):
        f.update(scale=scale, bias=bias, name=name)
        out.append(f)

    add(stem_filter(sd["visual.conv1.weight"]), "conv1", *bn_fold(sd, "visual.bn1"))
    add(same_filter(sd["visual.conv2.weight"]), "conv2", *bn_fold(sd, "visual.bn2"))
    add(same_filter(sd["visual.conv3.weight"]), "conv3", *bn_fold(sd, "visual.bn3"))
    for L, nb in enumerate(cfg["layers"]):
        for b in range(nb):
            p = f"visual.layer{L + 1}.{b}"
            pooled_in, stride2 = (L == 0 and b == 0), (L > 0 and b == 0)
            w1 = sd[p + ".conv1.weight"]
            add(pooled_filter(w1) if pooled_in else same_filter(w1), p + ".conv1",
                *bn_fold(sd, p + ".bn1", 0.25 if pooled_in else 1.0))
            add(same_filter(sd[p + ".conv2.weight"]), p + ".conv2", *bn_fold(sd, p + ".bn2"))
            w3 = sd[p + ".conv3.weight"]
            add(pooled_filter(w3) if stride2 else same_filter(w3), p + ".conv3",
                *bn_fold(sd, p + ".bn3", 0.25 if stride2 else 1.0))
            if b == 0:
                add(pooled_filter(sd[p + ".downsample.0.weight"]), p + ".downsample",
                    *bn_fold(sd, p + ".downsample.1", 0.25))
    a = "visual.attnpool."
    E = cfg["embed"]
    add(linear_filter(sd[a + "q_proj.weight"]), "q_proj", torch.ones(E), sd[a + "q_proj.bias"].float())
    add(linear_filter(torch.cat([sd[a + "k_proj.weight"], sd[a + "v_proj.weight"]])), "kv_proj", torch.ones(2 * E),
        torch.cat([sd[a + "k_proj.bias"], sd[a + "v_proj.bias"]]).float())
    add(linear_filter(sd[a + "c_proj.weight"]), "c_proj", torch.ones(cfg["out_dim"]), sd[a + "c_proj.bias"].float())
    return out


def emulate(X: torch.Tensor, f: dict, wp: int):
    """float64 [rows, n_out] of one launch on the rows X [rows, pitch] of a volume wp positions wide: tap j reads
    k_per_tap elements from row p + dh_j wp + dw_j on (zeros outside X); W_hi and W_lo passes summed (no lo_mask skip)."""
    rows, pitch = X.shape
    kpt, ktot = f["k_per_tap"], f["ntaps"] * f["k_per_tap"]
    offs = [dh * wp + dw for _, dh, dw in f["shifts"]]
    front = max(0, -min(offs)) * pitch
    flat = torch.cat([torch.zeros(front, dtype=torch.float64), X.double().reshape(-1),
                      torch.zeros(kpt + max(0, max(offs)) * pitch, dtype=torch.float64)])
    wt = f["Wt"].double()
    out = torch.zeros(rows, wt.shape[0], dtype=torch.float64)
    for j, off in enumerate(offs):
        A = flat.as_strided((rows, kpt), (pitch, 1), front + off * pitch)
        out += A @ (wt[:, j * kpt:(j + 1) * kpt] + wt[:, ktot + j * kpt:ktot + (j + 1) * kpt]).T
    return out
