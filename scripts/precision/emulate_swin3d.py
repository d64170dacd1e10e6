"""Float64 emulation of the Swin3D engine's declared rounding (DESIGN.md §4.14), to decide which tensor classes must be
carried as split-fp16 pairs.

    python scripts/precision/emulate_swin3d.py [--models swin3d_t swin3d_s swin3d_b] [--T 10] [--device cpu]

The stand-in network (oracle/swin3d_net.py) runs in float64 with the operands of each tensor class either kept exact
("split": a split-fp16 pair carries ~22 bits, far below the bar) or rounded to one fp16 value:
  w      every GEMM weight (patch embedding, qkv, proj, mlp.0, mlp.3, reduction)
  patch  the patch rows (the transformed clip)
  ln     the LayerNorm outputs that feed a GEMM (patch_embed.norm is fp32: it is the residual stream; norm1, norm2 and
         the patch-merging norm)
  qkv    q, k and v
  p      P = exp(s - max), the softmax numerator multiplied into v (the sum stays fp32)
  att    the attention output (proj's input)
  mlp    the MLP hidden layer after GELU (mlp.3's input)
For each model it prints, per scheme, the worst per-clip rel-L2 and max-abs / max at every stage and at the features
against the exact float64 forward: the all-fp16 scheme, each class alone in fp16, and the chosen scheme (SPLIT split,
everything else fp16).  The project bar is 1e-3 / 1e-3 at the features.
"""
import argparse
import os
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import swin3d_net as S  # noqa: E402

CLASSES = ("w", "patch", "ln", "qkv", "p", "att", "mlp")
# the engine's scheme: these classes are split-fp16 pairs, the others single fp16
SPLIT = ("w",)


def _q(x, cls, fp16):
    return x.half().double() if cls in fp16 else x


def _ln(sd, p, x):
    return F.layer_norm(x, x.shape[-1:], sd[p + ".weight"], sd[p + ".bias"], S.EPS)


def _lin(sd, p, x, fp16, bias=True):
    return F.linear(x, _q(sd[p + ".weight"], "w", fp16), sd[p + ".bias"] if bias else None)


def _attention(sd, p, x, heads, shifted, fp16):
    """The window attention with the engine's rounding points; padded positions are zero rows, so their qkv is the
    (rounded) bias, as in the engine."""
    b, t, h, w, c = x.shape
    win, sh = S.window_and_shift((t, h, w), shifted)
    pad = [(win[i] - (t, h, w)[i] % win[i]) % win[i] for i in range(3)]
    qkv = _q(_lin(sd, p + ".qkv", x, fp16), "qkv", fp16)
    bias = _q(sd[p + ".qkv.bias"], "qkv", fp16)
    qkv = F.pad(qkv - bias, (0, 0, 0, pad[2], 0, pad[1], 0, pad[0])) + bias
    tp, hp, wp = qkv.shape[1:4]
    if sum(sh):
        qkv = torch.roll(qkv, shifts=(-sh[0], -sh[1], -sh[2]), dims=(1, 2, 3))
    nw = (tp // win[0]) * (hp // win[1]) * (wp // win[2])
    vol = win[0] * win[1] * win[2]
    qkv = qkv.view(b, tp // win[0], win[0], hp // win[1], win[1], wp // win[2], win[2], 3 * c)
    qkv = qkv.permute(0, 1, 3, 5, 2, 4, 6, 7).reshape(b * nw, vol, 3, heads, c // heads)
    q, k, v = qkv.permute(2, 0, 3, 1, 4)
    s = (q * (c // heads) ** -0.5) @ k.transpose(-2, -1)
    s = s + sd[p + ".relative_position_bias_table"][S.bias_index(win).reshape(-1).to(x.device)].view(
        vol, vol, heads).permute(2, 0, 1)
    if sum(sh):
        reg = S.region_ids((tp, hp, wp), win, sh).to(x.device)
        reg = reg.view(tp // win[0], win[0], hp // win[1], win[1], wp // win[2], win[2]).permute(0, 2, 4, 1, 3, 5)
        reg = reg.reshape(nw, vol)
        mask = torch.where(reg[:, None, :] != reg[:, :, None], -100.0, 0.0).to(x.dtype)
        s = (s.view(b, nw, heads, vol, vol) + mask[None, :, None]).view(b * nw, heads, vol, vol)
    e = torch.exp(s - s.amax(-1, keepdim=True))
    y = (_q(e, "p", fp16) @ v) / e.sum(-1, keepdim=True)
    y = y.transpose(1, 2).reshape(b, tp // win[0], hp // win[1], wp // win[2], win[0], win[1], win[2], c)
    y = y.permute(0, 1, 4, 2, 5, 3, 6, 7).reshape(b, tp, hp, wp, c)
    if sum(sh):
        y = torch.roll(y, shifts=(sh[0], sh[1], sh[2]), dims=(1, 2, 3))
    return _lin(sd, p + ".proj", _q(y[:, :t, :h, :w], "att", fp16), fp16)


def forward(sd, x, fp16=()):
    """(features, {stage: activation}) of the stand-in with the classes in `fp16` rounded to one fp16 value."""
    sd = {k: v.to(x.device, torch.float64) if v.is_floating_point() else v for k, v in S._plain(sd).items()}
    _, depths = S.config(sd)
    st = {}
    xp = _q(F.pad(x, (0, 0, 0, 0, 0, x.shape[2] % 2)), "patch", fp16)
    y = F.conv3d(xp, _q(sd["patch_embed.proj.weight"], "w", fp16), sd["patch_embed.proj.bias"], stride=S.PATCH)
    y = _ln(sd, "patch_embed.norm", y.permute(0, 2, 3, 4, 1))
    st["embed"] = y
    for s in range(4):
        for d in range(depths[s]):
            p = f"features.{2 * s}.{d}"
            heads = y.shape[-1] // S.HEAD_DIM
            y = y + _attention(sd, p + ".attn", _q(_ln(sd, p + ".norm1", y), "ln", fp16), heads, d % 2 == 1, fp16)
            hdn = F.gelu(_lin(sd, p + ".mlp.0", _q(_ln(sd, p + ".norm2", y), "ln", fp16), fp16))
            y = y + _lin(sd, p + ".mlp.3", _q(hdn, "mlp", fp16), fp16)
        st[f"stage{s + 1}"] = y
        if s < 3:
            p = f"features.{2 * s + 1}"
            y = _lin(sd, p + ".reduction", _q(_ln(sd, p + ".norm", S.merge_rows(y)), "ln", fp16), fp16, bias=False)
    y = _ln(sd, "norm", y)
    st["norm"] = y
    return y.mean(dim=(1, 2, 3)), st


def errors(y, ref):
    """(worst per-clip rel-L2, worst per-clip max-abs / max)."""
    y, ref = y.flatten(1), ref.flatten(1)
    d = y - ref
    return (d.norm(dim=1) / ref.norm(dim=1)).max().item(), (d.abs().amax(dim=1) / ref.abs().amax(dim=1)).max().item()


def table(name, T, device, schemes):
    """{scheme label: {tap: (rel-L2, max-abs / max)}} for the stand-in of `name` on 2 calibration clips of T frames."""
    sd = S.stand_in_state_dict(name)
    x = S.calibration_clips(1, 2, T).double().to(device)
    with torch.no_grad():
        ref, rst = forward(sd, x)
        out = {}
        for label, fp16 in schemes.items():
            y, st = forward(sd, x, fp16)
            row = {k: errors(st[k], rst[k]) for k in S.STAGES}
            row["features"] = errors(y, ref)
            out[label] = row
    return out


def schemes():
    s = {"all fp16": CLASSES}
    s.update({f"{c} alone fp16": (c,) for c in CLASSES})
    s[f"engine ({'+'.join(SPLIT)} split)"] = tuple(c for c in CLASSES if c not in SPLIT)
    return s


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--models", nargs="+", default=list(S.MODELS))
    ap.add_argument("--T", type=int, default=10)
    ap.add_argument("--device", default="cpu")
    a = ap.parse_args()
    for name in a.models:
        tab = table(name, a.T, a.device, schemes())
        print(f"{name}, 2 clips of {a.T} frames (rel-L2 / max-abs÷max; stage4 | features):", flush=True)
        for label, row in tab.items():
            print(f"  {label:24s} stage4 {row['stage4'][0]:.2e} / {row['stage4'][1]:.2e} | features "
                  f"{row['features'][0]:.2e} / {row['features'][1]:.2e}", flush=True)


if __name__ == "__main__":
    main()
