"""Float64 emulation of the MViT engine's declared rounding (DESIGN.md §4.15), to decide which tensor classes must be
carried as split-fp16 pairs.

    python scripts/precision/emulate_mvit.py [--models mvit_v1_b mvit_v2_s] [--clips 1] [--device cpu]

The stand-in network (oracle/mvit_net.py) runs in float64 with the operands of each tensor class either kept exact
("split": a split-fp16 pair carries ~22 bits, far below the bar) or rounded to one fp16 value:
  w      every GEMM weight (patch conv, qkv, attn.project.0, project, mlp.0, mlp.3)
  patch  the patch rows (the transformed clip)
  ln     the norm1 / norm2 outputs (the GEMMs' inputs; the embedding and the residual stream stay fp32)
  qkv    the qkv GEMM output (the head pooling's input, and v1's unpooled q)
  pool   the pooled q / k / v after their LayerNorm (the attention's operands and v2's residual q)
  p      P = exp(s - max), the softmax numerator multiplied into v (the sum stays fp32)
  att    the attention output (attn.project.0's input)
  mlp    the MLP hidden layer after GELU (mlp.3's input)
For each model it prints, per scheme, the worst per-clip rel-L2 and max-abs / max at the last stage and at the
features against the exact float64 forward: the all-fp16 scheme, each class alone in fp16, and the engine's scheme
(SPLIT split, everything else fp16).  The project bar is 1e-3 / 1e-3 at the features.
"""
import argparse
import os
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import mvit_net as M  # noqa: E402

CLASSES = ("w", "patch", "ln", "qkv", "pool", "p", "att", "mlp")
# the engine's scheme: these classes are split-fp16 pairs, the others single fp16
SPLIT = ("w",)


def _q(x, cls, fp16):
    return x.half().double() if cls in fp16 else x


def _lin(sd, p, x, fp16):
    return F.linear(x, _q(sd[p + ".weight"], "w", fp16), sd[p + ".bias"])


def _attention(q, k, v, q_thw, k_thw, rel, resid, fp16):
    """oracle attention with P rounded where the engine rounds it (the rel-pos bias from the same unscaled q)."""
    s = (q * M.HEAD_DIM ** -0.5) @ k.transpose(2, 3)
    if rel is not None:
        s = s.clone()
        s[:, :, 1:, 1:] += M.rel_bias(q, q_thw, k_thw, *rel)
    e = torch.exp(s - s.amax(-1, keepdim=True))
    x = (_q(e, "p", fp16) @ v) / e.sum(-1, keepdim=True)
    if resid:
        x = x.clone()
        x[:, :, 1:] += q[:, :, 1:]
    return x


def _block(sd, name, i, x, s_in, fp16):
    p = f"blocks.{i}."
    v2 = name == "mvit_v2_s"
    cin, cout = M.CHANNELS[name][0][i], M.CHANNELS[name][1][i]
    ad, heads, sq, skv = (cout if v2 else cin), M.HEADS[i], M.STRIDE_Q[i], M.STRIDE_KV[i]
    thw = (M.T // 2, s_in, s_in)
    b, n, _ = x.shape
    xn1 = _q(M._ln(sd, p + "norm1", x), "ln", fp16)
    qkv = _q(_lin(sd, p + "attn.qkv", xn1, fp16), "qkv", fp16)
    q, k, v = qkv.reshape(b, n, 3, heads, M.HEAD_DIM).transpose(1, 3).unbind(dim=2)
    k, k_thw = M.head_pool(sd, p + "attn.pool_k", k, thw, skv)
    v, _ = M.head_pool(sd, p + "attn.pool_v", v, thw, skv)
    k, v = _q(k, "pool", fp16), _q(v, "pool", fp16)
    q_thw = thw
    if v2 or sq > 1:
        q, q_thw = M.head_pool(sd, p + "attn.pool_q", q, thw, sq)
        q = _q(q, "pool", fp16)
    rel = (sd[p + "attn.rel_pos_h"], sd[p + "attn.rel_pos_w"], sd[p + "attn.rel_pos_t"]) if v2 else None
    a = _q(_attention(q, k, v, q_thw, k_thw, rel, v2, fp16), "att", fp16)
    a = _lin(sd, p + "attn.project.0", a.transpose(1, 2).reshape(b, -1, ad), fp16)
    skip = x
    if v2 and cin != cout:
        skip = _lin(sd, p + "project", xn1, fp16)
    if sq > 1:
        skip = M.skip_pool(skip, thw)
    x = skip + a
    xn2 = _q(M._ln(sd, p + "norm2", x), "ln", fp16)
    if not v2 and cin != cout:
        x = _lin(sd, p + "project", xn2, fp16)
    h = _q(F.gelu(_lin(sd, p + "mlp.0", xn2, fp16)), "mlp", fp16)
    return x + _lin(sd, p + "mlp.3", h, fp16), M.pooled(s_in, sq)


def forward(sd, x, fp16=()):
    """(features, {stage: activation}) of the stand-in with the classes in `fp16` rounded to one fp16 value."""
    sd = {k: v.to(x.device, torch.float64) if v.is_floating_point() else v for k, v in M._plain(sd).items()}
    name = M.config(sd)
    esd = dict(sd)
    esd["conv_proj.weight"] = _q(sd["conv_proj.weight"], "w", fp16)
    st = {}
    y = M.embed(esd, _q(x, "patch", fp16))
    st["embed"] = y
    s = 56
    for i in range(16):
        y, s = _block(sd, name, i, y, s, fp16)
        if i in M.STAGE_END:
            st[f"stage{M.STAGE_END.index(i) + 1}"] = y
    y = M._ln(sd, "norm", y)
    st["norm"] = y
    return y[:, 0], st


def errors(y, ref):
    """(worst per-clip rel-L2, worst per-clip max-abs / max)."""
    y, ref = y.flatten(1), ref.flatten(1)
    d = y - ref
    return (d.norm(dim=1) / ref.norm(dim=1)).max().item(), (d.abs().amax(dim=1) / ref.abs().amax(dim=1)).max().item()


def table(name, clips, device, schemes):
    """{scheme label: {tap: (rel-L2, max-abs / max)}} for the stand-in of `name` on `clips` calibration clips (the
    clips the GPU test's 1-clip call uses)."""
    sd = M.stand_in_state_dict(name)
    x = M.calibration_clips(clips, clips).double().to(device)
    with torch.no_grad():
        ref, rst = forward(sd, x)
        out = {}
        for label, fp16 in schemes.items():
            y, st = forward(sd, x, fp16)
            row = {k: errors(st[k], rst[k]) for k in M.STAGES}
            row["features"] = errors(y, ref)
            out[label] = row
    return out


def engine_scheme():
    return tuple(c for c in CLASSES if c not in SPLIT)


def schemes():
    s = {"all fp16": CLASSES}
    s.update({f"{c} alone fp16": (c,) for c in CLASSES})
    s[f"engine ({'+'.join(SPLIT)} split)"] = engine_scheme()
    return s


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--models", nargs="+", default=list(M.MODELS))
    ap.add_argument("--clips", type=int, default=1)
    ap.add_argument("--device", default="cpu")
    a = ap.parse_args()
    torch.set_num_threads(os.cpu_count() or 1)
    for name in a.models:
        tab = table(name, a.clips, a.device, schemes())
        print(f"{name}, {a.clips} clip(s) of 16 frames (rel-L2 / max-abs÷max; stage4 | features):", flush=True)
        for label, row in tab.items():
            print(f"  {label:24s} stage4 {row['stage4'][0]:.2e} / {row['stage4'][1]:.2e} | features "
                  f"{row['features'][0]:.2e} / {row['features'][1]:.2e}", flush=True)


if __name__ == "__main__":
    main()
