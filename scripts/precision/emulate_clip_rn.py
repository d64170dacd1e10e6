"""Which operands of the CLIP ResNet towers could stay single fp16 (DESIGN.md §4.9)?

    python scripts/precision/emulate_clip_rn.py [--towers RN50 RN101 RN50x4 RN50x16] [--frames 2] [--tiny]

For each tower's calibrated stand-in (oracle/clip_resnet.py) and one operand class at a time, the forward in float64
with that class rounded to fp16 and every other operand stored as the engine's split pair, modelled exactly: hi =
fp16(v), lo = fp16(v - hi), subnormal lo halves included (for |v| < 0.125 lo is an fp16 subnormal with a spacing of
2^-24, so a pair of a small weight keeps about 19 bits, not fp32's 24), against the same forward with nothing rounded.  Classes: the stem input, the inputs of the 1x1 convs, of the 3x3 convs, of the
downsample convs, the residual stream (block outputs), all conv weights, the attention-pool tokens and their K / V, and
the attention output (c_proj's input); "pairs" rounds no class to fp16, so it is the cost of the pair representation
alone.  Reports the worst row's rel-L2 / max-abs÷max of the features; the project's
bar is 1e-3 against the fp32 oracle.  --tiny runs a one-block-per-stage tower of width 16 at 64 px (a smoke run).
"""
import argparse
import os
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import clip_resnet  # noqa: E402

CLASSES = ("none", "pairs", "stem_in", "1x1_in", "3x3_in", "down_in", "residual", "weights", "tokens_kv", "attn_out")


def forward(sd, x, cfg, cls):
    """The tower in float64 with operand class `cls` rounded to fp16 and every other class to fp32."""
    def r(c, t):
        if cls == "none":
            return t
        if c == cls:
            return t.half().double()
        hi = t.half()
        return hi.double() + (t - hi.double()).half().double()

    def conv(t, p, c, **kw):
        return F.conv2d(r(c, t), r("weights", sd[p + ".weight"]), **kw)

    def bn(t, p):
        return F.batch_norm(t, sd[p + ".running_mean"], sd[p + ".running_var"], sd[p + ".weight"], sd[p + ".bias"],
                            False, 0.0, 1e-5)

    x = F.relu(bn(conv(x, "visual.conv1", "stem_in", stride=2, padding=1), "visual.bn1"))
    x = F.relu(bn(conv(x, "visual.conv2", "3x3_in", padding=1), "visual.bn2"))
    x = F.relu(bn(conv(x, "visual.conv3", "3x3_in", padding=1), "visual.bn3"))
    x = F.avg_pool2d(x, 2)
    for L, nb in enumerate(cfg["layers"]):
        for b in range(nb):
            p = f"visual.layer{L + 1}.{b}"
            stride = 2 if (b == 0 and L > 0) else 1
            y = F.relu(bn(conv(x, p + ".conv1", "1x1_in"), p + ".bn1"))
            y = F.relu(bn(conv(y, p + ".conv2", "3x3_in", padding=1), p + ".bn2"))
            if stride > 1:
                y = F.avg_pool2d(y, 2)
            y = bn(conv(y, p + ".conv3", "1x1_in"), p + ".bn3")
            idn = x
            if b == 0:
                idn = F.avg_pool2d(x, 2) if stride > 1 else x
                idn = bn(conv(idn, p + ".downsample.0", "down_in"), p + ".downsample.1")
            x = r("residual", F.relu(idn + y))
    tok = r("tokens_kv", clip_resnet.pool_tokens(sd, x))
    a = "visual.attnpool."
    E, H = cfg["embed"], cfg["heads"]
    T, n = tok.shape[:2]
    q = F.linear(tok[:1], r("weights", sd[a + "q_proj.weight"]), sd[a + "q_proj.bias"]) * 0.125
    k = r("tokens_kv", F.linear(tok, r("weights", sd[a + "k_proj.weight"]), sd[a + "k_proj.bias"]))
    v = r("tokens_kv", F.linear(tok, r("weights", sd[a + "v_proj.weight"]), sd[a + "v_proj.bias"]))
    q, k, v = (t.reshape(t.shape[0], n * H, 64).transpose(0, 1) for t in (q, k, v))
    o = torch.softmax(q @ k.transpose(1, 2), -1) @ v                       # (n H, 1, 64)
    o = r("attn_out", o.transpose(0, 1).reshape(n, E))
    return F.linear(o, r("weights", sd[a + "c_proj.weight"]), sd[a + "c_proj.bias"])


def row_err(y, ref):
    rel = ((y - ref).norm(dim=1) / ref.norm(dim=1)).max().item()
    mx = ((y - ref).abs().amax(dim=1) / ref.abs().amax(dim=1)).max().item()
    return rel, mx


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--towers", nargs="+", default=list(clip_resnet.TOWERS))
    ap.add_argument("--frames", type=int, default=2)
    ap.add_argument("--tiny", action="store_true")
    a = ap.parse_args()
    if a.tiny:
        clip_resnet.TOWERS["tiny"] = ((1, 1, 1, 1), 16, 64, 32)
        a.towers, a.frames = ["tiny"], 1
    dev = torch.device("cuda", 0) if torch.cuda.is_available() else torch.device("cpu")
    print("tower    " + "".join(f"{c:>20s}" for c in CLASSES[1:]))
    for name in a.towers:
        sd = clip_resnet.stand_in_state_dict(name)
        cfg = clip_resnet.config(sd)
        sdd = {k: v.double().to(dev) for k, v in sd.items()}
        x = clip_resnet.calibration_images(cfg["n_px"], seed=11, n=a.frames).double().to(dev)
        with torch.no_grad():
            ref = forward(sdd, x, cfg, "none")
            errs = [row_err(forward(sdd, x, cfg, c), ref) for c in CLASSES[1:]]
        print(f"{name:8s} " + "".join(f"{e[0]:9.1e} / {e[1]:7.1e} " for e in errs), flush=True)
    print("(each cell: worst row rel-L2 / max-abs÷max of the features against float64)")


if __name__ == "__main__":
    main()
