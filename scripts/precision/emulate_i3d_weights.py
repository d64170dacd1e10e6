"""CPU emulation: which I3D convolutions tolerate SINGLE fp16 weights (one MMA pass instead of the hi + lo pair)?
Activations are rounded as the engine rounds them (single fp16 inputs for the 3x3x3 convs and the stem, pair = ~fp32
elsewhere); on top of that the weights of the named layer groups are rounded to fp16.  Trained rgb / flow checkpoints,
uniform-noise clip (the hardest input), T = 16.   python scripts/precision/emulate_i3d_weights.py [rgb|flow] [seed]"""
import os, sys
import torch, torch.nn.functional as F
ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import i3d_net as N


def main(mod="rgb", seed=116):
    torch.set_num_threads(os.cpu_count() or 1)
    sd = torch.load(os.path.join(ROOT, "oracle", "_ref", "checkpoints", f"i3d_{mod}.pt"), map_location="cpu")
    cin = 3 if mod == "rgb" else 2
    x = torch.rand(1, cin, 16, 224, 224, generator=torch.Generator().manual_seed(seed)) * 2 - 1
    ref = N.forward_features(sd, x)
    orig = N._unit

    def run(w16):
        def unit(sd_, name, xx, k, stride=1):
            if k == 3 or k == 7:
                xx = xx.half().float()                      # the engine's single-fp16 activation operands
            w = sd_[f"{name}.conv3d.weight"]
            if w16(name, k):
                w = w.half().float()
            pt, pb = N._same_pad(k, stride)
            if k > 1:
                xx = F.pad(xx, (pt, pb, pt, pb, pt, pb))
            y = F.conv3d(xx, w, None, stride=stride)
            y = F.batch_norm(y, sd_[f"{name}.batch3d.running_mean"], sd_[f"{name}.batch3d.running_var"],
                             sd_[f"{name}.batch3d.weight"], sd_[f"{name}.batch3d.bias"], False, 0.0, N.BN_EPS)
            return F.relu(y)
        N._unit = unit
        try:
            y = N.forward_features(sd, x)
        finally:
            N._unit = orig
        return "rel-L2 %.3e  max %.3e" % (float((y - ref).norm() / ref.norm()), float((y - ref).abs().max() / ref.abs().max()))

    cases = {
        "engine today (hi+lo weights everywhere)": lambda n, k: False,
        "fp16 weights: Mixed 3x3x3 of stage 3 (3b, 3c)": lambda n, k: k == 3 and n.startswith("mixed_3"),
        "fp16 weights: Mixed 3x3x3 of stage 4": lambda n, k: k == 3 and n.startswith("mixed_4"),
        "fp16 weights: Mixed 3x3x3 of stage 5": lambda n, k: k == 3 and n.startswith("mixed_5"),
        "fp16 weights: all Mixed 3x3x3": lambda n, k: k == 3 and n.startswith("mixed"),
        "fp16 weights: conv3d_2c only": lambda n, k: n == "conv3d_2c_3x3",
        "fp16 weights: all 3x3x3 (Mixed + 2c)": lambda n, k: k == 3,
        "fp16 weights: stem only": lambda n, k: k == 7,
        "fp16 weights: all 3x3x3 + stem": lambda n, k: k >= 3,
        "fp16 weights: everything": lambda n, k: True,
    }
    if os.environ.get("VF_EMU_COMBOS"):
        cases = {
            "engine today (hi+lo weights everywhere)": lambda n, k: False,
            "fp16 weights: stem": lambda n, k: k == 7,
            "fp16 weights: stem + stage-5 3x3x3": lambda n, k: k == 7 or (k == 3 and n.startswith("mixed_5")),
            "fp16 weights: stem + stage-3 3x3x3": lambda n, k: k == 7 or (k == 3 and n.startswith("mixed_3")),
            "fp16 weights: stem + stage-3 + stage-5 3x3x3": lambda n, k: k == 7 or (k == 3 and (n.startswith("mixed_3") or n.startswith("mixed_5"))),
            "fp16 weights: stem + 3b only": lambda n, k: k == 7 or (k == 3 and n.startswith("mixed_3b")),
            "fp16 weights: stem + 3c only": lambda n, k: k == 7 or (k == 3 and n.startswith("mixed_3c")),
        }
    if os.environ.get("VF_EMU_COMBOS") == "2":     # what could be added to the policy the engine ships (stem + stage 3)
        cur = lambda n, k: k == 7 or (k == 3 and n.startswith("mixed_3"))
        cases = {
            "engine today (stem + stage-3 3x3x3 single)": cur,
            "  + conv3d_2c": lambda n, k: cur(n, k) or n == "conv3d_2c_3x3",
            "  + stage-5 3x3x3": lambda n, k: cur(n, k) or (k == 3 and n.startswith("mixed_5")),
            "  + conv3d_2c + stage-5 3x3x3": lambda n, k: cur(n, k) or n == "conv3d_2c_3x3" or (k == 3 and n.startswith("mixed_5")),
            "  + mixed_4b/4c 3x3x3": lambda n, k: cur(n, k) or (k == 3 and (n.startswith("mixed_4b") or n.startswith("mixed_4c"))),
        }
    for tag, fn in cases.items():
        print(f"{mod} seed {seed}: {tag:55s} {run(fn)}", flush=True)


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else "rgb", int(sys.argv[2]) if len(sys.argv) > 2 else 116)
