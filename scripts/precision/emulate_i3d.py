"""CPU emulation behind DESIGN.md §2 (I3D): which fp16-rounded tensors make up the feature error of the trained rgb
checkpoint on a uniform-noise clip (T = 16).  Needs oracle/_ref/checkpoints/i3d_rgb.pt.

Measured in the build container (rel-L2 / max-abs relative to max |feature|, weights fp32, seed 1 / seed 116):
    every conv input rounded to fp16                       8.1e-04 / 8.6e-04      8.0e-04 / 7.4e-04
    only the inputs of the 3x3x3 convs of the Mixed blocks 2.7e-04 / 2.7e-04      3.2e-04 / 4.7e-04
    only the inputs of the 1x1x1 convs (concat, pools)     6.8e-04 / 6.3e-04      6.9e-04 / 9.6e-04
    only the stem input                                    1.2e-04 / 1.9e-04
    only conv3d_2b's input (the stem pool output)          4.1e-04 / 4.0e-04
    only conv3d_2c's input                                 1.8e-04 / 1.7e-04
    single fp16 only for: Mixed 3x3x3 inputs + 2c input + stem input (what the engine does)   2.9e-04 / 2.8e-04
Hence "pair tensors" (split-fp16) for everything the 1x1x1 convs and the pools read, single fp16 for the 3x3x3 inputs."""
import os, sys
import torch, torch.nn.functional as F
ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import i3d_net as N


def main(seed=116):
    torch.set_num_threads(os.cpu_count() or 1)
    sd = torch.load(os.path.join(ROOT, "oracle", "_ref", "checkpoints", "i3d_rgb.pt"), map_location="cpu")
    x = torch.rand(1, 3, 16, 224, 224, generator=torch.Generator().manual_seed(seed)) * 2 - 1
    ref = N.forward_features(sd, x)
    orig = N._unit

    def run(round_in):
        def unit(sd_, name, xx, k, stride=1):
            if round_in(name, k):
                xx = xx.half().float()
            pt, pb = N._same_pad(k, stride)
            if k > 1:
                xx = F.pad(xx, (pt, pb, pt, pb, pt, pb))
            y = F.conv3d(xx, sd_[f"{name}.conv3d.weight"], None, stride=stride)
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
        "every conv input": lambda n, k: True,
        "Mixed 3x3x3 inputs only": lambda n, k: k == 3 and n.startswith("mixed"),
        "1x1x1 inputs only (Mixed)": lambda n, k: k == 1 and n.startswith("mixed"),
        "stem input only": lambda n, k: k == 7,
        "conv3d_2b input only": lambda n, k: n == "conv3d_2b_1x1",
        "conv3d_2c input only": lambda n, k: n == "conv3d_2c_3x3",
        "engine: single fp16 only for 3x3x3 inputs and the stem input": lambda n, k: k == 3 or k == 7,
    }
    for tag, fn in cases.items():
        print(f"{tag:70s} {run(fn)}", flush=True)


if __name__ == "__main__":
    main(int(sys.argv[1]) if len(sys.argv) > 1 else 116)
