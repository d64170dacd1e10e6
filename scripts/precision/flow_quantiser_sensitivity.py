"""How sensitive is the reference's OWN I3D flow feature to its OWN optical flow?  (DESIGN.md §2, precision note 2.)

The flow stream of the reference is RAFT -> crop -> clamp(+-20) -> round(128 + 255/40 f) -> 2x/255-1 -> I3D
(models/i3d/extract_i3d.py:67-73, transforms/transforms.py:31-51).  The 8-bit quantiser is a staircase: a flow
perturbation far below any sensible RAFT tolerance moves a fraction of the pixels across a step, and on a clip with
little motion (few grey levels in use, small input norm) that is a large relative change of the I3D input.

This script runs the fp32 oracle (CPU) on the two clips the -m gpu composite tests use and reports, for Gaussian flow
perturbations of sigma px (seeded, 3 draws each), the relative L2 change of the oracle's own 1024-d feature:
    python scripts/precision/flow_quantiser_sensitivity.py            # prints a table and the JSON report
`feature_sensitivity()` is what tests/test_extract_i3d_raft_gpu.py imports to derive its bar from the engine's measured
flow error.  Needs oracle/_ref/checkpoints/{raft-sintel.pth,i3d_flow.pt} (oracle/fetch_ref.py) and cv2.
"""
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import i3d_net, raft_net  # noqa: E402

CLIPS = {                     # name -> per-frame shift of the synthetic texture (px at 120x160, before the 256-resize)
    "low_motion": (0.8, 0.5),
    "high_motion": (4.5, -3.0),
}


def write_clip(path, shift, n=20, h=120, w=160, fps=25.0, seed=11):
    import cv2
    fr = raft_net.synthetic_frames(n, h, w, seed=seed, shift=shift).permute(0, 2, 3, 1).numpy().astype(np.uint8)
    vw = cv2.VideoWriter(path, cv2.VideoWriter_fourcc(*"mp4v"), fps, (w, h))
    assert vw.isOpened()
    for f in fr:
        vw.write(f)
    vw.release()


def feature_sensitivity(sd_flow, flow, sigmas, draws=3, seed=0):
    """flow: the oracle's (T,2,H,W) flow field.  -> {sigma: max over draws of ||f(flow + N(0,sigma)) - f(flow)|| / ||f(flow)||}
    and the fraction of cropped pixels whose 8-bit level changed."""
    base_in = i3d_net.flow_transform(flow)
    base = i3d_net.forward_features(sd_flow, base_in)
    out = {}
    g = torch.Generator(device="cpu").manual_seed(seed)
    for s in sigmas:
        worst, flipped = 0.0, 0.0
        for _ in range(draws):
            noise = torch.randn(flow.shape, generator=g).to(flow.device) * s
            x = i3d_net.flow_transform(flow + noise)
            y = i3d_net.forward_features(sd_flow, x)
            worst = max(worst, float((y - base).norm() / base.norm()))
            flipped = max(flipped, float((x != base_in).float().mean()))
        out[float(s)] = {"feature_rel": worst, "levels_changed_frac": flipped}
    return out


def main():
    from PIL import Image
    import cv2
    torch.set_num_threads(os.cpu_count() or 1)
    sd_raft = torch.load(os.path.join(ROOT, "oracle", "_ref", "checkpoints", "raft-sintel.pth"), map_location="cpu")
    sd_flow = torch.load(os.path.join(ROOT, "oracle", "_ref", "checkpoints", "i3d_flow.pt"), map_location="cpu")
    report = {}
    for name, shift in CLIPS.items():
        path = f"/tmp/_flow_sens_{name}.mp4"
        write_clip(path, shift)
        cap, frames = cv2.VideoCapture(path), []
        while True:
            ok, f = cap.read()
            if not ok:
                break
            frames.append(f)
        # the reference resamples a 20-frame video to 65 indices (extract_i3d.py:250-255); first stack of 12 (+1)
        ix = np.linspace(1, len(frames) - 1, 65).astype(int)[:13]
        rs = torch.stack([torch.from_numpy(np.asarray(Image.fromarray(frames[i]).resize((341, 256), Image.BILINEAR)).copy())
                          for i in ix]).permute(0, 3, 1, 2).float()
        xp = raft_net.pad(rs)
        flow = raft_net.forward(sd_raft, xp[:-1], xp[1:], 20)
        # the reference against itself: the same fp32 RAFT with another summation order (1 thread instead of all)
        nthreads = torch.get_num_threads()
        torch.set_num_threads(1)
        flow_1t = raft_net.forward(sd_raft, xp[:-1], xp[1:], 20)
        torch.set_num_threads(nthreads)
        f_all = i3d_net.forward_features(sd_flow, i3d_net.flow_transform(flow))
        f_1t = i3d_net.forward_features(sd_flow, i3d_net.flow_transform(flow_1t))
        self_noise = {"flow_rms_diff_px": float((flow - flow_1t).pow(2).mean().sqrt()),
                      "feature_rel": float((f_all - f_1t).norm() / f_all.norm())}
        x = i3d_net.flow_transform(flow)
        levels = torch.unique(((x + 1) * 255 / 2).round()).numel()
        sens = feature_sensitivity(sd_flow, flow, [1e-5, 3e-5, 1e-4, 3e-4, 1e-3])
        report[name] = {"shift_px_per_frame": shift, "flow_rms_px": float(flow.pow(2).mean().sqrt()),
                        "grey_levels_in_use": int(levels), "i3d_input_rms": float(x.pow(2).mean().sqrt()),
                        "oracle_1_thread_vs_all_threads": self_noise,
                        "sensitivity": {f"{k:g}": v for k, v in sens.items()}}
        print(f"{name}: flow rms {report[name]['flow_rms_px']:.3f} px, {levels} grey levels, input rms {report[name]['i3d_input_rms']:.4f}")
        print(f"   the fp32 oracle against itself (1 thread vs {nthreads}): flow differs by {self_noise['flow_rms_diff_px']:.2e} px rms "
              f"-> feature rel-L2 {self_noise['feature_rel']:.3e}")
        for k, v in sens.items():
            print(f"   sigma {k:g} px -> feature rel-L2 {v['feature_rel']:.3e}   ({100 * v['levels_changed_frac']:.3f} % of levels changed)")
    print(json.dumps(report, indent=1))


if __name__ == "__main__":
    main()
