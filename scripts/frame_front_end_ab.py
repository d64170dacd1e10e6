"""Bit identity of the frame towers between two builds of libvfeat.so (say, a commit and its parent).

    python scripts/frame_front_end_ab.py --old /path/to/old/libvfeat.so [--new video_features_b200/libvfeat.so]

Every build runs in its own process (VF_LIBVFEAT selects it), once with CUDA graphs and once under VF_NO_GRAPH=1.  Each
process drives CLIP ViT-B/32 and B/16, ViT-L/14 at 224 and 336 px, CLIP RN50 and DINOv2 ViT-S/14 and ViT-B/14-reg
(synthetic or seeded stand-in weights) on small handles: fp32 frames, then u8 frames of two odd sizes (the second
larger, so the resize scratch is re-allocated), every call larger than one chunk and made three times (eager, capture
and replay where the tower captures on the second sighting); for ViT-B also the host-buffer entries (_host, _host_dev,
_host_async).  Every output and every call's launch count must be equal between the builds.  Prints one line per
mode and exits non-zero on a difference."""
import argparse
import os
import subprocess
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

SIZES = ((161, 203), (243, 317))     # u8 frame sizes: odd, the second larger than the first
REPEAT = 3


def _frames(n, h, w, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, 256, (n, h, w, 3), dtype=torch.uint8, generator=g)


def _f32(n, npx, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn((n, 3, npx, npx), generator=g)


def _calls(results, name, eng, count, entries):
    """entries: (label, fn) pairs; fn() returns a tensor.  Each runs REPEAT times."""
    for label, fn in entries:
        for r in range(REPEAT):
            before = count(eng)
            y = fn()
            torch.cuda.synchronize()
            results[f"{name} {label} #{r}"] = (y.detach().cpu().clone(), count(eng) - before)


def worker(out_path):
    from oracle import clip_resnet, dinov2_net
    from video_features_b200 import synthetic_weights
    from video_features_b200.clip_engine import ClipEngine
    from video_features_b200.clip_resnet_engine import ClipResNetEngine
    from video_features_b200.clip_vitl_engine import ClipViTLEngine
    from video_features_b200.dinov2_engine import DINOv2Engine
    dev = torch.device("cuda", 0)
    n = 5            # every handle below holds 3 or 4 frames: two chunks per call
    results = {}
    launches = lambda e: e.launch_count                                            # noqa: E731

    for patch, sd in ((32, synthetic_weights.clip_vit_b32_state_dict(0)), (16, synthetic_weights.clip_vit_b16_state_dict(0))):
        eng = ClipEngine(sd, 0, chunk_frames=4)
        entries = [("f32", lambda: eng.encode_image(_f32(n, 224, 1).to(dev)))]
        for i, (h, w) in enumerate(SIZES):
            u8 = _frames(n, h, w, 10 + i)
            pinned = u8.pin_memory()
            entries += [(f"u8 {h}x{w}", lambda u8=u8: eng.encode_frames_u8(u8.to(dev))),
                        (f"host {h}x{w}", lambda u8=u8: eng.encode_frames_u8_host(u8)),
                        (f"host_dev {h}x{w}", lambda u8=u8: eng.encode_frames_u8_host_dev(u8)),
                        (f"host_async {h}x{w}", lambda p=pinned: _async(eng, p))]
        _calls(results, f"ViT-B/{patch}", eng, launches, entries)
        eng.close()

    for npx in (224, 336):
        eng = ClipViTLEngine(synthetic_weights.clip_vit_l14_state_dict(0, n_px=npx), 0, max_frames=3)
        entries = [("f32", lambda: eng.encode_image(_f32(n, npx, 2).to(dev)))]
        entries += [(f"u8 {h}x{w}", lambda u8=_frames(n, h, w, 20 + i): eng.encode_frames_u8(u8.to(dev)))
                    for i, (h, w) in enumerate(SIZES)]
        _calls(results, f"ViT-L/14@{npx}", eng, launches, entries)
        eng.close()

    eng = ClipResNetEngine(clip_resnet.stand_in_state_dict("RN50"), 0, max_frames=3)
    entries = [("f32", lambda: eng.encode_image(_f32(n, 224, 3).to(dev)))]
    entries += [(f"u8 {h}x{w}", lambda u8=_frames(n, h, w, 30 + i): eng.encode_frames_u8(u8.to(dev)))
                for i, (h, w) in enumerate(SIZES)]
    _calls(results, "RN50", eng, launches, entries)
    eng.close()

    for name in ("dinov2_vits14", "dinov2_vitb14_reg"):
        eng = DINOv2Engine(dinov2_net.stand_in_state_dict(name), 0, max_frames=4)
        entries = [("f32", lambda: eng.encode_f32(_f32(n, 224, 4).to(dev)))]
        entries += [(f"u8 {h}x{w}", lambda u8=_frames(n, h, w, 40 + i): eng.encode_u8(u8.to(dev)))
                    for i, (h, w) in enumerate(SIZES)]
        _calls(results, name, eng, launches, entries)
        eng.close()
    torch.save(results, out_path)


def _async(eng, pinned):
    out = torch.empty((pinned.shape[0], 512), dtype=torch.float32).pin_memory()
    ticket, dev = eng.encode_frames_u8_host_async(pinned, out, out_dev=True)
    eng.wait(ticket)
    torch.cuda.synchronize()
    return torch.cat([out, dev.cpu()], 1)


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--old", help="the build to compare against")
    ap.add_argument("--new", default=os.path.join(ROOT, "video_features_b200", "libvfeat.so"))
    ap.add_argument("--worker", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.worker:
        return worker(args.worker)
    bad = 0
    with tempfile.TemporaryDirectory() as tmp:
        for no_graph in ("0", "1"):
            got = {}
            for tag, lib in (("old", args.old), ("new", args.new)):
                path = os.path.join(tmp, f"{tag}{no_graph}.pt")
                env = dict(os.environ, VF_LIBVFEAT=os.path.abspath(lib), VF_NO_GRAPH=no_graph)
                subprocess.check_call([sys.executable, os.path.abspath(__file__), "--worker", path], env=env, cwd=ROOT)
                got[tag] = torch.load(path)
            old, new = got["old"], got["new"]
            diff = [k for k in old if k not in new or not torch.equal(old[k][0], new[k][0]) or old[k][1] != new[k][1]]
            for k in diff:
                print(f"  DIFF {k}: launches {old[k][1]} vs {new[k][1] if k in new else 'missing'}")
            print(f"VF_NO_GRAPH={no_graph}: {len(got['old'])} calls, {len(diff)} differ")
            bad += len(diff)
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main())
