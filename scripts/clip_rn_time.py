"""CLIP ResNet tower timing on one GPU (numbers for the README / DESIGN.md §4.9).

    python scripts/clip_rn_time.py [--towers RN50 RN101 RN50x4 RN50x16] [--json OUT]

Prints, with the GPU's name, power limit and max SM clock:
  * per tower: engine frames/s at 64 and 256 device-resident 240x320 uint8 frames per call (bicubic resize, crop and
    normalisation included), the GEMM launches' achieved TFLOP/s executed and algorithmic (vf_gemm_profile; the
    algorithmic FLOPs are computed from the shapes below), and the oracle (oracle/clip_resnet.py) in torch on the same
    GPU and frame count: fp32 with TF32 off (the reference's --cpu arithmetic), TF32, and fp16 (what clip.load runs on
    a GPU);
  * ExtractCLIP with CLIP-RN50 end to end on 100 frames of tests/golden/v_GGSY1Qvo990.mp4 (decode + transform +
    tower).
Weights are the calibrated stand-ins: speed does not depend on the values.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import clip_resnet  # noqa: E402
from video_features_b200 import ops  # noqa: E402
from video_features_b200.clip_resnet_engine import ClipResNetEngine  # noqa: E402


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name(0)


def timed(fn, frames, reps):
    """frames/s of `fn` (processing `frames` frames per call) over `reps` calls after 2 warm-up calls."""
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return frames * reps / (a.elapsed_time(b) / 1e3)


def gemm_flops(cfg):
    """Algorithmic multiply-add FLOPs per frame of every conv and linear (2 x MACs), from the shapes."""
    w, E, T, npx = cfg["width"], cfg["embed"], cfg["tokens"], cfg["n_px"]
    s = npx // 2
    f = 2 * s * s * 9 * ((w // 2) * 3 + (w // 2) * (w // 2) + w * (w // 2))
    cin, side = w, npx // 4
    for L, nb in enumerate(cfg["layers"]):
        planes = w << L
        for b in range(nb):
            hc = side * 2 if (b == 0 and L > 0) else side      # conv1 / conv2 run before the block's pool
            ho = side
            ci = cin if b == 0 else 4 * planes
            f += 2 * hc * hc * (planes * ci + planes * planes * 9) + 2 * ho * ho * 4 * planes * planes
            if b == 0:
                f += 2 * ho * ho * 4 * planes * ci
        cin = 4 * planes
        side //= 2
    return f + 2 * (T * 2 * E * E + E * E + E * cfg["out_dim"])


def frames_u8(n, device):
    g = torch.Generator().manual_seed(1)
    return torch.randint(0, 256, (n, 240, 320, 3), dtype=torch.uint8, generator=g).to(device)


def torch_rates(sd, x, reps):
    out = {}
    dev = x.device
    with torch.no_grad():
        sdg = {k: v.to(dev) for k, v in sd.items()}
        for label, tf32 in (("torch_fp32", False), ("torch_tf32", True)):
            torch.backends.cudnn.allow_tf32 = tf32
            torch.backends.cuda.matmul.allow_tf32 = tf32
            out[label] = timed(lambda: clip_resnet.forward(sdg, x), x.shape[0], reps)
        torch.backends.cudnn.allow_tf32 = False
        torch.backends.cuda.matmul.allow_tf32 = False
        sdh = {k: v.half() for k, v in sdg.items()}
        xh = x.half()
        out["torch_fp16"] = timed(lambda: clip_resnet.forward(sdh, xh), x.shape[0], reps)
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--towers", nargs="+", default=list(clip_resnet.TOWERS))
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    dev = torch.device("cuda", 0)
    res = {"gpu": gpu_info(), "towers": {}}
    print(f"GPU: {res['gpu']} (name, power limit, max SM clock)", flush=True)
    frames = frames_u8(256, dev)
    for name in a.towers:
        sd = clip_resnet.stand_in_state_dict(name)
        cfg = clip_resnet.config(sd)
        alg = gemm_flops(cfg)
        r = {"gflop_per_frame": alg / 1e9}
        eng = ClipResNetEngine(sd, 0)
        r["max_frames"] = eng.max_frames
        for c in (64, 256):
            x = frames[:c]
            r[f"engine_{c}"] = timed(lambda: eng.encode_frames_u8(x), c, max(3, 1024 // c))
        ops.gemm_profile(True)
        eng.encode_frames_u8(frames[:64])
        ms, launches, executed = ops.gemm_profile_read()
        ops.gemm_profile(False)
        r["gemm_launches"], r["gemm_ms"] = launches, ms
        r["gemm_tflops_executed"] = executed / (ms / 1e3) / 1e12
        r["gemm_tflops_algorithmic"] = alg * 64 / (ms / 1e3) / 1e12
        eng.close()
        torch.cuda.empty_cache()
        xn = clip_resnet.calibration_images(cfg["n_px"], seed=1, n=64).to(dev)
        r.update(torch_rates(sd, xn, 3))
        res["towers"][name] = r
        print(f"{name}: {r['gflop_per_frame']:.2f} GFLOP/frame, workspace {r['max_frames']} frames | engine "
              f"{r['engine_64']:.0f} frames/s (64/call), {r['engine_256']:.0f} (256/call) | GEMM {launches} launches "
              f"at 64 frames, {r['gemm_tflops_executed']:.0f} TFLOP/s executed ({r['gemm_tflops_algorithmic']:.0f} "
              f"algorithmic) | torch at 64 frames: fp32 {r['torch_fp32']:.0f}, tf32 {r['torch_tf32']:.0f}, fp16 "
              f"{r['torch_fp16']:.0f} frames/s", flush=True)

    # ---- ExtractCLIP end to end on the sample video
    from video_features_b200.extract.extract_clip import ExtractCLIP
    video = os.path.join(ROOT, "tests", "golden", "v_GGSY1Qvo990.mp4")
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "RN50.pt")
        torch.save(clip_resnet.stand_in_state_dict("RN50"), path)
        os.environ["VF_CLIP_CKPT"] = path
        args = argparse.Namespace(feature_type="CLIP-RN50", video_paths=[video], flow_paths=None,
                                  file_with_video_paths=None, video_dir=None, flow_dir=None, extraction_fps=None,
                                  extract_method="uni_100", on_extraction="print", output_path=d, output_direct=True,
                                  tmp_path=d)
        ex = ExtractCLIP(args, external_call=True)
        idx = torch.zeros([1], dtype=torch.long, device=dev)
        ex(idx)                                          # warm-up: engine, graphs
        t0 = time.perf_counter()
        reps = 3
        for _ in range(reps):
            n = ex(idx)[0]["CLIP-RN50"].shape[0]
        dt = (time.perf_counter() - t0) / reps
        res["extract_rn50"] = n / dt
        print(f"ExtractCLIP CLIP-RN50 end to end: {n} frames in {dt * 1e3:.0f} ms = {n / dt:.0f} frames/s", flush=True)
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
