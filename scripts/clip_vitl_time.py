"""Throughput of the CLIP ViT-L/14 towers on one GPU (README, DESIGN.md §4.13).

    python scripts/clip_vitl_time.py [--reps 10] [--out result.json]

For each tower (224 px / 257 tokens, 336 px / 577 tokens), seeded synthetic weights, device-resident transformed frames:
  * frames/s at 64 and 256 frames per call (graph replay, CUDA events around `reps` calls after a warm-up);
  * GEMM time, executed and algorithmic TFLOP/s (one eager call of 256 frames with the GEMM profiler on; executed counts
    the patch GEMM's padded K of 592, algorithmic the FLOPs tests/clip_vitl_ref.py counts per frame);
  * the attention kernel's time per layer on a 256-frame chunk (its own entry, CUDA events) and its share of a call;
  * the reference's torch modules (tests/clip_vitl_ref.py, cuBLAS / cuDNN) in fp16 on the same GPU, 64 frames per call.
The GPU's name and power limit are read in the same run.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import clip_vitl_ref  # noqa: E402
from video_features_b200 import synthetic_weights  # noqa: E402
from video_features_b200._lib import check, lib  # noqa: E402
from video_features_b200.clip_vitl_engine import ClipViTLEngine  # noqa: E402


def timed(fn, reps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps          # ms per call


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("clip_vitl_time.py measures on a CUDA device; none is present")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True).stdout.strip()
    res = {"gpu": gpu, "towers": {}}
    print(f"GPU: {gpu}", flush=True)
    dev = torch.device("cuda", 0)
    for n_px in (224, 336):
        sd = synthetic_weights.clip_vit_l14_state_dict(0, n_px=n_px)
        eng = ClipViTLEngine(sd, 0)
        r = {"max_frames": eng.max_frames, "tokens": eng.tokens}
        x = torch.randn(256, 3, n_px, n_px, generator=torch.Generator().manual_seed(0)).to(dev)
        for n in (64, 256):
            for _ in range(3):
                eng.encode_image(x[:n])                       # eager, capture, replay
            ms = timed(lambda: eng.encode_image(x[:n]), a.reps)
            r[f"frames_per_s_{n}"] = n / ms * 1e3
            r[f"ms_per_call_{n}"] = ms
        check(lib().vf_gemm_profile(1))
        eng.encode_image(x)
        gms, glaunch, gflops = C.c_double(), C.c_int64(), C.c_double()
        check(lib().vf_gemm_profile_read(C.byref(gms), C.byref(glaunch), C.byref(gflops)))
        check(lib().vf_gemm_profile(0))
        alg = clip_vitl_ref.gemm_flops_per_frame(n_px) * 256
        r.update(gemm_ms_256=gms.value, gemm_launches=glaunch.value, gemm_tflops_executed=gflops.value / gms.value / 1e9,
                 gemm_tflops_algorithmic=alg / gms.value / 1e9, gemm_gflop_per_frame=alg / 256 / 1e9,
                 attention_gflop_per_frame=clip_vitl_ref.attention_flops_per_frame(n_px) / 1e9)
        qkv = (torch.randn(256, eng.tokens, 3072, device=dev) * 1.5).half()
        eng.attention(qkv)
        att_ms = timed(lambda: eng.attention(qkv), a.reps)
        r["attention_us_per_layer_256"] = att_ms * 1e3
        r["attention_share_256"] = 24 * att_ms / r["ms_per_call_256"]
        r["attention_tflops"] = clip_vitl_ref.attention_flops_per_frame(n_px) / 24 * 256 / att_ms / 1e9
        eng.close()
        sd16 = {k: v.to(dev, torch.float16) for k, v in sd.items()}
        x16 = x[:64].half()
        with torch.no_grad():
            for _ in range(2):
                clip_vitl_ref.encode_image(sd16, x16, dtype=torch.float16)
            ms = timed(lambda: clip_vitl_ref.encode_image(sd16, x16, dtype=torch.float16), max(2, a.reps // 2))
        r["torch_fp16_frames_per_s_64"] = 64 / ms * 1e3
        del sd16
        torch.cuda.empty_cache()
        res["towers"][f"{n_px}"] = r
        print(json.dumps({n_px: r}), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
