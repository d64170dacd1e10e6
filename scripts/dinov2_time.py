"""DINOv2 frame-feature timing on one GPU (numbers for the README / DESIGN.md §4.17).

    python scripts/dinov2_time.py [--models dinov2_vits14 ...] [--frames 64 256] [--json OUT]

Prints, with the GPU's name and power limit:
  * engine frames/s for each frames-per-call count (device-resident decoded 240 x 320 BGR frames through the fused
    transform, vf_dinov2_encode_u8): the median of --repeats timed windows, with their lowest and highest;
  * the GEMM launches' share of the call and their TFLOP/s (vf_gemm_profile), executed (split weights count twice) and
    algorithmic (oracle/dinov2_net.flops: all tokens through every block, one weight pass);
  * the attention kernel's share (the kernel alone, vf_dinov2_attention, once per block) and, for g/14, the SwiGLU
    kernel's share (vf_dinov2_swiglu, once per block but the last on all rows);
  * the oracle module on the same frames and GPU: fp32 with TF32 off, TF32, and fp16 autocast.
Weights are the seeded stand-ins (oracle/dinov2_net.py): speed does not depend on the values.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import dinov2_net as D  # noqa: E402
from video_features_b200 import ops  # noqa: E402
from video_features_b200.dinov2_engine import DINOv2Engine, attention, swiglu  # noqa: E402


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name(0)


def timed_ms(fn, reps):
    """ms per call of `fn` over `reps` calls after 2 warm-up calls."""
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps


def torch_rates(sd, x, reps):
    """frames/s of the oracle's forward on x (n, 3, 224, 224): fp32, TF32, fp16 autocast."""
    p = D.prepare(sd, torch.float32, x.device)
    out = {}
    with torch.no_grad():
        for label, tf32 in (("torch_fp32", False), ("torch_tf32", True)):
            torch.backends.cuda.matmul.allow_tf32 = tf32
            out[label] = x.shape[0] / (timed_ms(lambda: D.forward(p, x), reps) / 1e3)
        torch.backends.cuda.matmul.allow_tf32 = False
        with torch.autocast("cuda", dtype=torch.float16):
            out["torch_fp16_autocast"] = x.shape[0] / (timed_ms(lambda: D.forward(p, x), reps) / 1e3)
    del p
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--models", nargs="+", default=list(D.MODELS))
    ap.add_argument("--frames", type=int, nargs="+", default=[64, 256])
    ap.add_argument("--repeats", type=int, default=5, help="timed windows per engine measurement")
    ap.add_argument("--no-torch", action="store_true", help="skip the torch bars")
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    dev = torch.device("cuda", 0)
    res = {"gpu": gpu_info(), "models": {}}
    print(f"GPU: {res['gpu']} (name, power limit, max SM clock)", flush=True)
    g = torch.Generator().manual_seed(1)
    nmax = max(a.frames)
    frames = torch.randint(0, 256, (nmax, 240, 320, 3), dtype=torch.uint8, generator=g).to(dev)
    for name in a.models:
        d, depth, ffn, reg = D.shape_of(name)
        sd = D.stand_in_state_dict(name)
        fl = D.flops(name)
        executed = D.executed_gemm_flops(name)
        res["models"][name] = {"gemm_gflop_per_frame": fl["gemm"] / 1e9, "executed_gemm_gflop_per_frame": executed / 1e9}
        eng = DINOv2Engine(sd, 0)
        S = eng.tokens
        for n in a.frames:
            r = {"max_frames": eng.max_frames}
            reps = max(3, 1024 // (n * max(1, d // 384)))
            runs = sorted(timed_ms(lambda: eng.encode_u8(frames[:n]), reps) for _ in range(a.repeats))
            ms = runs[len(runs) // 2]
            r["frames_per_s"] = n / (ms / 1e3)
            r["frames_per_s_range"] = [n / (runs[-1] / 1e3), n / (runs[0] / 1e3)]
            ops.gemm_profile(True)
            eng.encode_u8(frames[:n])
            gms, launches, flops_run = ops.gemm_profile_read()
            ops.gemm_profile(False)
            r["gemm_share"] = gms / ms
            r["gemm_tflops_executed"] = flops_run / (gms / 1e3) / 1e12
            r["gemm_tflops_algorithmic"] = fl["gemm"] * n / (gms / 1e3) / 1e12
            # kernels alone, at the chunk size the engine runs
            c = -(-n // -(-n // eng.max_frames))
            chunks = -(-n // c)
            qkv = torch.randn(c, S, 3 * d, device=dev).half()
            att_ms = timed_ms(lambda: attention(qkv, d // 64), reps) * depth * chunks
            del qkv
            r["attention_share"] = att_ms / ms
            r["attention_tflops"] = fl["attention"] * n / (att_ms / 1e3) / 1e12
            if ffn == "swiglu":
                ab = torch.randn(c * S, 2 * D.SWIGLU_HIDDEN, device=dev)
                sw_ms = timed_ms(lambda: swiglu(ab), reps) * (depth - 1) * chunks
                del ab
                r["swiglu_share"] = sw_ms / ms
            if not a.no_torch:
                x = torch.randn(min(n, 64), 3, 224, 224, device=dev)
                r.update(torch_rates(sd, x, max(2, reps // 2)))
                del x
            res["models"][name][n] = r
            line = (f"{name} {n} frames/call: engine {r['frames_per_s']:.0f} frames/s "
                    f"({r['frames_per_s_range'][0]:.0f}-{r['frames_per_s_range'][1]:.0f}) | GEMM {100 * r['gemm_share']:.0f} %, "
                    f"{r['gemm_tflops_executed']:.0f} TFLOP/s executed, {r['gemm_tflops_algorithmic']:.0f} algorithmic "
                    f"({launches} launches) | attention {100 * r['attention_share']:.1f} %, {r['attention_tflops']:.0f} "
                    f"TFLOP/s")
            if "swiglu_share" in r:
                line += f" | SwiGLU {100 * r['swiglu_share']:.1f} %"
            if "torch_fp32" in r:
                line += (f" | torch fp32 {r['torch_fp32']:.0f}, tf32 {r['torch_tf32']:.0f}, fp16 autocast "
                         f"{r['torch_fp16_autocast']:.0f} frames/s")
            print(line, flush=True)
        eng.close()
        torch.cuda.empty_cache()
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
