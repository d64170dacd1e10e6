"""VideoMAE timing on one GPU, seeded stand-in weights: clips/s of the engine at 4 and 16 clips per call (f32 entry,
graphs warm), with the SM clock read right after; the GEMM launches' share of a call and their executed TFLOP/s (split
weights count twice; vf_gemm_profile, an eager run); the attention kernel's share of a call (its time alone x depth
over the call time), the attention kernel's TFLOP/s against torch's scaled_dot_product_attention (flash
backend, fp16) on the same q / k / v at S = 1568, and the feature error of the oracle run by torch in fp32, TF32 and
fp16 autocast against float64.  Prints one JSON line per model; the card and its power limit come first."""
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import videomae_net as V  # noqa: E402
from video_features_b200 import ops  # noqa: E402
from video_features_b200.videomae_engine import VideoMAEEngine, attention  # noqa: E402


def timed(fn, iters):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / iters


def sm_clock():
    q = ["nvidia-smi", "--query-gpu=clocks.sm", "--format=csv,noheader,nounits"]
    return subprocess.run(q, capture_output=True, text=True).stdout.strip()


def rel(y, ref):
    return ((y.double() - ref).norm(dim=1) / ref.norm(dim=1)).max().item()


def main():
    names = sys.argv[1:] or list(V.SHAPES)
    q = ["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"]
    print(json.dumps({"gpu": subprocess.run(q, capture_output=True, text=True).stdout.strip()}), flush=True)
    from torch.nn.attention import SDPBackend, sdpa_kernel
    for name in names:
        d, depth, heads, f = V.SHAPES[name]
        res = {"model": name}
        eng = VideoMAEEngine(V.stand_in_state_dict(name), V.config_dict(name), device=0, max_clips=16)
        for n in (4, 16):
            x = V.calibration_clips(0, 1).cuda().expand(n, -1, -1, -1, -1).contiguous()
            ms = timed(lambda: eng.forward_f32(x), 10)
            res[f"sm_mhz_after_{n}"] = sm_clock()
            res[f"clips_per_s_{n}"] = round(n * 1000 / ms, 1)
            res[f"ms_per_call_{n}"] = round(ms, 3)
            ops.gemm_profile(True)
            eng.forward_f32(x)
            gms, _, gfl = ops.gemm_profile_read()
            ops.gemm_profile(False)
            res[f"gemm_share_{n}"] = round(gms / ms, 3)
            res[f"gemm_tflops_executed_{n}"] = round(gfl / gms / 1e9, 1)
        # the attention alone at 4 clips, every head
        n = 4
        qkv = (torch.randn(n, V.TOKENS, 3 * d, device="cuda") * 1.5).half()
        ms_att = timed(lambda: attention(qkv, heads), 50)
        fl = 4 * V.TOKENS * V.TOKENS * d * n
        res["attention_tflops"] = round(fl / ms_att / 1e9, 1)
        qh, kh, vh = (t.view(n, V.TOKENS, heads, 64).transpose(1, 2).contiguous() for t in qkv.split(d, -1))
        with sdpa_kernel(SDPBackend.FLASH_ATTENTION):
            ms_sdpa = timed(lambda: torch.nn.functional.scaled_dot_product_attention(qh, kh, vh), 50)
        res["sdpa_flash_tflops"] = round(fl / ms_sdpa / 1e9, 1)
        res["attention_share"] = round(depth * ms_att / res["ms_per_call_4"], 3)
        w = V.flops(name)
        res["model_tflops_4"] = round(4 * (w["gemm"] + w["attention"]) / res["ms_per_call_4"] / 1e9, 1)
        # torch bars of the oracle
        p64 = V.prepare(V.stand_in_state_dict(name), torch.float64, "cuda")
        p32 = V.prepare(V.stand_in_state_dict(name), torch.float32, "cuda")
        x = V.calibration_clips(1, 2).cuda()
        with torch.no_grad():
            ref = V.forward(p64, x.double())
            res["engine_vs_f64"] = rel(eng.forward_f32(x), ref)
            torch.backends.cuda.matmul.allow_tf32 = False
            res["torch_fp32_vs_f64"] = rel(V.forward(p32, x), ref)
            torch.backends.cuda.matmul.allow_tf32 = True
            res["torch_tf32_vs_f64"] = rel(V.forward(p32, x), ref)
            torch.backends.cuda.matmul.allow_tf32 = False
            with torch.autocast("cuda", dtype=torch.float16):
                res["torch_fp16_autocast_vs_f64"] = rel(V.forward(p32, x).float(), ref)
        eng.close()
        print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
