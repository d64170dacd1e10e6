"""MViT clip-feature timing on one GPU (numbers for the README / DESIGN.md §4.15).

    python scripts/mvit_time.py [--models mvit_v1_b mvit_v2_s] [--clips 1 4 8] [--json OUT]

Prints, with the GPU's name and power limit:
  * engine clips/s at 16 x 224 x 224 for each clips-per-call count (device-resident decoded 240 x 320 frames through
    the fused transform, vf_mvit_forward_u8);
  * the pooling-attention kernel's share of the forward time and its achieved TFLOP/s (the kernel alone through
    vf_mvit_attention on every block's geometry, FLOPs counted from shapes by oracle/mvit_net.flops);
  * the GEMM launches' achieved TFLOP/s (vf_gemm_profile);
  * the same clips through torchvision's module on the same GPU: fp32 with TF32 off, TF32, and fp16 autocast.
Weights are the seeded stand-ins (oracle/mvit_net.py): speed does not depend on the values.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import mvit_net  # noqa: E402
from video_features_b200 import ops  # noqa: E402
from video_features_b200.mvit_engine import MViTEngine, pool_attention  # noqa: E402

T = 16


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


def attention_ms(name, n, reps):
    """The pooling-attention kernel alone on every block of one forward of n clips, in ms: each block's q and k / v
    grids (393 keys, or 1569 at the q-stride blocks 1, 3 and 14), v2's rel-pos tables and residual."""
    v2 = name == "mvit_v2_s"
    total, S = 0.0, 56
    for i in range(16):
        sq, skv = mvit_net.pooled(S, mvit_net.STRIDE_Q[i]), mvit_net.pooled(S, mvit_net.STRIDE_KV[i])
        heads = mvit_net.HEADS[i]
        c = heads * 96
        q = torch.randn(n, 1 + 8 * sq * sq, c, device="cuda").half()
        k = torch.randn(n, 1 + 8 * skv * skv, c, device="cuda").half()
        rel = None
        if v2:
            sp = 2 * max(sq, skv) - 1
            rel = (torch.zeros(sp, 96, device="cuda"), torch.zeros(sp, 96, device="cuda"), torch.zeros(15, 96, device="cuda"))
        total += timed_ms(lambda: pool_attention(q, k, k, (8, sq, sq), (8, skv, skv), rel, resid=v2), reps)
        del q, k
        S = sq
    return total


def torch_rates(name, sd, x, reps):
    net = mvit_net.torchvision_model(name)
    net.load_state_dict(sd)
    net = net.eval().to(x.device)
    out = {}
    with torch.no_grad():
        for label, tf32 in (("torch_fp32", False), ("torch_tf32", True)):
            torch.backends.cuda.matmul.allow_tf32 = tf32
            torch.backends.cudnn.allow_tf32 = tf32
            out[label] = x.shape[0] / (timed_ms(lambda: net(x), reps) / 1e3)
        torch.backends.cuda.matmul.allow_tf32 = False
        torch.backends.cudnn.allow_tf32 = False
        with torch.autocast("cuda", dtype=torch.float16):
            out["torch_fp16_autocast"] = x.shape[0] / (timed_ms(lambda: net(x), reps) / 1e3)
    del net
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--models", nargs="+", default=list(mvit_net.MODELS))
    ap.add_argument("--clips", type=int, nargs="+", default=[1, 4, 8])
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    dev = torch.device("cuda", 0)
    res = {"gpu": gpu_info(), "T": T, "models": {}}
    print(f"GPU: {res['gpu']} (name, power limit, max SM clock)", flush=True)
    g = torch.Generator().manual_seed(1)
    nmax = max(a.clips)
    frames = torch.randint(0, 256, (nmax * T, 240, 320, 3), dtype=torch.uint8, generator=g).to(dev)
    for name in a.models:
        sd = mvit_net.stand_in_state_dict(name)
        att_gf, tot_gf = mvit_net.flops(name)
        res["models"][name] = {"gflop_per_clip": tot_gf, "attention_gflop_per_clip": att_gf}
        eng = MViTEngine(sd, 0, max_clips=nmax)
        for n in a.clips:
            r = {}
            starts = [i * T for i in range(n)]
            reps = max(4, 32 // n)
            ms = timed_ms(lambda: eng.forward_u8(frames, starts, T), reps)
            r["clips_per_s"] = n / (ms / 1e3)
            att = attention_ms(name, n, reps)
            r["attention_share"] = att / ms
            r["attention_tflops"] = att_gf * n / att            # GFLOP / ms = TFLOP/s
            ops.gemm_profile(True)
            eng.forward_u8(frames, starts, T)
            gms, launches, executed = ops.gemm_profile_read()
            ops.gemm_profile(False)
            r["gemm_share"] = gms / ms
            r["gemm_tflops"] = executed / (gms / 1e3) / 1e12
            x = torch.randn(n, 3, T, 224, 224, device=dev)
            r.update(torch_rates(name, sd, x, max(2, reps // 2)))
            del x
            res["models"][name][n] = r
            print(f"{name} {n} x {T} frames: engine {r['clips_per_s']:.1f} clips/s | pooling attention "
                  f"{100 * r['attention_share']:.0f} % of the time, {r['attention_tflops']:.0f} TFLOP/s | GEMM "
                  f"{100 * r['gemm_share']:.0f} %, {r['gemm_tflops']:.0f} TFLOP/s ({launches} launches) | torch fp32 "
                  f"{r['torch_fp32']:.1f}, tf32 {r['torch_tf32']:.1f}, fp16 autocast {r['torch_fp16_autocast']:.1f} "
                  f"clips/s", flush=True)
        eng.close()
        torch.cuda.empty_cache()
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
