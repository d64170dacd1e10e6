"""PWC-Net timing on one GPU (numbers for the README / DESIGN.md §4).

    python scripts/pwc_time.py [--pairs 16] [--json OUT]

Prints, with the GPU's name and power limit:
  * engine pairs/s at 256x341 (I3D's frame size) and 436x1024 (Sintel), `pairs` pairs per call;
  * the GEMM launches' executed and algorithmic TFLOP/s (vf_gemm_profile), the algorithmic FLOPs counted from the layer
    shapes (extractor once per frame, decoders, transposed convs and refiner per pair);
  * the oracle (oracle/pwc_net.py: torch convolutions, the 81-slice cost volume, grid_sample) on the same GPU in fp32
    with TF32 off -- the reference's arithmetic -- and with TF32;
  * I3D flow-stream stacks/s (65 frames at 256x341 -> flow -> quantiser -> I3D) with PWC and with RAFT (20 iterations).
Weights: pwc_net_sintel.pt from oracle/_ref/checkpoints/ when present (build() copies it), else the seeded stand-in --
speed does not depend on the values.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import pwc_net, raft_net  # noqa: E402
from video_features_b200 import ops  # noqa: E402
from video_features_b200.pwc_engine import PWCEngine  # noqa: E402

FEAT_C = [3, 16, 32, 64, 96, 128, 196]


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name(0)


def timed(fn, items, reps):
    """items/s of `fn` (processing `items` per call) over `reps` calls after 2 warm-up calls."""
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return items * reps / (a.elapsed_time(b) / 1e3)


def algorithmic_flops(hp, wp, frames, pairs):
    """2 x MACs of every convolution at the /64 size (hp, wp): the extractor per frame, the rest per pair."""
    ext = 0
    for l in range(1, 7):
        hw = (hp >> l) * (wp >> l)
        ext += 2 * hw * 9 * (FEAT_C[l - 1] * FEAT_C[l] + 2 * FEAT_C[l] * FEAT_C[l])
    dec = 0
    for l in range(6, 1, -1):
        hw = (hp >> l) * (wp >> l)
        cin = 81 if l == 6 else 81 + FEAT_C[l] + 4
        for co in (128, 128, 96, 64, 32, 2):
            dec += 2 * hw * 9 * cin * co
            cin += co if co != 2 else 0
        if l < 6:
            coarse = (hp >> (l + 1)) * (wp >> (l + 1))
            prev = (81 if l + 1 == 6 else 81 + FEAT_C[l + 1] + 4) + 448
            dec += 2 * coarse * 16 * 2 * (2 + prev)               # ConvTranspose2d(4, 2, 1) of flow and feature
    hw2 = (hp >> 2) * (wp >> 2)
    ch = [565, 128, 128, 128, 96, 64, 32, 2]
    dec += sum(2 * hw2 * 9 * ch[k] * ch[k + 1] for k in range(7))
    return ext * frames + dec * pairs


def load_weights():
    path = os.path.join(ROOT, "oracle", "_ref", "checkpoints", pwc_net.CHECKPOINT)
    if os.path.exists(path):
        return torch.load(path, map_location="cpu"), "pwc_net_sintel.pt"
    return pwc_net.stand_in_state_dict(), "seeded stand-in"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=16)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    dev = torch.device("cuda", 0)
    sd, label = load_weights()
    res = {"gpu": gpu_info(), "weights": label, "pairs_per_call": a.pairs}
    print(f"GPU: {res['gpu']} (name, power limit, max SM clock); weights: {label}", flush=True)
    n = a.pairs + 1
    for h, w in ((256, 341), (436, 1024)):
        hp, wp = (h + 63) // 64 * 64, (w + 63) // 64 * 64
        x = raft_net.synthetic_frames(n, h, w, seed=1).to(dev)
        u8 = x.permute(0, 2, 3, 1).contiguous().to(torch.uint8)
        eng = PWCEngine(sd, 0, max_frames=n, max_h=h, max_w=w)
        r = {"engine_pairs_per_s": timed(lambda: eng.flow(u8), a.pairs, 10)}
        ops.gemm_profile(True)
        eng.flow(u8)
        ms, launches, executed = ops.gemm_profile_read()
        ops.gemm_profile(False)
        alg = algorithmic_flops(hp, wp, n, a.pairs)
        r.update(gemm_launches=launches, gemm_ms=ms, gflop_per_pair=alg / a.pairs / 1e9,
                 gemm_tflops_executed=executed / (ms / 1e3) / 1e12, gemm_tflops_algorithmic=alg / (ms / 1e3) / 1e12)
        eng.close()
        sdg = {k: v.to(dev) for k, v in sd.items()}
        with torch.no_grad():
            for name, tf32 in (("torch_fp32", False), ("torch_tf32", True)):
                torch.backends.cudnn.allow_tf32 = tf32
                torch.backends.cuda.matmul.allow_tf32 = tf32
                r[name] = timed(lambda: pwc_net.forward(sdg, x[:-1], x[1:]), a.pairs, 3)
        torch.backends.cudnn.allow_tf32 = False
        torch.backends.cuda.matmul.allow_tf32 = False
        res[f"{h}x{w}"] = r
        print(f"{h}x{w} ({hp}x{wp}): engine {r['engine_pairs_per_s']:.0f} pairs/s | {r['gflop_per_pair']:.1f} GFLOP/pair "
              f"algorithmic | GEMM {launches} launches, {r['gemm_tflops_executed']:.0f} TFLOP/s executed "
              f"({r['gemm_tflops_algorithmic']:.0f} algorithmic) | oracle torch fp32 {r['torch_fp32']:.1f}, "
              f"tf32 {r['torch_tf32']:.1f} pairs/s", flush=True)
        del sdg
        torch.cuda.empty_cache()

    # ---- I3D flow stream: one 65-frame stack -> flow -> quantiser -> I3D
    from oracle import stand_in
    from video_features_b200.i3d_engine import I3DEngine
    from video_features_b200.raft_engine import RAFTEngine
    i3d = I3DEngine(stand_in.state_dict("i3d_flow.pt"), "flow", 0, max_stacks=1, max_T=64)
    u8 = raft_net.synthetic_frames(65, 256, 341, seed=2).permute(0, 2, 3, 1).contiguous().to(torch.uint8).to(dev)
    pwc = PWCEngine(sd, 0, max_frames=65, max_h=256, max_w=341)
    res["i3d_flow_stacks_per_s_pwc"] = timed(lambda: i3d.forward_flow(pwc.flow(u8)[None]), 1, 5)
    pwc.close()
    raft = RAFTEngine(stand_in.state_dict("raft-sintel.pth"), 0, max_frames=65, max_h=256, max_w=341)
    res["i3d_flow_stacks_per_s_raft"] = timed(lambda: i3d.forward_flow(raft.flow(u8, iters=20, unpad=False)[None]), 1, 3)
    raft.close()
    i3d.close()
    print(f"I3D flow stream, 65-frame stacks at 256x341: {res['i3d_flow_stacks_per_s_pwc']:.2f} stacks/s with PWC, "
          f"{res['i3d_flow_stacks_per_s_raft']:.2f} with RAFT", flush=True)
    if a.json:
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
