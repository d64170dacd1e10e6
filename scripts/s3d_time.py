"""S3D clip-feature timing on one GPU (numbers for the README / DESIGN.md §4.12).

    python scripts/s3d_time.py [--clips 1 4 8] [--json OUT]

Prints, with the GPU's name and power limit:
  * engine clips/s at 64 x 224 x 224 for each clips-per-call count (device-resident decoded 240 x 320 frames through the
    fused transform, vf_s3d_forward_u8), and for the already-transformed fp32 entry;
  * the GEMM launches' executed / algorithmic FLOP ratio and achieved TFLOP/s (vf_gemm_profile);
  * the same network in torch on the same GPU: fp32 with TF32 off (the reference's arithmetic), TF32, and fp16
    channels_last_3d;
  * ExtractS3D end to end on tests/golden/v_GGSY1Qvo990.mp4 (decode + network + one copy back).
Weights are the calibrated stand-in (oracle/s3d_net.py): speed does not depend on the values.
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

from oracle import s3d_net  # noqa: E402
from video_features_b200 import ops  # noqa: E402
from video_features_b200.extract import extract_s3d  # noqa: E402
from video_features_b200.s3d_engine import S3DEngine  # noqa: E402

T = 64


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name(0)


def timed(fn, clips, reps):
    """clips/s of `fn` (processing `clips` clips per call) over `reps` calls after 2 warm-up calls."""
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return clips * reps / (a.elapsed_time(b) / 1e3)


def algorithmic_flops():
    from torch.utils.flop_counter import FlopCounterMode
    sd = s3d_net.stand_in_state_dict()
    with FlopCounterMode(display=False) as fc:
        s3d_net.forward({k: v.to("meta") for k, v in sd.items()}, torch.zeros(1, 3, T, 224, 224, device="meta"))
    return float(fc.get_total_flops())


def torch_rates(x, reps):
    import torchvision
    net = torchvision.models.video.s3d(weights=None)
    net.load_state_dict(s3d_net.stand_in_state_dict())
    net = net.eval().to(x.device)
    out = {}
    with torch.no_grad():
        for label, tf32 in (("torch_fp32", False), ("torch_tf32", True)):
            torch.backends.cudnn.allow_tf32 = tf32
            torch.backends.cuda.matmul.allow_tf32 = tf32
            out[label] = timed(lambda: net(x), x.shape[0], reps)
        torch.backends.cudnn.allow_tf32 = False
        torch.backends.cuda.matmul.allow_tf32 = False
        h = net.half().to(memory_format=torch.channels_last_3d)
        xh = x.half().contiguous(memory_format=torch.channels_last_3d)
        out["torch_fp16_channels_last_3d"] = timed(lambda: h(xh), x.shape[0], reps)
    del net
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--clips", type=int, nargs="+", default=[1, 4, 8])
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    dev = torch.device("cuda", 0)
    res = {"gpu": gpu_info(), "T": T, "clips_per_call": extract_s3d.CLIPS_PER_CALL}
    print(f"GPU: {res['gpu']} (name, power limit, max SM clock)", flush=True)
    sd = s3d_net.stand_in_state_dict()
    alg = algorithmic_flops()
    res["gflop_per_clip"] = alg / 1e9
    g = torch.Generator().manual_seed(1)
    nmax = max(a.clips)
    frames = torch.randint(0, 256, (nmax * T, 240, 320, 3), dtype=torch.uint8, generator=g).to(dev)
    res["engine"] = {}
    for n in a.clips:
        r = {}
        eng = S3DEngine(sd, 0, max_clips=n, max_T=T)
        starts = [i * T for i in range(n)]
        reps = max(4, 32 // n)
        r["u8_clips_per_s"] = timed(lambda: eng.forward_u8(frames, starts, T), n, reps)
        x = torch.randn(n, 3, T, 224, 224, device=dev)
        r["f32_clips_per_s"] = timed(lambda: eng.forward_f32(x), n, reps)
        ops.gemm_profile(True)
        eng.forward_f32(x)
        ms, launches, executed = ops.gemm_profile_read()
        ops.gemm_profile(False)
        r["gemm_launches"], r["gemm_ms"] = launches, ms
        r["executed_over_algorithmic"] = executed / (alg * n)
        r["gemm_tflops_executed"] = executed / (ms / 1e3) / 1e12
        r["gemm_tflops_algorithmic"] = alg * n / (ms / 1e3) / 1e12
        eng.close()
        torch.cuda.empty_cache()
        r.update(torch_rates(x, reps))
        res["engine"][n] = r
        print(f"s3d {n:3d} clips/call: engine {r['u8_clips_per_s']:.1f} clips/s (u8 entry), {r['f32_clips_per_s']:.1f} "
              f"(f32 entry) | GEMM {launches} launches, executed/algorithmic {r['executed_over_algorithmic']:.2f}, "
              f"{r['gemm_tflops_executed']:.0f} TFLOP/s executed ({r['gemm_tflops_algorithmic']:.0f} algorithmic) | "
              f"torch fp32 {r['torch_fp32']:.1f}, tf32 {r['torch_tf32']:.1f}, fp16 channels_last_3d "
              f"{r['torch_fp16_channels_last_3d']:.1f} clips/s", flush=True)

    # ---- ExtractS3D end to end on the sample video
    video = os.path.join(ROOT, "tests", "golden", "v_GGSY1Qvo990.mp4")
    with tempfile.TemporaryDirectory() as d:
        torch.save(sd, os.path.join(d, "s3d-standin.pth"))
        os.environ["VF_CKPT_DIR"] = d
        args = argparse.Namespace(feature_type="s3d", video_paths=[video], flow_paths=None,
                                  file_with_video_paths=None, video_dir=None, flow_dir=None, extraction_fps=None,
                                  on_extraction="print", output_path=d, tmp_path=d, show_pred=False,
                                  keep_tmp_files=False, stack_size=None, step_size=None)
        ex = extract_s3d.ExtractS3D(args)
        ex.extract(dev, None, None, video)                 # warm-up: engine, graphs, pinned buffers
        t0 = time.perf_counter()
        reps = 3
        for _ in range(reps):
            n = ex.extract(dev, None, None, video)["s3d"].shape[0]
        dt = (time.perf_counter() - t0) / reps
        res["extract_stacks_per_s"] = n / dt
        print(f"ExtractS3D end to end: {n} stacks (355 frames) in {dt * 1e3:.0f} ms = {n / dt:.1f} stacks/s",
              flush=True)
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
