"""ResNet frame-feature timing on one GPU (numbers for the README / DESIGN.md §4.6).

    python scripts/resnet_time.py [--depths 18 34 50 101 152] [--json OUT]

Prints, with the GPU's name and power limit:
  * the frames-per-call sweep of ResNet-50 (calls of `chunk` device-resident frames), which sets
    extract_resnet.FRAMES_PER_CALL;
  * per depth: engine frames/s at FRAMES_PER_CALL frames per call and at 1000 frames per call (chunked inside the call),
    the GEMM launches' executed / algorithmic FLOP ratio and achieved TFLOP/s (vf_gemm_profile), and the same network in
    torch on the same GPU: fp32 with TF32 off (the reference's arithmetic), TF32, fp16 channels_last;
  * ExtractResNet end to end on tests/golden/v_GGSY1Qvo990.mp4 (decode + resize + network + one copy back).
Weights are the calibrated stand-in (oracle/resnet_net.py): speed does not depend on the values.
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

from oracle import resnet_net  # noqa: E402
from video_features_b200 import ops  # noqa: E402
from video_features_b200.extract import extract_resnet  # noqa: E402
from video_features_b200.resnet_engine import ResNetEngine  # noqa: E402


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


def resized_frames(n, device):
    g = torch.Generator().manual_seed(1)
    return torch.randint(0, 256, (n, 256, 341, 3), dtype=torch.uint8, generator=g).to(device)


def algorithmic_flops(depth):
    from torch.utils.flop_counter import FlopCounterMode
    sd = resnet_net.stand_in_state_dict(depth)
    with FlopCounterMode(display=False) as fc:
        resnet_net.forward({k: v.to("meta") for k, v in sd.items()}, torch.zeros(1, 3, 224, 224, device="meta"), depth)
    return float(fc.get_total_flops())


def torch_rates(depth, x, reps):
    import torchvision
    net = getattr(torchvision.models, f"resnet{depth}")(weights=None)
    net.load_state_dict(resnet_net.stand_in_state_dict(depth))
    net.fc = torch.nn.Identity()
    net = net.eval().to(x.device)
    out = {}
    with torch.no_grad():
        for label, tf32 in (("torch_fp32", False), ("torch_tf32", True)):
            torch.backends.cudnn.allow_tf32 = tf32
            torch.backends.cuda.matmul.allow_tf32 = tf32
            out[label] = timed(lambda: net(x), x.shape[0], reps)
        torch.backends.cudnn.allow_tf32 = False
        torch.backends.cuda.matmul.allow_tf32 = False
        h = net.half().to(memory_format=torch.channels_last)
        xh = x.half().contiguous(memory_format=torch.channels_last)
        out["torch_fp16_channels_last"] = timed(lambda: h(xh), x.shape[0], reps)
    del net
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--depths", type=int, nargs="+", default=[18, 34, 50, 101, 152])
    ap.add_argument("--sweep", type=int, nargs="+", default=[16, 32, 64, 128, 256])
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    dev = torch.device("cuda", 0)
    res = {"gpu": gpu_info(), "frames_per_call": extract_resnet.FRAMES_PER_CALL}
    print(f"GPU: {res['gpu']} (name, power limit, max SM clock)", flush=True)
    frames1000 = resized_frames(1000, dev)

    # ---- frames-per-call sweep (ResNet-50)
    sd50 = resnet_net.stand_in_state_dict(50)
    res["sweep_resnet50"] = {}
    for c in a.sweep:
        eng = ResNetEngine(sd50, 50, 0, max_frames=c)
        x = frames1000[:c]
        fps = timed(lambda: eng.forward_u8(x), c, max(4, 2048 // c))
        res["sweep_resnet50"][c] = fps
        print(f"sweep resnet50: {c:4d} frames per call: {fps:8.0f} frames/s", flush=True)
        eng.close()
        torch.cuda.empty_cache()

    # ---- per depth
    chunk = extract_resnet.FRAMES_PER_CALL
    res["depths"] = {}
    for depth in a.depths:
        r = {}
        sd = resnet_net.stand_in_state_dict(depth)
        eng = ResNetEngine(sd, depth, 0, max_frames=chunk)
        x = frames1000[:chunk]
        r["engine_chunk"] = timed(lambda: eng.forward_u8(x), chunk, max(4, 2048 // chunk))
        r["engine_1000"] = timed(lambda: eng.forward_u8(frames1000), 1000, 3)
        ops.gemm_profile(True)
        eng.forward_u8(x)
        ms, launches, executed = ops.gemm_profile_read()
        ops.gemm_profile(False)
        alg = algorithmic_flops(depth) * chunk
        r["gemm_launches"], r["gemm_ms"] = launches, ms
        r["executed_over_algorithmic"] = executed / alg
        r["gemm_tflops_executed"] = executed / (ms / 1e3) / 1e12
        r["gemm_tflops_algorithmic"] = alg / (ms / 1e3) / 1e12
        r["gflop_per_frame"] = alg / chunk / 1e9
        eng.close()
        torch.cuda.empty_cache()
        xn = torch.randn(chunk, 3, 224, 224, device=dev)
        r.update(torch_rates(depth, xn, max(4, 1024 // chunk)))
        res["depths"][depth] = r
        print(f"resnet{depth}: {r['gflop_per_frame']:.2f} GFLOP/frame | engine {r['engine_chunk']:.0f} frames/s "
              f"({chunk}/call), {r['engine_1000']:.0f} frames/s (1000/call) | GEMM {launches} launches, executed/"
              f"algorithmic {r['executed_over_algorithmic']:.2f}, {r['gemm_tflops_executed']:.0f} TFLOP/s executed "
              f"({r['gemm_tflops_algorithmic']:.0f} algorithmic) | torch fp32 {r['torch_fp32']:.0f}, tf32 "
              f"{r['torch_tf32']:.0f}, fp16 channels_last {r['torch_fp16_channels_last']:.0f} frames/s", flush=True)

    # ---- ExtractResNet end to end on the sample video
    video = os.path.join(ROOT, "tests", "golden", "v_GGSY1Qvo990.mp4")
    with tempfile.TemporaryDirectory() as d:
        for depth in (18, 50):
            torch.save(resnet_net.stand_in_state_dict(depth), os.path.join(d, f"resnet{depth}-standin.pth"))
        os.environ["VF_CKPT_DIR"] = d
        res["extract"] = {}
        for depth in (18, 50):
            args = argparse.Namespace(feature_type=f"resnet{depth}", video_paths=[video], flow_paths=None,
                                      file_with_video_paths=None, video_dir=None, flow_dir=None, extraction_fps=None,
                                      on_extraction="print", output_path=d, tmp_path=d, show_pred=False,
                                      keep_tmp_files=False, batch_size=1)
            ex = extract_resnet.ExtractResNet(args)
            ex.extract(dev, None, None, video)                 # warm-up: engine, graphs, pinned buffers
            t0 = time.perf_counter()
            reps = 3
            for _ in range(reps):
                n = ex.extract(dev, None, None, video)[f"resnet{depth}"].shape[0]
            dt = (time.perf_counter() - t0) / reps
            res["extract"][depth] = n / dt
            print(f"ExtractResNet resnet{depth} end to end: {n} frames in {dt * 1e3:.0f} ms = {n / dt:.0f} frames/s",
                  flush=True)
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
