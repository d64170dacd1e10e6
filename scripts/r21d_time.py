"""R(2+1)D clip-feature timing on one GPU (numbers for the README / DESIGN.md §4.7).

    python scripts/r21d_time.py [--clips 1 8 32] [--json OUT] [--model_name NAME]

--model_name (extract_r21d.MODELS) times that network at its default stack size; without it, r2plus1d_18 at 16 frames.

Prints, with the GPU's name and power limit:
  * engine clips/s at 16 x 112 x 112 for each clips-per-call count (device-resident decoded 240 x 320 frames through the
    fused transform, vf_r21d_forward_u8), and for the already-transformed fp32 entry;
  * the GEMM launches' executed / algorithmic FLOP ratio and achieved TFLOP/s (vf_gemm_profile);
  * the same network in torch on the same GPU: fp32 with TF32 off (the reference's arithmetic), TF32, and fp16
    channels_last_3d;
  * ExtractR21D end to end on tests/golden/v_GGSY1Qvo990.mp4 (decode + network + one copy back).
Weights are the calibrated stand-in (oracle/r21d_net.py; tests/r21d_34_ref.py for the R(2+1)D-34 models): speed
does not depend on the values.
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
sys.path.insert(0, os.path.join(ROOT, "tests"))

import r21d_34_ref as ref34  # noqa: E402
from oracle import r21d_net  # noqa: E402
from video_features_b200 import ops  # noqa: E402
from video_features_b200.extract import extract_r21d  # noqa: E402
from video_features_b200.r21d_engine import R21DEngine  # noqa: E402

T = 16
NET = dict(eps=1e-5, layers=ref34.LAYERS_18)        # ref34.forward's network arguments


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


def algorithmic_flops(sd):
    from torch.utils.flop_counter import FlopCounterMode
    with FlopCounterMode(display=False) as fc:
        ref34.forward({k: v.to("meta") for k, v in sd.items()}, torch.zeros(1, 3, T, 112, 112, device="meta"), **NET)
    return float(fc.get_total_flops())


def torch_rates(sd, x, reps):
    import torchvision
    net = torchvision.models.video.r2plus1d_18(weights=None) if NET["layers"] == ref34.LAYERS_18 \
        else ref34.r2plus1d_34()
    net.load_state_dict(sd)
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
        h = net.half().to(memory_format=torch.channels_last_3d)
        xh = x.half().contiguous(memory_format=torch.channels_last_3d)
        out["torch_fp16_channels_last_3d"] = timed(lambda: h(xh), x.shape[0], reps)
    del net
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--clips", type=int, nargs="+", default=[1, 8, 32])
    ap.add_argument("--json", default=None)
    ap.add_argument("--model_name", choices=list(extract_r21d.MODELS), default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    global T
    model = extract_r21d.MODELS[a.model_name or extract_r21d.DEFAULT_MODEL]
    if model["layers"] == ref34.LAYERS_18:
        sd = r21d_net.stand_in_state_dict()
    else:
        sd = ref34.stand_in_state_dict_34()
        T = model["stack"]
        NET.update(eps=model["bn_eps"], layers=model["layers"])
    dev = torch.device("cuda", 0)
    res = {"gpu": gpu_info(), "model_name": a.model_name or extract_r21d.DEFAULT_MODEL, "T": T,
           "clips_per_call": extract_r21d.CLIPS_PER_CALL}
    print(f"GPU: {res['gpu']} (name, power limit, max SM clock); {res['model_name']}, {T} frames", flush=True)
    alg = algorithmic_flops(sd)
    res["gflop_per_clip"] = alg / 1e9
    g = torch.Generator().manual_seed(1)
    nmax = max(a.clips)
    frames = torch.randint(0, 256, (nmax * T, 240, 320, 3), dtype=torch.uint8, generator=g).to(dev)
    res["engine"] = {}
    for n in a.clips:
        r = {}
        eng = R21DEngine(sd, 0, max_clips=n, max_T=T, bn_eps=NET["eps"])
        starts = [i * T for i in range(n)]
        reps = max(4, 256 // n)
        r["u8_clips_per_s"] = timed(lambda: eng.forward_u8(frames, starts, T), n, reps)
        x = torch.randn(n, 3, T, 112, 112, device=dev)
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
        r.update(torch_rates(sd, x, reps))
        res["engine"][n] = r
        print(f"r21d {n:3d} clips/call ({alg / 1e9:.1f} GFLOP per clip): engine {r['u8_clips_per_s']:.1f} clips/s (u8 entry), {r['f32_clips_per_s']:.1f} "
              f"(f32 entry) | GEMM {launches} launches, executed/algorithmic {r['executed_over_algorithmic']:.2f}, "
              f"{r['gemm_tflops_executed']:.0f} TFLOP/s executed ({r['gemm_tflops_algorithmic']:.0f} algorithmic) | "
              f"torch fp32 {r['torch_fp32']:.1f}, tf32 {r['torch_tf32']:.1f}, fp16 channels_last_3d "
              f"{r['torch_fp16_channels_last_3d']:.1f} clips/s", flush=True)

    # ---- ExtractR21D end to end on the sample video
    video = os.path.join(ROOT, "tests", "golden", "v_GGSY1Qvo990.mp4")
    with tempfile.TemporaryDirectory() as d:
        torch.save(sd, os.path.join(d, model["pattern"].replace("*", "-standin-")))
        os.environ["VF_CKPT_DIR"] = d
        args = argparse.Namespace(feature_type="r21d_rgb", video_paths=[video], flow_paths=None,
                                  file_with_video_paths=None, video_dir=None, flow_dir=None, extraction_fps=None,
                                  on_extraction="print", output_path=d, tmp_path=d, show_pred=False,
                                  keep_tmp_files=False, stack_size=None, step_size=None, model_name=a.model_name)
        ex = extract_r21d.ExtractR21D(args)
        ex.extract(dev, None, None, video)                 # warm-up: engine, graphs, pinned buffers
        t0 = time.perf_counter()
        reps = 3
        for _ in range(reps):
            n = ex.extract(dev, None, None, video)["r21d_rgb"].shape[0]
        dt = (time.perf_counter() - t0) / reps
        res["extract_stacks_per_s"] = n / dt
        print(f"ExtractR21D end to end ({T}-frame stacks): {n} stacks (355 frames) in {dt * 1e3:.0f} ms = {n / dt:.1f} stacks/s",
              flush=True)
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
