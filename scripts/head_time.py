"""Cost of --show_pred on one GPU: the classifier-head call (vf_head_forward, two launches) timed with CUDA events
around back-to-back calls from Python (host dispatch included) and, kernel by kernel, from the profiler's device records, at
n = 64 for 1000 x 2048 (ResNet-50) and 400 x 1024 (I3D), and ExtractResNet(resnet50) / ExtractI3D (rgb + PWC flow) on
the sample video with and without --show_pred (seeded stand-in weights; the printing goes to /dev/null).  Prints the
card name and power limit read in the same run.

    python scripts/head_time.py
"""
import argparse
import contextlib
import os
import subprocess
import sys
import tempfile
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
VIDEO = os.path.join(ROOT, "tests", "golden", "v_GGSY1Qvo990.mp4")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def head_ms(C, K, n=64, reps=200):
    from video_features_b200.class_head import ClassHead
    g = torch.Generator().manual_seed(0)
    head = ClassHead(torch.randn(C, K, generator=g) * 0.02, torch.zeros(C), 0)
    x = torch.rand(n, K, generator=g).cuda()
    for _ in range(20):
        head.forward(x)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        head.forward(x)
    b.record()
    torch.cuda.synchronize()
    # the two kernels alone: their device durations from the profiler's CUDA activity records
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(50):
            head.forward(x)
        torch.cuda.synchronize()
    kern = {}
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA and "head_" in e.name:
            key = "logits" if "logits" in e.name else "softmax_topk"
            kern[key] = kern.get(key, 0.0) + e.device_time_total / 50
    head.close()
    return a.elapsed_time(b) / reps, kern


def _ns(**kw):
    d = dict(video_paths=[VIDEO], flow_paths=None, file_with_video_paths=None, video_dir=None, flow_dir=None,
             extraction_fps=None, on_extraction='print', keep_tmp_files=False, batch_size=1, stack_size=None,
             step_size=None, streams=None, flow_type='pwc', output_direct=False, extract_method=None)
    d.update(kw)
    return argparse.Namespace(**d)


def extract_s(cls, reps=3, **kw):
    """median wall time of one extract() of the sample video (engines built and warmed up first)"""
    d = tempfile.mkdtemp()
    ex = cls(_ns(output_path=d, tmp_path=d, **kw))
    dev = torch.device("cuda", 0)
    times = []
    with open(os.devnull, "w") as null, contextlib.redirect_stdout(null):
        models = ex._load(dev) if hasattr(ex, "_load") else None
        for i in range(reps + 1):
            torch.cuda.synchronize()
            t = time.perf_counter()
            ex.extract(dev, None, models, VIDEO)
            torch.cuda.synchronize()
            if i:
                times.append(time.perf_counter() - t)
    return sorted(times)[len(times) // 2]


def main():
    from helpers import checkpoint_dir
    from oracle import pwc_net, resnet_net
    from video_features_b200.extract import extract_i3d
    from video_features_b200.extract.extract_i3d import ExtractI3D
    from video_features_b200.extract.extract_resnet import ExtractResNet
    print("card, power limit:", card())
    for C, K in ((1000, 2048), (400, 1024)):
        ms, kern = head_ms(C, K)
        print(f"head {C} x {K}, n = 64: {ms * 1000:.1f} us per call from Python (2 launches); kernels alone: "
              + ", ".join(f"{k} {v:.1f} us" for k, v in kern.items()))
    d = tempfile.mkdtemp()
    torch.save(resnet_net.stand_in_state_dict(50), os.path.join(d, "resnet50-standin.pth"))
    os.environ["VF_CKPT_DIR"] = d
    for flag in (False, True):
        print(f"ExtractResNet resnet50, sample video (355 frames), show_pred={flag}: "
              f"{extract_s(ExtractResNet, feature_type='resnet50', show_pred=flag):.3f} s")
    cd = checkpoint_dir()
    torch.save(pwc_net.stand_in_state_dict(), os.path.join(cd, pwc_net.CHECKPOINT))
    extract_i3d._CKPT_DIRS = [cd]
    for flag in (False, True):
        print(f"ExtractI3D rgb + pwc flow, sample video (5 stacks), show_pred={flag}: "
              f"{extract_s(ExtractI3D, feature_type='i3d', show_pred=flag):.3f} s")


if __name__ == "__main__":
    main()
