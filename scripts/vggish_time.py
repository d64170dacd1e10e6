"""Throughput of the VGGish engine on one GPU (calibrated stand-in weights; the trunk's cost does not depend on them).

    python scripts/vggish_time.py [--json OUT]

Prints, with the GPU's name, power limit and max SM clock read in the same run:
  - examples/s of the trunk (vf_vggish_forward_logmel_f32) at 1, 10, 64 and 625 examples per call;
  - end-to-end seconds for a 10-minute 44.1 kHz stereo PCM-16 WAV (625 examples): read from disk, upload, resample,
    log-mel and trunk, and the front end's share (the same call minus the trunk on the same examples);
  - the fp32 torch oracle (oracle/vggish_net.py forward, TF32 off) on the same card at 64 and 625 examples.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time
import wave

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import vggish_net  # noqa: E402
from video_features_b200 import audio  # noqa: E402
from video_features_b200.vggish_engine import VGGishEngine  # noqa: E402


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    t = time.perf_counter()
    for _ in range(reps):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    res = {"gpu": gpu_info()}
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    sd = vggish_net.stand_in_state_dict()
    eng = VGGishEngine(sd, 0, max_examples=64)
    g = torch.Generator().manual_seed(0)
    lm = (torch.randn(625, 96, 64, generator=g) - 2.0).cuda()
    res["trunk_examples_per_s"] = {}
    for n in (1, 10, 64, 625):
        t = timed(lambda: eng.forward_logmel(lm[:n]), max(3, 640 // n))
        res["trunk_examples_per_s"][n] = n / t
    sdc = {k: v.cuda() for k, v in sd.items()}
    res["oracle_fp32_examples_per_s"] = {}
    with torch.no_grad():
        for n in (64, 625):
            t = timed(lambda: vggish_net.forward(sdc, lm[:n]), 3)
            res["oracle_fp32_examples_per_s"][n] = n / t
    x = vggish_net.synthetic_audio(600.0, 44100, 2, seed=1)
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "ten_minutes.wav")
        with wave.open(path, "wb") as w:
            w.setnchannels(2)
            w.setsampwidth(2)
            w.setframerate(44100)
            w.writeframes(x.astype("<i2").tobytes())

        def end_to_end():
            s, sr = audio.read_wav_pcm16(path)
            return eng.forward_pcm16(s, sr)
        y = end_to_end()
        t_e2e = timed(end_to_end, 3)
    t_pcm = timed(lambda: eng.forward_pcm16(torch.from_numpy(x).cuda(), 44100), 3)
    t_trunk = timed(lambda: eng.forward_logmel(lm[:y.shape[0]]), 3)
    res["ten_minute_wav"] = {"examples": int(y.shape[0]), "end_to_end_s": t_e2e, "device_call_s": t_pcm,
                             "trunk_s": t_trunk, "front_end_s": t_pcm - t_trunk}
    eng.close()
    print(json.dumps(res, indent=1))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
