"""The VGGish oracle against the reference's own outputs (tests/golden/vggish_outputs.npz, scripts/make_golden.py
vggish), the resampler restatement's properties, the kernel's time register, the stand-in's calibration and the WAV
reader."""
import os
import wave

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import vggish_net
from video_features_b200 import audio

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "vggish_outputs.npz")


def write_wav(path, samples: np.ndarray, rate: int, width: int = 2):
    ch = 1 if samples.ndim == 1 else samples.shape[1]
    with wave.open(str(path), "wb") as w:
        w.setnchannels(ch)
        w.setsampwidth(width)
        w.setframerate(rate)
        w.writeframes(np.ascontiguousarray(samples).tobytes())


def test_logmel_matches_reference_bit_for_bit():
    g = np.load(GOLDEN)
    ex = vggish_net.examples(g["samples"], int(g["sample_rate"]))
    assert ex.dtype == np.float32 and ex.shape == g["examples"].shape == (7, 96, 64)
    assert np.array_equal(ex.view(np.int32), g["examples"].view(np.int32))
    assert np.any(ex == np.float32(np.log(0.01)))             # the silent stretch


def test_vgg_forward_matches_reference():
    g = np.load(GOLDEN)
    with torch.no_grad():
        f = vggish_net.forward(vggish_net.stand_in_state_dict(), torch.from_numpy(g["examples"])).numpy()
    ref = g["vggish_torch"]
    assert f.shape == ref.shape == (7, 128)
    assert np.abs(f - ref).max() <= 1e-5 * np.abs(ref).max()


@pytest.mark.parametrize("sr", [44100, 48000, 22050, 8000])
def test_resampler_length_constant_and_sine(sr):
    n = int(1.5 * sr) + 7
    c = vggish_net.resample(np.full(n, 0.25), sr)
    assert c.shape[0] == int(n * (16000.0 / sr)) == audio.resampled_length(n, sr)
    inner = c[100:-100]                                        # the filter reaches 64 zero crossings into each edge
    assert np.abs(inner - 0.25).max() < 0.25 * 5e-3
    t = np.arange(n) / sr
    y = vggish_net.resample(0.5 * np.sin(2 * np.pi * 1000.0 * t), sr)[200:-200]
    amp = np.sqrt(2 * np.mean(y * y))
    assert abs(amp - 0.5) < 0.5 * 5e-3, amp


@pytest.mark.parametrize("sr", [44100, 48000, 22050, 8000, 11025, 32000, 7999])
def test_time_register_is_the_sequential_sum(sr):
    from video_features_b200.vggish_engine import time_register
    n = int(3_000_000 * 16000 / sr)
    ref = vggish_net.time_register(n, 16000.0 / sr)
    assert np.array_equal(time_register(sr, 0, n), ref)
    assert np.array_equal(time_register(sr, n - 1000, 1000), ref[-1000:])


def test_stand_in_is_deterministic_and_calibrated():
    a, b = vggish_net.stand_in_state_dict(), vggish_net.stand_in_state_dict()
    assert all(torch.equal(a[k], b[k]) for k in a)
    x = torch.from_numpy(vggish_net.calibration_examples()).double()[:, None]
    h = x
    sd = {k: v.double() for k, v in a.items()}
    for i, _, _ in vggish_net.CONVS:
        pre = F.conv2d(h, sd[f"features.{i}.weight"], sd[f"features.{i}.bias"], padding=1)
        assert 0.3 <= (pre > 0).double().mean() <= 0.7 and 0.5 <= pre.std() <= 2
        h = F.relu(pre)
        if i in vggish_net.POOL_AFTER:
            h = F.max_pool2d(h, 2, 2)
    h = h.permute(0, 2, 3, 1).reshape(h.shape[0], -1)
    for i, _, _ in vggish_net.LINEARS:
        pre = F.linear(h, sd[f"embeddings.{i}.weight"], sd[f"embeddings.{i}.bias"])
        assert 0.3 <= (pre > 0).double().mean() <= 0.7 and 0.5 <= pre.std() <= 2
        h = F.relu(pre)
    assert bool((h > 0).any(dim=1).all())                      # no feature row is all zero


def test_wav_reader(tmp_path):
    mono = vggish_net.synthetic_audio(0.1, 16000, 1)
    stereo = vggish_net.synthetic_audio(0.1, 44100, 2)
    write_wav(tmp_path / "m.wav", mono.astype("<i2"), 16000)
    write_wav(tmp_path / "s.wav", stereo.astype("<i2"), 44100)
    x, sr = audio.read_wav_pcm16(tmp_path / "m.wav")
    assert sr == 16000 and x.dtype == np.int16 and np.array_equal(x, mono)
    x, sr = audio.read_wav_pcm16(tmp_path / "s.wav")
    assert sr == 44100 and x.shape == stereo.shape and np.array_equal(x, stereo)
    write_wav(tmp_path / "u8.wav", np.zeros(100, np.uint8), 16000, width=1)
    write_wav(tmp_path / "s24.wav", np.zeros(300, np.uint8), 16000, width=3)
    for name, bits in (("u8.wav", "8-bit"), ("s24.wav", "24-bit")):
        with pytest.raises(ValueError, match=bits):
            audio.read_wav_pcm16(tmp_path / name)
    f = tmp_path / "f32.wav"                                   # IEEE-float WAV: format tag 3
    data = np.zeros(100, "<f4").tobytes()
    fmt = (3).to_bytes(2, "little") + (1).to_bytes(2, "little") + (16000).to_bytes(4, "little") + \
        (64000).to_bytes(4, "little") + (4).to_bytes(2, "little") + (32).to_bytes(2, "little")
    body = b"WAVE" + b"fmt " + len(fmt).to_bytes(4, "little") + fmt + b"data" + len(data).to_bytes(4, "little") + data
    f.write_bytes(b"RIFF" + len(body).to_bytes(4, "little") + body)
    with pytest.raises(ValueError, match="PCM-16"):
        audio.read_wav_pcm16(f)


def test_example_counts():
    assert audio.MIN_SAMPLES == 15600
    assert audio.num_examples(15600) == 1 and audio.num_examples(15599) == 0 and audio.num_examples(0) == 0
    assert audio.num_examples(2 * 15360 + 240) == 2 and audio.num_examples(2 * 15360 + 239) == 1
