"""Float64 / plain-torch restatement of the reference's VGGish (models/vggish_torch: vggish_input.waveform_to_examples,
mel_features, VGG with postprocess=False) -- the checker of the VGGish engine, never the thing run.

  front end: int16 -> /32768 (float64) -> mean over channels -> resampy 0.2.2 resample(kaiser_best) to 16 kHz (the
  numba loop resample_f restated: a sequential float64 time register, left wing then right wing, no FMA) -> frames of
  400, hop 160 -> periodic Hann -> |rfft 512| -> mel (257 x 64) -> log(. + 0.01) -> examples of 96 frames, hop 96,
  cast to fp32.
  VGG: 3x3 pad 1 convs 1-64, M, 64-128, M, 128-256, 256-256, M, 256-512, 512-512, M (ReLU after each conv, max-pool
  2x2/2), flatten in (H, W, C) order, 12288-4096-4096-128 with ReLU after each.

The interpolation filter, Hann window and mel matrix are video_features_b200.audio's (the log-mel's bit-for-bit match
with the reference's own examples, tests/golden/vggish_outputs.npz, holds them to the reference's)."""
from __future__ import annotations

import functools

import numpy as np
import torch
import torch.nn.functional as F

from video_features_b200 import audio

CONVS = ((0, 1, 64), (3, 64, 128), (6, 128, 256), (8, 256, 256), (11, 256, 512), (13, 512, 512))   # features.<i>
POOL_AFTER = (0, 3, 8, 13)
LINEARS = ((0, 12288, 4096), (2, 4096, 4096), (4, 4096, 128))                                    # embeddings.<i>


def mono(samples: np.ndarray) -> np.ndarray:
    """int16 (n,) or (n, ch) -> float64 mono: samples / 32768.0, then np.mean over the channels."""
    x = samples / 32768.0
    return np.mean(x, axis=1) if x.ndim > 1 else x


def time_register(n_out: int, ratio: float) -> np.ndarray:
    """resampy's time register for each output: 0, then a sequential float64 sum of 1 / ratio."""
    reg = np.zeros(n_out)
    if n_out > 1:
        reg[1:] = np.add.accumulate(np.full(n_out - 1, 1.0 / ratio))
    return reg


def resample(x: np.ndarray, sr: int, chunk: int = 4096) -> np.ndarray:
    """resampy 0.2.2 resample(x, sr, 16000, filter='kaiser_best') of a float64 mono signal, restated: each output is a
    sequential float64 sum of the left wing's products, then the right wing's (np.add.accumulate along the taps, so
    nothing is reordered or contracted)."""
    if sr == audio.SAMPLE_RATE:
        return x.copy()
    ratio = float(audio.SAMPLE_RATE) / sr
    n_out = int(x.shape[0] * ratio)
    win, num_table = audio.kaiser_best()
    if ratio < 1:
        win = win * ratio
    delta = np.zeros_like(win)
    delta[:-1] = np.diff(win)
    scale = min(1.0, ratio)
    step = int(scale * num_table)
    nwin, n_orig = win.shape[0], x.shape[0]
    reg = time_register(n_out, ratio)
    y = np.zeros(n_out)
    for t0 in range(0, n_out, chunk):
        r = reg[t0:t0 + chunk]
        n = r.astype(np.int64)
        frac = scale * (r - n)
        idx = frac * num_table
        off_l = idx.astype(np.int64)
        eta_l = idx - off_l
        frac = scale - frac
        idx = frac * num_table
        off_r = idx.astype(np.int64)
        eta_r = idx - off_r
        i_max = np.minimum(n + 1, (nwin - off_l) // step)
        k_max = np.minimum(n_orig - n - 1, (nwin - off_r) // step)
        taps_l, taps_r = int(i_max.max()), int(max(k_max.max(), 0))
        i = np.arange(taps_l)[None, :]
        k = np.arange(taps_r)[None, :]
        jl = np.minimum(off_l[:, None] + i * step, nwin - 1)
        jr = np.minimum(off_r[:, None] + k * step, nwin - 1)
        wl = win[jl] + eta_l[:, None] * delta[jl]
        wr = win[jr] + eta_r[:, None] * delta[jr]
        pl = wl * x[np.clip(n[:, None] - i, 0, n_orig - 1)]
        pr = wr * x[np.clip(n[:, None] + k + 1, 0, n_orig - 1)]
        pl[i >= i_max[:, None]] = 0.0
        pr[k >= k_max[:, None]] = 0.0
        y[t0:t0 + chunk] = np.add.accumulate(np.concatenate([pl, pr], axis=1), axis=1)[:, -1]
    return y


def log_mel(x16: np.ndarray) -> np.ndarray:
    """float64 16 kHz waveform -> (frames, 64) float64 log-mel (complete frames only)."""
    n_frames = 1 + (x16.shape[0] - audio.WINDOW) // audio.HOP if x16.shape[0] >= audio.WINDOW else 0
    frames = np.lib.stride_tricks.as_strided(x16, shape=(n_frames, audio.WINDOW),
                                             strides=(x16.strides[0] * audio.HOP, x16.strides[0]))
    spec = np.abs(np.fft.rfft(frames * audio.periodic_hann(), audio.FFT))
    return np.log(np.dot(spec, audio.mel_matrix()) + audio.LOG_OFFSET)


def examples_f64(samples: np.ndarray, sr: int) -> np.ndarray:
    """int16 samples -> (n_examples, 96, 64) float64 log-mel examples (before the fp32 cast)."""
    lm = log_mel(resample(mono(samples), sr))
    n = lm.shape[0] // audio.EXAMPLE_FRAMES
    return lm[:n * audio.EXAMPLE_FRAMES].reshape(n, audio.EXAMPLE_FRAMES, audio.MEL_BANDS)


def examples(samples: np.ndarray, sr: int) -> np.ndarray:
    """The network input: examples_f64 cast to fp32."""
    return examples_f64(samples, sr).astype(np.float32)


def forward(sd, x: torch.Tensor, taps: bool = False, rounding=None):
    """VGG forward of x (n, 96, 64) in x's dtype / device -> (n, 128); taps=True returns (features, [pool1..pool4 as
    NCHW, fc1, fc2, fc3]).  rounding: optional {tensor class: dtype} for precision emulation, the classes 'input',
    'conv_w', 'conv_act' (conv2..6 inputs), 'fc_w', 'fc_act' (fc1..3 inputs) rounded to that dtype."""
    rd = rounding or {}
    r = (lambda t, c: t.to(rd[c]).to(t.dtype) if c in rd else t)
    dt = x.dtype
    w = {k: v.to(device=x.device, dtype=dt) for k, v in sd.items()}
    h = r(x[:, None], "input")
    stages = []
    for i, _, _ in CONVS:
        h = F.relu(F.conv2d(h, r(w[f"features.{i}.weight"], "conv_w"), w[f"features.{i}.bias"], padding=1))
        if i in POOL_AFTER:
            h = F.max_pool2d(h, 2, 2)
            stages.append(h)
        if i != CONVS[-1][0]:
            h = r(h, "conv_act")
    h = h.permute(0, 2, 3, 1).reshape(h.shape[0], -1)
    for i, _, _ in LINEARS:
        h = F.relu(F.linear(r(h, "fc_act"), r(w[f"embeddings.{i}.weight"], "fc_w"), w[f"embeddings.{i}.bias"]))
        stages.append(h)
    return (h, stages) if taps else h


def synthetic_audio(seconds: float, sr: int, channels: int = 1, seed: int = 0) -> np.ndarray:
    """Seeded int16 test audio, (n,) or (n, channels): a chirp, a harmonic tone, amplitude-modulated noise, a stretch of
    digital silence (log-mel exactly log 0.01) and a clipped burst at +32767 / -32768, in turn."""
    g = np.random.default_rng(seed)
    n = int(round(seconds * sr))
    t = np.arange(n) / sr
    out = np.zeros((n, channels))
    for c in range(channels):
        f0 = 150.0 * (1 + c) + 50 * g.random()
        chirp = np.sin(2 * np.pi * (f0 * t + 0.5 * (3000.0 / max(seconds, 1e-3)) * t * t))
        tone = sum(np.sin(2 * np.pi * f0 * 2 * k * t + g.random() * 6) / k for k in range(1, 6)) / 2.3
        am = (0.5 + 0.5 * np.sin(2 * np.pi * 3.0 * t)) * g.standard_normal(n) * 0.5
        parts = [chirp, tone, am]
        y = np.zeros(n)
        edges = np.linspace(0, n, 6).astype(int)
        for j in range(5):
            a, b = edges[j], edges[j + 1]
            if j < 3:
                y[a:b] = parts[j][a:b] * 0.6
            elif j == 3:
                y[a:b] = 0.0                                    # digital silence
            else:
                y[a:b] = parts[0][a:b] * 1.6                    # clipped burst
        out[:, c] = y
    q = np.clip(np.round(out * 32768.0), -32768, 32767).astype(np.int16)
    return q[:, 0].copy() if channels == 1 else q


@functools.lru_cache(maxsize=None)
def _stand_in(seed: int):
    g = torch.Generator().manual_seed(3000 + seed)
    x = torch.from_numpy(calibration_examples(seed)).double()
    sd = {}
    h = x[:, None]
    for i, ci, co in CONVS:
        wgt = torch.randn(co, ci, 3, 3, generator=g, dtype=torch.float64)
        pre = F.conv2d(h, wgt, padding=1)
        s = 1.0 / pre.std().item()
        med = pre.transpose(0, 1).reshape(co, -1).median(dim=1).values
        sd[f"features.{i}.weight"] = (wgt * s).float()
        sd[f"features.{i}.bias"] = (-med * s).float()
        h = F.relu(F.conv2d(h, sd[f"features.{i}.weight"].double(), sd[f"features.{i}.bias"].double(), padding=1))
        if i in POOL_AFTER:
            h = F.max_pool2d(h, 2, 2)
    h = h.permute(0, 2, 3, 1).reshape(h.shape[0], -1)
    for i, ci, co in LINEARS:
        wgt = torch.randn(co, ci, generator=g, dtype=torch.float64)
        pre = h @ wgt.t()
        s = 1.0 / pre.std().item()
        med = pre.median(dim=0).values
        sd[f"embeddings.{i}.weight"] = (wgt * s).float()
        sd[f"embeddings.{i}.bias"] = (-med * s).float()
        h = F.relu(F.linear(h, sd[f"embeddings.{i}.weight"].double(), sd[f"embeddings.{i}.bias"].double()))
    return sd


def calibration_examples(seed: int = 0) -> np.ndarray:
    """(17, 96, 64) fp32 log-mel examples of seeded 16 kHz calibration audio (mono and a stereo mix)."""
    a = examples(synthetic_audio(9.0, 16000, 1, seed=100 + seed), 16000)
    b = examples(synthetic_audio(8.0, 16000, 2, seed=200 + seed), 16000)
    return np.concatenate([a, b])


def stand_in_state_dict(seed: int = 0):
    """Calibrated seeded stand-in for torchvggish's vggish-10086976.pth (no trained weights exist offline; VGGish has no
    BatchNorm to calibrate): each layer's weights ~ N(0, 1) (seeded), scaled so that its pre-activations over the
    calibration examples have unit standard deviation, and its bias set to minus each output channel's median
    pre-activation, so that about half of every channel is positive after the ReLU.  Keys and shapes of the reference's
    VGG state_dict (features.{0,3,6,8,11,13}, embeddings.{0,2,4}).  Returns a fresh copy."""
    return {k: v.clone() for k, v in _stand_in(seed).items()}
