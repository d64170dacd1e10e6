"""Host side of the VGGish audio front end: the PCM-16 WAV reader and the float64 tables the GPU front end uses (the
periodic Hann window, the HTK mel matrix, resampy's ``kaiser_best`` interpolation filter).  The tables are computed
with the numpy / scipy calls that define them, so the device receives the same float64 values the reference's
numpy pipeline uses."""
from __future__ import annotations

import wave
from typing import Tuple

import numpy as np

SAMPLE_RATE = 16000
WINDOW = 400                    # 25 ms
HOP = 160                       # 10 ms
FFT = 512
BINS = FFT // 2 + 1
MEL_BANDS = 64
MEL_LO_HZ, MEL_HI_HZ = 125.0, 7500.0
LOG_OFFSET = 0.01
EXAMPLE_FRAMES = 96             # frames per example, hop 96: a partial tail is dropped
MIN_SAMPLES = WINDOW + (EXAMPLE_FRAMES - 1) * HOP      # 15600 samples at 16 kHz: the shortest input with one example


def read_wav_pcm16(path: str) -> Tuple[np.ndarray, int]:
    """PCM-16 WAV -> (int16 samples, rate): shape (n,) for mono, (n, channels) interleaved as stored otherwise (what
    ``soundfile.read(path, dtype='int16')`` returns).  Any other sample format raises ValueError naming it."""
    try:
        with wave.open(str(path), "rb") as w:
            ch, width, rate = w.getnchannels(), w.getsampwidth(), w.getframerate()
            data = w.readframes(w.getnframes())
    except wave.Error as e:          # e.g. IEEE-float or A-law WAVs ("unknown format: 3")
        raise ValueError(f"{path}: not a PCM-16 WAV ({e}); only 16-bit PCM WAV input is read") from e
    if width != 2:
        raise ValueError(f"{path}: {8 * width}-bit PCM samples; only 16-bit PCM WAV input is read")
    x = np.frombuffer(data, dtype="<i2").astype(np.int16)
    return (x.reshape(-1, ch) if ch > 1 else x), rate


def periodic_hann() -> np.ndarray:
    """0.5 - 0.5 cos(2 pi n / 400), n < 400, float64."""
    return 0.5 - (0.5 * np.cos(2 * np.pi / WINDOW * np.arange(WINDOW)))


def hz_to_mel(f):
    """HTK mel scale: 1127 ln(1 + f / 700)."""
    return 1127.0 * np.log(1.0 + (f / 700.0))


def mel_matrix() -> np.ndarray:
    """(257, 64) float64: triangular HTK bands between 125 and 7500 Hz, equally spaced in mel, over the 257 bins of a
    512-point FFT at 16 kHz; the DC row is zero."""
    bins_mel = hz_to_mel(np.linspace(0.0, SAMPLE_RATE / 2.0, BINS))
    edges = np.linspace(hz_to_mel(MEL_LO_HZ), hz_to_mel(MEL_HI_HZ), MEL_BANDS + 2)
    m = np.empty((BINS, MEL_BANDS))
    for i in range(MEL_BANDS):
        lo, c, hi = edges[i:i + 3]
        rise = (bins_mel - lo) / (c - lo)
        fall = (hi - bins_mel) / (hi - c)
        m[:, i] = np.maximum(0.0, np.minimum(rise, fall))
    m[0, :] = 0.0
    return m


def kaiser_best() -> Tuple[np.ndarray, int]:
    """resampy 0.2.2's ``kaiser_best`` filter, regenerated: the right half of a Kaiser-windowed sinc (64 zero crossings,
    2^9 table entries per crossing, rolloff 0.9475937, Kaiser beta 14.769656), 32769 float64 entries.  Returns (table,
    entries per crossing)."""
    import scipy.signal
    num_zeros, precision = 64, 512
    rolloff, beta = 0.9475937167399596, 14.769656459379492
    n = precision * num_zeros
    sinc = rolloff * np.sinc(rolloff * np.linspace(0, num_zeros, num=n + 1, endpoint=True))
    taper = scipy.signal.windows.kaiser(2 * n + 1, beta)[n:]
    return taper * sinc, precision


def resampled_length(n: int, rate: int) -> int:
    """Samples after resampling n samples at `rate` to 16 kHz (resampy: int(n * ratio))."""
    return n if rate == SAMPLE_RATE else int(n * (float(SAMPLE_RATE) / rate))


def num_examples(n16: int) -> int:
    """Complete 96-frame examples in n16 samples at 16 kHz."""
    frames = 1 + (n16 - WINDOW) // HOP if n16 >= WINDOW else 0
    return frames // EXAMPLE_FRAMES
