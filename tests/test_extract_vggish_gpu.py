"""ExtractVGGish and main.py end to end on synthetic WAVs with the stand-in weights (VF_CKPT_DIR)."""
import os
import wave

import numpy as np
import pytest
import torch

import main
from oracle import vggish_net

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "vggish_outputs.npz")


def write_wav(path, samples: np.ndarray, rate: int):
    ch = 1 if samples.ndim == 1 else samples.shape[1]
    with wave.open(str(path), "wb") as w:
        w.setnchannels(ch)
        w.setsampwidth(2)
        w.setframerate(rate)
        w.writeframes(np.ascontiguousarray(samples, dtype="<i2").tobytes())


@pytest.fixture(scope="module")
def ckpt_dir(tmp_path_factory):
    d = tmp_path_factory.mktemp("vggish_ckpt")
    torch.save(vggish_net.stand_in_state_dict(), str(d / "vggish-10086976.pth"))
    return str(d)


def _run(paths, out, monkeypatch, ckpt_dir, *extra):
    monkeypatch.setenv("VF_CKPT_DIR", ckpt_dir)
    args = main.make_parser().parse_args(["--feature_type", "vggish_torch", "--on_extraction", "save_numpy",
                                          "--output_path", str(out), "--video_paths", *map(str, paths), *extra])
    ex = main.build_extractor(args)
    ex(torch.arange(len(paths), device="cuda"))
    return ex


def test_saves_golden_features_and_skips_bad_files(tmp_path, monkeypatch, capsys, ckpt_dir):
    g = np.load(GOLDEN)
    good = tmp_path / "clip.wav"
    write_wav(good, g["samples"], int(g["sample_rate"]))
    short = tmp_path / "short.wav"
    write_wav(short, vggish_net.synthetic_audio(0.5, 16000, 1), 16000)
    corrupt = tmp_path / "corrupt.wav"
    corrupt.write_bytes(b"RIFF\x10\x00\x00\x00WAVEjunk")
    stereo = tmp_path / "stereo.wav"
    xs = vggish_net.synthetic_audio(2.5, 44100, 2, seed=9)
    write_wav(stereo, xs, 44100)
    out = tmp_path / "out"
    _run([short, corrupt, good, stereo], out, monkeypatch, ckpt_dir)
    text = capsys.readouterr().out
    assert f"Extraction failed at: {short}" in text and f"Extraction failed at: {corrupt}" in text
    d = out / "vggish_torch"
    assert sorted(os.listdir(d)) == ["clip_vggish_torch.npy", "stereo_vggish_torch.npy"]
    f = np.load(d / "clip_vggish_torch.npy")
    assert f.dtype == np.float32 and f.shape == g["vggish_torch"].shape
    ref = g["vggish_torch"].astype(np.float64)
    assert (np.linalg.norm(f - ref, axis=1) / np.linalg.norm(ref, axis=1)).max() <= 1e-3
    assert (np.abs(f - ref).max(axis=1) / np.abs(ref).max(axis=1)).max() <= 1e-3
    fs = np.load(d / "stereo_vggish_torch.npy")
    with torch.no_grad():
        rs = vggish_net.forward(vggish_net.stand_in_state_dict(), torch.from_numpy(vggish_net.examples(xs, 44100))).numpy()
    assert fs.shape == rs.shape == (2, 128)
    assert (np.linalg.norm(fs - rs, axis=1) / np.linalg.norm(rs, axis=1)).max() <= 1e-3


def test_resume_skips_finished_files(tmp_path, monkeypatch, capsys, ckpt_dir):
    a, b = tmp_path / "a.wav", tmp_path / "b.wav"
    write_wav(a, vggish_net.synthetic_audio(1.5, 16000, 1, seed=1), 16000)
    write_wav(b, vggish_net.synthetic_audio(1.5, 22050, 2, seed=2), 22050)
    out = tmp_path / "out"
    _run([a], out, monkeypatch, ckpt_dir)
    target = out / "vggish_torch" / "a_vggish_torch.npy"
    target.write_bytes(target.read_bytes())           # unchanged content, new mtime
    before = target.stat().st_mtime_ns
    monkeypatch.setenv("VF_RESUME", "1")
    _run([a, b], out, monkeypatch, ckpt_dir)
    assert target.stat().st_mtime_ns == before
    assert (out / "vggish_torch" / "b_vggish_torch.npy").exists()
