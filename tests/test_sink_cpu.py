"""Output sink (utils/utils.py:50-114 semantics) and the opt-in extras of SURVEY 8(f) rank 2: the writer thread and the
resume check.  CPU only."""
import os
import pickle

import numpy as np
import pytest

from video_features_b200.utils import (AsyncSink, action_on_extraction, already_extracted, form_list_from_user_input,
                                       form_slices, sink_targets)


def _feats(key, n=4):
    return {key: np.arange(n * 3, dtype=np.float32).reshape(n, 3), 'fps': np.array(25.0), 'timestamps_ms': np.arange(n)}


def test_sink_file_names_follow_the_reference(tmp_path):
    out = str(tmp_path / "o")
    action_on_extraction(_feats('rgb'), "/v/clip_a.mp4", out, 'save_numpy')
    action_on_extraction(_feats('CLIP'), ("/v/clip_b.mp4", "/f/clip_b"), out, 'save_numpy', output_direct=True)
    action_on_extraction(_feats('flow'), "/v/clip_c.avi", out, 'save_pickle')
    assert sorted(os.listdir(out)) == ["clip_a_rgb.npy", "clip_b.npy", "clip_c_flow.pkl"]        # fps / timestamps never saved
    assert np.array_equal(np.load(os.path.join(out, "clip_a_rgb.npy")), _feats('rgb')['rgb'])
    assert np.array_equal(pickle.load(open(os.path.join(out, "clip_c_flow.pkl"), "rb")), _feats('flow')['flow'])
    with pytest.raises(NotImplementedError):
        action_on_extraction(_feats('rgb'), "/v/x.mp4", out, 'save_hdf5')
    # the reference's quirk 4: a key with '/' points into a directory that does not exist
    with pytest.raises(FileNotFoundError):
        action_on_extraction(_feats('CLIP-ViT-B/32'), "/v/x.mp4", out, 'save_numpy')


def test_print_sink_writes_nothing(tmp_path, capsys):
    action_on_extraction(_feats('rgb'), "/v/a.mp4", str(tmp_path / "o"), 'print')
    assert not (tmp_path / "o").exists()
    text = capsys.readouterr().out
    assert text.startswith("rgb\n") and "max: 11.00000000; mean: 5.50000000; min: 0.00000000" in text


def test_resume_check_and_targets(tmp_path):
    out = str(tmp_path / "o")
    assert sink_targets(['rgb', 'flow', 'fps'], "/v/a.mp4", out, 'save_numpy') == [os.path.join(out, "a_rgb.npy"),
                                                                                  os.path.join(out, "a_flow.npy")]
    assert sink_targets(['rgb'], "/v/a.mp4", out, 'print') == []
    assert not already_extracted(['rgb', 'flow'], "/v/a.mp4", out, 'save_numpy')
    action_on_extraction(_feats('rgb'), "/v/a.mp4", out, 'save_numpy')
    assert not already_extracted(['rgb', 'flow'], "/v/a.mp4", out, 'save_numpy')          # flow still missing
    action_on_extraction(_feats('flow'), "/v/a.mp4", out, 'save_numpy')
    assert already_extracted(['rgb', 'flow'], "/v/a.mp4", out, 'save_numpy')
    open(os.path.join(out, "a_flow.npy"), "w").close()                                     # truncated file = not done
    assert not already_extracted(['rgb', 'flow'], "/v/a.mp4", out, 'save_numpy')
    assert not already_extracted(['rgb'], "/v/a.mp4", out, 'print')


def test_async_sink_writes_the_same_files_and_survives_a_failed_write(tmp_path, capsys):
    out = str(tmp_path / "o")
    with AsyncSink(max_pending=2) as sink:
        for i in range(6):
            sink.submit(_feats('rgb', n=i + 1), f"/v/clip{i}.mp4", out, 'save_numpy')
        sink.submit(_feats('bad/key'), "/v/clipX.mp4", out, 'save_numpy')                  # write fails, extraction goes on
        sink.submit(_feats('flow'), "/v/clip0.mp4", out, 'save_numpy')
    assert sink.written == 7 and len(sink.errors) == 1 and sink.errors[0][0] == "/v/clipX.mp4"
    assert "Saving failed at: /v/clipX.mp4" in capsys.readouterr().out
    for i in range(6):
        assert np.load(os.path.join(out, f"clip{i}_rgb.npy")).shape == (i + 1, 3)
    assert os.path.exists(os.path.join(out, "clip0_flow.npy"))
    with pytest.raises(RuntimeError):
        sink.submit(_feats('rgb'), "/v/late.mp4", out, 'save_numpy')


def test_path_listing_and_slices(tmp_path):
    import argparse
    (tmp_path / "v").mkdir(); (tmp_path / "f").mkdir()
    for n in ("b.mp4", "a.mp4"):
        (tmp_path / "v" / n).write_bytes(b"x")
    for n in ("a", "b"):
        (tmp_path / "f" / n).mkdir()
    ns = argparse.Namespace(file_with_video_paths=None, video_dir=str(tmp_path / "v"), flow_dir=str(tmp_path / "f"),
                            video_paths=None, flow_paths=None)
    assert form_list_from_user_input(ns) == [(str(tmp_path / "v" / "a.mp4"), str(tmp_path / "f" / "a")),
                                             (str(tmp_path / "v" / "b.mp4"), str(tmp_path / "f" / "b"))]
    lst = tmp_path / "list.txt"
    lst.write_text(f"{tmp_path / 'v' / 'a.mp4'}\n\n{tmp_path / 'v' / 'b.mp4'}\n")
    ns = argparse.Namespace(file_with_video_paths=str(lst), video_dir=None, flow_dir=None, video_paths=None, flow_paths=None)
    assert form_list_from_user_input(ns) == [str(tmp_path / "v" / "a.mp4"), str(tmp_path / "v" / "b.mp4")]
    ns = argparse.Namespace(file_with_video_paths=None, video_dir=None, flow_dir=None, video_paths=[str(tmp_path / "nope.mp4")],
                            flow_paths=None)
    with pytest.raises(ValueError, match="path not exist"):
        form_list_from_user_input(ns)
    with pytest.raises(ValueError, match="no video provided"):
        form_list_from_user_input(argparse.Namespace())
    assert form_slices(65, 64, 64) == [(0, 64)] and form_slices(130, 64, 32) == [(0, 64), (32, 96), (64, 128)]


# ---- the forward loops of the three extractors, with the GPU work stubbed out (host logic only)
class _FakeIndices(list):
    """iterable of ints with a `.device` whose type is 'cuda' (the extractors take the device from the indices)."""
    class _Dev:
        type, index = 'cuda', 0
    device = _Dev()


def _ns(tmp_path, **kw):
    import argparse
    vids = []
    for n in ("a.mp4", "b.mp4", "c.mp4"):
        p = tmp_path / n
        p.write_bytes(b"x")
        vids.append(str(p))
    d = dict(feature_type='i3d', video_paths=vids, flow_paths=None, file_with_video_paths=None, video_dir=None, flow_dir=None,
             extraction_fps=None, extract_method='uni_4', on_extraction='save_numpy', output_path=str(tmp_path / "out"),
             output_direct=False, tmp_path=str(tmp_path / "tmp"), streams=['rgb'], flow_type='raft', stack_size=None,
             step_size=None, show_pred=False, keep_tmp_files=False, batch_size=1, resize_to_smaller_edge=True, side_size=None)
    d.update(kw)
    return argparse.Namespace(**d)


@pytest.mark.parametrize("mode", ["default", "async", "resume"])
def test_extractor_forward_loops_with_stubbed_engines(tmp_path, monkeypatch, capsys, mode):
    from video_features_b200.extract.extract_clip import ExtractCLIP
    from video_features_b200.extract.extract_i3d import ExtractI3D
    from video_features_b200.extract.extract_raft import ExtractRAFT
    from video_features_b200.extract.extract_s3d import ExtractS3D
    from video_features_b200.extract.extract_vggish import ExtractVGGish
    monkeypatch.delenv("VF_ASYNC_SINK", raising=False)
    monkeypatch.delenv("VF_RESUME", raising=False)
    if mode == "async":
        monkeypatch.setenv("VF_ASYNC_SINK", "1")
    calls = []

    def fake_extract(key):
        def f(self, *a, **k):
            video = a[-1] if a else k.get('video_path')
            video = k.get('video_path', video)
            calls.append((key, os.path.basename(str(video))))
            if os.path.splitext(os.path.basename(str(video)))[0] == "b":
                raise RuntimeError("decoder says no")                  # per-video catch-print-continue
            return _feats(key)
        return f

    # CLIP (output_direct, the documented way to save CLIP features)
    ex = ExtractCLIP(_ns(tmp_path, feature_type='CLIP-ViT-B/32', output_direct=True))
    ex.batch_frames = 0                                # one engine call per video: the reference's loop shape
    monkeypatch.setattr(ExtractCLIP, "_engine", lambda self, device: object())
    monkeypatch.setattr(ExtractCLIP, "extract", fake_extract('CLIP-ViT-B/32'))
    out = tmp_path / "out"
    if mode == "resume":
        out.mkdir()
        np.save(out / "a.npy", np.zeros((1, 3), np.float32))
        monkeypatch.setenv("VF_RESUME", "1")
    assert ex(_FakeIndices([0, 1, 2])) == []
    assert sorted(os.listdir(out)) == ["a.npy", "c.npy"]
    assert [c[1] for c in calls] == (["b.mp4", "c.mp4"] if mode == "resume" else ["a.mp4", "b.mp4", "c.mp4"])
    # external_call=True returns the dicts and writes nothing
    calls.clear()
    exx = ExtractCLIP(_ns(tmp_path, feature_type='CLIP-ViT-B/32'), external_call=True)
    exx.batch_frames = 0
    got = exx(_FakeIndices([0, 2]))
    assert len(got) == 2 and set(got[0]) == {'CLIP-ViT-B/32', 'fps', 'timestamps_ms'}

    # I3D: files <stem>_<stream>.npy under <output_path>/i3d
    calls.clear()
    monkeypatch.delenv("VF_RESUME", raising=False)
    ei = ExtractI3D(_ns(tmp_path))
    monkeypatch.setattr(ExtractI3D, "_load", lambda self, device: {})
    monkeypatch.setattr(ExtractI3D, "extract", fake_extract('rgb'))
    assert ei(_FakeIndices([0, 1, 2])) == []
    assert sorted(os.listdir(out / "i3d")) == ["a_rgb.npy", "c_rgb.npy"] and len(calls) == 3

    # RAFT: forward returns None, files under <output_path>/raft
    calls.clear()
    er = ExtractRAFT(_ns(tmp_path, feature_type='raft'))
    monkeypatch.setattr(ExtractRAFT, "extract", fake_extract('raft'))
    assert er(_FakeIndices([0, 1, 2])) is None
    assert sorted(os.listdir(out / "raft")) == ["a_raft.npy", "c_raft.npy"] and len(calls) == 3

    # a stack extractor (S3D): files under <output_path>/s3d, and the kept feature dicts are returned
    calls.clear()
    es = ExtractS3D(_ns(tmp_path, feature_type='s3d'))
    monkeypatch.setattr(ExtractS3D, "extract", fake_extract('s3d'))
    es.keep_features = True
    capsys.readouterr()
    got = es(_FakeIndices([0, 1, 2]))
    assert sorted(os.listdir(out / "s3d")) == ["a_s3d.npy", "c_s3d.npy"] and len(calls) == 3
    assert len(got) == 2 and set(got[0]) == {'s3d', 'fps', 'timestamps_ms'}
    b = str(tmp_path / "b.mp4")
    assert f"Extraction failed at: {b} with error (↑). Continuing extraction" in capsys.readouterr().out

    # VGGish (output_direct: <output_path>/vggish_torch/<stem>.npy, for the resume check too)
    calls.clear()
    wavs = []
    for n in ("a.wav", "b.wav", "c.wav"):
        (tmp_path / n).write_bytes(b"x")
        wavs.append(str(tmp_path / n))
    ev = ExtractVGGish(_ns(tmp_path, feature_type='vggish_torch', video_paths=wavs, output_direct=True))
    monkeypatch.setattr(ExtractVGGish, "extract", fake_extract('vggish_torch'))
    if mode == "resume":
        (out / "vggish_torch").mkdir()
        np.save(out / "vggish_torch" / "a.npy", np.zeros((1, 3), np.float32))
        monkeypatch.setenv("VF_RESUME", "1")
    assert ev(_FakeIndices([0, 1, 2])) == []
    assert sorted(os.listdir(out / "vggish_torch")) == ["a.npy", "c.npy"]
    assert [c[1] for c in calls] == (["b.wav", "c.wav"] if mode == "resume" else ["a.wav", "b.wav", "c.wav"])
    assert f"Extraction failed at: {wavs[1]}. Continuing extraction" in capsys.readouterr().out


class _FakeClipEngine:
    """Stands in for ClipEngine: feature row i = (mean of frame i, number of frames in the call, ...)."""
    def __init__(self):
        self.calls = []

    def encode_frames_u8_host(self, frames, out=None):
        import torch
        if isinstance(frames, np.ndarray):
            frames = torch.from_numpy(frames)
        n = frames.shape[0]
        self.calls.append((n, tuple(frames.shape[1:3])))
        y = torch.zeros((n, 512), dtype=torch.float32)
        y[:, 0] = frames.reshape(n, -1).float().mean(dim=1)
        y[:, 1] = n
        return y

    # the asynchronous pair the batcher uses (ClipEngine.encode_frames_u8_host_async / wait)
    def encode_frames_u8_host_async(self, frames, out_host=None, out_dev=False):
        out_host.copy_(self.encode_frames_u8_host(frames))
        self.tickets = getattr(self, "tickets", 0) + 1
        return self.tickets - 1, None

    def wait(self, ticket):
        assert 0 <= ticket < self.tickets


def test_extract_clip_batches_consecutive_videos_into_one_engine_call(tmp_path, monkeypatch, capsys):
    """ExtractCLIP.forward over a list: frames of consecutive same-geometry videos share one engine call; results are
    cut back per video; a failing decode and a geometry change behave like the reference's per-video loop."""
    import argparse
    from video_features_b200.extract.extract_clip import ExtractCLIP
    vids = []
    for i in range(7):
        p = tmp_path / f"v{i}.mp4"
        p.write_bytes(b"x")
        vids.append(str(p))
    ns = argparse.Namespace(feature_type='CLIP-ViT-B/32', video_paths=vids, flow_paths=None, file_with_video_paths=None,
                            video_dir=None, flow_dir=None, extraction_fps=None, extract_method='uni_4',
                            on_extraction='save_numpy', output_path=str(tmp_path / "out"), output_direct=True,
                            tmp_path=str(tmp_path / "tmp"))

    def source(path, method):
        i = int(os.path.basename(path)[1])
        if i == 2:
            raise RuntimeError("decoder says no")
        hw = (24, 32) if i < 5 else (16, 16)                       # geometry changes at video 5
        n = 3 + i % 2
        return [np.full(hw + (3,), 10 * i + k, np.uint8) for k in range(n)] + [None], 25.0, list(range(n))

    eng = _FakeClipEngine()
    monkeypatch.setattr(ExtractCLIP, "_engine", lambda self, device: eng)
    ex = ExtractCLIP(ns)
    ex.frame_source = source
    ex.batch_frames = 8
    assert ex(_FakeIndices(range(7))) == []
    assert "Extraction failed at: " + vids[2] in capsys.readouterr().out
    out = tmp_path / "out"
    assert sorted(os.listdir(out)) == [f"v{i}.npy" for i in (0, 1, 3, 4, 5, 6)]
    for i in (0, 1, 3, 4, 5, 6):
        f = np.load(out / f"v{i}.npy")
        assert f.shape == (3 + i % 2, 512) and np.allclose(f[:, 0], [10 * i + k for k in range(3 + i % 2)])
    # videos 0,1 (3+4 frames) share a call; 3,4 (4+3) share the next; the geometry change splits 5,6 (4+3) off
    assert eng.calls == [(7, (24, 32)), (7, (24, 32)), (7, (16, 16))]
    # external_call returns the dicts in list order
    ex2 = ExtractCLIP(ns, external_call=True)
    ex2.frame_source = source
    ex2.batch_frames = 8
    got = ex2(_FakeIndices([6, 0, 1]))
    assert [g['CLIP-ViT-B/32'].shape[0] for g in got] == [3, 3, 4] and float(got[0]['CLIP-ViT-B/32'][0, 0]) == 60.0


def test_extract_clip_first_engine_call_of_a_list_is_small(tmp_path, monkeypatch):
    """The first call holds at most `first_batch_frames` frames (the GPU starts early), the following ones `batch_frames`."""
    import argparse
    from video_features_b200.extract.extract_clip import ExtractCLIP
    vids = []
    for i in range(30):
        p = tmp_path / f"w{i:02d}.mp4"
        p.write_bytes(b"x")
        vids.append(str(p))
    ns = argparse.Namespace(feature_type='CLIP-ViT-B/32', video_paths=vids, flow_paths=None, file_with_video_paths=None,
                            video_dir=None, flow_dir=None, extraction_fps=None, extract_method='uni_4',
                            on_extraction='save_numpy', output_path=str(tmp_path / "out"), output_direct=True,
                            tmp_path=str(tmp_path / "tmp"))

    def source(path, method):
        i = int(os.path.basename(path)[1:3])
        return [np.full((8, 8, 3), i, np.uint8) for _ in range(4)], 25.0, [0, 1, 2, 3]

    eng = _FakeClipEngine()
    monkeypatch.setattr(ExtractCLIP, "_engine", lambda self, device: eng)
    ex = ExtractCLIP(ns, external_call=True)
    ex.frame_source = source
    ex.batch_frames, ex.first_batch_frames = 40, 8
    got = ex(_FakeIndices(range(30)))
    assert [c[0] for c in eng.calls] == [8, 40, 40, 32]
    assert [float(g['CLIP-ViT-B/32'][0, 0]) for g in got] == [float(i) for i in range(30)]
