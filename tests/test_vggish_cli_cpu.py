"""main.py's vggish_torch: ExtractVGGish for .wav lists; .mp4 and the TF1 vggish type refused."""
import wave

import pytest

import main


def _wav(path):
    with wave.open(str(path), "wb") as w:
        w.setnchannels(1)
        w.setsampwidth(2)
        w.setframerate(16000)
        w.writeframes(b"\x00\x00" * 16)
    return str(path)


def test_wav_list_builds_extract_vggish(tmp_path):
    from video_features_b200.extract.extract_vggish import ExtractVGGish
    paths = [_wav(tmp_path / "a.wav"), _wav(tmp_path / "b.wav")]
    args = main.make_parser().parse_args(["--feature_type", "vggish_torch", "--video_paths", *paths,
                                          "--output_direct"])
    ex = main.build_extractor(args)
    assert isinstance(ex, ExtractVGGish)
    assert ex.feature_type == "vggish_torch" and ex.path_list == paths and ex.output_direct is True
    assert ex.output_path.endswith("vggish_torch") and ex.tmp_path.endswith("vggish_torch")
    assert ex.on_extraction == "print" and ex.keep_tmp_files is False
    assert "vggish_torch" in main.SUPPORTED and "vggish" not in main.SUPPORTED


def test_mp4_and_tf_vggish_refused(tmp_path):
    mp4 = tmp_path / "v.mp4"
    mp4.write_bytes(b"")
    args = main.make_parser().parse_args(["--feature_type", "vggish_torch", "--video_paths", _wav(tmp_path / "a.wav"),
                                          str(mp4)])
    with pytest.raises(NotImplementedError, match="ffmpeg"):
        main.build_extractor(args)
    args = main.make_parser().parse_args(["--feature_type", "vggish", "--video_paths", _wav(tmp_path / "a.wav")])
    with pytest.raises(NotImplementedError, match="PCA"):
        main.build_extractor(args)
