"""--device_ids dispatch on real GPUs: one process per GPU, NCCL group, ExtractCLIP over a shard each, ONE all-gather of
every video's (T, 512) block (reference: main.py:11-55 -- threads, no gather).  Needs >= 2 GPUs on the box
(`python -m pytest tests/test_dispatch_gpu.py -m gpu`); on a 1-GPU machine only the single-device form
(no process group) runs."""
import argparse
import functools
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _write_video(path, n, seed, h=120, w=160):
    import cv2
    vw = cv2.VideoWriter(path, cv2.VideoWriter_fourcc(*"mp4v"), 10.0, (w, h))
    assert vw.isOpened()
    base = np.random.default_rng(seed).integers(0, 256, (h, w, 3), dtype=np.uint8)
    for i in range(n):
        vw.write(np.roll(base, 5 * i, axis=1))
    vw.release()


def _ns(paths, out):
    return argparse.Namespace(feature_type='CLIP-ViT-B/32', video_paths=paths, flow_paths=None, file_with_video_paths=None,
                              video_dir=None, flow_dir=None, extraction_fps=None, extract_method='uni_4',
                              on_extraction='save_numpy', output_path=out, output_direct=True, tmp_path=os.path.join(out, 'tmp'))


def _make(ns):
    os.environ["VF_CLIP_SYNTHETIC"] = "0"
    from video_features_b200.extract.extract_clip import ExtractCLIP
    return ExtractCLIP(ns)


def _save(target, blocks):
    torch.save([b.clone() for b in blocks], target)


@pytest.mark.parametrize("n_dev", [1, 2])
def test_parallel_feature_extraction_nccl(cuda_device, tmp_path, n_dev):
    if torch.cuda.device_count() < n_dev:
        pytest.skip(f"needs {n_dev} GPUs, this box has {torch.cuda.device_count()} (run it on a machine with two GPUs)")
    from video_features_b200.dispatch import parallel_feature_extraction
    vids = []
    for i in range(7):
        v = str(tmp_path / f"d{i}.mp4")
        _write_video(v, 12 + i, seed=i)
        vids.append(v)
    out = str(tmp_path / f"out{n_dev}")
    target = str(tmp_path / f"gathered{n_dev}.pt")
    parallel_feature_extraction(functools.partial(_make, _ns(vids, out)), len(vids), list(range(n_dev)), backend="nccl",
                                gather_key='CLIP-ViT-B/32', on_gathered=functools.partial(_save, target))
    blocks = torch.load(target)
    assert [tuple(b.shape) for b in blocks] == [(4, 512)] * 7
    # the gathered blocks are the saved files, in list order, whichever rank produced them
    for i, b in enumerate(blocks):
        saved = np.load(os.path.join(out, f"d{i}.npy"))
        assert saved.shape == (4, 512) and np.array_equal(saved, b.numpy())
