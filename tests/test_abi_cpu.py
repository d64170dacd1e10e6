"""The C-ABI library loads without a GPU and exports every symbol include/vfeat.h declares."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared_symbols():
    text = open(os.path.join(ROOT, "include", "vfeat.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(vf_[a-z0-9_]+)\s*\(", text)))


def test_library_exports_every_declared_symbol():
    from video_features_b200 import _lib
    names = _declared_symbols()
    assert len(names) >= 10
    lib = ctypes.CDLL(_lib.LIB_PATH)
    for n in names:
        assert hasattr(lib, n), f"{n} declared in include/vfeat.h but not exported"
    assert set(names) == set(_lib.SIGNATURES), "ctypes signature table out of sync with include/vfeat.h"


def test_version_and_error_text():
    from video_features_b200 import _lib
    lib = _lib.lib()
    assert lib.vf_version() == 2
    b, e = ctypes.c_int64(), ctypes.c_int64()
    assert lib.vf_shard_range(10, 0, 0, ctypes.byref(b), ctypes.byref(e)) == 1
    assert b"shard_range" in lib.vf_last_error()


def test_engine_fails_loudly_without_gpu():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from oracle import clip_tower
    from video_features_b200.clip_engine import ClipEngine
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        ClipEngine(clip_tower.synthetic_state_dict(0))
