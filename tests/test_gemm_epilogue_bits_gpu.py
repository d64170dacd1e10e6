"""The GEMM epilogue's output bits stay what they were: every launch of tests/gemm_epilogue_cases.py (all activations on
fp16 / fp32 / split / reduce-add outputs, with and without scale / bias, every tile width, and two masked conv-mode
launches) hashes to the SHA-256 recorded in tests/golden/gemm_epilogue_sha256.json, which
scripts/make_gemm_epilogue_hashes.py wrote from the build before the epilogue was specialised per activation."""
import json
import os

import pytest
import torch

import gemm_epilogue_cases as gc

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "gemm_epilogue_sha256.json")


def test_gemm_epilogue_outputs_are_bit_identical(cuda_device):
    from video_features_b200 import _lib
    with open(GOLDEN) as fh:
        doc = json.load(fh)
    sms = torch.cuda.get_device_properties(cuda_device).multi_processor_count
    if sms != doc["sm_count"]:
        # the tile width of a launch depends on the SM count, and the cases are named for the widths on the device
        # the hashes were recorded on
        pytest.skip(f"hashes recorded on a {doc['sm_count']}-SM {doc['device']}; this device has {sms} SMs")
    with torch.cuda.device(cuda_device):
        got = gc.all_hashes(gc.open_lib(_lib.LIB_PATH), cuda_device)
    want = doc["sha256"]
    assert sorted(got) == sorted(want)
    bad = [k for k in want if got[k] != want[k]]
    assert not bad, f"{len(bad)} of {len(want)} launches changed bits: {bad}"
