"""The GEMM epilogue's output bits stay what they were when every CTA runs several tiles and its staging buffers are
reused across tiles: every launch of tests/gemm_multitile_cases.py hashes to the SHA-256 recorded in
tests/golden/gemm_epilogue_multitile_sha256.json, which scripts/make_gemm_multitile_hashes.py wrote from the build
before the epilogue was cut to one path per launch and its store staging deepened."""
import json
import os

import pytest
import torch

import gemm_epilogue_cases as gc
import gemm_multitile_cases as mc

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "gemm_epilogue_multitile_sha256.json")


def test_gemm_multitile_outputs_are_bit_identical(cuda_device):
    from video_features_b200 import _lib
    with open(GOLDEN) as fh:
        doc = json.load(fh)
    sms = torch.cuda.get_device_properties(cuda_device).multi_processor_count
    if sms != doc["sm_count"]:
        # tile widths and the tiles each CTA runs depend on the SM count
        pytest.skip(f"hashes recorded on a {doc['sm_count']}-SM {doc['device']}; this device has {sms} SMs")
    with torch.cuda.device(cuda_device):
        got = mc.all_hashes(gc.open_lib(_lib.LIB_PATH), cuda_device)
    want = doc["sha256"]
    assert sorted(got) == sorted(want)
    bad = [k for k in want if got[k] != want[k]]
    assert not bad, f"{len(bad)} of {len(want)} launches changed bits: {bad}"
