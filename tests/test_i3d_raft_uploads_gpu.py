"""Every conv the I3D and RAFT engines uploaded, read back (vf_i3d_conv / vf_raft_conv), against the layouts restated in
tests/conv_layout.py on the same weights, bit for bit: W_hi | W_lo (or W_hi alone for a single-fp16 conv), the padded
rows, lo_mask, the tap shifts and the fp32 scale / bias of the epilogue.

The float64 stage tests (test_i3d_raft_float64_gpu.py) see a lost lo class only where it costs more than the engine's
own noise; a single wrong lo_mask bit, gmap_lo column, lo-at-384 column of convc1, flow8 column or duplicated unmerged tap
costs less than that at most stages.  Here each of them changes a compared bit."""
import pytest
import torch

import conv_layout as cl
from oracle import i3d_net

pytestmark = pytest.mark.gpu


def _same(what, got, f):
    assert (got["n_out"], got["ntaps"], got["k_per_tap"], got["nsplit"]) == (
        f["n_out"], f["ntaps"], f["k_per_tap"], f["nsplit"]), what
    assert got["shifts"] == f["shifts"], what
    assert got["lo_mask"] == f["lo_mask"], (what, hex(got["lo_mask"]), hex(f["lo_mask"]))
    w = got["w"].cpu()
    assert torch.equal(w, f["Wt"]), (what, int((w != f["Wt"]).sum()))
    assert torch.equal(got["scale"].cpu(), f["scale"]), what
    assert torch.equal(got["bias"].cpu(), f["bias"]), what


def _vf_error():
    from video_features_b200._lib import VfError
    return VfError


@pytest.mark.parametrize("modality,single", [("rgb", "default"), ("flow", "default"), ("rgb", "none")])
def test_i3d_uploads_match_the_restated_filters(cuda_device, monkeypatch, modality, single):
    """All 57 units; VF_I3D_SINGLE=none uploads every unit split."""
    from helpers import checkpoint
    from video_features_b200.i3d_engine import I3DEngine
    sd = torch.load(checkpoint(f"i3d_{modality}.pt"), map_location="cpu")
    if single == "none":
        monkeypatch.setenv("VF_I3D_SINGLE", "none")
    eng = I3DEngine(sd, modality, 0, max_stacks=1, max_T=16)
    names = i3d_net.unit_names()
    want = cl.i3d_engine_filters(sd, names, single=() if single == "none" else cl.I3D_SINGLE_UNITS)
    for i, (n, f) in enumerate(zip(names, want)):
        _same(f"{i} {n}", eng.conv(i), f)
    assert sum(f["nsplit"] == 1 for f in want) == (0 if single == "none" else 5)
    with pytest.raises(_vf_error(), match="outside"):
        eng.conv(len(names))
    eng.close()


def test_raft_uploads_match_the_restated_filters(cuda_device):
    """Both encoders (stride-2 phase inversion, the down convs, pair rows) and the update block (convc1's lo half at
    column 384, convf1's flow8 columns, z|r stacked over gmap / gmap_lo, the duplicated unmerged taps of the flow and
    mask heads, the rows padded 2 -> 8 and 126 -> 128, mask.2's x 0.25, the single-fp16 mask head)."""
    from helpers import stand_in_state_dict
    from video_features_b200.raft_engine import RAFTEngine
    sd = stand_in_state_dict("raft-sintel.pth")
    eng = RAFTEngine(sd, 0, max_frames=2, max_h=128, max_w=128)
    want = cl.raft_engine_filters(sd)
    assert len(want) == 45
    for i, (n, f) in enumerate(want):
        _same(f"{i} {n}", eng.conv(i), f)
    with pytest.raises(_vf_error(), match="outside"):
        eng.conv(len(want))
    eng.close()
