"""oracle/pwc_net.py against the reference's own PWC-Net module (fixture made by scripts/make_pwc_golden.py, and live where
the reference checkout is readable), its cost volume against a literal transcription of the reference's CUDA kernel,
and the align_corners decision of the backward warp."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "pwc_outputs.npz")


def _golden():
    d = np.load(GOLDEN)
    return torch.from_numpy(d["frames"]).float(), torch.from_numpy(d["flow"])


def test_oracle_matches_reference_fixture():
    from oracle import pwc_net
    fr, flow = _golden()
    y = pwc_net.forward(pwc_net.stand_in_state_dict(), fr[:-1], fr[1:])
    assert y.shape == flow.shape == (2, 2, 72, 100)
    err = float((y - flow).abs().max())
    assert err <= 1e-5 * float(flow.abs().max()), err


def test_align_corners_true_is_the_pinned_choice():
    """The reference pins torch 1.2, whose grid_sample samples pixel (x + u, y + v) (align_corners=True); the same call
    under torch >= 1.3 lands elsewhere.  The difference is far above the comparison bars: the choice matters."""
    from oracle import pwc_net
    fr, flow = _golden()
    sd = pwc_net.stand_in_state_dict()
    y_false = pwc_net.forward(sd, fr[:-1], fr[1:], align_corners=False)
    diff = float((y_false - flow).abs().max()) / float(flow.abs().max())
    assert diff > 1e-2, diff


def test_float64_oracle_agrees_with_fp32():
    from oracle import pwc_net
    fr, flow = _golden()
    sd = {k: v.double() for k, v in pwc_net.stand_in_state_dict().items()}
    y = pwc_net.forward(sd, fr[:-1].double(), fr[1:].double(), torch.float64)
    rel = float((y - flow.double()).norm() / flow.double().norm())
    assert rel < 1e-4, rel


def _kernel_transcription(first, second):
    """kernel_Correlation_rearrange + kernel_Correlation_updateOutput (correlation.py:17-112) as float64 loops: rbot =
    NHWC copies padded by 4, one 'block' per (x, y, item), 32 'threads' summing channels ch_off, ch_off + 32, ..., thread
    0 adding the 32 partial sums and dividing by the channel count."""
    n, C, H, W = first.shape
    rbot0 = np.zeros((n, H + 8, W + 8, C))
    rbot1 = np.zeros((n, H + 8, W + 8, C))
    rbot0[:, 4:4 + H, 4:4 + W] = first.permute(0, 2, 3, 1).numpy()
    rbot1[:, 4:4 + H, 4:4 + W] = second.permute(0, 2, 3, 1).numpy()
    top = np.zeros((n, 81, H, W))
    for item in range(n):
        for by in range(H):
            for bx in range(W):
                x1, y1 = bx + 4, by + 4
                for top_channel in range(81):
                    s2o, s2p = top_channel % 9 - 4, top_channel // 9 - 4
                    sums = [0.0] * 32
                    for ch_off in range(32):
                        for ch in range(ch_off, C, 32):
                            sums[ch_off] += rbot0[item, y1, x1, ch] * rbot1[item, y1 + s2p, x1 + s2o, ch]
                    total = 0.0
                    for s in sums:
                        total += s
                    top[item, top_channel, by, bx] = total / C
    return torch.from_numpy(top)


def test_correlation_equals_kernel_transcription():
    from oracle import pwc_net
    g = torch.Generator().manual_seed(4)
    a = torch.randn(2, 40, 5, 7, generator=g, dtype=torch.float64)
    b = torch.randn(2, 40, 5, 7, generator=g, dtype=torch.float64)
    ref = _kernel_transcription(a, b)
    got = pwc_net.correlation(a, b)
    assert float((got - ref).abs().max()) < 1e-12


def test_stand_in_has_the_checkpoint_layout_and_scale():
    """Same keys and shapes as pwc_net_sintel.pt, and the trained level-6 extractor weights' tiny scale (|w| <= 1e-36 ..
    3e-14) kept: it is what the engine's per-channel weight scaling exists for."""
    import json
    from oracle import pwc_net
    sd = pwc_net.stand_in_state_dict()
    rows = json.load(open(pwc_net.STATS))
    assert [r[0] for r in rows] == list(sd) and all(list(sd[r[0]].shape) == r[1] for r in rows)
    assert len(sd) == 126 and sum(v.numel() for v in sd.values()) == 9374274
    assert float(sd["moduleExtractor.moduleSix.0.weight"].abs().max()) < 1e-34
    assert float(sd["moduleTwo.moduleOne.0.weight"].abs().max()) > 0.1


@pytest.mark.skipif(not os.path.exists(os.path.join(os.environ.get("VF_REFERENCE_DIR", "/root/reference"), "models",
                                                    "pwc", "pwc_src", "pwc_net.py")),
                    reason="the reference checkout is not readable here; the fixture test covers the same ground")
def test_oracle_matches_reference_module_live():
    sys.path.insert(0, os.path.join(ROOT, "scripts"))
    import make_pwc_golden
    from oracle import pwc_net
    fr = make_pwc_golden.golden_frames()[:, :, :64, :96]
    sd = pwc_net.stand_in_state_dict()
    ref = make_pwc_golden.reference_flow(fr, sd)
    y = pwc_net.forward(sd, fr[:-1], fr[1:])
    assert float((y - ref).abs().max()) <= 1e-5 * float(ref.abs().max())
