"""ExtractPWC and ExtractI3D's default ``--flow_type pwc`` (reference-facing classes) on synthetic videos with seeded
stand-in weights, against the oracle run on the same decoded frames."""
import argparse
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "scripts", "precision"))
from helpers import checkpoint, checkpoint_dir  # noqa: E402  (seeded stand-ins of the reference checkpoints)


def _pwc_checkpoint() -> str:
    """The PWC-Net stand-in, saved beside the others under the reference's file name."""
    from oracle import pwc_net
    path = os.path.join(checkpoint_dir(), pwc_net.CHECKPOINT)
    if not os.path.exists(path):
        torch.save(pwc_net.stand_in_state_dict(), path)
    return path


@pytest.fixture(autouse=True)
def _reference_weights(monkeypatch):
    """The extractors look their weights up in $VF_CKPT_DIR / ./checkpoints: point them at the stand-in files."""
    from video_features_b200.extract import extract_i3d
    _pwc_checkpoint()
    monkeypatch.setattr(extract_i3d, "_CKPT_DIRS", [checkpoint_dir()])
    monkeypatch.setattr(extract_i3d, "_STATE_DICTS", {})


def _write_video(path, n, h=120, w=160, fps=25.0, shift=(0.8, 0.5)):
    import cv2
    from oracle import raft_net
    fr = raft_net.synthetic_frames(n, h, w, seed=11, shift=shift).permute(0, 2, 3, 1).numpy().astype(np.uint8)
    vw = cv2.VideoWriter(path, cv2.VideoWriter_fourcc(*"mp4v"), fps, (w, h))
    assert vw.isOpened()
    for f in fr:
        vw.write(f)
    vw.release()


def _ns(**kw):
    d = dict(feature_type='pwc', video_paths=None, flow_paths=None, file_with_video_paths=None, video_dir=None,
             flow_dir=None, extraction_fps=None, extract_method=None, on_extraction='save_numpy', output_path='./output',
             output_direct=False, tmp_path='./tmp', streams=None, flow_type='pwc', stack_size=None, step_size=None,
             show_pred=False, keep_tmp_files=False, batch_size=1, resize_to_smaller_edge=True, side_size=None)
    d.update(kw)
    return argparse.Namespace(**d)


def _decoded_rgb(path):
    import cv2
    cap = cv2.VideoCapture(path)
    fr = []
    while True:
        ok, f = cap.read()
        if not ok:
            break
        fr.append(cv2.cvtColor(f, cv2.COLOR_BGR2RGB))
    return np.stack(fr)


def test_extract_pwc_writes_flow_and_skips_a_broken_file(cuda_device, tmp_path):
    from oracle import pwc_net
    from video_features_b200.extract.extract_pwc import ExtractPWC
    vid, bad = str(tmp_path / "clip2.mp4"), str(tmp_path / "broken.mp4")
    _write_video(vid, 6, h=128, w=160)
    with open(bad, "wb") as f:
        f.write(b"not a video")
    out = str(tmp_path / "out")
    ex = ExtractPWC(_ns(video_paths=[bad, vid], output_path=out, tmp_path=str(tmp_path / "tmp"), batch_size=2))
    assert ex.output_path == os.path.join(out, "pwc")
    assert ex(torch.arange(2, device=cuda_device)) is None
    flow = np.load(os.path.join(out, "pwc", "clip2_pwc.npy"))
    assert flow.shape == (5, 2, 128, 160) and flow.dtype == np.float64
    # the reference feeds RGB (extract_pwc.py:129); the model swaps channels itself
    x = torch.from_numpy(_decoded_rgb(vid)).permute(0, 3, 1, 2).double().to(cuda_device)
    sd = {k: v.to(cuda_device, torch.float64) for k, v in pwc_net.stand_in_state_dict().items()}
    ref = pwc_net.forward(sd, x[:-1], x[1:], torch.float64).cpu().numpy()
    rel = np.linalg.norm(flow - ref) / np.linalg.norm(ref)
    mx = np.abs(flow - ref).max() / np.abs(ref).max()
    print(f"ExtractPWC vs float64 oracle: rel-L2 {rel:.2e}, max-abs / max {mx:.2e}")
    assert rel <= 1e-3 and mx <= 1e-3


def test_extract_pwc_side_size(cuda_device, tmp_path):
    from video_features_b200.extract.extract_pwc import ExtractPWC
    vid = str(tmp_path / "clip3.mp4")
    _write_video(vid, 4, h=120, w=160)
    out = str(tmp_path / "out")
    ex = ExtractPWC(_ns(video_paths=[vid], output_path=out, tmp_path=str(tmp_path / "tmp"), side_size=96))
    res = ex.extract(cuda_device, None, vid)
    assert res['pwc'].shape == (3, 2, 96, 128) and res['pwc'].dtype == np.float64
    assert res['timestamps_ms'].shape == (4,)


@pytest.mark.parametrize("clip,shift", [("low_motion", (0.8, 0.5)), ("high_motion", (4.5, -3.0))])
def test_extract_i3d_default_flow_type_pwc_vs_oracle(cuda_device, tmp_path, clip, shift):
    """ExtractI3D with the CLI's default flow type: PWC on the stack's resized BGR frames, then the flow stream.  The
    composite bar is derived as test_extract_i3d_two_streams_vs_oracle derives it for RAFT: the flow stream's 8-bit
    quantiser is a staircase, so the features may differ by up to twice the oracle's own sensitivity to flow noise of
    the engine's measured flow error."""
    from PIL import Image
    from flow_quantiser_sensitivity import feature_sensitivity            # scripts/precision/
    from oracle import i3d_net, pwc_net
    from video_features_b200 import utils
    from video_features_b200.extract.extract_i3d import ExtractI3D
    from video_features_b200.pwc_engine import PWCEngine
    for n in ("i3d_rgb.pt", "i3d_flow.pt"):
        checkpoint(n)
    vid = str(tmp_path / "clip.mp4")
    _write_video(vid, 20, shift=shift)
    ex = ExtractI3D(_ns(feature_type='i3d', video_paths=[vid], output_path=str(tmp_path / "out"),
                        tmp_path=str(tmp_path / "tmp"), stack_size=12, step_size=12), external_call=True)
    assert ex.flow_type == 'pwc'
    res = ex(torch.zeros([1], dtype=torch.long, device=cuda_device))[0]
    assert res['rgb'].shape == (5, 1024) and res['flow'].shape == (5, 1024) and res['flow'].dtype == np.float64
    rd = utils.VideoReader(vid)
    ix = np.linspace(1, rd.frame_cnt - 1, 65).astype(int)[:13]
    frames = [rd.get_frame(int(i)) for i in ix]                            # BGR, as the reference keeps them
    rs = torch.stack([torch.from_numpy(np.asarray(Image.fromarray(f).resize((341, 256), Image.BILINEAR)).copy())
                      for f in frames]).permute(0, 3, 1, 2).float().to(cuda_device)
    sd_pwc_cpu = torch.load(_pwc_checkpoint())
    sd_pwc = {k: v.to(cuda_device, torch.float64) for k, v in sd_pwc_cpu.items()}
    flow = pwc_net.forward(sd_pwc, rs[:-1].double(), rs[1:].double(), torch.float64).float()   # (12, 2, 256, 341)
    eng = PWCEngine(sd_pwc_cpu, 0, max_frames=13, max_h=256, max_w=341)
    eflow = eng.flow(rs.permute(0, 2, 3, 1).contiguous().to(torch.uint8))
    eng.close()
    d = eflow.double() - flow.double()
    flow_rel, flow_rms = float(d.norm() / flow.double().norm()), float(d.pow(2).mean().sqrt())
    flow_max = float(d.abs().max()) / float(flow.abs().max())
    assert flow_rel <= 1e-3 and flow_max <= 1e-3, (flow_rel, flow_max)
    sd_flow = {k: v.to(cuda_device) for k, v in torch.load(checkpoint("i3d_flow.pt")).items()}
    ref_flow = i3d_net.forward_features(sd_flow, i3d_net.flow_transform(flow))
    rel = float((torch.from_numpy(res['flow'][:1]).to(cuda_device) - ref_flow).norm() / ref_flow.norm())
    sens = feature_sensitivity(sd_flow, flow, [flow_rms], draws=5)[flow_rms]["feature_rel"]
    bar = max(1e-3, 2.0 * sens)
    print(f"[{clip}] ExtractI3D flow (PWC -> quantiser -> I3D) vs oracle: {rel:.3e}; engine flow error {flow_rel:.2e} rel "
          f"(max {flow_max:.2e}) / {flow_rms:.2e} px rms; oracle's own sensitivity at that rms: {sens:.3e}; bar {bar:.3e}")
    assert rel <= bar, (rel, bar)
    sd_rgb = {k: v.to(cuda_device) for k, v in torch.load(checkpoint("i3d_rgb.pt")).items()}
    ref_rgb = i3d_net.forward_features(sd_rgb, i3d_net.rgb_transform(rs[:-1]))
    rel = float((torch.from_numpy(res['rgb'][:1]).to(cuda_device) - ref_rgb).norm() / ref_rgb.norm())
    assert rel < 1e-3


def test_main_i3d_with_default_flow_type_writes_both_streams(cuda_device, tmp_path):
    import main
    for n in ("i3d_rgb.pt", "i3d_flow.pt"):
        checkpoint(n)
    vid = os.path.join(ROOT, "tests", "golden", "v_GGSY1Qvo990.mp4")
    out = str(tmp_path / "out")
    args = main.make_parser().parse_args(["--feature_type", "i3d", "--video_paths", vid, "--on_extraction", "save_numpy",
                                          "--output_path", out, "--tmp_path", str(tmp_path / "tmp")])
    assert args.flow_type == "pwc" and args.streams is None
    ex = main.build_extractor(args)
    ex(torch.zeros([1], dtype=torch.long, device=cuda_device))
    rgb = np.load(os.path.join(out, "i3d", "v_GGSY1Qvo990_rgb.npy"))
    flow = np.load(os.path.join(out, "i3d", "v_GGSY1Qvo990_flow.npy"))
    assert rgb.ndim == 2 and rgb.shape[1] == 1024 and rgb.shape[0] >= 1
    assert flow.shape == rgb.shape and np.isfinite(flow).all() and np.abs(flow).max() > 0
