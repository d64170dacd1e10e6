"""The IG65M R(2+1)D-34 network on R21DEngine (vf_r21d_create2, BatchNorm eps 1e-3) with the calibrated stand-in
(tests/r21d_34_ref.py stand_in_state_dict_34): against the fp32 oracle and float64 at every stage, at T = 32, 8 and 7
(8 and 7 reach one frame at layer4) across a chunk boundary; every uploaded conv read back, the unequal conv1 / conv2
mid widths and the eps-1e-3 folding included; ExtractR21D, `main.py --model_name` and `--show_pred` on the sample
video against the oracle on the same decoded frames."""
import argparse
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import conv_layout as cl
import r21d_34_bars as b34
import r21d_34_ref as ref34
import split_engine_bars as bars
from oracle import class_heads, r21d_net

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
VIDEO = os.path.join(ROOT, "tests", "golden", "v_GGSY1Qvo990.mp4")
M32, M8 = "r2plus1d_34_32_ig65m_ft_kinetics", "r2plus1d_34_8_ig65m_ft_kinetics"
# (T, clips): a workspace of max_clips 1 x max_T 32 holds 34 frame slots, so every case runs as two chunks
CASES = [(32, 2), (8, 4), (7, 4)]


def _engine(sd, **kw):
    from video_features_b200.r21d_engine import R21DEngine
    return R21DEngine(sd, 0, **dict(dict(max_clips=1, max_T=32, bn_eps=ref34.EPS_34), **kw))


def _cast(sd, dev, dtype=None):
    return {k: (v.to(dtype) if dtype is not None and v.is_floating_point() else v).to(dev) for k, v in sd.items()}


@pytest.fixture(scope="module")
def sd34():
    return ref34.stand_in_state_dict_34()


@pytest.mark.parametrize("T,n", CASES)
def test_engine_vs_fp32_oracle(cuda_device, sd34, T, n):
    eng = _engine(sd34)
    per_chunk = 34 // (T + 2)
    x = r21d_net.calibration_clips(seed=T, n=n, T=T).to(cuda_device)
    y = eng.forward_f32(x)
    with torch.no_grad():
        ref, taps = ref34.forward(_cast(sd34, cuda_device), x, taps=True)
    rel, mx = bars.row_errors(y, ref)
    print(f"r21d-34 T={T} n={n}: features worst row rel-L2 {rel:.2e}, max-abs/max {mx:.2e}")
    m = n - (n - 1) // per_chunk * per_chunk                 # read_stage holds the last chunk
    errs = {}
    for sid, name in enumerate(r21d_net.STAGES):
        got, want = eng.read_stage(sid), taps[name][n - m:]
        assert got.shape == want.shape, (name, got.shape, want.shape)
        errs[name] = float((got.double() - want.double()).norm() / want.double().norm())
        print(f"  {name}: rel-L2 {errs[name]:.2e}")
    eng.close()
    assert rel <= 1e-3 and mx <= 1e-3, (rel, mx)
    assert all(errs[s] <= b34.STAGE_BAR_FP32[s] for s in errs), errs


def _stages(eng, y, ref, taps, rows):
    errs = {"features": bars.row_errors(y, ref)}
    for sid, s in enumerate(b34.R21D_34_STAGES[:-1]):
        errs[s] = bars.row_errors(eng.read_stage(sid), taps[s][rows])
    return errs


def _report(what, errs):
    for s, e in errs.items():
        bar = b34.R21D_34_BARS[s]
        print(f"{what} {s}: rel-L2 {e[0]:.2e}, max-abs/max {e[1]:.2e} (bar {bar[0]:.1e} / {bar[1]:.1e})")


@pytest.mark.parametrize("T,n", CASES)
def test_engine_vs_float64(cuda_device, sd34, T, n):
    eng = _engine(sd34)
    per_chunk = 34 // (T + 2)
    x = r21d_net.calibration_clips(seed=7, n=n, T=T).to(cuda_device)
    y = eng.forward_f32(x)
    with torch.no_grad():
        ref, taps = ref34.forward(_cast(sd34, cuda_device, torch.float64), x.double(), taps=True)
    errs = _stages(eng, y, ref, taps, slice(n - (n - 1) % per_chunk - 1, n))
    eng.close()
    _report(f"r21d-34-T{T}", errs)
    assert all(bars.within(e, b34.R21D_34_BARS[s]) for s, e in errs.items()), errs


def test_dropped_lo_half_is_caught(cuda_device, sd34):
    """Weights pre-rounded to fp16 (every W_lo zero), then the input pre-rounded to fp16 (the stem input's lo half
    zero): against float64 of the original operands each fails the stem's bar tenfold and the features' bar; against
    float64 of the rounded operands every stage passes."""
    x = r21d_net.calibration_clips(seed=8, n=2, T=8).to(cuda_device)
    sd16 = {k: (v.half().float() if v.is_floating_point() and v.dim() >= 4 else v) for k, v in sd34.items()}

    def f64(s, xx):
        with torch.no_grad():
            return ref34.forward(_cast(s, cuda_device, torch.float64), xx.double(), taps=True)
    for what, s_eng, x_eng in (("fp16-weights", sd16, x), ("fp16-input", sd34, x.half().float())):
        eng = _engine(s_eng, max_clips=2, max_T=8)
        y = eng.forward_f32(x_eng)
        lost = _stages(eng, y, *f64(sd34, x), slice(0, 2))
        kept = _stages(eng, y, *f64(s_eng, x_eng), slice(0, 2))
        eng.close()
        _report(f"r21d-34 {what} vs original", lost)
        _report(f"r21d-34 {what} vs rounded", kept)
        assert bars.beyond(lost["stem"], b34.R21D_34_BARS["stem"], 10), (what, lost["stem"])
        assert bars.beyond(lost["features"], b34.R21D_34_BARS["features"]), (what, lost["features"])
        assert all(bars.within(e, b34.R21D_34_BARS[s]) for s, e in kept.items()), (what, kept)


def _kinds_34():
    """(conv key, BatchNorm key, conv_layout kind) in vf_r21d_conv's order at depth 34."""
    out = [("stem.0", "stem.1", "stem"), ("stem.3", "stem.4", "temporal")]
    for L, nb in enumerate(ref34.LAYERS_34):
        for b in range(nb):
            p, s2 = f"layer{L + 1}.{b}", b == 0 and L > 0
            out += [(p + ".conv1.0.0", p + ".conv1.0.1", "stride2" if s2 else "same"),
                    (p + ".conv1.0.3", p + ".conv1.1", "temporal2" if s2 else "temporal"),
                    (p + ".conv2.0.0", p + ".conv2.0.1", "same"), (p + ".conv2.0.3", p + ".conv2.1", "temporal")]
            if s2:
                out.append((p + ".downsample.0", p + ".downsample.1", "point"))
    return out


def test_uploads_match_the_restated_filters(cuda_device, sd34):
    """Every conv as uploaded (vf_r21d_conv) equals conv_layout.engine_filter on the same weights bit for bit, with
    BatchNorm folded at eps 1e-3; layer2..4's first blocks read conv1 and conv2 at different mid widths."""
    from video_features_b200._lib import VfError
    eng = _engine(sd34, max_clips=1, max_T=1)
    vol = cl.Vol(1, 1, 1, 1, 0, 1, 0, 1, 0, 1)
    kinds = _kinds_34()
    assert len(kinds) == 2 + 4 * 16 + 3
    widths = {}
    for i, (conv, bn, kind) in enumerate(kinds):
        got = eng.conv(i)
        w = sd34[conv + ".weight"].double()
        co, ci = w.shape[:2]
        f = cl.engine_filter(kind, w, vol, ci_p=cl.pad8(ci), n_out=cl.pad8(co))
        what = f"{i} {conv} ({kind})"
        assert (got["n_out"], got["ntaps"], got["k_per_tap"]) == (cl.pad8(co), f["ntaps"], f["k_per_tap"]), what
        assert got["shifts"] == f["shifts"] and got["lo_mask"] == f["lo_mask"], what
        assert torch.equal(got["w"].cpu(), f["Wt"]), what
        s = sd34[bn + ".weight"].double() / torch.sqrt(sd34[bn + ".running_var"].double() + 1e-3)
        sh = sd34[bn + ".bias"].double() - sd34[bn + ".running_mean"].double() * s
        zeros = torch.zeros(cl.pad8(co) - co, dtype=torch.float32)
        assert torch.equal(got["scale"].cpu(), torch.cat([s.float(), zeros])), what
        assert torch.equal(got["bias"].cpu(), torch.cat([sh.float(), zeros])), what
        widths[conv] = got["n_out"]
    assert [(widths[f"layer{L}.0.conv1.0.0"], widths[f"layer{L}.0.conv2.0.0"]) for L in (2, 3, 4)] == \
        [(232, 288), (464, 576), (928, 1152)]
    with pytest.raises(VfError, match="outside"):
        eng.conv(len(kinds))
    eng.close()


def test_structure_errors(cuda_device, sd34):
    from video_features_b200._lib import VfError
    bad = dict(sd34)
    bad["layer3.0.conv2.0.0.weight"] = torch.zeros(577, 255, 1, 3, 3)
    with pytest.raises(VfError, match=r"'layer3.0.conv2.0.0.weight' has .* not a \(co, 256, 1, 3, 3\) weight"):
        _engine(bad)
    bad = dict(sd34)
    bad["layer3.0.conv2.0.3.weight"] = torch.zeros(256, 460, 3, 1, 1)      # conv1's width in conv2
    with pytest.raises(VfError, match="layer3.0.conv2.0.3.weight"):
        _engine(bad)
    bad = dict(sd34)
    bad["layer1.1.downsample.0.weight"] = torch.zeros(64, 64, 1, 1, 1)
    with pytest.raises(VfError, match="'layer1.1.downsample.0.weight' on a stride-1 block"):
        _engine(bad)
    with pytest.raises(VfError, match="eps"):
        _engine(sd34, bn_eps=0.0)


# ------------------------------------------------------------------------------------- ExtractR21D on the sample video
@pytest.fixture(scope="module")
def ckpt_dir(tmp_path_factory, sd34):
    """The stand-in under both IG65M release names (as recalled)."""
    d = tmp_path_factory.mktemp("ckpt34")
    torch.save(sd34, str(d / "r2plus1d_34_clip32_ft_kinetics_from_ig65m-standin.pth"))
    torch.save(sd34, str(d / "r2plus1d_34_clip8_ft_kinetics_from_ig65m-standin.pth"))
    return str(d)


@pytest.fixture
def weights(ckpt_dir, monkeypatch):
    from video_features_b200.extract import extract_r21d
    monkeypatch.setenv("VF_CKPT_DIR", ckpt_dir)
    monkeypatch.setattr(extract_r21d, "_STATE_DICTS_34", {})
    return ckpt_dir


def _ns(**kw):
    d = dict(feature_type='r21d_rgb', video_paths=[VIDEO], flow_paths=None, file_with_video_paths=None, video_dir=None,
             flow_dir=None, extraction_fps=None, on_extraction='save_numpy', output_path='./output', tmp_path='./tmp',
             show_pred=False, keep_tmp_files=False, stack_size=None, step_size=None)
    d.update(kw)
    return argparse.Namespace(**d)


def _extract(tmp_path, tag, capsys=None, **kw):
    from video_features_b200.extract.extract_r21d import ExtractR21D
    ex = ExtractR21D(_ns(output_path=str(tmp_path / tag), tmp_path=str(tmp_path / "tmp"), **kw))
    ex.keep_features = True
    if capsys is not None:
        capsys.readouterr()
    res = ex(torch.zeros([1], dtype=torch.long, device="cuda:0"))[0]
    return res, (capsys.readouterr().out if capsys is not None else None)


_REF = {}


def _oracle(stack, cuda_device, sd34):
    """(slices, features, logits) of the fp32 oracle on the decoded sample video at stack = step."""
    if stack not in _REF:
        from test_r21d_oracle_cpu import decoded_rgb
        x = r21d_net.transform(decoded_rgb())
        slices = r21d_net.form_slices(x.shape[1], stack, stack)
        sd = _cast(sd34, cuda_device)
        with torch.no_grad():
            feats = torch.cat([ref34.forward(sd, torch.stack([x[:, s:e] for s, e in slices[i:i + 4]]).to(cuda_device))
                               for i in range(0, len(slices), 4)])
            logits = class_heads.fc_logits(sd, feats)
        _REF[stack] = (slices, feats.cpu(), logits.cpu())
    return _REF[stack]


@pytest.mark.parametrize("model,stack,rows", [(M32, 32, 11), (M8, 8, 44)])
def test_extract_vs_oracle_cli_and_show_pred(cuda_device, sd34, weights, tmp_path, capsys, model, stack, rows):
    from test_show_pred_gpu import _check_block, _engine_head, _parse
    from video_features_b200.class_head import FC_KEYS
    from video_features_b200.utils import class_names
    slices, ref, ref_logits = _oracle(stack, cuda_device, sd34)
    assert len(slices) == rows
    res, _ = _extract(tmp_path, "plain", model_name=model)
    feats = res["r21d_rgb"]
    assert set(res) == {"r21d_rgb"} and feats.shape == (rows, 512) and feats.dtype == np.float64
    saved = np.load(str(tmp_path / "plain" / "r21d_rgb" / "v_GGSY1Qvo990_r21d_rgb.npy"))
    np.testing.assert_array_equal(saved, feats)
    rel, mx = bars.row_errors(torch.from_numpy(feats), ref)
    print(f"ExtractR21D {model} ({rows} stacks) vs fp32 oracle: rel-L2 {rel:.2e}, max-abs/max {mx:.2e}")
    assert rel <= 1e-3 and mx <= 1e-3
    # --show_pred: the same features, and per stack the oracle's top-5
    shown, out = _extract(tmp_path, "shown", capsys, model_name=model, show_pred=True)
    np.testing.assert_array_equal(shown["r21d_rgb"], feats)
    blocks = _parse(out)
    assert [h for h, _ in blocks] == [f"{VIDEO} @ frames ({s}, {e})" for s, e in slices]
    eng_l, eng_p = _engine_head(sd34, FC_KEYS, feats, cuda_device)
    names = class_names("kinetics")
    for i, ((_, printed), r) in enumerate(zip(blocks, ref_logits)):
        _check_block(printed, r, names, (eng_l[i], eng_p[i]))
    # main.py --model_name: the same features, saved under r21d_rgb
    out_dir = tmp_path / "cli"
    cmd = [sys.executable, os.path.join(ROOT, "main.py"), "--feature_type", "r21d_rgb", "--model_name", model,
           "--on_extraction", "save_numpy", "--output_path", str(out_dir), "--tmp_path", str(tmp_path / "tmp"),
           "--video_paths", VIDEO]
    r = subprocess.run(cmd, cwd=str(tmp_path), env=dict(os.environ, VF_CKPT_DIR=weights), capture_output=True,
                       text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    y = np.load(str(out_dir / "r21d_rgb" / "v_GGSY1Qvo990_r21d_rgb.npy"))
    np.testing.assert_array_equal(y, feats)
