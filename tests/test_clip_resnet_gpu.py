"""ClipResNetEngine (vf_clip_rn_*) on the calibrated stand-ins of oracle/clip_resnet.py: every read_stage stage and the
features against a float64 forward of the oracle on the GPU, the project's fp32 gate on the features, bit identity of
the u8 / f32 entries and of chunked calls, the uploaded convs read back bit for bit against tests/clip_rn_layout.py,
and the conv-GEMM at the towers' new widths against float64.

Bars (FLOAT64_BARS): worst rows, rel-L2 / max-abs÷max, set 1.5 .. 2.2x above the values measured on one H100 80GB HBM3
(700 W power limit) and printed by test_zz_report_measured (pytest -s).  The error grows with depth (RN50x16's layer4
3.3e-4 against its stem's 4.5e-6): it is the length of the tensor cores' fp32 accumulation chains, as for ResNet
(test_split_engines_float64_gpu.py), not a lost lo half -- the negative control, weights rounded to fp16, misses the
stem's bar by 96x (6.7e-4)."""
import ctypes as C

import numpy as np
import pytest
import torch

import clip_rn_layout as lay
from oracle import clip_resnet

pytestmark = pytest.mark.gpu

FRAMES = {"RN50": (3, 2), "RN101": (3, 2), "RN50x4": (2, 2), "RN50x16": (2, 2)}      # (frames, max_frames)
# bars on (rel-L2, max-abs / max) of the worst row against float64; measured (RN50, RN101, RN50x4, RN50x16):
#   stem 3.3e-6 .. 4.5e-6, layer1 6.8e-6 .. 1.3e-5, layer2 1.6e-5 .. 3.9e-5, layer3 4.2e-5 .. 1.5e-4,
#   layer4 / tokens 8.5e-5 .. 3.3e-4, pre_cproj 6.6e-5 .. 2.2e-4 (max-abs up to 5.3e-4), features 1.3e-4 .. 2.2e-4
FLOAT64_BARS = {
    "RN50": {"stem": (7e-6, 7e-6), "layer1": (1.5e-5, 1.5e-5), "layer2": (3.5e-5, 3e-5), "layer3": (9e-5, 6e-5),
             "layer4": (1.7e-4, 1.3e-4), "tokens": (1.7e-4, 1.3e-4), "pre_cproj": (1.4e-4, 1.5e-4),
             "features": (3e-4, 3e-4)},
    "RN101": {"stem": (7e-6, 7e-6), "layer1": (1.5e-5, 1.5e-5), "layer2": (3.5e-5, 3e-5), "layer3": (1.9e-4, 1.4e-4),
              "layer4": (3.3e-4, 2.6e-4), "tokens": (3.3e-4, 2.6e-4), "pre_cproj": (1.7e-4, 1.8e-4),
              "features": (4.4e-4, 4.9e-4)},
    "RN50x4": {"stem": (9e-6, 1.2e-5), "layer1": (2e-5, 2e-5), "layer2": (5e-5, 4.5e-5), "layer3": (1.6e-4, 1.3e-4),
               "layer4": (3.4e-4, 3.6e-4), "tokens": (3.4e-4, 3.6e-4), "pre_cproj": (2.5e-4, 3.5e-4),
               "features": (2.6e-4, 2.6e-4)},
    "RN50x16": {"stem": (9e-6, 9e-6), "layer1": (2.7e-5, 2.7e-5), "layer2": (8e-5, 7e-5), "layer3": (3.1e-4, 2.6e-4),
                "layer4": (6.6e-4, 5.3e-4), "tokens": (6.6e-4, 5.3e-4), "pre_cproj": (4.4e-4, 8e-4),
                "features": (4.4e-4, 5.5e-4)},
}
MEASURED = {}


def row_errors(got, want):
    g, w = got.double().reshape(got.shape[0], -1).cpu(), want.double().reshape(want.shape[0], -1).cpu()
    rel = ((g - w).norm(dim=1) / w.norm(dim=1)).max().item()
    mx = ((g - w).abs().amax(dim=1) / w.abs().amax(dim=1)).max().item()
    return rel, mx


def _f64(sd, dev):
    return {k: v.double().to(dev) for k, v in sd.items()}


def _stage_errors(name, eng, y, ref, taps, rows, record=True):
    errs = {"features": row_errors(y, ref)}
    for sid, s in enumerate(clip_resnet.STAGES):
        got = eng.read_stage(sid)
        want = taps[s][rows]
        assert got.shape == want.shape, (s, got.shape, want.shape)
        errs[s] = row_errors(got, want)
    for s, e in errs.items():
        print(f"{name} {s}: rel-L2 {e[0]:.2e}, max-abs/max {e[1]:.2e}")
        if record:
            old = MEASURED.get((name, s), (0.0, 0.0))
            MEASURED[(name, s)] = (max(old[0], e[0]), max(old[1], e[1]))
    return errs


@pytest.mark.parametrize("name", list(clip_resnet.TOWERS))
def test_engine_matches_float64(cuda_device, name):
    from video_features_b200.clip_resnet_engine import ClipResNetEngine
    sd = clip_resnet.stand_in_state_dict(name)
    cfg = clip_resnet.config(sd)
    n, chunk = FRAMES[name]
    eng = ClipResNetEngine(sd, 0, max_frames=chunk)
    assert (eng.out_dim, eng.n_px, eng.tokens, eng.layers) == (cfg["out_dim"], cfg["n_px"], cfg["tokens"], cfg["layers"])
    x = clip_resnet.calibration_images(cfg["n_px"], seed=7, n=n).to(cuda_device)
    y = eng.encode_image(x)
    with torch.no_grad():
        ref, taps = clip_resnet.forward(_f64(sd, cuda_device), x.double(), taps=True)
        ref32 = clip_resnet.forward({k: v.to(cuda_device) for k, v in sd.items()}, x)
    rel, mx = row_errors(y, ref32)
    print(f"{name} vs fp32 oracle: rel-L2 {rel:.2e}, max-abs/max {mx:.2e}")
    assert rel <= 1e-3 and mx <= 1e-3, (rel, mx)
    last = slice(n - (n - 1) % chunk - 1, n)
    errs = _stage_errors(name, eng, y, ref, taps, last)
    bars = FLOAT64_BARS[name]
    failures = [(s, e, bars[s]) for s, e in errs.items() if e[0] > bars[s][0] or e[1] > bars[s][1]]
    assert not failures, failures
    eng.close()


def test_fp16_weights_fail_the_stem_bar(cuda_device):
    """Negative control: weights pre-rounded to fp16 (every W_lo exactly zero) miss the stem's float64 bar by far."""
    from video_features_b200.clip_resnet_engine import ClipResNetEngine
    sd = clip_resnet.stand_in_state_dict("RN50")
    sd16 = {k: (v.half().float() if v.dim() >= 2 else v) for k, v in sd.items()}
    eng = ClipResNetEngine(sd16, 0, max_frames=2)
    x = clip_resnet.calibration_images(224, seed=8, n=2).to(cuda_device)
    y = eng.encode_image(x)
    with torch.no_grad():
        ref, taps = clip_resnet.forward(_f64(sd, cuda_device), x.double(), taps=True)
    errs = _stage_errors("RN50 fp16-weights", eng, y, ref, taps, slice(0, 2), record=False)
    bar = FLOAT64_BARS["RN50"]["stem"]
    assert errs["stem"][0] > 10 * bar[0], errs["stem"]
    eng.close()


def _frames_u8(n, h, w, seed):
    g = torch.Generator().manual_seed(seed)
    low = torch.rand(n, 3, 10, 12, generator=g)
    img = torch.nn.functional.interpolate(low, size=(h, w), mode="bilinear", align_corners=False)
    img = img * 0.85 + 0.15 * torch.rand(n, 3, h, w, generator=g)
    return img.mul(255).round().clamp(0, 255).to(torch.uint8).permute(0, 2, 3, 1).contiguous()


@pytest.mark.parametrize("name,hw", [("RN50", (240, 320)), ("RN50x4", (360, 270))])
def test_u8_entry_and_call_splits_are_bit_identical(cuda_device, name, hw):
    from video_features_b200.clip_resnet_engine import ClipResNetEngine
    sd = clip_resnet.stand_in_state_dict(name)
    eng = ClipResNetEngine(sd, 0, max_frames=3)
    u8 = _frames_u8(7, *hw, seed=3)
    a = eng.encode_frames_u8(u8.to(cuda_device))            # resize + crop + normalise fused, chunks of 3
    x = clip_resnet.preprocess_batch(u8.numpy(), eng.n_px).to(cuda_device)
    assert torch.equal(a, eng.encode_image(x))
    parts = torch.cat([eng.encode_frames_u8(u8[i:j].to(cuda_device)) for i, j in ((0, 2), (2, 3), (3, 7))])
    assert torch.equal(a, parts)
    host = eng.encode_frames_u8_host(u8)
    assert torch.equal(host, a.cpu())
    ticket, dev = eng.encode_frames_u8_host_async(u8.pin_memory(), torch.empty(7, eng.out_dim).pin_memory(), True)
    eng.wait(ticket)
    assert torch.equal(dev, a)
    eng.close()


@pytest.mark.parametrize("name", ["RN50", "RN50x4", "RN50x16"])
def test_uploads_match_the_restated_layout(cuda_device, name):
    from video_features_b200._lib import VfError
    from video_features_b200.clip_resnet_engine import ClipResNetEngine
    sd = clip_resnet.stand_in_state_dict(name)
    cfg = clip_resnet.config(sd)
    eng = ClipResNetEngine(sd, 0, max_frames=1)
    want = lay.engine_convs(sd, cfg)
    for i, f in enumerate(want):
        got = eng.conv(i)
        where = (i, f["name"])
        assert (got["n_out"], got["ntaps"], got["k_per_tap"]) == (f["Wt"].shape[0], f["ntaps"], f["k_per_tap"]), where
        assert got["shifts"] == f["shifts"], where
        assert got["lo_mask"] == f["lo_mask"], where
        assert torch.equal(got["w"].cpu().view(torch.int16), f["Wt"].view(torch.int16)), where
        assert torch.equal(got["scale"].cpu().view(torch.int32), f["scale"].view(torch.int32)), where
        assert torch.equal(got["bias"].cpu().view(torch.int32), f["bias"].float().view(torch.int32)), where
    with pytest.raises(VfError, match="outside"):
        eng.conv(len(want))
    eng.close()


def test_create_names_a_missing_or_missized_key(cuda_device):
    from video_features_b200._lib import VfError
    from video_features_b200.clip_resnet_engine import ClipResNetEngine
    sd = clip_resnet.stand_in_state_dict("RN50")
    bad = dict(sd)
    del bad["visual.layer3.2.bn2.running_var"]
    with pytest.raises(VfError, match="missing tensor 'visual.layer3.2.bn2.running_var'"):
        ClipResNetEngine(bad, 0, max_frames=1)
    bad = dict(sd)
    bad["visual.attnpool.k_proj.weight"] = torch.zeros(2048, 1024)
    with pytest.raises(VfError, match="visual.attnpool.k_proj.weight"):
        ClipResNetEngine(bad, 0, max_frames=1)


def _conv_gemm(X, pitch, P, f, N, region, out, split_off, bias, scale, dev):
    from video_features_b200 import _lib
    taps = (C.c_int * f["ntaps"])(*[dh * region[2] + dw for _, dh, dw in f["shifts"]])
    reg = (C.c_int * 9)(*region)
    ldd = out.shape[1]
    with torch.cuda.device(dev):
        _lib.check(_lib.lib().vf_conv_gemm_f16(
            X.data_ptr(), pitch, P, f["Wt"].to(dev).data_ptr(), N, f["ntaps"], f["k_per_tap"], taps, 2, f["lo_mask"],
            0, reg, out.data_ptr(), ldd, int(out.dtype == torch.float32), split_off, bias.data_ptr(), scale.data_ptr(),
            0, torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()


@pytest.mark.parametrize("kind,ci,co,S", [("stem", 3, 40, 18), ("stem", 3, 48, 18), ("same3", 40, 40, 18),
                                          ("same3", 48, 48, 14), ("same3", 40, 80, 14), ("pooled", 80, 320, 9),
                                          ("pooled", 48, 80, 7), ("same1", 80, 320, 9)])
def test_conv_gemm_at_clip_widths_matches_float64(cuda_device, kind, ci, co, S):
    """The conv-GEMM at the widths RN50x4 / RN50x16 bring (N = 40, 48, 80, 320; split rows of 80, 96, 160): a conv of
    the engine's layout against F.conv2d in float64 (pooled: after F.avg_pool2d), fp32 out and split out."""
    import torch.nn.functional as F
    g = torch.Generator().manual_seed(ci * 1000 + co)
    n = 2
    if kind == "stem":
        x = torch.randn(n, 3, 2 * S, 2 * S, generator=g)
        w = torch.randn(co, 3, 3, 3, generator=g) * 0.2
        V, f = lay.stem_phase_volume(x), lay.stem_filter(w)
        ref = F.conv2d(sum(lay.split(x)[i].double() for i in (0, 1)), sum(lay.split(w)[i].double() for i in (0, 1)),
                       stride=2, padding=1)
    else:
        x = torch.randn(n, ci, 2 * S if kind == "pooled" else S, 2 * S if kind == "pooled" else S, generator=g)
        k = 3 if kind == "same3" else 1
        w = torch.randn(co, ci, k, k, generator=g) / (ci * k * k) ** 0.5
        V = lay.volume(x)
        f = lay.pooled_filter(w) if kind == "pooled" else lay.same_filter(w)
        xe = sum(lay.split(x)[i].double() for i in (0, 1))
        we = sum(lay.split(w)[i].double() for i in (0, 1))
        if kind == "pooled":
            V = lay.phase_repack(V)
            ref = F.conv2d(F.avg_pool2d(xe, 2), we)
        else:
            ref = F.conv2d(xe, we, padding=k // 2)
    Hp = V.shape[1]
    pitch = V.shape[3]
    P = n * Hp * Hp
    X = torch.cat([V.reshape(P, pitch).half(), torch.zeros(64, pitch, dtype=torch.float16)]).to(cuda_device)
    scale = torch.full((co,), 0.25 if kind == "pooled" else 1.0, device=cuda_device)
    bias = torch.zeros(co, device=cuda_device)
    region = [1, Hp, Hp, 0, 1, 1, Hp - 1, 1, Hp - 1]
    want = torch.zeros(n, Hp, Hp, co, dtype=torch.float64)
    want[:, 1:Hp - 1, 1:Hp - 1] = ref.permute(0, 2, 3, 1)
    want = want.reshape(P, co)
    o32 = torch.zeros(P, co, device=cuda_device)
    _conv_gemm(X, pitch, P, f, co, region, o32, 0, bias, scale, cuda_device)
    osp = torch.zeros(P, 2 * co, dtype=torch.float16, device=cuda_device)
    _conv_gemm(X, pitch, P, f, co, region, osp, co, bias, scale, cuda_device)
    for what, got in (("f32", o32.double().cpu()), ("split", (osp[:, :co].double() + osp[:, co:].double()).cpu())):
        rel = float((got - want).norm() / want.norm())
        mx = float((got - want).abs().max() / want.abs().max())
        print(f"{kind} ci {ci} co {co} {what}: rel-L2 {rel:.2e}, max-abs/max {mx:.2e}")
        assert rel <= 2e-5 and mx <= 1e-4, (what, rel, mx)


def test_zz_report_measured(cuda_device):
    """Prints the worst row per tower and stage over test_engine_matches_float64 (run in the same session)."""
    for (name, s), (rel, mx) in sorted(MEASURED.items()):
        print(f"measured worst {name} {s}: rel-L2 {rel:.2e}, max-abs/max {mx:.2e}")
