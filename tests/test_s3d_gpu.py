"""S3DEngine (vf_s3d_*) against a float64 forward of torchvision's S3D (oracle/s3d_net.py) on the calibrated stand-in,
at every read_stage stage and the features; the fused transform against the preset; call splits; the uploaded convs
against their restated layout; and the classifier head against torchvision's ``model(x)``.

Bars: tests/s3d_bars.py (worst row: clip; rel-L2, max-abs / max|ref|), 1.5x .. 2.3x above the values measured on an
H100; test_s3d_bars_cpu.py shows that each lies well under every single-fp16 tensor class of the emulation.  The engine
is deterministic, so a rerun gives the same values."""
import numpy as np
import pytest
import torch

from oracle import s3d_net
from s3d_bars import BARS

pytestmark = pytest.mark.gpu
MEASURED = {}


def _f64(sd, dev):
    return {k: (v.double() if v.is_floating_point() else v).to(dev) for k, v in sd.items()}


def row_errors(y, ref):
    y = y.double().flatten(1)
    ref = ref.double().flatten(1).to(y.device)
    d = y - ref
    return (d.norm(dim=1) / ref.norm(dim=1)).max().item(), (d.abs().amax(dim=1) / ref.abs().amax(dim=1)).max().item()


def within(err, bar, factor=1.0):
    return err[0] <= factor * bar[0] and err[1] <= factor * bar[1]


def stage_errors(name, eng, y, ref, taps, record=True):
    """{stage: error}: the features of every clip, read_stage (the last chunk) of every other stage."""
    errs = {"features": row_errors(y, ref)}
    for sid, s in enumerate(s3d_net.STAGES):
        got = eng.read_stage(sid)
        want = taps[s][ref.shape[0] - got.shape[0]:]
        assert got.shape == want.shape, (s, got.shape, want.shape)
        errs[s] = row_errors(got, want)
    for s, e in errs.items():
        print(f"{name} {s}: rel-L2 {e[0]:.2e}, max-abs/max {e[1]:.2e} (bar {BARS[s][0]:.1e} / {BARS[s][1]:.1e})")
        if record:
            old = MEASURED.get(s, (0.0, 0.0))
            MEASURED[s] = (max(old[0], e[0]), max(old[1], e[1]))
    return errs


def frames_bgr(n, h=240, w=320, seed=0):
    """n smooth random uint8 BGR frames, slowly changing in time."""
    g = torch.Generator().manual_seed(seed)
    low = torch.rand(1, 3, max(n // 4, 2), 8, 10, generator=g)
    vid = torch.nn.functional.interpolate(low, size=(n, h, w), mode="trilinear", align_corners=False)[0]
    vid = vid * 0.85 + 0.15 * torch.rand(3, n, h, w, generator=g)
    return vid.mul(255).round().clamp(0, 255).to(torch.uint8).permute(1, 2, 3, 0).contiguous()


def clips_f32(u8_bgr, starts, T):
    """The preset (torchvision's own transform) of each clip of RGB frames: (n, 3, T, 224, 224)."""
    rgb = u8_bgr.numpy()[..., ::-1].copy()
    return torch.stack([s3d_net.transform_torchvision(rgb[s:s + T]) for s in starts])


@pytest.mark.parametrize("T,n,max_clips,max_T", [(64, 1, 1, 64), (16, 3, 1, 17), (13, 3, 1, 17), (17, 3, 2, 17)])
def test_matches_float64(cuda_device, T, n, max_clips, max_T):
    """Small workspaces, so three clips run as chunks inside the call."""
    from video_features_b200.s3d_engine import S3DEngine
    sd = s3d_net.stand_in_state_dict()
    eng = S3DEngine(sd, 0, max_clips=max_clips, max_T=max_T)
    x = s3d_net.calibration_clips(seed=7 + T, n=n, T=T).to(cuda_device)
    y = eng.forward_f32(x)
    with torch.no_grad():
        ref, taps = s3d_net.forward(_f64(sd, cuda_device), x.double(), taps=True)
    assert y.shape == (n, 1024) and y.dtype == torch.float32
    errs = stage_errors(f"s3d T={T} n={n}", eng, y, ref, taps)
    eng.close()
    failures = [(s, e) for s, e in errs.items() if not within(e, BARS[s])]
    assert not failures, failures


def test_negative_controls(cuda_device):
    """Weights pre-rounded to fp16, then the input pre-rounded to fp16: against float64 of the original operands each
    fails the stem's bar at least tenfold; against float64 of the rounded operands every stage passes."""
    from video_features_b200.s3d_engine import S3DEngine
    sd = s3d_net.stand_in_state_dict()
    x = s3d_net.calibration_clips(seed=8, n=1, T=16).to(cuda_device)
    sd16 = {k: (v.half().float() if v.is_floating_point() and v.dim() >= 4 else v) for k, v in sd.items()}
    x16 = x.half().float()

    def forward(s, xx):
        with torch.no_grad():
            return s3d_net.forward(_f64(s, cuda_device), xx.double(), taps=True)
    for what, s_eng, x_eng in (("fp16-weights", sd16, x), ("fp16-input", sd, x16)):
        eng = S3DEngine(s_eng, 0, max_clips=1, max_T=16)
        y = eng.forward_f32(x_eng)
        lost = stage_errors(f"s3d {what} vs original", eng, y, *forward(sd, x), record=False)
        kept = stage_errors(f"s3d {what} vs rounded", eng, y, *forward(s_eng, x_eng), record=False)
        eng.close()
        assert not within(lost["stem"], BARS["stem"], 10), (what, lost["stem"])
        assert all(within(e, BARS[s]) for s, e in kept.items()), (what, kept)


@pytest.mark.parametrize("hw", [(240, 320), (100, 60), (360, 480)])
def test_u8_equals_f32(cuda_device, hw):
    """The fused transform is the preset bit for bit, so both entries give identical features."""
    from video_features_b200.s3d_engine import S3DEngine
    T = 13
    eng = S3DEngine(s3d_net.stand_in_state_dict(), 0, max_clips=2, max_T=T)
    u8 = frames_bgr(T + 4, *hw, seed=hw[0])
    starts = [0, 4]
    y8 = eng.forward_u8(u8.to(cuda_device), starts, T)
    yf = eng.forward_f32(clips_f32(u8, starts, T).to(cuda_device))
    eng.close()
    assert torch.equal(y8, yf), (y8 - yf).abs().max().item()


def test_call_splits_are_bit_identical(cuda_device):
    """Any split of clips over calls, and the chunking inside a call, give the same bits."""
    from video_features_b200.s3d_engine import S3DEngine
    T = 13
    sd = s3d_net.stand_in_state_dict()
    u8 = frames_bgr(40, seed=3).to(cuda_device)
    starts = [0, 5, 10, 20, 27]
    big = S3DEngine(sd, 0, max_clips=5, max_T=T)
    small = S3DEngine(sd, 0, max_clips=1, max_T=T)
    whole = big.forward_u8(u8, starts, T)
    parts = torch.cat([big.forward_u8(u8, starts[:2], T), big.forward_u8(u8, starts[2:], T)])
    chunked = small.forward_u8(u8, starts, T)
    single = torch.cat([small.forward_u8(u8, [s], T) for s in starts])
    big.close()
    small.close()
    for other in (parts, chunked, single):
        assert torch.equal(whole, other)


def test_rejects_short_clips(cuda_device):
    from video_features_b200._lib import VfError
    from video_features_b200.s3d_engine import S3DEngine
    eng = S3DEngine(s3d_net.stand_in_state_dict(), 0, max_clips=1, max_T=16)
    with pytest.raises(VfError, match="T=12"):
        eng.forward_f32(torch.zeros(1, 3, 12, 224, 224, device=cuda_device))
    eng.close()


# ---- every uploaded conv against its restated layout, bit for bit
def _bn(sd, p):
    g, b = sd[p + ".weight"].double(), sd[p + ".bias"].double()
    m, v = sd[p + ".running_mean"].double(), sd[p + ".running_var"].double()
    s = g / torch.sqrt(v + 1e-3)
    return s.float(), (b - m * s).float()


def _restated(sd, p, ntaps, kpt, lo_off, col):
    """(W_hi | W_lo fp16 [co, 2 ntaps kpt], lo_mask, scale, bias) of Conv3dNormActivation p, as s3d.cu lays it out."""
    w = sd[p + ".0.weight"].float()
    co, ci, kt, kh, kw = w.shape
    ktot = ntaps * kpt
    hi = w.half()
    lo = (w - hi.float()).half()
    W = torch.zeros(co, 2 * ktot, dtype=torch.float16)
    has_hi = torch.zeros(ktot, dtype=torch.bool)
    for a in range(kt):
        for y in range(kh):
            for x in range(kw):
                cols = torch.tensor([col(a, y, x, c) for c in range(ci)])
                for kk in (cols, cols + lo_off):
                    W[:, kk] = hi[:, :, a, y, x]
                    W[:, ktot + kk] = lo[:, :, a, y, x]
                has_hi[cols] = True
    nb = (kpt + 63) // 64
    mask = 0
    for kk in range(nb):
        if not any(has_hi[t * kpt + kk * 64:t * kpt + min((kk + 1) * 64, kpt)].any() for t in range(ntaps)):
            mask |= 1 << kk
    return W, mask, *_bn(sd, p + ".1")


def _layouts(sd):
    """(name, ntaps, k_per_tap, shifts, lo_off, col) in vf_s3d_conv's order."""
    out = [("features.0.0", 4, 128, [(0, a - 2, -2) for a in range(4)], 16,
            lambda t, kh, kw, c: (kh + 1) // 2 * 128 + (kw + 1) // 2 * 32 + ((kh + 1) % 2 * 2 + (kw + 1) % 2) * 4 + c),
           ("features.0.1", 4, 256, [(a - 2, 0, 0) for a in range(4)], 64,
            lambda t, kh, kw, c: (t + 1) // 2 * 256 + (t + 1) % 2 * 128 + c)]

    def point(p, ci):
        return (p, 1, 2 * ci, [(0, 0, 0)], ci, lambda t, kh, kw, c: c)

    def spatial(p, ci):
        return (p, 3, 6 * ci, [(0, a - 1, -1) for a in range(3)], ci, lambda t, kh, kw, c: kh * 6 * ci + kw * 2 * ci + c)

    def temporal(p, ci):
        return (p, 3, 2 * ci, [(a - 1, 0, 0) for a in range(3)], ci, lambda t, kh, kw, c: t * 2 * ci + c)
    out += [point("features.2", 64), spatial("features.3.0", 64), temporal("features.3.1", 192)]
    for i, (cin, b0, b1m, b1, b2m, b2, b3) in s3d_net.MIXED.items():
        p = f"features.{i}"
        out += [point(p + ".branch0", cin), point(p + ".branch1.0", cin), spatial(p + ".branch1.1.0", b1m),
                temporal(p + ".branch1.1.1", b1), point(p + ".branch2.0", cin), spatial(p + ".branch2.1.0", b2m),
                temporal(p + ".branch2.1.1", b2), point(p + ".branch3.1", cin)]
    return out


def test_uploaded_convs_match_the_restated_layout(cuda_device):
    from video_features_b200._lib import VfError
    from video_features_b200.s3d_engine import S3DEngine
    sd = s3d_net.stand_in_state_dict()
    eng = S3DEngine(sd, 0, max_clips=1, max_T=13)
    layouts = _layouts(sd)
    assert len(layouts) == 77
    for idx, (p, ntaps, kpt, shifts, lo_off, col) in enumerate(layouts):
        got = eng.conv(idx)
        W, mask, scale, bias = _restated(sd, p, ntaps, kpt, lo_off, col)
        assert (got["n_out"], got["ntaps"], got["k_per_tap"]) == (W.shape[0], ntaps, kpt), p
        assert got["shifts"] == shifts, p
        assert got["lo_mask"] == mask, (p, hex(got["lo_mask"]), hex(mask))
        assert torch.equal(got["w"].cpu().view(torch.int16), W.view(torch.int16)), p
        assert torch.equal(got["scale"].cpu(), scale) and torch.equal(got["bias"].cpu(), bias), p
    with pytest.raises(VfError):
        eng.conv(77)
    eng.close()


def test_class_head_matches_torchvision(cuda_device):
    """ClassHead on the engine's features against torchvision's ``model(x)`` in float64."""
    import torchvision
    from video_features_b200.class_head import ClassHead
    from video_features_b200.s3d_engine import S3DEngine
    sd = s3d_net.stand_in_state_dict()
    x = s3d_net.calibration_clips(seed=11, n=2, T=16)
    net = torchvision.models.video.s3d()
    net.load_state_dict(sd)
    net = net.double().eval().to(cuda_device)
    with torch.no_grad():
        ref = net(x.double().to(cuda_device))
    eng = S3DEngine(sd, 0, max_clips=2, max_T=16)
    head = ClassHead.from_state_dict(sd, s3d_net.HEAD_KEYS, 0)
    logits = head.forward(eng.forward_f32(x.to(cuda_device)))[0]
    err = row_errors(logits, ref)
    print(f"s3d logits vs torchvision float64: rel-L2 {err[0]:.2e}, max-abs/max {err[1]:.2e}")
    eng.close()
    assert within(err, BARS["features"]), err


def test_zz_report_measured(cuda_device):
    """Prints the worst row per stage over test_matches_float64 (run in the same session)."""
    for k, (rel, mx) in MEASURED.items():
        print(f"measured worst s3d {k}: rel-L2 {rel:.2e}, max-abs/max {mx:.2e}")
