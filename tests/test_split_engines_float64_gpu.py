"""ResNetEngine and R21DEngine against a float64 forward of the same network on the GPU (oracle/resnet_net.py,
oracle/r21d_net.py with the stand-in state dict and the exact fp32 input cast to double), at every read_stage stage and
the features, worst row (frame or clip).

The engines carry every activation as a split-fp16 pair [hi C | lo C] and every weight as a hi + lo pair, and skip the
W_lo pass only on K blocks that meet nothing but lo halves (DESIGN.md §4.6, §4.7).  The fp32-oracle tests
(test_resnet_gpu.py, test_r21d_gpu.py) cannot see that scheme lose a part: their bars (1e-5 .. 1e-3) are set by the fp32
oracle's own summation noise, which is as large as what one tensor class left in single fp16 costs.  The bars here
(tests/split_engine_bars.py) sit 1.5x .. 3x above the engine and, at the stem through layer3, tenfold under every
single-fp16 class (test_split_engine_bars_cpu.py).  Two negative controls through the public API lose a lo half on
purpose: weights pre-rounded to fp16 (W_lo exactly zero) and an input pre-rounded to fp16 (the stem input's lo half
zero).  Against float64 of the original operands each fails the stem's bar 50x .. 110x; against float64 of the rounded
operands every stage passes.

Measured worst rows, one H100 80GB HBM3 (700 W power limit), rel-L2 / max-abs÷max:
  stage      ResNet-18          ResNet-50          ResNet-152         R(2+1)D-18 (T = 16, 7, 1)
  stem       1.2e-6 / 1.6e-6    1.3e-6 / 1.9e-6    1.3e-6 / 2.0e-6    2.2e-6 / 2.5e-6
  maxpool    1.1e-6 / 1.6e-6    1.1e-6 / 1.9e-6    1.2e-6 / 2.0e-6    -
  layer1     2.4e-6 / 2.0e-6    4.0e-6 / 3.6e-6    3.8e-6 / 5.1e-6    5.6e-6 / 4.9e-6
  layer2     6.2e-6 / 6.2e-6    1.1e-5 / 1.0e-5    1.5e-5 / 1.5e-5    1.2e-5 / 1.1e-5
  layer3     1.2e-5 / 1.1e-5    3.0e-5 / 3.0e-5    1.6e-4 / 1.8e-4    2.6e-5 / 2.4e-5
  layer4     2.1e-5 / 2.2e-5    5.6e-5 / 5.0e-5    3.0e-4 / 3.4e-4    6.6e-5 / 8.3e-5
  features   1.6e-5 / 2.9e-5    3.4e-5 / 6.2e-5    8.6e-5 / 1.7e-4    4.8e-5 / 8.3e-5
These are 10 .. 20x what a plain fp32 torch forward on the CPU measures (ResNet-18 layer4 1.1e-6, R(2+1)D layer4
1.8e-6), and far above the operand rounding the split scheme leaves (4e-8 .. 3e-7, the emulation).
test_conv_gemm_resnet_r21d_gpu.py shows it conv by conv, 8.6e-7 at K = 512 (the stems) up to 1.5e-5 at K = 4 x 4096
(layer4's stride-2 conv), no conv outside its fp32 bar, and isolates the cause: the same operands as four one-tap
launches summed in float64 measure 6.0e-6 against 1.6e-5 as one launch, so the error is the length of the tensor
cores' fp32 accumulation chain.  That every lo half, W_lo row and lo_mask bit is uploaded is checked exactly there,
conv by conv at every depth.  The
controls: fp16 weights 2.8e-4 / 4.9e-4 (ResNet-18 stem), 4.6e-4 / 5.0e-4 (R(2+1)D stem); fp16 input 2.6e-4 / 5.6e-4,
3.8e-4 / 4.6e-4.  test_zz_report_measured prints the worst rows of a run (pytest -s).
"""
import pytest
import torch

import split_engine_bars as bars
from oracle import r21d_net, resnet_net

pytestmark = pytest.mark.gpu

MEASURED = {}


def _f64(sd, dev):
    return {k: (v.double() if v.is_floating_point() else v).to(dev) for k, v in sd.items()}


def _fp16_weights(sd):
    """The conv weights (4-D / 5-D) rounded to fp16: the engine's W_lo of every conv is then exactly zero."""
    return {k: (v.half().float() if v.is_floating_point() and v.dim() >= 4 else v) for k, v in sd.items()}


def _compare(what, got, want, bar, record=True):
    err = bars.row_errors(got, want)
    print(f"{what}: rel-L2 {err[0]:.2e}, max-abs/max {err[1]:.2e} (bar {bar[0]:.1e} / {bar[1]:.1e})")
    if record:
        key = what.split(" ")[0] + " " + what.split(" ")[-1]
        old = MEASURED.get(key, (0.0, 0.0))
        MEASURED[key] = (max(old[0], err[0]), max(old[1], err[1]))
    return err


def _stage_errors(name, eng, y, ref, taps, stages, bar, last, record=True):
    """{stage: error}: the features of every row, read_stage (the last chunk: rows `last`) of every other stage."""
    errs = {"features": _compare(f"{name} features", y, ref, bar["features"], record)}
    for sid, s in enumerate(stages[:-1]):
        got = eng.read_stage(sid)
        want = taps[s][last]
        assert got.shape == want.shape, (s, got.shape, want.shape)
        errs[s] = _compare(f"{name} {s}", got, want, bar[s], record)
    return errs


def _check_stages(name, eng, y, ref, taps, stages, bar, last):
    errs = _stage_errors(name, eng, y, ref, taps, stages, bar, last)
    failures = [(s, e) for s, e in errs.items() if not bars.within(e, bar[s])]
    assert not failures, failures


@pytest.mark.parametrize("depth", [18, 50, 152])
def test_resnet_matches_float64(cuda_device, depth):
    from video_features_b200.resnet_engine import ResNetEngine
    sd = resnet_net.stand_in_state_dict(depth)
    n, chunk = (6, 4) if depth == 18 else (3, 3)        # ResNet-18: 6 frames in two internal chunks of 4
    eng = ResNetEngine(sd, depth, 0, max_frames=chunk)
    x = resnet_net.calibration_images(seed=7, n=n).to(cuda_device)
    y = eng.forward_f32(x)
    with torch.no_grad():
        ref, taps = resnet_net.forward(_f64(sd, cuda_device), x.double(), depth, taps=True)
    last = slice(n - (n - 1) % chunk - 1, n)
    _check_stages(f"resnet{depth}", eng, y, ref, taps, bars.RESNET_STAGES, bars.RESNET_BARS[depth], last)
    eng.close()


@pytest.mark.parametrize("T,n", [(16, 2), (7, 5), (1, 3)])
def test_r21d_matches_float64(cuda_device, T, n):
    from video_features_b200.r21d_engine import R21DEngine
    sd = r21d_net.stand_in_state_dict()
    eng = R21DEngine(sd, 0, max_clips=2, max_T=16)      # 36 frame slots: T = 7 runs 5 clips as chunks of 4 + 1
    per_chunk = 36 // (T + 2)
    x = r21d_net.calibration_clips(seed=7, n=n, T=T).to(cuda_device)
    y = eng.forward_f32(x)
    with torch.no_grad():
        ref, taps = r21d_net.forward(_f64(sd, cuda_device), x.double(), taps=True)
    last = slice(n - (n - 1) % per_chunk - 1, n)
    _check_stages(f"r21d-T{T}", eng, y, ref, taps, bars.R21D_STAGES, bars.R21D_BARS, last)
    eng.close()


def _negative_controls(name, make_engine, forward, sd, x, stages, bar):
    """Weights pre-rounded to fp16, then the input pre-rounded to fp16.  Against float64 of the original operands each
    fails the stem's bar at least tenfold (both enter the stem conv) and the features' bar; against float64 of the
    rounded operands every stage passes."""
    sd16 = _fp16_weights(sd)
    x16 = x.half().float()
    for what, s_eng, x_eng in (("fp16-weights", sd16, x), ("fp16-input", sd, x16)):
        eng = make_engine(s_eng)
        y = eng.forward_f32(x_eng)
        all_rows = slice(0, x.shape[0])
        lost = _stage_errors(f"{name} {what} vs original", eng, y, *forward(sd, x), stages, bar, all_rows, False)
        kept = _stage_errors(f"{name} {what} vs rounded", eng, y, *forward(s_eng, x_eng), stages, bar, all_rows, False)
        eng.close()
        assert bars.beyond(lost["stem"], bar["stem"], 10), (what, lost["stem"])
        assert bars.beyond(lost["features"], bar["features"]), (what, lost["features"])
        assert all(bars.within(e, bar[s]) for s, e in kept.items()), (what, kept)


def test_resnet18_negative_controls(cuda_device):
    from video_features_b200.resnet_engine import ResNetEngine
    sd = resnet_net.stand_in_state_dict(18)
    x = resnet_net.calibration_images(seed=8, n=4).to(cuda_device)

    def forward(s, xx):
        with torch.no_grad():
            return resnet_net.forward(_f64(s, cuda_device), xx.double(), 18, taps=True)
    _negative_controls("resnet18", lambda s: ResNetEngine(s, 18, 0, max_frames=4), forward, sd, x,
                       bars.RESNET_STAGES, bars.RESNET_BARS[18])


def test_r21d_negative_controls(cuda_device):
    from video_features_b200.r21d_engine import R21DEngine
    sd = r21d_net.stand_in_state_dict()
    x = r21d_net.calibration_clips(seed=8, n=2, T=8).to(cuda_device)

    def forward(s, xx):
        with torch.no_grad():
            return r21d_net.forward(_f64(s, cuda_device), xx.double(), taps=True)
    _negative_controls("r21d", lambda s: R21DEngine(s, 0, max_clips=2, max_T=8), forward, sd, x, bars.R21D_STAGES,
                       bars.R21D_BARS)


def test_zz_report_measured(cuda_device):
    """Prints the worst row per network and stage over the tests above (run in the same session)."""
    for k, (rel, mx) in sorted(MEASURED.items()):
        print(f"measured worst {k}: rel-L2 {rel:.2e}, max-abs/max {mx:.2e}")
