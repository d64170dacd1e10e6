"""The CLIP ViT towers piece by piece (ClipEngine.debug_embed / debug_blocks / debug_head: the functions encode_image
runs, one at a time) against a float64 reference with the tower's declared fp16 rounding (oracle/clip_tower.py:
embed / block / head / attention_core, DECLARED).  Each piece of the reference is fed the ENGINE's own input at that
depth, so rounding flips do not compound over the 12 blocks.  Bars and what they consist of: tests/split_engine_bars.py
(CLIP_VIT); the product gate stays test_clip_gpu.py's 1e-3 against the fp32 oracle.

Covered: embed through the fp32 and uint8 entries (B/32, B/16); each of the 12 blocks on plain and outlier weights at
1, 2, 5, 23 frames and one block at a full 250-frame chunk; the class-token-only last block; the head on outlier,
near-zero-variance and constant rows; the VF_CLIP_ATTN=split and VF_CLIP_RESID=y / mix handles against the reference of
their own rounding; embed -> blocks -> head == encode_image bit for bit (eager and graph replay); attention on inputs
with scores of 50 .. 150, the maximum at chosen keys, equal scores, and frames of different scale side by side (fused,
split, and B/16's two-half kernel); the features at 8 and 270 frames.  Controls: a handle with bf16-rounded weights, and
the reference with P unrounded, eps 1e-6, a QuickGELU constant of 1.7 or one in_proj bias column group zeroed.

test_zz_report_measured prints the worst value per bar over the session (pytest -s).
"""
import os

import pytest
import torch
import torch.nn.functional as F

import split_engine_bars as bars
from oracle import clip_tower

pytestmark = pytest.mark.gpu

MEASURED = {}
MEAN = torch.tensor([0.48145466, 0.4578275, 0.40821073])
STD = torch.tensor([0.26862954, 0.26130258, 0.27577711])
ATT = frozenset({"qkv", "p", "att"})


def _transform_224(frames_u8):
    x = frames_u8.permute(0, 3, 1, 2).to(torch.float32).div(255)
    return x.sub(MEAN[None, :, None, None]).div(STD[None, :, None, None])


def _frames(n, seed):
    g = torch.Generator().manual_seed(seed)
    fr = torch.randint(0, 256, (n, 224, 224, 3), dtype=torch.uint8, generator=g)
    fr[n // 2 + 1:] = fr[n // 2 + 1:] // 4 + 96            # the later frames low-contrast
    return fr


def _state_dict(weights, patch):
    from video_features_b200 import synthetic_weights
    if weights == "outlier":
        return synthetic_weights.clip_vit_b32_state_dict(5, outliers=True, patch=patch)
    sd = clip_tower.synthetic_state_dict(0 if patch == 32 else 1, patch=patch)
    if weights == "bf16":                                   # every GEMM weight rounded to bf16 (8 mantissa bits)
        sd = {k: (v.bfloat16().float() if v.dim() >= 2 and "positional" not in k else v) for k, v in sd.items()}
    return sd


@pytest.fixture(scope="module")
def engines(cuda_device):
    """get(weights, patch, **env) -> (float64 state dict on the device, engine); the environment is read at create."""
    from video_features_b200.clip_engine import ClipEngine
    made = {}

    def get(weights="plain", patch=32, **env):
        key = (weights, patch, tuple(sorted(env.items())))
        if key not in made:
            sd = _state_dict(weights, patch)
            old = {k: os.environ.get(k) for k in env}
            os.environ.update(env)
            try:
                eng = ClipEngine(sd, device=0)
            finally:
                for k, v in old.items():
                    os.environ.pop(k, None) if v is None else os.environ.__setitem__(k, v)
            made[key] = ({k: v.double().to(cuda_device) for k, v in sd.items()}, eng)
        return made[key]
    yield get
    for _, eng in made.values():
        eng.close()


def _compare(key, what, got, want, bar):
    assert got.shape == want.shape, (what, tuple(got.shape), tuple(want.shape))
    err = bars.row_errors(got, want)
    print(f"{what}: rel-L2 {err[0]:.2e}, max-abs/max {err[1]:.2e} (bar {bar[0]:.1e} / {bar[1]:.1e})")
    if key:
        old = MEASURED.get(key, (0.0, 0.0))
        MEASURED[key] = (max(old[0], err[0]), max(old[1], err[1]))
    return err


def _block_ref(sd64, k, x, T, **kw):
    kw.setdefault("declared_rounding", True)
    return clip_tower.block(sd64, k, x.double().view(-1, T, 768), **kw).reshape(-1, 768)


# ------------------------------------------------------------------------------------------------------ embed

@pytest.mark.parametrize("n", [1, 3, 13])
@pytest.mark.parametrize("patch", [32, 16])
def test_embed_matches_float64(engines, cuda_device, patch, n):
    """1, 3 and 13 frames: 13 x 50 = 650 and 13 x 197 = 2561 rows end inside a LayerNorm block of 8 rows.  The worst
    row is taken over every token row, so the class-token rows, the first and last patch of each frame and the last
    frame of the ragged count are all held to the bar (and are printed on their own)."""
    sd64, eng = engines("plain", patch)
    T = eng.tokens
    u8 = _frames(n, 10 + n)
    f32 = _transform_224(u8).to(cuda_device)
    x = eng.debug_embed(f32)
    assert torch.equal(x, eng.debug_embed(u8.to(cuda_device))), "uint8 and fp32 entries must agree bit for bit"
    ref = clip_tower.embed(sd64, f32.double(), declared_rounding=True).reshape(-1, 768)
    bar = bars.CLIP_VIT["embed"]
    err = _compare("embed", f"embed B/{patch} n={n}", x, ref, bar)
    edge = torch.tensor([f * T + t for f in (0, n - 1) for t in (0, 1, T - 1)], device=cuda_device)
    _compare(None, "  class token / first / last patch of the first and last frame", x[edge], ref[edge], bar)
    assert bars.within(err, bar), err


# ------------------------------------------------------------------------------------------------------ blocks

def _run_blocks(name, key, sd64, eng, x, resid="acc"):
    """Every block on its own from the engine's stream at that depth; returns the failures and the stream before block 11."""
    T = eng.tokens
    fails = []
    for k in range(12):
        got = eng.debug_blocks(x, k, k + 1)
        ref = _block_ref(sd64, k, x, T, resid=resid)
        bar = bars.CLIP_VIT[key[0]][key[1]]
        if k == 11:         # the class-token-only last block against the block evaluated on all rows
            err = _compare(" ".join(key), f"{name} block 11 (class rows)", got[::T], ref[::T], bar)
        else:
            err = _compare(" ".join(key), f"{name} block {k}", got, ref, bar)
            x = got
        if not bars.within(err, bar):
            fails.append((k, err))
    return fails, x


@pytest.mark.parametrize("weights,patch,n", [("plain", 32, 1), ("plain", 32, 2), ("plain", 32, 5), ("plain", 32, 23),
                                             ("outlier", 32, 1), ("outlier", 32, 2), ("outlier", 32, 5), ("outlier", 32, 23),
                                             ("plain", 16, 3)])
def test_each_block_matches_float64(engines, cuda_device, weights, patch, n):
    """23 frames: 12 tiles x 12 heads = one tile past a wave of the fused kernel, and a ragged last tile.  The outlier
    weights carry residual peaks above 50: a one-pass variance or an fp16 residual stream would show there."""
    sd64, eng = engines(weights, patch)
    x0 = eng.debug_embed(_transform_224(_frames(n, 20 + n)).to(cuda_device))
    if weights == "outlier":
        assert float(x0.abs().max()) > 50.0
    key = ("block", weights + ("16" if patch == 16 else ""))
    fails, x11 = _run_blocks(f"{weights} B/{patch} n={n}", key, sd64, eng, x0)
    assert torch.equal(x11, eng.debug_blocks(x0, 0, 11)), "one call over blocks 0..10 == the same blocks one by one"
    assert not fails, fails


def test_one_block_at_a_full_chunk(engines, cuda_device):
    """250 frames (the balanced chunk of a 1000-frame call): several tiles per CTA in every kernel."""
    sd64, eng = engines("plain")
    n = 250
    x5 = eng.debug_blocks(eng.debug_embed(_transform_224(_frames(n, 7)).to(cuda_device)), 0, 5)
    bar = bars.CLIP_VIT["block"]["plain"]
    err = _compare("block plain", "plain n=250 block 5", eng.debug_blocks(x5, 5, 6), _block_ref(sd64, 5, x5, 50), bar)
    assert bars.within(err, bar), err


@pytest.mark.parametrize("weights", ["plain", "outlier"])
@pytest.mark.parametrize("mode", ["split", "y", "mix"])
def test_other_paths_match_their_own_rounding(engines, cuda_device, weights, mode):
    """VF_CLIP_ATTN=split and VF_CLIP_RESID=y / mix (separate handles: the environment is read at create), every block
    against the reference of that path's declared rounding (y / mix: the fp16 increments), the class-token-only last
    block included -- there the increment rows are compact and the stream rows strided.  The split path gives the bits
    of the fused one: both accumulate q, k, v over K in the same order and share the attention arithmetic."""
    env = {"VF_CLIP_ATTN": "split"} if mode == "split" else {"VF_CLIP_RESID": mode}
    resid = "acc" if mode == "split" else mode
    sd64, eng = engines(weights, 32, **env)
    _, fused = engines(weights)
    n = 5
    f32 = _transform_224(_frames(n, 31)).to(cuda_device)
    x0 = eng.debug_embed(f32)
    fails, x11 = _run_blocks(f"{mode} {weights} n={n}", ("block" if resid == "acc" else "block y", weights), sd64, eng, x0,
                             resid)
    y = eng.debug_head(eng.debug_blocks(x0, 0, 12))
    assert torch.equal(y, eng.encode_image(f32)), "embed -> blocks -> head == encode_image on this handle"
    if mode == "split":
        assert torch.equal(x11, fused.debug_blocks(x0, 0, 11)), "split == fused, bit for bit"
        assert torch.equal(y, fused.encode_image(f32))
    assert not fails, fails


# ------------------------------------------------------------------------------------------------------ head

@pytest.mark.parametrize("weights", ["plain", "outlier"])
def test_head_matches_float64(engines, cuda_device, weights):
    """ln_post + projection on the class rows of a strided stream whose other rows are NaN (a row read from the wrong
    place cannot hide): rows of an engine stream (outlier channels above 50 with the outlier weights), a row of variance
    1e-6 (eps = 1e-5 is ten times the variance: the reference with eps = 1e-6 misses the bar more than a thousandfold)
    and a constant row (variance exactly 0; its own bar, see split_engine_bars.CLIP_VIT)."""
    sd64, eng = engines(weights)
    T, n = eng.tokens, 6
    g = torch.Generator().manual_seed(3)
    x = torch.full((n * T, 768), float("nan"))
    stream = eng.debug_blocks(eng.debug_embed(_transform_224(_frames(4, 5)).to(cuda_device)), 0, 11).cpu()
    x[0:4 * T:T] = stream[0:4 * T:T]
    x[4 * T] = 1e-3 * torch.randn(768, generator=g)
    x[5 * T] = 0.5
    x = x.to(cuda_device)
    got = eng.debug_head(x)
    cls = x[::T].double()
    ref = clip_tower.head(sd64, cls, declared_rounding=True)
    _compare(None, f"  head {weights}, engine stream rows", got[:4], ref[:4], bars.CLIP_VIT["head"])
    errs = {"head": _compare("head", f"head {weights}, stream rows and the row of variance 1e-6", got[:5], ref[:5],
                             bars.CLIP_VIT["head"]),
            "head constant row": _compare("head constant row", f"head {weights}, constant row", got[5:], ref[5:],
                                          bars.CLIP_VIT["head constant row"])}
    assert all(bars.within(e, bars.CLIP_VIT[k]) for k, e in errs.items()), errs
    what, factor = bars.CLIP_VIT_CONTROLS["eps 1e-6"]
    ctl = _compare(None, "  control: reference with eps 1e-6", got[:5],
                   clip_tower.head(sd64, cls[:5], declared_rounding=True, eps=1e-6), bars.CLIP_VIT[what])
    assert what == "head" and bars.beyond(ctl, bars.CLIP_VIT[what], factor), ctl


# ------------------------------------------------------------------------------------------------------ composition

@pytest.mark.parametrize("patch", [32, 16])
def test_pieces_compose_to_encode_image_bit_for_bit(engines, cuda_device, patch):
    """The diagnostics run the shipped code: embed -> blocks(0, 12) -> head == encode_image, on the eager first call of
    a size and on the graph replays that follow its second call; the uint8 entries likewise."""
    sd64, eng = engines("plain", patch)
    u8 = _frames(7, 40).to(cuda_device)
    f32 = _transform_224(u8.cpu()).to(cuda_device)
    want = eng.debug_head(eng.debug_blocks(eng.debug_embed(f32), 0, 12))
    for call in ("eager", "capture", "replay"):
        assert torch.equal(eng.encode_image(f32), want), call
    assert torch.equal(eng.encode_frames_u8(u8), eng.debug_head(eng.debug_blocks(eng.debug_embed(u8), 0, 12)))
    assert torch.equal(eng.encode_frames_u8(u8), want)


def test_diagnostics_reject_bad_arguments(engines, cuda_device):
    """More frames than a chunk and bad layer ranges are refused by argument checks, before any launch."""
    _, eng = engines("plain")
    x = torch.zeros((257 * 50, 768), device=cuda_device)
    before = eng.launch_count
    for call in (lambda: eng.debug_blocks(x, 0, 1), lambda: eng.debug_head(x),
                 lambda: eng.debug_embed(torch.zeros((257, 3, 224, 224), device=cuda_device)),
                 lambda: eng.debug_blocks(x[:50], 3, 3), lambda: eng.debug_blocks(x[:50], -1, 2),
                 lambda: eng.debug_blocks(x[:50], 5, 13)):
        with pytest.raises(RuntimeError):
            call()
    assert eng.launch_count == before


# ------------------------------------------------------------------------------------------------------ attention

def _attention_ref(sd64, layer, x, T):
    p = f"visual.transformer.resblocks.{layer}."
    w = sd64[p + "attn.in_proj_weight"].half().double()
    qkv = F.linear(x.double(), w, sd64[p + "attn.in_proj_bias"]).view(-1, T, 2304)
    return qkv, clip_tower.attention_core(qkv, rounding=ATT).reshape(-1, 768)


@pytest.mark.parametrize("patch,n", [(32, 1), (32, 2), (32, 5), (32, 23), (16, 1), (16, 3), (16, 7)])
def test_attention_on_hard_inputs(engines, cuda_device, patch, n):
    """Frames scaled 4, 5, 3, 6 side by side (scores grow with the square: a row taken from the neighbouring frame cannot
    hide), one token row per frame times 4 so that the largest score of about a quarter of the (head, query) rows -- row
    maxima of 20 .. 100 at the median, several hundred at most -- falls on that key: key 0, the last key, a key of the first half and, at 197 tokens, a key of the second half (the
    running maximum then changes after the first half and the rescale runs).  Frame 1 has 50 / 197 identical rows: every
    score of a query row is equal.  Reference: float64 with fp16 q / k / v, P and output.  At these scores one flipped
    rounding of a q or k element moves a score by ~1e-2, which is what the bar consists of."""
    sd64, eng = engines("plain", patch)
    T = eng.tokens
    g = torch.Generator().manual_seed(50 + n)
    x = torch.randn(n, T, 768, generator=g)
    keys = [0, T - 1, 60, 150] if T > 64 else [0, T - 1, 25]
    for f in range(n):
        x[f] *= (4.0, 5.0, 3.0, 6.0)[f % 4]
        x[f, keys[f % len(keys)]] *= 4.0
    if n > 1:
        x[1] = x[1, 7]
    x = x.reshape(-1, 768).half().to(cuda_device)
    qkv, ref = _attention_ref(sd64, 3, x, T)
    q, k, _ = (t.view(n, T, 12, 64).transpose(1, 2) for t in qkv.half().double().split(768, dim=-1))
    s = q @ k.transpose(-1, -2) * 0.125
    for f in range(n):
        if n > 1 and f == 1:
            assert float((s[1].amax(-1) - s[1].amin(-1)).max()) < 1e-9, "frame 1: all scores of a row equal"
            continue
        hit = (s[f].argmax(-1) == keys[f % len(keys)]).double().mean().item()
        top = s[f].amax(-1).median().item()
        assert hit > 0.15 and 15.0 < top < 400.0, (f, hit, top)
    bar = bars.CLIP_VIT["attention hard"]
    split = eng.block_attention(3, x, fused=False)
    err = _compare("attention hard", f"hard attention B/{patch} n={n} split", split, ref, bar)
    if T == 50:
        fused = eng.block_attention(3, x, fused=True)
        assert torch.equal(fused, split), "fused == split, bit for bit"
    assert bars.within(err, bar), err


# ------------------------------------------------------------------------------------------------------ features

@pytest.mark.parametrize("n", [8, 270])
def test_features_match_the_declared_float64_tower(engines, cuda_device, n):
    """End to end, where the flips of 12 blocks compound and the later blocks amplify them: 6.5x a block's error and
    2.7x under the 1e-3 product gate (measured 3.7e-4; the declared-rounding tower run in fp32 on the CPU lies 3.3e-4
    from the float64 one, so this is what fp32 arithmetic between fp16 rounding points costs, not a kernel's error)."""
    sd64, eng = engines("plain")
    u8 = _frames(n, 60 + n)
    y = eng.encode_frames_u8(u8.to(cuda_device))
    ref = torch.cat([clip_tower.encode_image(sd64, _transform_224(u8[i:i + 54]).to(cuda_device), dtype=torch.float64,
                                             declared_rounding=True) for i in range(0, n, 54)])
    bar = bars.CLIP_VIT["features"]
    err = _compare("features", f"features n={n}", y, ref, bar)
    assert bars.within(err, bar), err


# ------------------------------------------------------------------------------------------------------ controls

def test_controls(engines, cuda_device):
    """Block 5 at 5 frames.  A handle built from bf16-rounded weights fails the block bar against the reference of the
    original weights and passes against that of its own.  The reference changed on the CPU side -- P left unrounded,
    eps 1e-6, a QuickGELU constant of 1.7, the last in_proj bias column group zeroed -- : the engine's error carries
    none of that change's direction (split_engine_bars.defect_share), and the zeroed bias group fails the attention bar
    (the engine's own ln_1 output through block_attention, fused and split)."""
    sd64, eng = engines("plain")
    sdb, engb = engines("bf16")
    T, k = 50, 5
    x = eng.debug_blocks(eng.debug_embed(_transform_224(_frames(5, 70)).to(cuda_device)), 0, k)
    got, ref = eng.debug_blocks(x, k, k + 1), _block_ref(sd64, k, x, T)
    bar = bars.CLIP_VIT["block"]["plain"]
    assert bars.within(_compare(None, "block 5", got, ref, bar), bar)

    what, factor = bars.CLIP_VIT_CONTROLS["bf16 weights"]
    gotb = engb.debug_blocks(x, k, k + 1)
    lost = _compare(None, "control: bf16-weight handle vs the original weights", gotb, ref, bar)
    kept = _compare(None, "control: bf16-weight handle vs its own weights", gotb, _block_ref(sdb, k, x, T), bar)
    assert what == "block" and bars.beyond(lost, bar, factor) and bars.within(kept, bar), (lost, kept)

    p = f"visual.transformer.resblocks.{k}."
    sdz = dict(sd64)
    sdz[p + "attn.in_proj_bias"] = sd64[p + "attn.in_proj_bias"].clone()
    sdz[p + "attn.in_proj_bias"][-8:] = 0                     # the last column group: v of head 11, dims 56..63
    variants = {"P unrounded": dict(rounding=clip_tower.DECLARED - {"p"}), "eps 1e-6": dict(eps=1e-6),
                "QuickGELU 1.7": dict(gelu=1.7), "in_proj bias group zeroed": dict(sd=sdz)}
    shares = {}
    for name, kw in variants.items():
        refd = _block_ref(kw.pop("sd", sd64), k, x, T, **kw)
        err = _compare(None, f"control: reference with {name}", got, refd, bar)
        shares[name] = bars.defect_share(got, ref, refd)
        print(f"  {err[0] / bar[0]:.1f}x / {err[1] / bar[1]:.1f}x the block bar; the engine carries {shares[name]:+.3f} of it")
    assert all(abs(s) < bars.CLIP_VIT_SHARE[0] for s in shares.values()), shares

    h = clip_tower._r16(clip_tower._ln_d(x.double(), sd64[p + "ln_1.weight"], sd64[p + "ln_1.bias"], clip_tower.LN_EPS))
    h16 = h.half()
    abar = bars.CLIP_VIT["attention"]
    what, factor = bars.CLIP_VIT_CONTROLS["in_proj bias group zeroed"]
    for fused in (True, False):
        a = eng.block_attention(k, h16, fused=fused)
        err = _compare("attention", f"attention of block 5 ({'fused' if fused else 'split'})", a, _attention_ref(sd64, k, h16, T)[1], abar)
        ctl = _compare(None, "  control: reference with the bias group zeroed", a, _attention_ref(sdz, k, h16, T)[1], abar)
        assert bars.within(err, abar) and what == "attention" and bars.beyond(ctl, abar, factor), (err, ctl)


def test_zz_report_measured():
    for key, (rel, mx) in sorted(MEASURED.items()):
        print(f"measured {key:<22s} rel-L2 {rel:.2e}  max-abs/max {mx:.2e}")
