"""The VideoMAE engine on the GPU against float64: the wgmma attention kernel against the float64 reference of its
declared rounding on random and hard inputs; the fused tubelet transform bit for bit against the f32 entry and the
processor's PIL preset; the embedding, every block on the float64 chain's own stream, the head and the feature against
the exact float64 forward (oracle/videomae_net.py) on seeded stand-ins; --show_pred's top-5 against the float64
head's; a graph replayed across calls."""
import numpy as np
import pytest
import torch

import attention_ref as A
import videomae_bars as B
from oracle import videomae_net as V

pytestmark = pytest.mark.gpu
NAMES = ("videomae_vits16", "videomae_vitb16", "videomae_vitl16")


def _errors(y, ref):
    y, ref = y.double().flatten(1), ref.double().flatten(1)
    rel = ((y - ref).norm(dim=1) / ref.norm(dim=1)).max().item()
    mx = ((y - ref).abs().amax(dim=1) / ref.abs().amax(dim=1)).max().item()
    return rel, mx


def _check(name, got, want, bar):
    assert torch.isfinite(got.float()).all(), name
    e = _errors(got, want)
    print(f"\n{name}: {e[0]:.2e} / {e[1]:.2e}  (bar {bar[0]:.1e} / {bar[1]:.1e})")
    assert e[0] <= bar[0] and e[1] <= bar[1], (name, e)
    return e


def _hard(S, heads, seed):
    """Clips of scores in the tens to hundreds, one dominant key each: key 0, the last key of the first 64-key block,
    the first of the second and the last key (dinov2_hard's scheme at any S); the last clip has identical rows."""
    g = torch.Generator().manual_seed(seed)
    keys = sorted({0, min(63, S - 1), min(64, S - 1), S - 1})
    D = heads * 64
    qkv = torch.randn(len(keys) + 1, S, 3 * D, generator=g)
    for f, key in enumerate(keys):
        qkv[f, :, :2 * D] *= 3.0 + f
        qkv[f, key, D:2 * D] *= 4.0
    qkv[-1, :, :2 * D] *= 4.0
    qkv[-1] = qkv[-1, min(7, S - 1)].clone()
    return qkv.half(), keys


@pytest.mark.parametrize("heads", [6, 12, 16])
@pytest.mark.parametrize("S", [1, 63, 64, 65, 1000, 1568, 2048])
def test_attention(cuda_device, S, heads):
    from video_features_b200.videomae_engine import attention
    g = torch.Generator().manual_seed(S * 31 + heads)
    rnd = (torch.randn(2, S, 3 * heads * 64, generator=g) * 1.5).half().cuda()
    _check(f"videomae attention S={S} heads={heads} random", attention(rnd, heads), A.dinov2(rnd, heads, key_block=64),
           B.BARS["attention"])
    qkv, keys = _hard(S, heads, 1000 * heads + S)
    qkv = qkv.cuda()
    if S >= 64:
        s = A.dinov2_scores(qkv[:-1], heads)
        assert s.amax().item() > 100.0
        for f, key in enumerate(keys):
            dominant = torch.zeros(S, dtype=torch.bool, device=s.device)
            dominant[key] = True
            hit, med = A.hardness(s[f], dominant)
            assert hit >= 0.05 and med > 15.0, (key, hit, med)
    got = attention(qkv, heads)
    _check(f"videomae attention S={S} heads={heads} hard (keys {keys}, identical rows)", got,
           A.dinov2(qkv, heads, key_block=64), B.BARS["attention hard"])
    assert torch.equal(got[-1], got[-1, :1].expand(S, -1)), "identical rows give identical outputs"


def test_attention_refuses_long_sequences(cuda_device):
    from video_features_b200.videomae_engine import attention
    with pytest.raises(RuntimeError, match="2048"):
        attention(torch.zeros(1, 2049, 3 * 64, dtype=torch.float16, device="cuda"), 1)


@pytest.fixture(scope="module")
def engines():
    from video_features_b200.videomae_engine import VideoMAEEngine
    made = {}

    def get(name):
        if name not in made:
            made[name] = VideoMAEEngine(V.stand_in_state_dict(name), V.config_dict(name), device=0, max_clips=2)
        return made[name]
    yield get
    for e in made.values():
        e.close()


def _f64(name):
    return V.prepare(V.stand_in_state_dict(name), torch.float64, "cuda")


def test_tubelets_u8_bits(cuda_device, engines):
    """u8 frames of an odd-margin size (240 x 321 -> 224 x 299, crop from column 37): the fused transform equals the
    f32 entry on the PIL preset's pixel_values, and both equal the oracle's tubelet rows rounded to fp16."""
    eng = engines("videomae_vits16")
    g = np.random.default_rng(5)
    frames = g.integers(0, 256, (20, 240, 321, 3), dtype=np.uint8)
    starts = [0, 4]
    got = eng.tubelets_u8(torch.from_numpy(frames).cuda(), starts)
    x = torch.stack([V.preset_clip(frames[s:s + 16]) for s in starts])
    f32 = eng.tubelets_f32(x.cuda())
    assert torch.equal(got, f32)
    assert torch.equal(f32.cpu(), V.tubelets(x).half())


@pytest.mark.parametrize("name", NAMES)
def test_embed_blocks_head_feature(cuda_device, engines, name):
    eng = engines(name)
    p = _f64(name)
    x = V.calibration_clips(0, 2).cuda()
    rows = V.tubelets(x).half()
    with torch.no_grad():
        emb = V.embed(p, rows.double())
        _check(f"{name} embed", eng.embed(rows), emb, B.BARS["embed"])
        h = emb
        for i in range(p["depth"]):
            nxt = V.block(p, i, h)
            got = eng.blocks(h.float(), i, i + 1)
            _check(f"{name} block {i} update", got.double() - h.float().double(), nxt - h.float().double(),
                   B.BARS["block"])
            h = nxt
        _check(f"{name} head", eng.head(h.float()), V.head(p, h.float().double()), B.BARS["head"])
        d = V.SHAPES[name][0]
        _check(f"{name} feature", eng.forward_f32(x), V.forward(p, x.double()), B.FEATURES[d])


def test_show_pred_top5(cuda_device, engines):
    from video_features_b200.class_head import ClassHead
    name = "videomae_vitb16"
    eng = engines(name)
    p = _f64(name)
    x = V.calibration_clips(3, 2).cuda()
    feat = eng.forward_f32(x)
    head = ClassHead.from_state_dict(V.stand_in_state_dict(name), ("classifier.weight", "classifier.bias"), 0, "t")
    top_idx = head.top_k_host(feat, 5)[0]
    ref = V.logits(p, V.forward(p, x.double())).softmax(-1).topk(5, -1).indices.cpu()
    assert torch.equal(torch.as_tensor(top_idx).long(), ref), (top_idx, ref)


def test_graph_reused_across_calls(cuda_device, engines):
    """The same clip count replays one graph: identical bits and launch counts on every call, and the f32 entry on the
    preset's pixel_values gives the same bits."""
    eng = engines("videomae_vits16")
    g = np.random.default_rng(9)
    frames = torch.from_numpy(g.integers(0, 256, (24, 256, 340, 3), dtype=np.uint8)).cuda()
    outs, counts = [], []
    for _ in range(3):
        c0 = eng.launch_count
        outs.append(eng.forward_u8(frames, [0, 8]).clone())
        counts.append(eng.launch_count - c0)
    torch.cuda.synchronize()
    assert all(torch.equal(o, outs[0]) for o in outs) and len(set(counts)) == 1, counts
    x = torch.stack([V.preset_clip(frames.cpu().numpy()[s:s + 16]) for s in (0, 8)]).cuda()
    assert torch.equal(eng.forward_f32(x), outs[0])


@pytest.mark.parametrize("name", ["videomae_vits16", "videomae_vitl16"])
def test_a_lost_lo_half_is_caught(cuda_device, name):
    """The engine with the lo half of every weight zeroed (plain fp16 weights) fails the embedding and feature bars by
    SEPARATION: the bars above would catch a split weight that lost its lo half."""
    from video_features_b200.videomae_engine import VideoMAEEngine
    eng = VideoMAEEngine(V.stand_in_state_dict(name), V.config_dict(name), device=0, max_clips=2)
    eng.drop_lo()
    p = _f64(name)
    x = V.calibration_clips(0, 2).cuda()
    rows = V.tubelets(x).half()
    with torch.no_grad():
        e_emb = _errors(eng.embed(rows), V.embed(p, rows.double()))
        e_feat = _errors(eng.forward_f32(x), V.forward(p, x.double()))
    eng.close()
    d = V.SHAPES[name][0]
    print(f"\n{name} lo halves dropped: embed {e_emb[0]:.2e} / {e_emb[1]:.2e}, feature {e_feat[0]:.2e} / {e_feat[1]:.2e}")
    for e, bar in ((e_emb, B.BARS["embed"]), (e_feat, B.FEATURES[d])):
        assert e[0] >= B.SEPARATION * bar[0] and e[1] >= B.SEPARATION * bar[1], (e, bar)
