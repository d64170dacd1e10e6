"""The MViT engine against the float64 oracle (oracle/mvit_net.py) at every read_stage tap and at the features, for the
v1_b and v2_s stand-ins with 1 and 3 clips per call (3 exceeds the 2-clip workspace: one call of 2 + 1); the u8 entry
against the f32 entry, graph replay against eager, and the pooling-attention, head-pooling and skip-pool kernels alone
on every block geometry of both variants against float64 / exactly, and a control with fp16-rounded weights."""
import pytest
import torch

from oracle import mvit_net as M
from mvit_bars import BARS, SEPARATION

pytestmark = pytest.mark.gpu

ATTN_BAR = (6e-4, 9e-4)
POOL_BAR = (1e-3, 1.5e-3)


def _errors(y, ref):
    """(worst per-clip rel-L2, worst per-clip max-abs / max) over the leading dimension."""
    y, ref = y.double().flatten(1), ref.double().flatten(1)
    rel = ((y - ref).norm(dim=1) / ref.norm(dim=1)).max().item()
    mx = ((y - ref).abs().amax(dim=1) / ref.abs().amax(dim=1)).max().item()
    return rel, mx


def _sd64(sd):
    return {k: (v.double() if v.is_floating_point() else v).cuda() for k, v in sd.items()}


@pytest.fixture(scope="module", params=list(M.MODELS))
def model(request):
    from video_features_b200.mvit_engine import MViTEngine
    name = request.param
    sd = M.stand_in_state_dict(name)
    eng = MViTEngine(sd, 0, max_clips=2)
    assert eng.name == name and eng.out_dim == 768 and eng.T == 16
    yield name, sd, _sd64(sd), eng
    eng.close()


@pytest.mark.parametrize("n", [1, 3])
def test_engine_vs_float64(cuda_device, model, n):
    name, sd, sd64, eng = model
    x = M.calibration_clips(n, n).cuda()
    y = eng.forward_f32(x)
    assert tuple(y.shape) == (n, 768)
    with torch.no_grad():
        ref, taps = M.forward(sd64, x.double(), taps=True)
    worst = {"features": _errors(y, ref)}
    last = 2 if n == 3 else 0                          # the stages hold the last chunk
    for i, st in enumerate(M.STAGES):
        got = eng.read_stage(i)
        want = taps[st][last:]
        assert got.shape == want.shape, (st, got.shape, want.shape)
        worst[st] = _errors(got, want)
    print(f"\n{name} n={n}: " + ", ".join(f"{k} {r:.2e}/{m:.2e}" for k, (r, m) in worst.items()))
    for k, (r, m) in worst.items():
        assert r <= BARS[k][0] and m <= BARS[k][1], (k, r, m)


def test_u8_entry_equals_f32_entry(cuda_device):
    from video_features_b200.mvit_engine import MViTEngine
    sd = M.stand_in_state_dict("mvit_v2_s")
    eng = MViTEngine(sd, 0, max_clips=2)
    g = torch.Generator().manual_seed(11)
    for hw in [(240, 320), (360, 270)]:
        bgr = torch.randint(0, 256, (24,) + hw + (3,), dtype=torch.uint8, generator=g)
        starts = [0, 5, 8]
        yu = eng.forward_u8(bgr.cuda(), starts)
        rgb = bgr.numpy()[..., ::-1].copy()
        x = torch.stack([M.transform(rgb[s:s + 16]) for s in starts]).cuda()
        yf = eng.forward_f32(x)
        assert torch.equal(yu, yf), hw
    eng.close()


def test_graph_replay_equals_eager(cuda_device, monkeypatch):
    from video_features_b200.mvit_engine import MViTEngine
    for name in M.MODELS:
        sd = M.stand_in_state_dict(name)
        x = M.calibration_clips(2, 2).cuda()
        eng = MViTEngine(sd, 0, max_clips=2)
        first, second = eng.forward_f32(x), eng.forward_f32(x)        # captured, then replayed
        eng.close()
        monkeypatch.setenv("VF_NO_GRAPH", "1")
        eager_eng = MViTEngine(sd, 0, max_clips=2)
        eager = eager_eng.forward_f32(x)
        eager_eng.close()
        monkeypatch.delenv("VF_NO_GRAPH")
        assert torch.equal(first, second) and torch.equal(second, eager), name


def test_refuses_other_clip_lengths(cuda_device):
    from video_features_b200._lib import VfError
    from video_features_b200.mvit_engine import MViTEngine
    eng = MViTEngine(M.stand_in_state_dict("mvit_v1_b"), 0, max_clips=1)
    with pytest.raises(VfError, match="16 frames"):
        eng.forward_f32(torch.zeros(1, 3, 8, 224, 224, device="cuda"))
    eng.close()


def test_refuses_other_shapes(cuda_device):
    from video_features_b200._lib import VfError
    from video_features_b200.mvit_engine import MViTEngine
    sd = M.stand_in_state_dict("mvit_v2_s")
    bad = dict(sd)
    bad["blocks.3.attn.rel_pos_h"] = torch.zeros(13, 96)
    with pytest.raises(VfError, match="blocks.3.attn.rel_pos_h"):
        MViTEngine(bad, 0, max_clips=1)
    bad = {k: v for k, v in sd.items() if not k.startswith("blocks.7.mlp.3")}
    with pytest.raises(VfError, match="blocks.7.mlp.3.weight"):
        MViTEngine(bad, 0, max_clips=1)
    bad = dict(M.stand_in_state_dict("mvit_v1_b"))
    bad["blocks.0.attn.qkv.weight"] = torch.zeros(3 * 192, 96)
    with pytest.raises(VfError, match="blocks.0.attn.qkv.weight"):
        MViTEngine(bad, 0, max_clips=1)
    eng = MViTEngine({"module." + k: v for k, v in sd.items()}, 0, max_clips=1)
    assert eng.name == "mvit_v2_s"
    eng.close()


# every block geometry of both variants: (q extent, kv extent, heads), T' = 8: blocks 0, 2, 4-13 and 15 hold 393 keys,
# the q-stride blocks 1, 3 and 14 pool k / v from the unstrided grid (1569 keys, streamed through shared memory)
ATTN_CASES = [(56, 7, 1), (28, 14, 2), (28, 7, 2), (14, 14, 4), (14, 7, 4), (7, 14, 8), (7, 7, 8)]


@pytest.mark.parametrize("v2", [False, True])
@pytest.mark.parametrize("S,K,heads", ATTN_CASES)
def test_pool_attention_vs_float64(cuda_device, S, K, heads, v2):
    from video_features_b200.mvit_engine import pool_attention
    g = torch.Generator().manual_seed(S * 10 + K * 1000 + heads + 100 * v2)
    c, n = heads * 96, 2 if S >= 28 else 3
    nq, nk = 1 + 8 * S * S, 1 + 8 * K * K
    # q as the column slice of qkv rows (v1's unpooled q) at S = 56, contiguous pooled rows otherwise
    qkv = (torch.randn(n, nq, 3 * c, generator=g)).half().cuda()
    q = qkv[..., :c] if S == 56 else qkv[..., :c].contiguous()
    k = torch.randn(n, nk, c, generator=g).half().cuda()
    v = torch.randn(n, nk, c, generator=g).half().cuda()
    rel = None
    if v2:
        sp = 2 * max(S, K) - 1
        rel = tuple((torch.randn(r, 96, generator=g) * 0.1).cuda() for r in (sp, sp, 15))
    y = pool_attention(q, k, v, (8, S, S), (8, K, K), rel, resid=v2)
    assert tuple(y.shape) == (n, nq, c)

    def heads_of(t):
        return t.double().reshape(t.shape[0], t.shape[1], heads, 96).transpose(1, 2)

    ref = M.attention(heads_of(q), heads_of(k), heads_of(v), (8, S, S), (8, K, K),
                      tuple(r.double() for r in rel) if rel else None, resid=v2)
    ref = ref.transpose(1, 2).reshape(n, nq, c)
    rel_err, mx = _errors(y, ref)
    print(f"\nattention q {S} kv {K} heads {heads} v2 {v2}: {rel_err:.2e}/{mx:.2e}")
    assert rel_err <= ATTN_BAR[0] and mx <= ATTN_BAR[1], (rel_err, mx)


# (input extent, stride, heads): the kv strides 8 / 4 / 2 / 1 and the q strides 2 and 1 of both variants
POOL_CASES = [(56, 8, 1), (56, 2, 1), (56, 1, 1), (28, 4, 2), (28, 2, 2), (28, 1, 2), (14, 2, 4), (14, 1, 4),
              (7, 1, 8), (56, 8, 2), (28, 4, 4), (14, 2, 8)]


@pytest.mark.parametrize("S,stride,heads", POOL_CASES)
def test_head_pool_vs_float64(cuda_device, S, stride, heads):
    from video_features_b200.mvit_engine import head_pool
    g = torch.Generator().manual_seed(S * 100 + stride * 10 + heads)
    c, n = heads * 96, 2
    rows = 1 + 8 * S * S
    qkv = torch.randn(n, rows, 3 * c, generator=g).half().cuda()
    src = qkv[..., c:2 * c]                                  # the k slice, read in place
    w = torch.randn(96, 1, 3, 3, 3, generator=g) / 27 ** 0.5
    gm, bt = torch.rand(96, generator=g) + 0.5, torch.randn(96, generator=g) * 0.1
    y = head_pool(src, (8, S, S), stride, w, gm, bt)
    sd = {"p.pool.weight": w.double().cuda(), "p.norm_act.0.weight": gm.double().cuda(),
          "p.norm_act.0.bias": bt.double().cuda()}
    x = src.double().reshape(n, rows, heads, 96).transpose(1, 2)
    ref, thw = M.head_pool(sd, "p", x, (8, S, S), stride)
    ref = ref.transpose(1, 2).reshape(n, -1, c)
    assert thw == (8, M.pooled(S, stride), M.pooled(S, stride)) and y.shape == ref.shape
    rel, mx = _errors(y, ref)
    assert rel <= POOL_BAR[0] and mx <= POOL_BAR[1], (rel, mx)


@pytest.mark.parametrize("S,C", [(56, 96), (56, 192), (28, 192), (28, 384), (14, 384), (14, 768)])
def test_skip_pool_exact(cuda_device, S, C):
    from video_features_b200.mvit_engine import skip_pool
    g = torch.Generator().manual_seed(S + C)
    x = torch.randn(2, 1 + 8 * S * S, C, generator=g).cuda()
    y = skip_pool(x, (8, S, S))
    assert torch.equal(y, M.skip_pool(x, (8, S, S)))


@pytest.mark.parametrize("name", list(M.MODELS))
def test_lost_lo_half_raises_the_error(cuda_device, name):
    """Control: every GEMM weight rounded to one fp16 value (its lo half zero, as a lost W_lo half or pass would leave
    it) raises the feature error on the same clips by SEPARATION.  scripts/precision/emulate_mvit.py predicts 2.1x (v1)
    and 2.0x (v2): the fp16 activations carry about half the engine's error, so a lost lo half roughly doubles it
    rather than clearing the bar by a wide margin (DESIGN.md §4.15, tests/test_mvit_bars_cpu.py)."""
    from video_features_b200.mvit_engine import MViTEngine
    sd = M.stand_in_state_dict(name)
    gemm_w = [k for k in sd if k.endswith("weight") and sd[k].dim() >= 2 and ".pool." not in k and k != "head.1.weight"]
    assert len(gemm_w) == 1 + 16 * 4 + 3          # patch conv, qkv / project.0 / mlp.0 / mlp.3, three projects
    hi = {k: (v.half().float() if k in gemm_w else v) for k, v in sd.items()}
    x = M.calibration_clips(1, 2).cuda()
    ys = []
    for w in (sd, hi):
        eng = MViTEngine(w, 0, max_clips=2)
        ys.append(eng.forward_f32(x))
        eng.close()
    with torch.no_grad():
        ref = M.forward(_sd64(sd), x.double())
    (rs, ms), (rh, mh) = _errors(ys[0], ref), _errors(ys[1], ref)
    print(f"\n{name} features: split weights {rs:.2e} / {ms:.2e}, fp16 weights {rh:.2e} / {mh:.2e}")
    assert rs <= BARS["features"][0] and rh >= SEPARATION * rs, (rs, rh)
