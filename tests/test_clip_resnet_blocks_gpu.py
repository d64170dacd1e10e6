"""The CLIP ResNet towers Bottleneck by Bottleneck, and their attention pool kernel by kernel, against float64.

Every Bottleneck of RN50, RN101, RN50x4 and RN50x16 (115 blocks) runs on its own through ClipResNetEngine.debug_block
(the trunk's own kernels and buffers) on a split-fp16 pair input: the float64 trunk's real input to it, and for the
first and last block of every layer synthetic non-negative inputs with about half their elements exactly zero at n = 1,
3 (one frame scaled 50x: the bars are per frame) and max_frames.  The input is canonical (hi = fp16(v), lo = fp16(v -
hi)) and the reference reads exactly hi + lo.  The output, the residual branch (bn3's output before the add) and the
shortcut (the downsample's output) are each compared against a float64 block with the ORIGINAL weights, worst frame,
rel-L2 and max-abs / max; the error against float64 with the uploaded hi + lo weights is printed beside it, so the share
of the weights' subnormal lo halves is on record.  Every border row must be exactly zero: the next conv reads it as
padding.

The attention pool: the tokens bit for bit against a CPU float32 restatement of tokens_kernel; K|V, Q and c_proj
against float64 of the engine's own inputs; the attention core against a float64 softmax of the engine's own fp32 K|V
and Q, at each tower's T and n = 1, 3, max_frames, and through the stateless entry at T = 1 .. 257 and on hard inputs
(scores of +-30 .. +-100, exact ties for the maximum).

Composition: the stem (read_pairs 0) -> every debug_block -> debug_attnpool equals encode_image bit for bit, and the
chained layer outputs equal read_stage 1 .. 4.

Past layer1 the bars sit within 3 .. 10x of a lo half lost inside a block (clip_rn_block_bars.SEPARATION), so there
the engine must also carry at most a third of the direction of every single-fp16 defect (split_engine_bars.defect_share
against the exact-pair emulation, clip_rn_block_bars.SHARE).

Controls: one conv's weights pre-rounded to fp16 fail that block's branch or shortcut bar by its layer's SEPARATION,
carry their own direction, and leave every other block bit-identical; an input with its lo half dropped fails every
block by its layer's SEPARATION; K|V rounded to fp16 fails the attention-core bar tenfold.  Bars: tests/clip_rn_block_bars.py; test_zz_report_measured prints the session's worst values (pytest -s)."""
import pytest
import torch
import torch.nn.functional as F

import clip_rn_block_bars as rb
import split_engine_bars as bars
from oracle import clip_resnet

pytestmark = pytest.mark.gpu

TOWERS = list(clip_resnet.TOWERS)
MAX_FRAMES = 5
PARTS = ("branch", "shortcut", "out")
MEASURED = {}          # (tower, layer, part) -> worst (rel-L2, max-abs / max) against the original weights
MEASURED_UP = {}       # the same against the uploaded hi + lo weights
ATTN_MEASURED = {}     # attention-pool piece -> worst (rel-L2, max-abs / max)
SHARES = {}            # (tower, defect) -> largest |defect_share| of the intact engine over the session


def _f64(sd, dev):
    return {k: v.double().to(dev) for k, v in sd.items()}


def _uploaded(sd64):
    """The weights as the engine holds them: every conv weight replaced by fp16(w) + fp16(w - fp16(w)) (the
    difference in fp32), BatchNorm untouched."""
    out = dict(sd64)
    for k, v in sd64.items():
        if v.dim() == 4:
            w = v.float()
            hi = w.half()
            out[k] = hi.double() + (w - hi.float()).half().double()
    return out


def to_pairs(v):
    """float64 (n, C, S, S) -> (its exact hi + lo value, the pair volume (n, S + 2, S + 2, 2C), zero border)."""
    hi = v.half()
    lo = (v - hi.double()).half()
    n, c, s, _ = v.shape
    x = torch.zeros(n, s + 2, s + 2, 2 * c, dtype=torch.float16, device=v.device)
    x[:, 1:-1, 1:-1, :c] = hi.permute(0, 2, 3, 1)
    x[:, 1:-1, 1:-1, c:] = lo.permute(0, 2, 3, 1)
    return hi.double() + lo.double(), x


def from_pairs(y):
    """Pair volume (n, S + 2, S + 2, 2c) -> float64 (n, c, S, S) of hi + lo over the valid region."""
    c = y.shape[-1] // 2
    inner = y[:, 1:-1, 1:-1].double()
    return (inner[..., :c] + inner[..., c:]).permute(0, 3, 1, 2)


def border_nonzero(y):
    m = torch.ones(y.shape[:3], dtype=torch.bool, device=y.device)
    m[:, 1:-1, 1:-1] = False
    return int((y[m].view(torch.int16) != 0).sum())


def _record(store, key, e):
    old = store.get(key, (0.0, 0.0))
    store[key] = (max(old[0], e[0]), max(old[1], e[1]))


def layer_of(cfg, i):
    return clip_resnet.blocks(cfg)[i][2]


def check_block(tower, eng, sd64, sdu64, cfg, i, v, label, record=True):
    """Block i on v (float64 NCHW) -> (failures, {part: error}).  The engine's output, branch and shortcut against
    float64 with the original weights (recorded and asserted) and with the uploaded weights (recorded, printed)."""
    xv, x = to_pairs(v)
    out, branch, short = eng.debug_block(i, x)
    got = {"out": out, "branch": branch, "shortcut": short}
    with torch.no_grad():
        ref = dict(zip(("out", "branch", "shortcut"), clip_resnet.block(sd64, cfg, i, xv)))
        ref_up = dict(zip(("out", "branch", "shortcut"), clip_resnet.block(sdu64, cfg, i, xv)))
    L = layer_of(cfg, i)
    fails, errs = [], {}
    for part in PARTS:
        if got[part] is None:
            continue
        g = from_pairs(got[part])
        e, eu = bars.row_errors(g, ref[part]), bars.row_errors(g, ref_up[part])
        errs[part] = e
        if record:
            _record(MEASURED, (tower, L, part), e)
            _record(MEASURED_UP, (tower, L, part), eu)
        bar = rb.BLOCK[tower][L][part]
        print(f"{tower} {label} block {i} {part}: rel-L2 {e[0]:.2e}, max-abs/max {e[1]:.2e} (bar {bar[0]:.1e} / "
              f"{bar[1]:.1e}); uploaded weights {eu[0]:.2e} / {eu[1]:.2e}")
        if record and not bars.within(e, bar):
            fails.append((tower, label, i, part, e))
        nz = border_nonzero(got[part])
        if nz:
            fails.append((tower, label, i, part, "border", nz))
    if label == "real" and L > 0:
        # past layer1 the bars do not separate a lost lo half tenfold: the engine must carry at most SHARE[0] of the
        # direction of each single-fp16 defect, measured against the exact-pair emulation
        with torch.no_grad():
            clean = rb.emulated_block(sd64, cfg, i, xv)
            for d in rb.DEFECTS:
                if d[1] == "downsample.0" and not rb.has_downsample(sd64, cfg, i):
                    continue
                part = rb.PART[d[1]]
                share = bars.defect_share(from_pairs(got[part]), clean[part], rb.emulated_block(sd64, cfg, i, xv, d)[part])
                SHARES[(tower, d)] = max(SHARES.get((tower, d), 0.0), abs(share))
                if abs(share) > rb.SHARE[0]:
                    fails.append((tower, label, i, d, "share", share))
    return fails, errs


def synthetic(eng, i, n, seed, dev, scaled=None):
    """Non-negative, about half exactly zero, O(1): a post-ReLU-like block input; frame `scaled` times 50."""
    s_in, cin, _, _ = eng.block_geometry(i)
    g = torch.Generator().manual_seed(seed)
    v = torch.relu(torch.randn(n, cin, s_in, s_in, generator=g, dtype=torch.float64))
    if scaled is not None:
        v[scaled] *= 50
    return v.to(dev)


@pytest.fixture(scope="module", params=TOWERS)
def tower(request, cuda_device):
    """(name, engine, float64 weights, uploaded float64 weights, cfg, the float64 trunk's input to every block for two
    frames), once per tower."""
    from video_features_b200.clip_resnet_engine import ClipResNetEngine
    name = request.param
    sd = clip_resnet.stand_in_state_dict(name)
    cfg = clip_resnet.config(sd)
    eng = ClipResNetEngine(sd, 0, max_frames=MAX_FRAMES)
    sd64 = _f64(sd, cuda_device)
    x = clip_resnet.calibration_images(cfg["n_px"], seed=7, n=2).double().to(cuda_device)
    with torch.no_grad():
        ins = clip_resnet.block_inputs(sd64, x, cfg)
    yield name, eng, sd64, _uploaded(sd64), cfg, ins
    eng.close()


def test_every_block_matches_float64(tower, cuda_device):
    name, eng, sd64, sdu64, cfg, ins = tower
    fails = []
    ends = {j for L in range(4) for j in (sum(cfg["layers"][:L]), sum(cfg["layers"][:L + 1]) - 1)}
    for i in range(len(ins)):
        f, errs = check_block(name, eng, sd64, sdu64, cfg, i, ins[i], "real")
        fails += f
        # the same input with its lo half dropped: every block fails its output bar by its layer's SEPARATION
        _, x = to_pairs(ins[i].half().double())
        out = eng.debug_block(i, x)[0]
        with torch.no_grad():
            ref_o = clip_resnet.block(sd64, cfg, i, to_pairs(ins[i])[0])[0]
        e = bars.row_errors(from_pairs(out), ref_o)
        L = layer_of(cfg, i)
        bar = rb.BLOCK[name][L]["out"]
        print(f"{name} lo dropped block {i}: out {e[0]:.2e} / {e[1]:.2e} ({e[0] / bar[0]:.1f}x / {e[1] / bar[1]:.1f}x)")
        if not bars.beyond(e, bar, rb.SEPARATION[name][L]):
            fails.append((name, "lo dropped", i, e))
        if i in ends:
            for n, scaled in ((1, None), (3, 1), (MAX_FRAMES, None)):
                v = synthetic(eng, i, n, 1000 * i + n, cuda_device, scaled)
                fails += check_block(name, eng, sd64, sdu64, cfg, i, v, f"synthetic n={n}")[0]
    assert not fails, fails


def test_debug_block_rejects_bad_calls(cuda_device):
    from video_features_b200._lib import VfError, check, lib
    from video_features_b200.clip_resnet_engine import ClipResNetEngine
    sd = clip_resnet.stand_in_state_dict("RN50")
    eng = ClipResNetEngine(sd, 0, max_frames=2)
    x = torch.zeros(1, 114, 114, 128, dtype=torch.float16, device=cuda_device)
    with pytest.raises(ValueError):
        eng.debug_block(16, x)
    with pytest.raises(ValueError):
        eng.debug_block(0, x.float())
    with pytest.raises(ValueError):
        eng.debug_block(1, x)                                     # block 1 takes layer1's 56 x 56 x 256
    with pytest.raises(ValueError):
        eng.debug_block(0, torch.zeros(3, 114, 114, 128, dtype=torch.float16, device=cuda_device))
    with pytest.raises(ValueError):
        eng.debug_block(0, x.cpu())
    stream = torch.cuda.current_stream().cuda_stream
    y = torch.empty(1, 58, 58, 512, dtype=torch.float16, device=cuda_device)
    for block, n in ((-1, 1), (16, 1), (0, 0), (0, 3)):
        with pytest.raises(VfError, match="debug_block"):
            check(lib().vf_clip_rn_debug_block(eng._h, block, x.data_ptr(), n, y.data_ptr(), y.data_ptr(), None,
                                               stream))
    with pytest.raises(VfError, match="debug_attnpool"):
        check(lib().vf_clip_rn_debug_attnpool(eng._h, x.data_ptr(), 3, y.data_ptr(), stream))
    eng.close()


def test_read_stage_fails_after_a_debug_call(cuda_device):
    from video_features_b200._lib import VfError
    from video_features_b200.clip_resnet_engine import ClipResNetEngine
    sd = clip_resnet.stand_in_state_dict("RN50")
    eng = ClipResNetEngine(sd, 0, max_frames=2)
    x = clip_resnet.calibration_images(224, seed=3, n=2).to(cuda_device)
    launches = eng.launch_count
    y = eng.encode_image(x)
    per_call = eng.launch_count - launches
    first = [eng.read_stage(s).clone() for s in range(7)]
    x4 = eng.read_pairs(4)
    for call in (lambda: eng.debug_block(0, eng.read_pairs(0)), lambda: eng.debug_attnpool(x4)):
        call()
        for s in range(7):
            with pytest.raises(VfError) as e:
                eng.read_stage(s)
            assert e.value.code == 1
        with pytest.raises(VfError):
            eng.read_pairs(0)
        launches = eng.launch_count
        assert torch.equal(eng.encode_image(x), y)
        assert eng.launch_count - launches == per_call
        assert all(torch.equal(eng.read_stage(s), first[s]) for s in range(7))
    eng.close()


# ---- the attention pool
def tokens_f32(x4_pairs, pos):
    """CPU float32 restatement of tokens_kernel: per (frame, channel) the sequential row-major fp32 sum of hi + lo, an
    IEEE division by T - 1, + pos, then the split; token t = position t - 1 + pos[t].  -> (n, T, 2E) fp16 pairs."""
    y = x4_pairs[:, 1:-1, 1:-1].cpu()
    n, s, _, e2 = y.shape
    E = e2 // 2
    T = s * s + 1
    pos = pos.float().cpu()
    out = torch.empty(n, T, 2 * E, dtype=torch.float16)

    def put(t, v):
        hi = v.half()
        out[:, t, :E] = hi
        out[:, t, E:] = (v - hi.float()).half()
    acc = torch.zeros(n, E, dtype=torch.float32)
    for r in range(s):
        for c in range(s):
            xv = y[:, r, c, :E].float() + y[:, r, c, E:].float()
            acc = acc + xv
            t = r * s + c + 1
            put(t, xv + pos[t])
    put(0, acc / torch.tensor(T - 1, dtype=torch.float32) + pos[0])
    return out


def attention_ref(kv, q):
    """float64 softmax((q / 8) . k) v per head of 64 on the engine's own fp32 K|V (n, T, 2E) and Q (n, E) -> (n, E)."""
    n, T, e2 = kv.shape
    E = e2 // 2
    kv, q = kv.double(), q.double()
    k = kv[..., :E].reshape(n, T, E // 64, 64)
    v = kv[..., E:].reshape(n, T, E // 64, 64)
    s = torch.einsum("nhd,nthd->nht", (q * 0.125).reshape(n, E // 64, 64), k)
    return torch.einsum("nht,nthd->nhd", torch.softmax(s, -1), v).reshape(n, E)


def pair_value(p):
    E = p.shape[-1] // 2
    return p[..., :E].double() + p[..., E:].double()


def _attn_record(key, e, bar):
    _record(ATTN_MEASURED, key, e)
    print(f"attention pool {key}: rel-L2 {e[0]:.2e}, max-abs/max {e[1]:.2e} (bar {bar[0]:.1e} / {bar[1]:.1e})")
    return bars.within(e, bar)


@pytest.mark.parametrize("n", [1, 3, MAX_FRAMES])
def test_attention_pool_piece_by_piece(tower, cuda_device, n):
    name, eng, sd64, _, cfg, ins = tower
    a = "visual.attnpool."
    E, T = cfg["embed"], cfg["tokens"]
    # a layer4 input: the real trunk's last block output (two frames) for n <= 2, synthetic beyond
    with torch.no_grad():
        x4 = clip_resnet.block(sd64, cfg, len(ins) - 1, ins[-1])[0]
    if n > 2:
        g = torch.Generator().manual_seed(n)
        extra = torch.relu(torch.randn(n - 2, E, *x4.shape[2:], generator=g, dtype=torch.float64)).to(cuda_device)
        x4 = torch.cat([x4, extra])
    _, xp = to_pairs(x4[:n])
    r = eng.debug_attnpool(xp)
    fails = []
    # tokens, bit for bit
    want = tokens_f32(xp, sd64[a + "positional_embedding"])
    diff = int((r["tokens"].cpu().view(torch.int16) != want.view(torch.int16)).sum())
    print(f"{name} n={n} tokens: {diff} differing halves of {want.numel()}")
    if diff:
        fails.append(("tokens", diff))
    tok = pair_value(r["tokens"])
    with torch.no_grad():
        kv = torch.cat([F.linear(tok, sd64[a + "k_proj.weight"], sd64[a + "k_proj.bias"]),
                        F.linear(tok, sd64[a + "v_proj.weight"], sd64[a + "v_proj.bias"])], -1)
        q = F.linear(tok[:, 0], sd64[a + "q_proj.weight"], sd64[a + "q_proj.bias"])
        core = attention_ref(r["kv"], r["q"])
        feats = F.linear(pair_value(r["att"]), sd64[a + "c_proj.weight"], sd64[a + "c_proj.bias"])
    for key, got, ref in (("kv", r["kv"], kv), ("q", r["q"], q), ("core", pair_value(r["att"]), core),
                          ("cproj", r["features"], feats)):
        if not _attn_record(key, bars.row_errors(got, ref), rb.ATTN[key]):
            fails.append((name, n, key))
    assert not fails, fails


def _kv_q(n, T, E, seed, dev, hard=False):
    g = torch.Generator().manual_seed(seed)
    kv = torch.randn(n, T, 2 * E, generator=g)
    q = torch.randn(n, E, generator=g)
    if hard:
        # per head: keys along +-q at 30 .. 100 / |q|^2 x 8, so scores (q / 8) . k spread over +-30 .. +-100, and the
        # first key copied to the last position with the largest score: an exact tie for the maximum
        qh = q.reshape(n, 1, E // 64, 64)
        mag = (torch.rand(n, T, E // 64, 1, generator=g) * 70 + 30) * torch.sign(torch.randn(n, T, E // 64, 1,
                                                                                             generator=g))
        k = qh * (8 * mag / (qh * qh).sum(-1, keepdim=True)) + 0.01 * torch.randn(n, T, E // 64, 64, generator=g)
        k[:, 0] = qh[:, 0] * (8 * 110 / (qh[:, 0] * qh[:, 0]).sum(-1, keepdim=True))
        if T > 1:
            k[:, T - 1] = k[:, 0]
        kv[..., :E] = k.reshape(n, T, E)
    return kv.to(dev), q.to(dev)


@pytest.mark.parametrize("T", [1, 2, 127, 128, 129, 256, 257])
@pytest.mark.parametrize("hard", [False, True])
def test_attention_core_stateless(cuda_device, T, hard):
    from video_features_b200._lib import debug_clip_rn_attention
    E = 128
    kv, q = _kv_q(3, T, E, T * 7 + hard, cuda_device, hard)
    out = debug_clip_rn_attention(kv, q)
    ref = attention_ref(kv, q)
    key = "core hard" if hard else "core"
    e = bars.row_errors(pair_value(out), ref)
    assert _attn_record(key, e, rb.ATTN[key]), (T, hard, e)
    # control: K|V rounded to fp16 fails the bar tenfold
    e16 = bars.row_errors(pair_value(debug_clip_rn_attention(kv.half().float(), q)), ref)
    print(f"attention T={T} hard={hard}: K|V in fp16 {e16[0]:.2e} / {e16[1]:.2e}")
    assert bars.beyond(e16, rb.ATTN[key], rb.KV_FP16_FACTOR), (T, hard, e16)


def test_attention_core_rejects_bad_shapes(cuda_device):
    from video_features_b200._lib import VfError, check, lib
    kv, q = _kv_q(1, 8, 64, 0, cuda_device)
    out = torch.empty(1, 128, dtype=torch.float16, device=cuda_device)
    stream = torch.cuda.current_stream().cuda_stream
    with pytest.raises(VfError, match="multiple of 64"):
        check(lib().vf_debug_clip_rn_attention(kv.data_ptr(), q.data_ptr(), 1, 8, 96, out.data_ptr(), stream))
    big = torch.zeros(1, 20000, 128, device=cuda_device)
    with pytest.raises(VfError, match="tokens"):
        check(lib().vf_debug_clip_rn_attention(big.data_ptr(), q.data_ptr(), 1, 20000, 64, out.data_ptr(), stream))
    with pytest.raises(VfError, match="tokens"):
        check(lib().vf_debug_clip_rn_attention(kv.data_ptr(), q.data_ptr(), 1, 0, 64, out.data_ptr(), stream))


# ---- composition
@pytest.mark.parametrize("n", [2, MAX_FRAMES])
def test_chained_pieces_equal_encode(cuda_device, n):
    from video_features_b200.clip_resnet_engine import ClipResNetEngine
    sd = clip_resnet.stand_in_state_dict("RN50")
    cfg = clip_resnet.config(sd)
    eng = ClipResNetEngine(sd, 0, max_frames=MAX_FRAMES)
    x = clip_resnet.calibration_images(224, seed=11, n=n).to(cuda_device)
    y = eng.encode_image(x)
    pairs = [eng.read_pairs(s).clone() for s in range(5)]
    stages = [eng.read_stage(s).clone() for s in range(5)]
    h = pairs[0]
    for i, (p, _, L) in enumerate(clip_resnet.blocks(cfg)):
        h = eng.debug_block(i, h)[0]
        if i + 1 == sum(cfg["layers"][:L + 1]):
            assert torch.equal(h.view(torch.int16), pairs[L + 1].view(torch.int16)), p
            assert torch.equal(from_pairs(h).float(), stages[L + 1]), p
    assert torch.equal(eng.debug_attnpool(h)["features"], y)
    eng.close()


# ---- controls
@pytest.mark.parametrize("ctl", rb.CONTROLS, ids=[f"{c[0]}-{c[1]}-{c[2][1]}" for c in rb.CONTROLS])
def test_control_fp16_weights_of_one_conv(cuda_device, ctl):
    """One conv's weights pre-rounded to fp16 (its W_lo pass multiplies zeros): that block fails its branch or shortcut
    bar by its layer's SEPARATION and carries its own defect direction (defect_share >= SHARE[1], the intact engine
    <= SHARE[0]); every other block is bit-identical to the intact engine's."""
    from video_features_b200.clip_resnet_engine import ClipResNetEngine
    name, block, defect, part = ctl
    sd = clip_resnet.stand_in_state_dict(name)
    cfg = clip_resnet.config(sd)
    key = f"{clip_resnet.blocks(cfg)[block][0]}.{defect[1]}.weight"
    bad_sd = dict(sd)
    bad_sd[key] = sd[key].half().float()
    eng = ClipResNetEngine(sd, 0, max_frames=1)
    bad = ClipResNetEngine(bad_sd, 0, max_frames=1)
    sd64 = _f64(sd, cuda_device)
    x = clip_resnet.calibration_images(cfg["n_px"], seed=7, n=1).double().to(cuda_device)
    with torch.no_grad():
        v = clip_resnet.block_inputs(sd64, x, cfg)[block]
    xv, xp = to_pairs(v)
    got = dict(zip(("out", "branch", "shortcut"), bad.debug_block(block, xp)))
    ok = dict(zip(("out", "branch", "shortcut"), eng.debug_block(block, xp)))
    with torch.no_grad():
        ref = dict(zip(("out", "branch", "shortcut"), clip_resnet.block(sd64, cfg, block, xv)))
        clean = rb.emulated_block(sd64, cfg, block, xv)[part]
        with_defect = rb.emulated_block(sd64, cfg, block, xv, defect)[part]
    L = layer_of(cfg, block)
    bar = rb.BLOCK[name][L]
    for p in PARTS:
        if got[p] is None:
            continue
        e = bars.row_errors(from_pairs(got[p]), ref[p])
        print(f"control {name} {key}: {p} {e[0]:.2e} / {e[1]:.2e} ({e[0] / bar[p][0]:.1f}x / {e[1] / bar[p][1]:.1f}x)")
    e = bars.row_errors(from_pairs(got[part]), ref[part])
    assert bars.beyond(e, bar[part], rb.SEPARATION[name][L]), e
    share_bad = bars.defect_share(from_pairs(got[part]), clean, with_defect)
    share_ok = bars.defect_share(from_pairs(ok[part]), clean, with_defect)
    print(f"control {name} {key}: defect_share {share_bad:+.3f}, intact engine {share_ok:+.3f}")
    assert share_bad >= rb.SHARE[1] and abs(share_ok) <= rb.SHARE[0], (share_bad, share_ok)
    for i in range(sum(cfg["layers"])):
        if i == block:
            continue
        _, xi = to_pairs(synthetic(eng, i, 1, 50 + i, cuda_device))
        a, b = eng.debug_block(i, xi), bad.debug_block(i, xi)
        assert all((u is None and w is None) or torch.equal(u.view(torch.int16), w.view(torch.int16))
                   for u, w in zip(a, b)), i
    eng.close()
    bad.close()


def test_zz_report_measured(cuda_device):
    """Prints the worst values over the session (pytest -s), against the original and the uploaded weights."""
    name = torch.cuda.get_device_name(0)
    try:
        import subprocess
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        pl = "unknown"
    print(f"measured on {name}, power limit {pl}")
    for k, (rel, mx) in sorted(MEASURED.items()):
        ru, mu = MEASURED_UP.get(k, (0.0, 0.0))
        print(f"measured worst {k[0]} layer{k[1] + 1} {k[2]}: rel-L2 {rel:.2e}, max-abs/max {mx:.2e}; "
              f"uploaded weights {ru:.2e} / {mu:.2e}")
    print("measured dict:", {k: (float(f"{v[0]:.3g}"), float(f"{v[1]:.3g}")) for k, v in sorted(MEASURED.items())})
    for (t, d), share in sorted(SHARES.items()):
        print(f"measured largest |defect_share| {t} {d[0]} {d[1]}: {share:.3f}")
    for k, (rel, mx) in sorted(ATTN_MEASURED.items()):
        print(f"measured worst attention pool {k}: rel-L2 {rel:.2e}, max-abs/max {mx:.2e}")
