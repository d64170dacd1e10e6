"""Seeded wgmma GEMM launches in which every CTA runs several tiles, hashed bit for bit
(tests/test_gemm_epilogue_multitile_gpu.py against tests/golden/gemm_epilogue_multitile_sha256.json, written by
scripts/make_gemm_multitile_hashes.py).

The launches of tests/gemm_epilogue_cases.py run at most one tile per CTA, so they never reuse a staging buffer across
tiles.  These do: the CLIP tower's four GEMMs on a 250-frame chunk at full K and at K = 64, a reduce-add launch of
exactly three tiles per CTA (the two warpgroups of a ping-pong CTA then run different tile counts), and multi-tile
conv-mode launches with ReLU, the row mask and split output."""
import numpy as np
import torch

import conv_layout as cl
import gemm_epilogue_cases as gc

QUICKGELU = 1
# name, M, N, K, mode (f16 / f32 / acc), bias, scale, act
TOWER = [
    ("fc1", 12500, 3072, 768, "f16", True, False, QUICKGELU),
    ("out-proj", 12500, 768, 768, "acc", True, False, 0),
    ("fc2", 12500, 768, 3072, "acc", True, False, 0),
    ("patch-embed", 12250, 768, 3072, "f32", False, False, 0),
]
PLAIN = TOWER + [(name + "-k64", M, N, 64, mode, bias, scale, act) for (name, M, N, K, mode, bias, scale, act) in TOWER]
# 99 row blocks x 4 column tiles of 192 = 396 tiles = 3 per CTA on 132 SMs; K = 3 blocks + a tail of 8
PLAIN.append(("acc-3-tiles-per-cta", 6300, 768, 200, "acc", True, True, 0))
# 36000 rows of 128-row tiles x one 192-wide column tile = 282 tiles: 2 or 3 per CTA
CONV = cl._i3d3(64, 192, 4, 8, 28, "split")


def run_plain(l, name, M, N, K, mode, has_bias, has_scale, act, seed, dev) -> str:
    rng = np.random.default_rng(seed)
    a = torch.from_numpy((rng.standard_normal((M, K), dtype=np.float32) * 0.5).astype(np.float16)).to(dev)
    b = torch.from_numpy((rng.standard_normal((N, K), dtype=np.float32) * K ** -0.5).astype(np.float16)).to(dev)
    bias = torch.from_numpy(rng.standard_normal(N, dtype=np.float32)).to(dev) if has_bias else None
    scale = torch.from_numpy((1 + 0.1 * rng.standard_normal(N, dtype=np.float32))).to(dev) if has_scale else None
    bp = None if bias is None else bias.data_ptr()
    sp = None if scale is None else scale.data_ptr()
    stream = torch.cuda.current_stream(dev).cuda_stream
    ld = N + 8
    if mode == "acc":
        D = torch.from_numpy(rng.standard_normal((M + 8, ld), dtype=np.float32) * 3).to(dev)
        st = l.vf_gemm_f16_accumulate(a.data_ptr(), K, b.data_ptr(), K, M, N, K, D.data_ptr(), ld, bp, sp, act, stream)
    else:
        f32 = mode == "f32"
        D = torch.full((M + 8, ld), -3.5 if f32 else 7.0, dtype=torch.float32 if f32 else torch.float16, device=dev)
        st = l.vf_gemm_f16(a.data_ptr(), K, b.data_ptr(), K, M, N, K, D.data_ptr(), ld, int(f32), bp, sp, act, stream)
    assert st == 0, f"{name}: libvfeat error {st}"
    torch.cuda.synchronize(dev)
    return gc._sha(D)


def all_hashes(l, dev) -> dict:
    out = {}
    for i, case in enumerate(PLAIN):
        out[case[0]] = run_plain(l, *case, seed=1000 + i, dev=dev)
    for nsplit in (1, 2):
        out[f"conv-{CONV['id']}-nsplit{nsplit}-relu-mask-split"] = gc.run_conv(l, CONV, nsplit, 2000 + nsplit, dev)
    return out
