"""Seeded wgmma GEMM launches whose outputs are hashed bit for bit (tests/test_gemm_epilogue_bits_gpu.py against
tests/golden/gemm_epilogue_sha256.json, written by scripts/make_gemm_epilogue_hashes.py).

Each launch goes through the C ABI of a given libvfeat.so, so the same cases run against any build of the library.
They cover every activation on fp16, fp32, split-fp16 and reduce-add outputs, with and without scale / bias, on each
of the four tile widths (three of them with an N tail inside the tile, all with a K tail), plus two conv-mode launches
with the row mask, ReLU and split output.  The output buffers are wider than N and longer than M, filled with a
sentinel, and hashed whole, so a write outside M x N changes the hash too."""
import ctypes as C
import hashlib

import numpy as np
import torch

import conv_layout as cl

ACT_NAMES = ["none", "quickgelu", "relu", "sigmoid", "tanh"]
# tile width -> (M, N) that the width rule of run_gemm (64-row ping-pong tiles) maps to it on a 132-SM H100
SHAPES = {64: (500, 200), 128: (6400, 120), 192: (4200, 376), 256: (8448, 248)}
MODES = ["f16", "f32", "split", "acc"]
K = 136                                      # two full K blocks and a tail of 8


def open_lib(path: str) -> C.CDLL:
    l = C.CDLL(path)
    p, i, f = C.c_void_p, C.c_int, C.c_void_p
    l.vf_gemm_f16.argtypes = [p, i, p, i, i, i, i, p, i, i, f, f, i, p]
    l.vf_gemm_f16_accumulate.argtypes = [p, i, p, i, i, i, i, p, i, f, f, i, p]
    l.vf_gemm_f16_split.argtypes = [p, i, p, i, i, i, i, p, i, i, f, f, i, p]
    l.vf_conv_gemm_f16.argtypes = [p, i, C.c_int64, p, i, i, i, p, i, C.c_uint64, i, p, p, i, i, i, f, f, i, p]
    for fn in (l.vf_gemm_f16, l.vf_gemm_f16_accumulate, l.vf_gemm_f16_split, l.vf_conv_gemm_f16):
        fn.restype = C.c_int
    return l


def tile_width(M: int, N: int, sms: int, bm: int = 64) -> int:
    """run_gemm's choice: the width whose busiest SM computes the fewest columns; the widest wins a tie."""
    num_m = -(-M // bm)
    best, bn = None, 256
    for cand in (256, 192, 128, 64):
        cost = -(-(num_m * -(-N // cand)) // sms) * cand
        if best is None or cost < best:
            best, bn = cost, cand
    return bn


def plain_cases():
    out = []
    for a in range(5):
        for mi, mode in enumerate(MODES):
            bn = (64, 128, 192, 256)[(a + mi) % 4]
            out.append(dict(name=f"{mode}-{ACT_NAMES[a]}-bn{bn}", mode=mode, act=a, bn=bn,
                            scale=(a + mi) % 2 == 0, bias=(a + mi) % 3 != 2, seed=100 * a + mi))
    # fc1's epilogue (bias + QuickGELU, fp16 out) at every width
    for bn in (64, 128, 192, 256):
        out.append(dict(name=f"f16-quickgelu-bias-bn{bn}", mode="f16", act=1, bn=bn, scale=False, bias=True, seed=bn))
    return out


CONV_CASES = [(cl.RAFT_CASES[0], 2, 3), (cl.I3D_CASES[2], 1, 4)]     # (case, nsplit, seed): ReLU, row mask, split out


def _sha(t: torch.Tensor) -> str:
    return hashlib.sha256(t.contiguous().cpu().numpy().tobytes()).hexdigest()


def _dev(x: np.ndarray, dev) -> torch.Tensor:
    return torch.from_numpy(x).to(dev)


def run_plain(l, case, dev) -> str:
    M, N = SHAPES[case["bn"]]
    rng = np.random.default_rng(case["seed"])
    a = _dev((rng.standard_normal((M, K)) * 0.5).astype(np.float16), dev)
    b = _dev((rng.standard_normal((N, K)) * K ** -0.5).astype(np.float16), dev)
    bias = _dev(rng.standard_normal(N).astype(np.float32), dev) if case["bias"] else None
    scale = _dev((1 + 0.1 * rng.standard_normal(N)).astype(np.float32), dev) if case["scale"] else None
    bp = None if bias is None else bias.data_ptr()
    sp = None if scale is None else scale.data_ptr()
    mode, act = case["mode"], case["act"]
    stream = torch.cuda.current_stream(dev).cuda_stream
    if mode == "split":
        off, ld = N + 8, 2 * N + 24
        D = torch.full((M + 8, ld), 7.0, dtype=torch.float16, device=dev)
        st = l.vf_gemm_f16_split(a.data_ptr(), K, b.data_ptr(), K, M, N, K, D.data_ptr(), ld, off, bp, sp, act, stream)
    elif mode == "acc":
        ld = N + 8
        D = _dev((rng.standard_normal((M + 8, ld)) * 3).astype(np.float32), dev)
        st = l.vf_gemm_f16_accumulate(a.data_ptr(), K, b.data_ptr(), K, M, N, K, D.data_ptr(), ld, bp, sp, act, stream)
    else:
        f32 = mode == "f32"
        ld = N + 8
        D = torch.full((M + 8, ld), -3.5 if f32 else 7.0, dtype=torch.float32 if f32 else torch.float16, device=dev)
        st = l.vf_gemm_f16(a.data_ptr(), K, b.data_ptr(), K, M, N, K, D.data_ptr(), ld, int(f32), bp, sp, act, stream)
    assert st == 0, f"{case['name']}: libvfeat error {st}"
    torch.cuda.synchronize(dev)
    return _sha(D)


def run_conv(l, case, nsplit, seed, dev) -> str:
    d = cl.build_case(case, nsplit, seed=seed)
    vol, f = d["vol"], d["f"]
    P, N, ctot, c0 = vol.P, case["N"], case["ctot"], case["c_off"]
    X, Wt = d["X"].to(dev), f["Wt"].to(dev)
    bias, scale = d["bias"].float().to(dev), d["scale"].float().to(dev)
    D = torch.full((P + 8, 2 * ctot), 7.0, dtype=torch.float16, device=dev)
    nt = f["ntaps"]
    taps = (C.c_int * nt)(*f["tap_off"])
    reg = (C.c_int * 9)(*vol.region())
    st = l.vf_conv_gemm_f16(X.data_ptr(), d["pitch"], P, Wt.data_ptr(), N, nt, f["k_per_tap"], taps, f["nsplit"],
                            f["lo_mask"], vol.row0, reg, D.data_ptr() + 2 * c0, 2 * ctot, 0, ctot, bias.data_ptr(),
                            scale.data_ptr(), d["act"], torch.cuda.current_stream(dev).cuda_stream)
    assert st == 0, f"{case['id']}: libvfeat error {st}"
    torch.cuda.synchronize(dev)
    return _sha(D)


def all_hashes(l, dev) -> dict:
    out = {}
    for case in plain_cases():
        out[case["name"]] = run_plain(l, case, dev)
    for case, nsplit, seed in CONV_CASES:
        out[f"conv-{case['id']}-nsplit{nsplit}-relu-mask-split"] = run_conv(l, case, nsplit, seed, dev)
    return out
