"""A/B timing of the wgmma GEMM from one or more builds of the library on the CLIP tower's exact launches (development
aid), with cuBLAS (`a @ b.t()` in fp16) on the same shapes as a ceiling.
usage: gemm_ab.py libA.so [libB.so ...]

Rows (a 250-frame chunk of ViT-B/32): fc1 (fp16 out, bias + QuickGELU), out-proj and fc2 (fp32 reduce-add into the
residual stream through vf_gemm_f16_accumulate), patch-embed (fp32 out), each also at K = 64, where the time is mostly
the epilogue."""
import ctypes as C, sys, torch
torch.cuda.init()
QUICKGELU = 1
shapes = [  # name, M, N, K, mode (fp16 / acc / f32), bias, act
    ("fc1", 12500, 3072, 768, "fp16", True, QUICKGELU),
    ("out-proj", 12500, 768, 768, "acc", True, 0),
    ("fc2", 12500, 768, 3072, "acc", True, 0),
    ("patch-embed", 12250, 768, 3072, "f32", False, 0),
]
shapes += [(name + " K=64", M, N, 64, mode, bias, act) for (name, M, N, K, mode, bias, act) in shapes]
libs = []
for p in sys.argv[1:]:
    l = C.CDLL(p)
    l.vf_gemm_f16.restype = C.c_int
    l.vf_gemm_f16.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int,
                              C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]
    l.vf_gemm_f16_accumulate.restype = C.c_int
    l.vf_gemm_f16_accumulate.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int,
                                         C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]
    libs.append((p, l))


def timeit(fn, n=50):
    for _ in range(5): fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n): fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def cell(label, ms, flop):
    return f"{label}: {ms*1e3:7.1f} us {flop/ms/1e9:6.1f} TF"


for rep in range(2):
    for (name, M, N, K, mode, has_bias, act) in shapes:
        g = torch.Generator(device="cuda").manual_seed(0)
        a = (torch.randn(M, K, device="cuda", generator=g) * 0.1).half()
        b = (torch.randn(N, K, device="cuda", generator=g) * 0.1).half()
        bias = torch.randn(N, device="cuda", generator=g) if has_bias else None
        out = torch.zeros(M, N, device="cuda", dtype=torch.float16 if mode == "fp16" else torch.float32)
        stream = torch.cuda.current_stream().cuda_stream
        bptr = bias.data_ptr() if has_bias else None
        flop = 2.0 * M * N * K
        row = []
        for p, l in libs:
            if mode == "acc":
                def run():
                    assert l.vf_gemm_f16_accumulate(a.data_ptr(), K, b.data_ptr(), K, M, N, K, out.data_ptr(), N, bptr, None,
                                                    act, stream) == 0
            else:
                def run():
                    assert l.vf_gemm_f16(a.data_ptr(), K, b.data_ptr(), K, M, N, K, out.data_ptr(), N, int(mode == "f32"),
                                         bptr, None, act, stream) == 0
            row.append(cell(p, timeit(run), flop))
        c = torch.empty(M, N, device="cuda", dtype=torch.float16)
        row.append(cell("cuBLAS", timeit(lambda: torch.matmul(a, b.t(), out=c)), flop))
        print(f"{name:16s} {M}x{N}x{K} {mode:4s} | " + " | ".join(row), flush=True)
