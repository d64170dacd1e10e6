"""Generates tests/golden/pwc_outputs.npz by running the REFERENCE's own PWC-Net module (models/pwc/pwc_src/pwc_net.py,
imported from the reference checkout, never copied) on the seeded stand-in weights.

Under the torch this project runs, the module needs three shims, each pinned by a test:
1. its version assert (pwc_net.py:21) parses "2.11.0+cu128" with int() and raises: it is given "1.2.0", the version
   the reference pins (conda_env_pwc.yml:60);
2. its cost volume (correlation.py) is CuPy-only and raises on the CPU: `correlation.FunctionCorrelation` is
   oracle.pwc_net.correlation, which tests/test_pwc_oracle_cpu.py holds to a literal float64 transcription of
   kernel_Correlation_updateOutput;
3. torch 1.2's grid_sample has no align_corners argument and behaves as align_corners=True; later releases default to
   False.  The module's grid_sample is called with align_corners=True.

    python scripts/make_pwc_golden.py            # needs the reference checkout ($VF_REFERENCE_DIR)
"""
import os
import sys
import types

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
REF = os.environ.get("VF_REFERENCE_DIR", "/root/reference")
OUT = os.path.join(ROOT, "tests", "golden", "pwc_outputs.npz")


def load_reference_pwc():
    """The reference's pwc_net module, executed from its source with the three shims above."""
    from oracle import pwc_net
    src = open(os.path.join(REF, "models", "pwc", "pwc_src", "pwc_net.py")).read()
    corr = types.ModuleType("models.pwc.pwc_src.correlation")
    corr.FunctionCorrelation = lambda tensorFirst, tensorSecond, device=None: pwc_net.correlation(tensorFirst, tensorSecond)
    saved = {k: sys.modules.get(k) for k in ("models", "models.pwc", "models.pwc.pwc_src", "models.pwc.pwc_src.correlation")}
    for name in ("models", "models.pwc", "models.pwc.pwc_src"):
        m = types.ModuleType(name)
        m.__path__ = []
        sys.modules[name] = m
    sys.modules["models.pwc.pwc_src.correlation"] = corr
    try:
        fn = types.SimpleNamespace(**{k: getattr(F, k) for k in dir(F) if not k.startswith("__")})
        fn.grid_sample = lambda *a, **k: F.grid_sample(*a, align_corners=True, **k)
        nn = types.SimpleNamespace(**{k: getattr(torch.nn, k) for k in dir(torch.nn) if not k.startswith("__")})
        nn.functional = fn
        shim_torch = types.SimpleNamespace(**{k: getattr(torch, k) for k in dir(torch) if not k.startswith("__")})
        shim_torch.nn = nn
        shim_torch.__version__ = "1.2.0"
        mod = types.ModuleType("models.pwc.pwc_src.pwc_net")
        mod.__dict__["torch"] = shim_torch
        src = src.replace("import torch\n", "")       # the module's own `import torch` would replace the shim
        exec(compile(src, os.path.join(REF, "models", "pwc", "pwc_src", "pwc_net.py"), "exec"), mod.__dict__)
    finally:
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v
    return mod


def golden_frames() -> torch.Tensor:
    """3 frames of 72 x 100 (neither a multiple of 64: the model's own resize runs), float in [0,255]."""
    from oracle import raft_net
    return raft_net.synthetic_frames(3, 72, 100, seed=21, shift=(1.6, -0.8))


def reference_flow(frames: torch.Tensor, sd) -> torch.Tensor:
    mod = load_reference_pwc()
    net = mod.PWCNet()
    net.load_state_dict(sd)
    net.eval()
    with torch.no_grad():
        return net(frames[:-1], frames[1:])


def main() -> None:
    from oracle import pwc_net
    sd = pwc_net.stand_in_state_dict()
    fr = golden_frames()
    flow = reference_flow(fr, sd)
    np.savez_compressed(OUT, frames=fr.numpy().astype(np.uint8), flow=flow.numpy())
    print("wrote", OUT, tuple(flow.shape), float(flow.abs().max()))


if __name__ == "__main__":
    main()
