"""Seeded stand-ins for the reference's pretrained checkpoints (i3d_rgb.pt, i3d_flow.pt, raft-sintel.pth), for machines
that do not have the real files: the tests always use them, bench.py falls back to them.  Test infrastructure, never
imported by the product."""
import os

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
# RAFT's refinement is contractive only with trained update weights: with the random stand-in every one of the 20
# iterations adds ~18 px and the flow runs off the image.  Attenuating the flow head by 0.01 brings the increments to the
# trained model's order (mean |flow| 0.55 px on the test clips, 1.2 px with raft-sintel.pth).  The factor is split
# as 0.1 on conv1 (weight and bias: ReLU is positively homogeneous) and 0.1 on conv2, so that no weight gets so small
# that the lo half of its split-fp16 form (~2^-12 of it) falls into the fp16 subnormals -- a scale trained weights
# never have.  The GRU's six gate convs are scaled by 0.3: the random recurrence is otherwise about twice as sensitive
# to perturbations as the trained one (max |flow| 2.0 px against 1.65 px with raft-sintel.pth).
_FLOW_HEAD = "module.update_block.flow_head."
_ATTENUATE = {("raft-sintel.pth", _FLOW_HEAD + "conv1.weight"): 0.1, ("raft-sintel.pth", _FLOW_HEAD + "conv1.bias"): 0.1,
              ("raft-sintel.pth", _FLOW_HEAD + "conv2.weight"): 0.1}
_ATTENUATE.update({("raft-sintel.pth", f"module.update_block.gru.conv{g}{i}.weight"): 0.3 for g in "zrq" for i in (1, 2)})


def state_dict(name: str) -> "dict[str, torch.Tensor]":
    """Seeded stand-in for one of the reference's pretrained checkpoints (i3d_rgb.pt, i3d_flow.pt, raft-sintel.pth):
    the same keys, shapes and dtypes, every tensor drawn with the mean and standard deviation of the trained tensor it
    replaces (tests/golden/checkpoint_stats.json; BatchNorm variances log-normal, so they stay positive; RAFT's flow head
    attenuated, see _ATTENUATE).  Each tensor
    has its own generator (seeded from its name), so the values do not depend on the order of the keys."""
    import json
    import math
    import zlib
    from collections import OrderedDict
    rows = json.load(open(os.path.join(GOLDEN, "checkpoint_stats.json")))[name]
    sd = OrderedDict()
    for key, shape, dtype, mean, std in rows:
        if dtype != "float32":
            sd[key] = torch.full(shape, int(round(mean)), dtype=getattr(torch, dtype))
            continue
        g = torch.Generator().manual_seed(zlib.crc32(f"{name}/{key}".encode()))
        z = torch.randn(shape, generator=g, dtype=torch.float64)
        if key.endswith("running_var"):
            s2 = math.log1p((std / mean) ** 2)
            v = torch.exp(math.log(mean) - s2 / 2 + math.sqrt(s2) * z)
        else:
            v = mean + std * z
        sd[key] = (v * _ATTENUATE.get((name, key), 1.0)).float()
    return sd
