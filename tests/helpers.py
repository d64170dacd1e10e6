"""Shared test helpers (weights files, module trees).  Test infrastructure only."""
import os

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
from oracle.stand_in import state_dict as stand_in_state_dict  # noqa: E402,F401  (seeded stand-in checkpoints)

_CKPT_DIR = None


def checkpoint_dir() -> str:
    """A per-process directory holding the stand-in checkpoints under the reference's file names."""
    global _CKPT_DIR
    if _CKPT_DIR is None:
        import atexit
        import shutil
        import tempfile
        d = tempfile.mkdtemp(prefix="vf_ckpt_")
        atexit.register(shutil.rmtree, d, True)
        for n in ("i3d_rgb.pt", "i3d_flow.pt", "raft-sintel.pth"):
            torch.save(stand_in_state_dict(n), os.path.join(d, n))
        _CKPT_DIR = d
    return _CKPT_DIR


def checkpoint(name: str) -> str:
    """Path of the stand-in for the reference checkpoint `name` (see stand_in_state_dict)."""
    return os.path.join(checkpoint_dir(), name)


class _Node(torch.nn.Module):
    def forward(self, x):
        return x


def module_tree(state_dict) -> torch.nn.Module:
    """A module whose parameters carry exactly the dotted names of `state_dict` (for TorchScript archives shaped like
    the ones `clip.load` downloads)."""
    root = _Node()
    for key, value in state_dict.items():
        parts = key.split('.')
        m = root
        for p in parts[:-1]:
            if not hasattr(m, p):
                m.add_module(p, _Node())
            m = getattr(m, p)
        m.register_parameter(parts[-1], torch.nn.Parameter(value.clone(), requires_grad=False))
    return root
