"""``ExtractResNet`` -- drop-in for the reference's models/resnet/extract_resnet.py on the H100 engine.

Same constructor attributes / ``forward(indices)`` / ``extract(...)`` surface; output key ``feature_type`` is a float64
``(n_frames, D)`` array (D = 512 for resnet18/34, 2048 for resnet50/101/152; the reference builds it with ``.tolist()``)
plus 'fps' and 'timestamps_ms', saved under ``{output_path}/{feature_type}``.  Every frame is read as
base.FrameExtractor reads it; each chunk is resized on the GPU (Pillow-exact bilinear, short side 256), then runs the
fused BGR->RGB swap + CenterCrop(224) + ToTensor + Normalize + ResNet trunk (vf_resnet_forward_u8).
``--show_pred``: after every engine call the checkpoint's ``fc`` runs on its device features (class_head.py) and the
ImageNet top-5 of each frame is printed in frame order, as the reference prints per batch (extract_resnet.py:105-114).
"""
from __future__ import annotations

from typing import Dict

import torch

from .. import ops
from .._lib import VF_FILTER_BILINEAR
from ..class_head import FC_KEYS, ClassHead
from ..resnet_engine import DEPTHS, ResNetEngine
from ..utils import print_top_predictions
from .base import FRAMES_PER_CALL, FrameExtractor, load_first

RESIZE_SIZE = 256
CENTER_CROP_SIZE = 224
_STATE_DICTS: Dict[int, Dict[str, torch.Tensor]] = {}


def load_resnet_weights(depth: int) -> Dict[str, torch.Tensor]:
    """The first ``resnet{depth}-*.pth`` found in base.checkpoint_dirs(); read from disk once per process."""
    if depth not in _STATE_DICTS:
        _STATE_DICTS[depth] = load_first(f"resnet{depth}-*.pth")
    return _STATE_DICTS[depth]


class ExtractResNet(FrameExtractor):
    float64 = True

    def __init__(self, args):
        depth = int(args.feature_type[len("resnet"):]) if args.feature_type.startswith("resnet") else None
        if depth not in DEPTHS:
            raise NotImplementedError(args.feature_type)
        super().__init__(args)
        self.depth = depth
        self.batch_size = args.batch_size
        self.central_crop_size = CENTER_CROP_SIZE

    def _engine(self, device: torch.device) -> ResNetEngine:
        return self.per_device("engine", device, lambda idx: ResNetEngine(load_resnet_weights(self.depth), self.depth,
                                                                          idx, max_frames=FRAMES_PER_CALL))

    def _head(self, device: torch.device) -> ClassHead:
        return self.per_device("head", device, lambda idx: ClassHead.from_state_dict(
            load_resnet_weights(self.depth), FC_KEYS, idx, f"resnet{self.depth} checkpoint"))

    def encoder(self, device, preds):
        eng = self._engine(device)
        head = self._head(device) if self.show_pred else None

        def encode(x: torch.Tensor) -> torch.Tensor:
            h, w = x.shape[1:3]
            oh, ow = ops.resize_geometry(h, w, RESIZE_SIZE, True)
            if (oh, ow) != (h, w):
                x = torch.ops.vfeat.resize_u8(x, oh, ow, VF_FILTER_BILINEAR)      # ToPILImage -> Resize(256)
            y = eng.forward_u8(x)
            if head is not None:
                preds.submit([(head, y)], lambda tops: print_top_predictions(*tops[0], 'imagenet'))
            return y
        return encode
