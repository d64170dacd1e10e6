"""VideoMAE clip-feature handle: Hugging Face ``VideoMAEForVideoClassification`` (Kinetics-400 fine-tuned ViT-S / B / L
with 16 x 16 patches, 2-frame tubelets, 16 frames at 224 px), the classifier's input
``fc_norm(last_hidden_state.mean(1))``, with the processor's transform fused into the u8 entry."""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass
from typing import Dict, Optional, Sequence, Tuple

import numpy as np
import torch

from ._lib import check, lib, named_tensors

T, CROP, TUBELET, PATCH = 16, 224, 2, 16
TOKENS = (T // TUBELET) * (CROP // PATCH) ** 2          # 1568
# hidden size -> (depth, heads, MLP width) of the fine-tuned checkpoints
SHAPES = {384: (12, 6, 1536), 768: (12, 12, 3072), 1024: (24, 16, 4096)}
FEATURE_TYPES = {"videomae_vits16": "videomae-small-finetuned-kinetics",
                 "videomae_vitb16": "videomae-base-finetuned-kinetics",
                 "videomae_vitl16": "videomae-large-finetuned-kinetics"}
WIDTHS = {"videomae_vits16": 384, "videomae_vitb16": 768, "videomae_vitl16": 1024}
# ImageNet's statistics, which the original VideoMAE normalises with.  The processor class itself defaults to
# (0.5, 0.5, 0.5) / (0.5, 0.5, 0.5); a checkpoint's preprocessor_config.json, when present, says which one it used.
IMAGENET_MEAN = (0.485, 0.456, 0.406)
IMAGENET_STD = (0.229, 0.224, 0.225)
PIL_BILINEAR = 2


@dataclass(frozen=True)
class VideoMAEConfig:
    """The fields of a checkpoint's config.json the engine reads."""
    hidden_size: int
    depth: int
    heads: int
    intermediate_size: int
    layer_norm_eps: float
    qkv_bias: bool
    id2label: Optional[Dict[int, str]] = None

    @staticmethod
    def from_dict(cfg: dict) -> "VideoMAEConfig":
        """Refuses, naming the field, whatever the engine does not build: a head dim other than 64, no mean pooling,
        another tubelet, patch, clip length or image size, another activation."""
        def get(key, default=None):
            v = cfg.get(key, default)
            if v is None:
                raise ValueError(f"VideoMAE config.json has no '{key}'")
            return v
        d, heads = int(get("hidden_size")), int(get("num_attention_heads"))
        if d % heads or d // heads != 64:
            raise ValueError(f"VideoMAE config.json: hidden_size {d} / num_attention_heads {heads} gives head dim "
                             f"{d / heads:g}; only head dim 64 is built (ViT-S, B and L)")
        if d not in SHAPES:
            raise ValueError(f"VideoMAE config.json: hidden_size {d} is not built (384, 768, 1024)")
        if not get("use_mean_pooling", True):
            raise ValueError("VideoMAE config.json: use_mean_pooling = false (a final layernorm and no fc_norm) is not "
                             "built; the Kinetics checkpoints pool by mean")
        for key, want in (("tubelet_size", TUBELET), ("num_frames", T), ("image_size", CROP), ("patch_size", PATCH),
                          ("num_channels", 3), ("hidden_act", "gelu")):
            if get(key, want) != want:
                raise ValueError(f"VideoMAE config.json: {key} = {cfg[key]!r} is not built ({want!r} is)")
        labels = cfg.get("id2label")
        return VideoMAEConfig(d, int(get("num_hidden_layers")), heads, int(get("intermediate_size")),
                              float(get("layer_norm_eps", 1e-12)), bool(get("qkv_bias", True)),
                              {int(k): str(v) for k, v in labels.items()} if labels else None)

    def class_names(self, n: int) -> Optional[list]:
        """The id2label names of classes 0 .. n-1, or None when the config does not name every one of them (HF fills a
        bare config with LABEL_i)."""
        if not self.id2label or any(i not in self.id2label for i in range(n)):
            return None
        names = [self.id2label[i] for i in range(n)]
        return None if all(v == f"LABEL_{i}" for i, v in enumerate(names)) else names


@dataclass(frozen=True)
class Preset:
    """The processor's transform: Resize(shortest_edge, Pillow ``resample``), center crop, rescale, Normalize."""
    mean: Tuple[float, float, float] = IMAGENET_MEAN
    std: Tuple[float, float, float] = IMAGENET_STD
    shortest_edge: int = CROP
    crop: int = CROP
    resample: int = PIL_BILINEAR

    @staticmethod
    def from_dict(cfg: Optional[dict]) -> "Preset":
        """preprocessor_config.json; None (no file) gives ImageNet's mean / std, the original VideoMAE's.  Refuses a
        resize, crop or filter other than the 224-px bilinear preset, and a rescale other than 1 / 255."""
        if cfg is None:
            return Preset()
        size, crop = cfg.get("size", {"shortest_edge": CROP}), cfg.get("crop_size", {"height": CROP, "width": CROP})
        edge = size.get("shortest_edge") if isinstance(size, dict) else size
        ch, cw = (crop.get("height"), crop.get("width")) if isinstance(crop, dict) else (crop, crop)
        p = Preset(tuple(float(v) for v in cfg.get("image_mean", IMAGENET_MEAN)),
                   tuple(float(v) for v in cfg.get("image_std", IMAGENET_STD)), edge, ch, int(cfg.get("resample", 2)))
        if p.shortest_edge != CROP or ch != CROP or cw != CROP:
            raise ValueError(f"VideoMAE preprocessor_config.json: size {size} / crop_size {crop} is not built "
                             f"(shortest_edge 224, crop 224 x 224)")
        if p.resample != PIL_BILINEAR:
            raise ValueError(f"VideoMAE preprocessor_config.json: resample {p.resample} is not built (2, bilinear)")
        if not cfg.get("do_rescale", True) or abs(float(cfg.get("rescale_factor", 1 / 255)) - 1 / 255) > 1e-12 or \
                not cfg.get("do_normalize", True) or not cfg.get("do_resize", True) or \
                not cfg.get("do_center_crop", True):
            raise ValueError("VideoMAE preprocessor_config.json: only resize, center crop, rescale 1 / 255 and "
                             "Normalize, all on, are built")
        if len(p.mean) != 3 or len(p.std) != 3:
            raise ValueError("VideoMAE preprocessor_config.json: image_mean / image_std need 3 values")
        return p


def sinusoid_table(n_position: int = TOKENS, d_hid: int = 768) -> np.ndarray:
    """VideoMAE's fixed positional table, (n_position, d_hid) fp32: float64 angles position / 10000^(2 (j // 2) / d),
    sin on even and cos on odd columns, rounded to fp32 once."""
    # each denominator as one scalar power, as the reference builds it element by element
    denom = np.array([np.power(10000, 2 * (j // 2) / d_hid) for j in range(d_hid)], dtype=np.float64)
    table = np.arange(n_position, dtype=np.float64)[:, None] / denom[None, :]
    table[:, 0::2] = np.sin(table[:, 0::2])
    table[:, 1::2] = np.cos(table[:, 1::2])
    return table.astype(np.float32)


def check_state_dict(sd: Dict[str, torch.Tensor], cfg: VideoMAEConfig) -> None:
    """Every tensor the engine reads, with its shape from the config; refuses the first missing or mis-shaped key."""
    d, f = cfg.hidden_size, cfg.intermediate_size
    want = {"videomae.embeddings.patch_embeddings.projection.weight": (d, 3, TUBELET, PATCH, PATCH),
            "videomae.embeddings.patch_embeddings.projection.bias": (d,),
            "fc_norm.weight": (d,), "fc_norm.bias": (d,)}
    for i in range(cfg.depth):
        p = f"videomae.encoder.layer.{i}."
        a = p + "attention.attention."
        want.update({a + "query.weight": (d, d), a + "key.weight": (d, d), a + "value.weight": (d, d),
                     p + "attention.output.dense.weight": (d, d), p + "attention.output.dense.bias": (d,),
                     p + "intermediate.dense.weight": (f, d), p + "intermediate.dense.bias": (f,),
                     p + "output.dense.weight": (d, f), p + "output.dense.bias": (d,)})
        for n in ("layernorm_before", "layernorm_after"):
            want.update({p + n + ".weight": (d,), p + n + ".bias": (d,)})
        if cfg.qkv_bias:
            want.update({a + "q_bias": (d,), a + "v_bias": (d,)})
        elif a + "q_bias" in sd or a + "v_bias" in sd:
            raise ValueError(f"VideoMAE checkpoint: tensor '{a}q_bias' / 'v_bias' present, but config.json has "
                             f"qkv_bias = false")
    for k, shape in want.items():
        if k not in sd:
            raise ValueError(f"VideoMAE checkpoint: missing tensor '{k}'")
        if tuple(sd[k].shape) != shape:
            raise ValueError(f"VideoMAE checkpoint: tensor '{k}' has shape {tuple(sd[k].shape)}, not {shape}")
    if f"videomae.encoder.layer.{cfg.depth}.layernorm_before.weight" in sd:
        raise ValueError(f"VideoMAE checkpoint: tensor 'videomae.encoder.layer.{cfg.depth}.layernorm_before.weight' "
                         f"beyond the config's {cfg.depth} layers")


class VideoMAEEngine:
    """``state_dict``: the HF keys (``videomae.*``, ``fc_norm.*``; ``classifier.*`` is ignored here), any float dtype;
    ``config``: the checkpoint's config.json as a dict; ``preset``: its transform.  ``max_clips``: the workspace, about
    31 MB per clip at ViT-B (vf_videomae_create); a larger call runs in chunks, one CUDA graph per chunk size."""

    def __init__(self, state_dict: Dict[str, torch.Tensor], config: dict, preset: Preset = Preset(), device: int = 0,
                 max_clips: int = 16):
        if not torch.cuda.is_available():
            raise RuntimeError("VideoMAEEngine needs a CUDA device (sm_90a); there is no CPU fallback")
        self.config = VideoMAEConfig.from_dict(config)
        check_state_dict(state_dict, self.config)
        self.device = torch.device("cuda", device)
        self.preset = preset
        c = self.config
        extra = {"position_embeddings": torch.from_numpy(sinusoid_table(TOKENS, c.hidden_size)),
                 "image_mean": torch.tensor(preset.mean, dtype=torch.float32),
                 "image_std": torch.tensor(preset.std, dtype=torch.float32)}
        keys = [(k, v) for k, v in state_dict.items() if k.startswith(("videomae.", "fc_norm."))]
        arr, n, keep = named_tensors(keys + list(extra.items()))
        cfg = (C.c_float * 6)(c.hidden_size, c.depth, c.heads, c.intermediate_size, c.layer_norm_eps, float(c.qkv_bias))
        h = C.c_void_p()
        check(lib().vf_videomae_create(C.byref(h), arr, n, cfg, device, max_clips))
        self._h = h
        del keep
        info = (C.c_int * 5)()
        check(lib().vf_videomae_info(self._h, info))
        self.out_dim, self.depth, self.heads, self.hidden, self.max_clips = tuple(info)
        self.T = T

    def _stream(self) -> int:
        return torch.cuda.current_stream(self.device).cuda_stream

    def forward_f32(self, x: torch.Tensor) -> torch.Tensor:
        """x: (n, 16, 3, 224, 224) fp32 (the processor's pixel_values) on this device -> (n, D) fp32."""
        if not x.is_cuda:
            raise RuntimeError("VideoMAEEngine expects CUDA input (no CPU fallback)")
        x = x.to(torch.float32).contiguous()
        assert x.dim() == 5 and tuple(x.shape[2:]) == (3, CROP, CROP), x.shape
        out = torch.empty((x.shape[0], self.out_dim), device=x.device, dtype=torch.float32)
        with torch.cuda.device(self.device):
            check(lib().vf_videomae_forward_f32(self._h, x.data_ptr(), x.shape[0], x.shape[1], out.data_ptr(),
                                                self._stream()))
        return out

    def forward_u8(self, frames: torch.Tensor, starts: Sequence[int], T: int = T, out: torch.Tensor = None) -> torch.Tensor:
        """frames: (F, H, W, 3) uint8 BGR decoded frames of any size on this device; clip i is frames
        ``starts[i] .. starts[i] + 15`` -> (len(starts), D) fp32.  Asynchronous on the current stream.  ``out``: an
        optional (len(starts), D) fp32 device tensor to write into."""
        if not frames.is_cuda:
            raise RuntimeError("VideoMAEEngine expects CUDA frames (no CPU fallback)")
        assert frames.dtype == torch.uint8 and frames.dim() == 4 and frames.shape[3] == 3, frames.shape
        frames = frames.contiguous()
        nf, hh, ww, _ = frames.shape
        n = len(starts)
        st = (C.c_int * max(n, 1))(*[int(s) for s in starts])
        if out is None:
            out = torch.empty((n, self.out_dim), device=frames.device, dtype=torch.float32)
        assert out.is_contiguous() and tuple(out.shape) == (n, self.out_dim) and out.dtype == torch.float32
        with torch.cuda.device(self.device):
            check(lib().vf_videomae_forward_u8(self._h, frames.data_ptr(), nf, hh, ww, st, n, T, out.data_ptr(),
                                               self._stream()))
        return out

    # ---- diagnostics (eager, the caller's stream)
    def tubelets_u8(self, frames: torch.Tensor, starts: Sequence[int]) -> torch.Tensor:
        """(F, H, W, 3) uint8 BGR -> (len(starts), 1568, 1536) fp16 tubelet rows."""
        frames = frames.contiguous()
        n = len(starts)
        out = torch.empty((n, TOKENS, 3 * TUBELET * PATCH * PATCH), device=self.device, dtype=torch.float16)
        st = (C.c_int * n)(*[int(s) for s in starts])
        with torch.cuda.device(self.device):
            check(lib().vf_videomae_debug_tubelets_u8(self._h, frames.data_ptr(), frames.shape[0], frames.shape[1],
                                                      frames.shape[2], st, n, out.data_ptr(), self._stream()))
        return out

    def tubelets_f32(self, x: torch.Tensor) -> torch.Tensor:
        """(n, 16, 3, 224, 224) fp32 -> (n, 1568, 1536) fp16 tubelet rows."""
        x = x.to(torch.float32).contiguous()
        out = torch.empty((x.shape[0], TOKENS, 3 * TUBELET * PATCH * PATCH), device=self.device, dtype=torch.float16)
        with torch.cuda.device(self.device):
            check(lib().vf_videomae_debug_tubelets_f32(self._h, x.data_ptr(), x.shape[0], out.data_ptr(),
                                                       self._stream()))
        return out

    def embed(self, tubelets: torch.Tensor) -> torch.Tensor:
        """(n, 1568, 1536) fp16 -> the embedding (n, 1568, D) fp32."""
        tubelets = tubelets.to(torch.float16).contiguous()
        out = torch.empty((tubelets.shape[0], TOKENS, self.out_dim), device=self.device, dtype=torch.float32)
        with torch.cuda.device(self.device):
            check(lib().vf_videomae_debug_embed(self._h, tubelets.data_ptr(), tubelets.shape[0], out.data_ptr(),
                                                self._stream()))
        return out

    def blocks(self, x: torch.Tensor, begin: int, end: int) -> torch.Tensor:
        """Blocks [begin, end) on a copy of x (n, 1568, D) fp32."""
        y = x.to(torch.float32).contiguous().clone()
        with torch.cuda.device(self.device):
            check(lib().vf_videomae_debug_blocks(self._h, y.data_ptr(), y.shape[0], begin, end, self._stream()))
        return y

    def head(self, x: torch.Tensor) -> torch.Tensor:
        """fc_norm of the token mean of x (n, 1568, D) fp32 -> (n, D) fp32."""
        x = x.to(torch.float32).contiguous()
        out = torch.empty((x.shape[0], self.out_dim), device=self.device, dtype=torch.float32)
        with torch.cuda.device(self.device):
            check(lib().vf_videomae_debug_head(self._h, x.data_ptr(), x.shape[0], out.data_ptr(), self._stream()))
        return out

    def drop_lo(self) -> None:
        """Precision control: the lo half of every split-fp16 weight set to zero (plain fp16 weights), for good."""
        check(lib().vf_videomae_debug_drop_lo(self._h))

    @property
    def launch_count(self) -> int:
        return int(lib().vf_videomae_launch_count(self._h))

    def close(self):
        if getattr(self, "_h", None):
            lib().vf_videomae_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def attention(qkv: torch.Tensor, heads: int) -> torch.Tensor:
    """The blocks' wgmma attention alone (vf_videomae_attention): qkv (n, S, 3 heads 64) fp16 -> (n, S, heads 64)."""
    assert qkv.is_cuda and qkv.dtype == torch.float16 and qkv.dim() == 3 and qkv.shape[2] == 3 * heads * 64
    qkv = qkv.contiguous()
    n, S, _ = qkv.shape
    out = torch.empty((n, S, heads * 64), device=qkv.device, dtype=torch.float16)
    with torch.cuda.device(qkv.device):
        check(lib().vf_videomae_attention(qkv.data_ptr(), n, S, heads, out.data_ptr(),
                                          torch.cuda.current_stream().cuda_stream))
    return out
