"""video_features_b200 -- H100-native (sm_90a) engine for the per-frame / per-clip inference hot path of
Kamino666/video_features.  Host side mirrors the reference's Extract* classes; the compute lives in
libvfeat.so (hand-written CUDA behind a C ABI, see include/vfeat.h)."""
__version__ = "0.1.0"

from . import ops  # noqa: E402,F401  (registers the torch.library custom ops)
