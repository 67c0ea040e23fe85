"""x_clip_b200: H100-native (sm_90a) CLIP contrastive-training hot path behind the
lucidrains/x-clip `CLIP(...)` surface.  `import x_clip_b200 as x_clip` is the drop-in."""
from .clip import CLIP, TextTransformer, VisionTransformer, Unsupported  # noqa: F401

__all__ = ["CLIP", "TextTransformer", "VisionTransformer", "Unsupported"]
