"""`src.models.tokenizer.qwen_visual.*` -> H100 engine classes (reference: src/models/tokenizer/qwen_visual.py)."""
from seedx_b200.agent import Resampler  # noqa: F401
from seedx_b200.vit import VisionTransformerWithAttnPool  # noqa: F401
