"""`src.models.detokenizer.resampler.ResamplerXLV2` -> H100 engine (reference: src/models/detokenizer/resampler.py:226-286)."""
from seedx_b200.resampler_xl import ResamplerXLV2  # noqa: F401
