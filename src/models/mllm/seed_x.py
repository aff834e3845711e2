"""`src.models.mllm.seed_x.ContinuousLVLM` -> H100 engine (reference: src/models/mllm/seed_x.py:22-234)."""
from seedx_b200.agent import BOI_TOKEN, EOI_TOKEN, IMG_TOKEN, ContinuousLVLM  # noqa: F401
