"""`src.models.mllm.generation.AutoImageTokenGenerationProcessor` -> H100 engine (reference: src/models/mllm/generation.py:9-31)."""
from seedx_b200.agent import BOI_TOKEN, EOI_TOKEN, IMG_TOKEN  # noqa: F401
from seedx_b200.llm import AutoImageTokenGenerationProcessor  # noqa: F401
