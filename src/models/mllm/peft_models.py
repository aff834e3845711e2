"""`src.models.mllm.peft_models.get_peft_model_with_resize_embedding` -> H100 engine (reference: src/models/mllm/peft_models.py:27-106).
The LoRA adapters are merged into the packed fp16 weights at load time (seedx_b200/lora.py)."""
from seedx_b200.lora import LoraConfig, get_peft_model_with_resize_embedding  # noqa: F401
