"""`src.models.mllm.modeling_llama_xformer.LlamaForCausalLM` -> H100 engine (reference: modeling_llama_xformer.py:612-779)."""
from seedx_b200.llm import LlamaForCausalLM  # noqa: F401
