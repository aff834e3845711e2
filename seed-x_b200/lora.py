"""LoRA-tuned checkpoints ("Inference with your own model", /root/reference/README.md:144-167).

The reference keeps the adapters un-merged at inference: ``configs/clm_models/llm_seed_x_lora.yaml`` builds
``get_peft_model_with_resize_embedding(model=LlamaForCausalLM, peft_config=LoraConfig(r=32, lora_alpha=32, target_modules=[q,k,v,o,gate,
down,up], modules_to_save=[input_layernorm, post_attention_layernorm, norm]), vocab_size=32330)``
(/root/reference/src/models/mllm/peft_models.py:27-106) and ``ContinuousLVLM.from_pretrained`` then loads the fine-tuned
``pytorch_model.bin`` whose ``llm.base_model.model.*`` keys carry ``lora_A.default`` / ``lora_B.default`` / ``modules_to_save.default``
tensors (PEFT 0.4.0 vendored under /root/reference/proj/peft; forward: ``W x + (alpha/r) B A x``, proj/peft/src/peft/tuners/lora.py:808-832).

Here the adapters are folded into the packed fp16 weights **once at load time** (``W' = W + (alpha/r) B A`` in fp32, rounded to fp16):
the decode loop is weight-bandwidth bound, so an un-merged path would add 2 extra launches and r·(in+out) extra weight bytes per
projection per token for the same result.  Dropout (0.05) is inactive in eval mode.
"""
import json
import os

import torch

from ._lib import SeedxError

PEFT_PREFIX = "base_model.model."
LLAMA_TARGETS = ("q_proj", "k_proj", "v_proj", "o_proj", "gate_proj", "up_proj", "down_proj")


class LoraConfig:
    """Stand-in for ``peft.LoraConfig`` (the `_target_` of llm_seed_x_lora.yaml:6-25): holds the hyper-parameters the merge needs."""

    def __init__(self, r=8, lora_alpha=8, target_modules=None, modules_to_save=None, lora_dropout=0.0, task_type=None, bias="none",
                 fan_in_fan_out=False, **kw):
        if bias != "none":
            raise SeedxError("LoRA bias training is not used by any SEED-X config")
        if fan_in_fan_out:
            raise SeedxError("fan_in_fan_out LoRA layers (Conv1D) do not occur in LLaMA")
        self.r, self.lora_alpha = int(r), float(lora_alpha)
        self.target_modules = list(target_modules) if target_modules is not None else list(LLAMA_TARGETS)
        self.modules_to_save = list(modules_to_save) if modules_to_save is not None else []
        self.lora_dropout, self.task_type = lora_dropout, task_type

    @property
    def scaling(self):
        return self.lora_alpha / self.r

    @classmethod
    def from_pretrained(cls, path):
        c = json.load(open(os.path.join(path, "adapter_config.json")))
        return cls(r=c["r"], lora_alpha=c["lora_alpha"], target_modules=c.get("target_modules"), modules_to_save=c.get("modules_to_save"),
                   lora_dropout=c.get("lora_dropout", 0.0), task_type=c.get("task_type"), bias=c.get("bias", "none"),
                   fan_in_fan_out=c.get("fan_in_fan_out", False))


def split_peft_state_dict(sd, adapter="default"):
    """Sort the keys of a PEFT-wrapped model's state dict (names as produced by PEFT 0.4.0 ``get_peft_model``; the adapter name may be
    absent, as in a saved ``adapter_model.bin``) into
      base   {hf_name: tensor}          plain parameters (``original_module.`` copies of modules_to_save are dropped)
      lora   {hf_module: (A [r,in], B [out,r])}
      saved  {hf_name: tensor}          ``modules_to_save`` replacements (they win over the base value)
    with the ``base_model.model.`` prefix removed."""
    base, saved, la, lb = {}, {}, {}, {}
    for k, v in sd.items():
        if k.startswith(PEFT_PREFIX):
            k = k[len(PEFT_PREFIX):]
        if ".lora_A." in k or ".lora_B." in k:
            mod, rest = k.split(".lora_A." if ".lora_A." in k else ".lora_B.")
            if rest not in ("weight", adapter + ".weight"):
                continue                                   # another adapter's weights
            (la if ".lora_A." in k else lb)[mod] = v
        elif ".modules_to_save." in k:
            mod, rest = k.split(".modules_to_save.")
            parts = rest.split(".")
            if len(parts) == 2 and parts[0] != adapter:
                continue
            saved[mod + "." + parts[-1]] = v
        elif ".original_module." in k:
            continue
        elif ".lora_embedding_" in k or ".lora_dropout." in k:
            raise SeedxError(f"unsupported LoRA parameter {k!r} (embedding adapters are not used by SEED-X)")
        else:
            base[k] = v
    if la.keys() != lb.keys():
        raise SeedxError("LoRA checkpoint has lora_A without lora_B (or the reverse): " + ", ".join(sorted(set(la) ^ set(lb))[:4]))
    return base, {m: (la[m], lb[m]) for m in la}, saved


def lora_delta(a, b, scaling):
    """(alpha/r) * B @ A in fp32 — the dense update PEFT's ``merge`` adds to ``weight`` (lora.py:798-806)."""
    if a.shape[0] != b.shape[1]:
        raise SeedxError(f"LoRA rank mismatch: A {tuple(a.shape)} vs B {tuple(b.shape)}")
    return (b.float() @ a.float()) * float(scaling)


def merge_lora_state_dict(sd, scaling, adapter="default"):
    """PEFT-named state dict that contains the base weights -> plain HF-named state dict with the adapters folded in (fp32)."""
    base, lora, saved = split_peft_state_dict(sd, adapter)
    out = dict(base)
    for mod, (a, b) in lora.items():
        w = mod + ".weight"
        if w not in out:
            raise SeedxError(f"LoRA pair for {mod} but no base weight in the same state dict; use LlamaForCausalLM.apply_peft_state_dict")
        out[w] = out[w].float() + lora_delta(a, b, scaling).to(out[w].device)
    out.update(saved)
    return out


def get_peft_model_with_resize_embedding(model, peft_config=None, model_id=None, vocab_size=None, torch_dtype="bf16"):
    """Factory behind ``configs/clm_models/llm_seed_x_lora.yaml`` (reference: peft_models.py:27-106).

    ``model``: a built LlamaForCausalLM or its `_target_` mapping.  Exactly one of ``peft_config`` (adapters arrive later with the agent
    checkpoint, README.md:150-160) and ``model_id`` (a PEFT adapter directory: adapter_config.json + adapter_model.bin/.safetensors, merged
    now) must be given.  ``vocab_size``: rows are appended to both embeddings — input rows = mean of the old rows, output rows = 3x the
    mean (peft_models.py:62-82).  ``torch_dtype`` is accepted for signature parity; operands are fp16."""
    if isinstance(model, dict) and "_target_" in model:
        from .compat import instantiate
        model = instantiate(model)
    if (peft_config is None) + (model_id is None) != 1:
        raise AssertionError("give exactly one of peft_config and model_id")           # the reference asserts (peft_models.py:57)
    if vocab_size is not None:
        model.resize_token_embeddings(int(vocab_size))
    if peft_config is not None:
        if isinstance(peft_config, dict):
            from .compat import instantiate
            peft_config = instantiate(peft_config) if "_target_" in peft_config else LoraConfig(**peft_config)
        model.peft_config = peft_config
    else:
        cfg = LoraConfig.from_pretrained(model_id)
        model.peft_config = cfg
        f = os.path.join(model_id, "adapter_model.safetensors")
        if os.path.exists(f):
            from safetensors.torch import load_file
            sd = load_file(f)
        else:
            sd = torch.load(os.path.join(model_id, "adapter_model.bin"), map_location="cpu")
        model.apply_peft_state_dict(sd)
    return model
