"""Import the UNMODIFIED reference modules on CPU from the reference tree (SEEDX_REFERENCE, default /root/reference), where it exists.
Three import stubs are needed (SURVEY.md §8c): deepspeed, transformers.deepspeed, xformers.ops."""
import importlib
import os
import sys
import types

import torch
import torch.nn.functional as F

REF = os.environ.get("SEEDX_REFERENCE", "/root/reference")


def install_stubs():
    if "deepspeed" not in sys.modules:
        ds = types.ModuleType("deepspeed")
        ds.zero = types.SimpleNamespace(GatheredParameters=None)
        sys.modules["deepspeed"] = ds
    if "transformers.deepspeed" not in sys.modules:
        td = types.ModuleType("transformers.deepspeed")
        td.is_deepspeed_zero3_enabled = lambda: False
        sys.modules["transformers.deepspeed"] = td
    if "xformers" not in sys.modules:
        xf = types.ModuleType("xformers")
        xo = types.ModuleType("xformers.ops")

        class LowerTriangularMask:  # marker type, as in xformers
            pass

        def memory_efficient_attention(q, k, v, attn_bias=None, p=0.0, scale=None):
            # q,k,v: [B,S,H,D] -> exact softmax attention (xformers semantics)
            causal = isinstance(attn_bias, LowerTriangularMask)
            o = F.scaled_dot_product_attention(q.transpose(1, 2), k.transpose(1, 2), v.transpose(1, 2), is_causal=causal, scale=scale)
            return o.transpose(1, 2)

        xo.memory_efficient_attention = memory_efficient_attention
        xo.LowerTriangularMask = LowerTriangularMask
        xf.ops = xo
        sys.modules["xformers"] = xf
        sys.modules["xformers.ops"] = xo
    if REF not in sys.path:
        sys.path.insert(0, REF)
    # the reference's `src` is a namespace package (no __init__.py) while this repo ships a regular `src` shim package, which would win
    # the import regardless of sys.path order: bind `src` to the reference tree explicitly
    cur = sys.modules.get("src")
    if cur is None or list(getattr(cur, "__path__", [])) != [REF + "/src"]:
        for k in [k for k in sys.modules if k == "src" or k.startswith("src.")]:
            del sys.modules[k]
        pkg = types.ModuleType("src")
        pkg.__path__ = [REF + "/src"]
        sys.modules["src"] = pkg


def ref_module(dotted):
    install_stubs()
    m = importlib.import_module(dotted)
    assert m.__file__.startswith(REF + "/"), f"{dotted} resolved to {m.__file__}, not the reference"
    return m


def install_diffusers_stub():
    """diffusers (==0.25.0, requirements.txt:4) is not installable offline.  The reference's OWN pipeline file
    (src/models/detokenizer/pipeline_stable_diffusion_xl_t2i_edit.py) and adapter file only need a handful of names from it at import time and a
    tiny `DiffusionPipeline` base (module registry, progress bar, execution device).  These stand-ins carry NO arithmetic: UNet / VAE / scheduler
    objects are passed in by the caller (make_golden.py backs them with oracle/sdxl.py)."""
    import contextlib
    if "diffusers" in sys.modules and getattr(sys.modules["diffusers"], "_seedx_stub", False):
        return

    def mod(name, **attrs):
        m = types.ModuleType(name)
        m.__dict__.update(attrs)
        sys.modules[name] = m
        return m

    class _Any:
        def __init__(self, *a, **k):
            pass

    class VaeImageProcessor:
        def __init__(self, vae_scale_factor=8, **k):
            self.vae_scale_factor = vae_scale_factor

        def preprocess(self, image):          # diffusers: latents (4 channels) and tensors already in [-1, 1] pass through unchanged
            assert torch.is_tensor(image)
            return image

        def postprocess(self, image, output_type="pil"):
            return image

    class DiffusionPipeline:
        def register_modules(self, **kw):
            for k, v in kw.items():
                setattr(self, k, v)

        def register_to_config(self, **kw):
            self.config = types.SimpleNamespace(**kw)

        @property
        def _execution_device(self):
            return torch.device("cpu")

        def to(self, *a, **k):
            return self

        def maybe_free_model_hooks(self):
            pass

        @contextlib.contextmanager
        def progress_bar(self, total=None):
            yield types.SimpleNamespace(update=lambda *a: None)

    class Output:
        def __init__(self, images):
            self.images = images

    def randn_tensor(shape, generator=None, device=None, dtype=None):
        return torch.randn(shape, generator=generator, dtype=dtype)

    logging = types.SimpleNamespace(get_logger=lambda name: types.SimpleNamespace(warning=lambda *a, **k: None, info=lambda *a, **k: None))
    d = mod("diffusers", StableDiffusionXLPipeline=_Any, _seedx_stub=True)
    mod("diffusers.image_processor", PipelineImageInput=object, VaeImageProcessor=VaeImageProcessor)
    mod("diffusers.loaders", FromSingleFileMixin=type("FromSingleFileMixin", (), {}), StableDiffusionXLLoraLoaderMixin=type("L", (), {}),
        TextualInversionLoaderMixin=type("T", (), {}))
    mod("diffusers.models", AutoencoderKL=_Any, UNet2DConditionModel=_Any)
    mod("diffusers.models.attention_processor", AttnProcessor2_0=_Any, LoRAAttnProcessor2_0=_Any, LoRAXFormersAttnProcessor=_Any, XFormersAttnProcessor=_Any)
    mod("diffusers.models.lora", adjust_lora_scale_text_encoder=lambda *a, **k: None)
    mod("diffusers.schedulers", KarrasDiffusionSchedulers=_Any)
    mod("diffusers.utils", USE_PEFT_BACKEND=False, deprecate=lambda *a, **k: None, is_invisible_watermark_available=lambda: False,
        is_torch_xla_available=lambda: False, logging=logging, replace_example_docstring=lambda doc: (lambda f: f), scale_lora_layers=lambda *a, **k: None)
    mod("diffusers.utils.torch_utils", randn_tensor=randn_tensor)
    mod("diffusers.pipelines")
    mod("diffusers.pipelines.pipeline_utils", DiffusionPipeline=DiffusionPipeline)
    mod("diffusers.pipelines.stable_diffusion_xl")
    mod("diffusers.pipelines.stable_diffusion_xl.pipeline_output", StableDiffusionXLPipelineOutput=Output)
    return d
