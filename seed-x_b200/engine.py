"""End-to-end engine: 448x448 image + prompt -> ViT -> LLaMA (prompt ending in <img>: 64 forced image tokens) -> output resampler ->
ResamplerXLV2 -> 50-step Euler/CFG SDXL UNet -> VAE -> 1024x1024 uint8 image, on one GPU, for a batch of independent requests.

This is the composition the reference's src/inference/eval_text2img_seed_x_i.py / eval_img2edit_seed_x_edit.py scripts perform
(SURVEY.md §3.5) expressed over the drop-in classes; bench.py drives it with synthetic full-size weights.
"""
import time

import torch

from . import synth, trace
from .adapter import SDXLAdapter, SDXLAdapterWithLatentImage
from .agent import ContinuousLVLM, Resampler
from .llm import LLAMA_13B, LlamaForCausalLM
from .resampler_xl import ResamplerXLV2
from .sdxl import SDXL_UNET, SDXL_VAE, AutoencoderKL, EulerDiscreteScheduler, UNet2DConditionModel
from .vit import VisionTransformerWithAttnPool

VIT_G = dict(width=1664, layers=48, heads=16, mlp_width=8192, output_dim=4096, n_queries=256, patch=14)


class SeedXEngine:
    def __init__(self, vit_cfg=None, llm_cfg=None, unet_cfg=None, vae_cfg=None, rxl_cfg=None, device_weights=True, vit_sd=None,
                 max_len=1024, log=None, edit=False, llm_weight_format="fp16", unet_weight_format="fp16"):
        """edit=True builds the SEED-X-Edit pipe (eval_img2edit_seed_x_edit.py): 8-channel conv_in UNet behind SDXLAdapterWithLatentImage and
        the VAE encoder for the source image.  llm_weight_format: "fp16" or "fp8_e4m3" (LlamaForCausalLM's weight_format: FP8 projection
        weights with per-row scales, half the bytes per decode step).  unet_weight_format: "fp16", "fp8_e4m3" or "fp8_e4m3_conv"
        (UNet2DConditionModel's weight_format: the transformer-block projections run as FP8 GEMMs with per-row scales; "fp8_e4m3_conv" also
        runs the ResnetBlock2D and upsampler 3x3 convs as FP8 convs with per-image scales)."""
        log = log or (lambda *a: None)
        t0 = time.time()
        vit_cfg = dict(VIT_G if vit_cfg is None else vit_cfg)
        llm_cfg = dict(LLAMA_13B if llm_cfg is None else llm_cfg)
        unet_cfg = dict(SDXL_UNET if unet_cfg is None else unet_cfg)
        if edit:
            unet_cfg["in_channels"] = 8
        self.edit = edit
        vae_cfg = dict(SDXL_VAE if vae_cfg is None else vae_cfg)
        rxl_cfg = dict(synth.RESAMPLER_XL if rxl_cfg is None else rxl_cfg)
        self.vit_cfg, self.llm_cfg = vit_cfg, llm_cfg
        if vit_sd is None:
            if device_weights:
                synth.set_device("cuda")
            vit_sd = synth.vit_state_dict(**vit_cfg)
        if device_weights:
            synth.set_device("cuda")
        try:
            self.vit = VisionTransformerWithAttnPool(image_size=448, patch_size=vit_cfg["patch"], width=vit_cfg["width"], layers=vit_cfg["layers"],
                                                     heads=vit_cfg["heads"], mlp_ratio=vit_cfg["mlp_width"] / vit_cfg["width"] + 1e-6,
                                                     n_queries=vit_cfg["n_queries"], output_dim=vit_cfg["output_dim"])
            self.vit.mlp_width = vit_cfg["mlp_width"]
            self.vit.load_state_dict(vit_sd)
            del vit_sd
            log(f"vit ready {time.time() - t0:.1f}s")
            self.llm = LlamaForCausalLM(llm_cfg, max_len=max_len, weight_format=llm_weight_format)
            self.llm.load_state_dict(synth.llama_state_dict(llm_cfg))
            log(f"llm ready {time.time() - t0:.1f}s")
            D, V = llm_cfg["hidden"], vit_cfg["output_dim"]
            heads_in = 32 if D == 5120 else 2
            heads_out = V // 128 if V >= 256 else 2
            self.agent = ContinuousLVLM.from_pretrained(llm=self.llm, input_resampler=Resampler(8, D, heads_in, V),
                                                        output_resampler=Resampler(8, V, heads_out, D), add_patch_pos=True, vit_down=True)
            self.agent.load_state_dict(synth.agent_state_dict(D, V))
            unet = UNet2DConditionModel(unet_cfg, weight_format=unet_weight_format)
            unet.load_state_dict(synth.unet_state_dict(unet_cfg))
            log(f"unet ready {time.time() - t0:.1f}s")
            self.vae = AutoencoderKL(vae_cfg)
            self.vae.load_state_dict({k: v for k, v in synth.vae_state_dict(vae_cfg).items()
                                      if edit or not k.startswith(("encoder.", "quant_conv"))})
            rxl = ResamplerXLV2(normalize=False, **rxl_cfg)
            rxl.load_state_dict(synth.resampler_xl_state_dict(rxl_cfg))
            if edit:
                self.adapter = SDXLAdapterWithLatentImage(unet=unet, resampler=rxl, vit_down=True)
                self.adapter.init_pipe(vae=self.vae, scheduler=EulerDiscreteScheduler(), visual_encoder=self.vit, image_transform=None)
            else:
                self.adapter = SDXLAdapter(unet=unet, resampler=rxl, vit_down=True)
                self.adapter.init_pipe(vae=self.vae, scheduler=EulerDiscreteScheduler(), visual_encoder=self.vit, image_transform=None)
        finally:
            synth.set_device("cpu")
        self.tok = synth.SynthTokenizer(vocab=llm_cfg["vocab"])
        log(f"engine ready {time.time() - t0:.1f}s")

    # ---- prompt layout (SURVEY.md A.2; eval_img2text_seed_x_i.py:142-162) ---------------------------------------------------
    def build_prompt(self, n_views, text_ids, force_image=True):
        t = self.tok
        img = "".join("<img_{:05d}>".format(i) for i in range(64))
        s = ("<patch>" + img + "</patch>") * (n_views - 1) + "<img>" + img + "</img>"
        ids = [t.bos_token_id] + t.encode("[INST] ") + t.encode(s) + list(text_ids) + t.encode(" [/INST]\n")
        if force_image:
            ids = ids + t.encode("<img>")          # the processor then emits <img_00000..00063></img> (eval_text2img_seed_x.py:23)
        ids_t = torch.tensor(ids)
        first = t.tok2id["<img_00000>"]
        mask = (ids_t >= first) & (ids_t < first + 64)
        return ids_t, mask

    def _ev(self):
        e = torch.cuda.Event(enable_timing=True)
        e.record()
        return e

    def _requests(self, feats, patch_pos, text_ids, n_views, extra_ids=None, force_image=True):
        reqs = []
        for b in range(len(text_ids)):
            ids, mask = self.build_prompt(n_views, text_ids[b], force_image=False)
            tail = (list(extra_ids[b]) if extra_ids is not None else []) + (self.tok.encode("<img>") if force_image else [])
            if tail:
                ids = torch.cat([ids, torch.tensor(tail, dtype=ids.dtype)])
                mask = torch.cat([mask, torch.zeros(len(tail), dtype=torch.bool)])
            reqs.append(dict(input_ids=ids.unsqueeze(0), image_embeds=feats[b * n_views:(b + 1) * n_views],
                             embeds_cmp_mask=torch.ones((n_views, 64), dtype=torch.bool), ids_cmp_mask=mask.unsqueeze(0),
                             patch_positions=patch_pos[b * n_views:(b + 1) * n_views]))
        return reqs

    def _image_feats(self, reqs):
        outs = self.agent.generate_batch(self.tok, reqs, max_new_tokens=66, suppress_eos=True)   # lock-step decode of the B requests
        if not all(o["has_img_output"] for o in outs):
            raise RuntimeError("the forced image span was not produced")
        return torch.cat([o["img_gen_feat"] for o in outs], dim=0)                # [B, 64, 4096] fp32

    def generate(self, views, patch_pos, text_ids, steps=50, guidance=7.5, noise=None, n_views=2, source_images=None, text_tokens=0):
        """views: float32 [B*n_views, 3, 448, 448] (host pinned or device); patch_pos [B*n_views, 2]; text_ids: list of B lists.
        Returns the uint8 device tensor [B, 1024, 1024, 3]; per-stage CUDA events are kept in self._events.
          source_images (edit engine): fp32 NCHW [B, 3, 1024, 1024] in [-1, 1] -> VAE encode -> 3-way CFG edit loop
            (eval_img2edit_seed_x_edit.py:137-149)
          text_tokens > 0 (eval_img2text_seed_x_i.py:169-176 followed by an image turn): the agent first answers with `text_tokens` free-running
            greedy tokens (kept in self.last_text_ids), then the image span is opened behind that answer and the image is generated."""
        B = len(text_ids)
        e0 = self._ev()
        trace.mark("start")
        feats = self.vit(views)                                                   # [B*n_views, 256, 4096] fp16
        e1 = self._ev()
        trace.mark("vit")
        extra = None
        if text_tokens:
            outs = self.agent.generate_batch(self.tok, self._requests(feats, patch_pos, text_ids, n_views, force_image=False),
                                             max_new_tokens=text_tokens, suppress_eos=True)
            extra = [o["ids"] for o in outs]
            self.last_text_ids = extra
            trace.mark("llm.text_answer")
        img_feats = self._image_feats(self._requests(feats, patch_pos, text_ids, n_views, extra_ids=extra))
        e2 = self._ev()
        if source_images is not None:
            if not self.edit:
                raise RuntimeError("source_images need SeedXEngine(edit=True)")
            u8 = self.adapter.generate(image_embeds=img_feats, latent_image=source_images, num_inference_steps=steps, guidance_scale=guidance,
                                       latents=noise, output_type="uint8")
        else:
            u8 = self.adapter.generate(image_embeds=img_feats, num_inference_steps=steps, guidance_scale=guidance, latents=noise,
                                       output_type="uint8")
        e3 = self._ev()
        self._events = (e0, e1, e2, e3)
        return u8

    def stage_ms(self):
        torch.cuda.synchronize()
        e0, e1, e2, e3 = self._events
        return dict(vit_ms=e0.elapsed_time(e1), llm_ms=e1.elapsed_time(e2), detok_ms=e2.elapsed_time(e3))
