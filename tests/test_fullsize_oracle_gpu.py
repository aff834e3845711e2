"""Oracle parity at BASELINE.json dimensions for the stages that dominate the step (VERDICT r01, 'what's weak' 1-4): the full-size SDXL UNet
sample-forward (128x128 latents, 64 x 2048 context, 4- and 8-channel conv_in), short full-size t2i / edit walks under the CUDA graph, the full-size
VAE decode (one 128x128 latent -> 1024x1024) and encode, four LLaMA layers at 13B width (hidden 5120, 40 heads, FFN 13824, vocab 32330; prefill
P=174 + 8 greedy tokens) and the full-width ViT at 448x448 (interpolated position tables).  The CPU side is oracle/ (the reference restated,
fp32) run on the GPU box's host cores: one UNet sample-forward is 6.75 TFLOP = 10-20 s of CPU, so these tests take a few CPU-minutes in total.

Weights are random-init at the real architecture sizes, drawn ON THE DEVICE in fp16 (seconds instead of minutes for 2.6 B parameters) and copied
to the host for the oracle, so both sides start from bit-identical fp16 values.  Tolerances are the ones of the small-config tests:
UNet eps <= 5e-3 and latents <= 1e-2 relative Frobenius (fp16 activations between layers, as the reference runs the UNet), decoded pixels
PSNR >= 40 dB, ViT features / LLM logits <= 1e-3, greedy ids exact."""
import math
import time

import pytest
import torch

from seedx_b200 import synth

pytestmark = pytest.mark.gpu
_ORACLE_CACHE = {}


def rel(a, b):
    return ((a.float().cpu() - b.float().cpu()).norm() / b.float().cpu().norm()).item()


def psnr(a, b):
    a = (a.float().cpu() / 2 + 0.5).clamp(0, 1)
    b = (b.float().cpu() / 2 + 0.5).clamp(0, 1)
    return 10 * math.log10(1.0 / max((a - b).pow(2).mean().item(), 1e-20))


@pytest.fixture(scope="module")
def cpu_threads():
    """the thread count at which torch's CPU GEMMs are fastest on this host (a container's os.cpu_count() can be 10x its real core budget)"""
    import bench
    n, avail = bench.pick_threads()
    print(f"[fullsize] oracle runs on {n} of {avail} schedulable CPUs")
    return n


def device_state_dict(fn, *a, **k):
    """draw a synthetic state dict on the GPU (fp16) and return (device dict, fp32 host copy for the oracle)"""
    synth.set_device("cuda")
    try:
        sd = fn(*a, **k)
    finally:
        synth.set_device("cpu")
    host = {kk: v.cpu().float() for kk, v in sd.items()}
    return sd, host


# ------------------------------------------------------------------------------------------------------------------------------------------
# SDXL UNet
# ------------------------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def full_unet(cpu_threads):
    from seedx_b200.sdxl import SDXL_UNET, UNet2DConditionModel
    cfg = dict(SDXL_UNET, in_channels=8)
    t0 = time.time()
    sd_dev, sd = device_state_dict(synth.unet_state_dict, cfg)
    # the image-latent half of the widened conv_in starts at zero and is fine-tuned to small values (adapter_modules.py:183-198)
    sd_dev["conv_in.weight"][:, 4:] *= 0.25
    sd["conv_in.weight"] = sd_dev["conv_in.weight"].float().cpu()
    m = UNet2DConditionModel(cfg)
    m.load_state_dict(sd_dev)
    del sd_dev
    torch.cuda.empty_cache()
    print(f"[fullsize] SDXL UNet ready in {time.time() - t0:.1f}s ({sum(v.numel() for v in sd.values()) / 1e9:.2f} B parameters)")
    return m, cfg, sd


def _unet_inputs(B, in_ch, tag):
    x = synth.randn(tag + "x", (B, in_ch, 128, 128))
    ctx = synth.randn(tag + "ctx", (B, 64, 2048))
    te = synth.randn(tag + "te", (B, 1280))
    tid = torch.tensor([[1024.0, 1024.0, 0.0, 0.0, 1024.0, 1024.0]]).repeat(B, 1)
    return x, ctx, te, tid


@pytest.mark.parametrize("in_ch", [8, 4])
def test_unet_full_size_sample_forward_matches_oracle(full_unet, in_ch):
    """one SDXL UNet sample-forward at BASELINE dimensions (pipeline_stable_diffusion_xl_t2i_edit.py:915-922): 128x128 latents, 64 x 2048 context,
    every GEMM / conv / attention / norm shape the bench runs (C = 320/640/1280, K up to 11 520, 10-deep transformers)."""
    from oracle import sdxl as osd
    m, cfg, sd = full_unet
    x, ctx, te, tid = _unet_inputs(1, in_ch, f"fs_unet{in_ch}_")
    sd_o, cfg_o = sd, cfg
    if in_ch == 4:   # the t2i UNet = the same weights with the 4-channel conv_in; on the device the partial checkpoint is merged in place
        sd_o = dict(sd, **{"conv_in.weight": sd["conv_in.weight"][:, :4].contiguous()})
        cfg_o = dict(cfg, in_channels=4)
        m.load_state_dict({"conv_in.weight": sd_o["conv_in.weight"]})
    try:
        t0 = time.time()
        with torch.no_grad():
            ref = osd.unet_forward(sd_o, cfg_o, x, 601.0, ctx, te, tid)
        t_cpu = time.time() - t0
        out = m(x.cuda(), 601.0, ctx.cuda(), added_cond_kwargs=dict(text_embeds=te.cuda(), time_ids=tid.cuda()))
    finally:
        if in_ch == 4:
            m.load_state_dict({"conv_in.weight": sd["conv_in.weight"]})
    e = rel(out, ref)
    print(f"full-size UNet sample-forward (in_channels={in_ch}): eps rel vs oracle = {e:.3e}  (oracle {t_cpu:.1f}s on the host)")
    assert torch.isfinite(out).all() and e < 5e-3, e


def _walk_inputs(tag):
    lat = synth.randn(tag + "lat", (1, 4, 128, 128))
    p, n = synth.randn(tag + "p", (1, 64, 2048)), synth.randn(tag + "n", (1, 64, 2048))
    pp, npool = synth.randn(tag + "pp", (1, 1280)), synth.randn(tag + "np", (1, 1280))
    return lat, p, pp, n, npool


def test_t2i_full_size_walk_under_the_cuda_graph_matches_oracle(full_unet):
    """4 Euler steps of the 2-way CFG loop (adapter_modules.py:156-167 -> StableDiffusionXLPipeline) at full size, UNet replayed as a CUDA graph
    exactly as adapter.generate runs it; the 8-channel engine input carries zeros in the image-latent half = the 4-channel t2i UNet."""
    from oracle import sdxl as osd
    from seedx_b200.sampler import DenoiseLoop
    from seedx_b200.sdxl import EulerDiscreteScheduler
    m, cfg, sd = full_unet
    lat, p, pp, n, npool = _walk_inputs("fs_t2i_")
    steps = 4
    sd4 = dict(sd, **{"conv_in.weight": sd["conv_in.weight"][:, :4].contiguous()})
    t0 = time.time()
    with torch.no_grad():
        ref = osd.t2i_sample(sd4, dict(cfg, in_channels=4), lat, p, pp, n, npool, steps=steps, guidance=7.5)
    t_cpu = time.time() - t0
    loop = DenoiseLoop(m, EulerDiscreteScheduler(), 1, (128, 128), 2, use_graph=True)
    tid = torch.tensor([[1024.0, 1024.0, 0.0, 0.0, 1024.0, 1024.0]]).repeat(2, 1).cuda()
    loop.set_condition(torch.cat([n, p]).cuda(), torch.cat([npool, pp]).cuda(), tid)
    out = loop.run(lat.cuda(), steps=steps, guidance=7.5).clone()
    assert loop.graph is not None
    again = loop.run(lat.cuda(), steps=steps, guidance=7.5)          # second request through the captured graph: bitwise repeatable
    assert torch.equal(out, again)
    e = rel(out, ref)
    print(f"full-size t2i walk, {steps} steps, CUDA graph: latents rel vs oracle = {e:.3e}  (oracle {t_cpu:.1f}s)")
    assert e < 1e-2, e


def test_edit_full_size_walk_under_the_cuda_graph_matches_oracle(full_unet):
    """3 steps of the edit loop (pipeline_stable_diffusion_xl_t2i_edit.py:884-963: [text, image, uncond], un-scaled source latents in channels
    4..7, sigma-space 3-way CFG) at full size with the UNet under the CUDA graph — the configuration adapter.generate(latent_image=...) uses."""
    from oracle import sdxl as osd
    from seedx_b200.sampler import DenoiseLoop
    from seedx_b200.sdxl import EulerDiscreteScheduler
    m, cfg, sd = full_unet
    lat, p, pp, n, npool = _walk_inputs("fs_edit_")
    img_lat = synth.randn("fs_edit_img", (1, 4, 128, 128), 4.0)       # un-scaled VAE-mode latents of a real image are O(1/0.13)
    steps = 3
    t0 = time.time()
    with torch.no_grad():
        ref = osd.edit_sample(sd, cfg, lat, img_lat, p, pp, n, npool, steps=steps, guidance=7.5, image_guidance=1.5)
    t_cpu = time.time() - t0
    loop = DenoiseLoop(m, EulerDiscreteScheduler(), 1, (128, 128), 3, use_graph=True)
    tid = torch.tensor([[1024.0, 1024.0, 0.0, 0.0, 1024.0, 1024.0]]).repeat(3, 1).cuda()
    loop.set_condition(torch.cat([p, n, n]).cuda(), torch.cat([pp, npool, npool]).cuda(), tid, image_latents=img_lat.cuda())
    out = loop.run(lat.cuda(), steps=steps, guidance=7.5, image_guidance=1.5)
    assert loop.graph is not None
    e = rel(out, ref)
    print(f"full-size edit walk, {steps} steps, CUDA graph: latents rel vs oracle = {e:.3e}  (oracle {t_cpu:.1f}s)")
    assert e < 1e-2, e


# ------------------------------------------------------------------------------------------------------------------------------------------
# SDXL VAE
# ------------------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("force_upcast", [False, True])
def test_vae_full_size_decode_and_encode_match_oracle(cpu_threads, force_upcast):
    """AutoencoderKL at full size: decode of one 128x128 latent to 1024x1024 (PSNR >= 40 dB on the [0,1] image, north_star) and encode of that
    1024x1024 image (latent_dist.mode(), pipeline...edit.py:523), plain fp16 stream and the force_upcast scaled stream."""
    from oracle import sdxl as osd
    from seedx_b200.sdxl import SDXL_VAE, AutoencoderKL
    cfg = dict(SDXL_VAE)
    sd_dev, sd = device_state_dict(synth.vae_state_dict, cfg)
    vae = AutoencoderKL(dict(cfg, force_upcast=force_upcast))
    vae.load_state_dict(sd_dev)
    z = synth.randn("fs_vae_z", (1, 4, 128, 128))
    out = vae.decode(z.cuda(), scale=1.0 / cfg["scaling_factor"])
    if "vae" not in _ORACLE_CACHE:   # same weights and inputs in both parametrisations: the oracle runs once
        t0 = time.time()
        with torch.no_grad():
            ref = osd.vae_decode(sd, cfg, z / cfg["scaling_factor"])
            img = ref.clamp(-1, 1)
            ref_lat = osd.vae_encode_mode(sd, cfg, img)
        print(f"[fullsize] VAE oracle decode+encode {time.time() - t0:.1f}s")
        _ORACLE_CACHE["vae"] = (ref, ref_lat, img)
    ref, ref_lat, img = _ORACLE_CACHE["vae"]
    p = psnr(out, ref)
    lat = vae.encode_mode(img.cuda())
    e = rel(lat, ref_lat)
    print(f"full-size VAE (force_upcast={force_upcast}): decode 1024^2 PSNR = {p:.1f} dB (rel {rel(out, ref):.3e}), encode rel = {e:.3e}")
    assert out.shape == (1, 3, 1024, 1024) and torch.isfinite(out).all() and p >= 40.0, p
    assert lat.shape == (1, 4, 128, 128) and e < 5e-3, e


# ------------------------------------------------------------------------------------------------------------------------------------------
# LLaMA at 13B width
# ------------------------------------------------------------------------------------------------------------------------------------------
def test_llama_13b_width_four_layers_prefill_and_greedy_match_oracle(cpu_threads):
    """modeling_llama_xformer.py:643-746 at hidden 5120 / 40 heads / FFN 13824 / vocab 32330, 4 layers: prefill of P=174 rows (wgmma GEMMs +
    causal wgmma attention at d=128) and 8 greedy tokens (GEMV token loop over the paged KV cache, CUDA graph)."""
    from oracle import llm as ollm
    from seedx_b200.llm import LLAMA_13B, LlamaForCausalLM
    cfg = dict(LLAMA_13B, layers=4)
    sd_dev, sd = device_state_dict(synth.llama_state_dict, cfg)
    m = LlamaForCausalLM(cfg, max_len=512)
    m.load_state_dict(sd_dev)
    del sd_dev
    P, new = 174, 8
    ids = ((synth.randn("fs_llm_ids", (P,)).abs() * 1000).long() % 30000 + 3).tolist()
    emb = sd["model.embed_tokens.weight"][torch.tensor(ids)]
    tok = synth.SynthTokenizer(vocab=cfg["vocab"])
    img_ids = tok.encode("".join(["<img>"] + ["<img_{:05d}>".format(i) for i in range(64)] + ["</img>"]))   # the processor's id list at full vocabulary
    with torch.no_grad():
        ref_logits, ref_hid, _ = ollm.llama_forward(sd, cfg, emb, 0, None)
        ref_ids, ref_gen_hid = ollm.greedy_generate(sd, cfg, ids, emb, img_ids, new)
    logits, hid = m.logits_all(m.prefill(emb.cuda()))
    e1, e2 = rel(logits, ref_logits), rel(hid, ref_hid)
    out = m.generate_greedy(ids, emb.cuda(), img_ids=img_ids, max_new_tokens=new)
    got = out.sequences[0][P:].tolist()
    e3 = rel(out.last_hidden_states, ref_gen_hid)
    print(f"LLaMA 13B width x 4 layers: prefill logits rel = {e1:.3e}, hidden rel = {e2:.3e}; {new} greedy ids {'exact' if got == ref_ids else 'DIFFER'}, "
          f"decode hidden rel = {e3:.3e}")
    assert e1 < 1e-3 and e2 < 1e-3 and e3 < 1e-3, (e1, e2, e3)
    assert got == ref_ids, (got, ref_ids)


# ------------------------------------------------------------------------------------------------------------------------------------------
# ViT at full width, 448 x 448
# ------------------------------------------------------------------------------------------------------------------------------------------
def test_vit_full_width_448_matches_oracle(cpu_threads):
    """qwen_visual.py:387-417 at width 1664 / 16 heads x 104 / MLP 8192 / pool to 4096, 4 layers, 448x448 input: 1024 patch tokens, the trunk's and
    the attention pool's position tables bicubic-interpolated from 16x16 to 32x32 (qwen_visual.py:24-40)."""
    from oracle import vit as ovit
    from seedx_b200.vit import VisionTransformerWithAttnPool
    cfg = dict(width=1664, layers=4, heads=16, mlp_width=8192, output_dim=4096, n_queries=256, patch=14)
    sd = synth.vit_state_dict(**cfg)
    x = synth.image("vit_full_in_448", 1, 448)
    with torch.no_grad():
        ref = ovit.vit_forward(sd, x, 16)
    m = VisionTransformerWithAttnPool(image_size=448, patch_size=14, width=1664, layers=4, heads=16, mlp_ratio=4.9231, n_queries=256, output_dim=4096)
    m.load_state_dict(sd)
    out = m(x.cuda())
    e = rel(out, ref)
    print(f"vit full width, 4 layers, 448x448: rel err vs oracle = {e:.3e}")
    assert out.shape == (1, 256, 4096) and e < 1e-3, e
