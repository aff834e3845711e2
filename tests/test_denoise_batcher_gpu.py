"""Continuous batching of the denoising loop on the GPU: seedx_cfg_euler_slots bit for bit against seedx_cfg_euler_step slot by slot, and
`serving.DenoiseBatcher` (staggered arrivals, mixed step counts and guidance, under the CUDA graph) bit for bit against the lock-step
`sampler.DenoiseLoop` and `adapter.generate` given the same request in the same slot."""
import ctypes as C

import pytest
import torch

from seedx_b200 import _lib, ops, synth

pytestmark = pytest.mark.gpu


def mk(shape, seed, scale=1.0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).cuda()


def bits(t):
    return t.contiguous().view(torch.int32 if t.element_size() == 4 else torch.int16).clone()


# ---- 1. the kernel ---------------------------------------------------------------------------------------------------------------------
def _tables(S, M, ns, seed):
    from seedx_b200.sdxl import EulerDiscreteScheduler
    sig = torch.zeros((S, M + 1))
    ts = torch.zeros((S, M))
    scal = torch.zeros((S, 3))
    for s, n in enumerate(ns):
        if n:
            sch = EulerDiscreteScheduler().set_timesteps(n)
            sig[s, :n + 1], ts[s, :n] = torch.tensor(sch.sigmas), torch.tensor(sch.timesteps)
            scal[s] = torch.tensor([3.0 + 1.5 * s, 1.1 + 0.3 * s, sch.init_noise_sigma])
    return sig.cuda(), ts.cuda(), scal.cuda()


@pytest.mark.parametrize("branches", [2, 3])
def test_slots_kernel_matches_lockstep_kernel_bit_for_bit(branches):
    S, h, w, M = 5, 16, 24, 12
    ns = [6, 4, 9, 0, 3]                     # slot 3 parked (count 0)
    idx = [2, 4, 0, 0, 2]                    # slot 1 finished (index == count), slot 2 at its first step, slot 4 at its last
    sig, ts, scal = _tables(S, M, ns, branches)
    state = torch.tensor([[i, n] for i, n in zip(idx, ns)], dtype=torch.int32).cuda()
    x = mk((S, 4, h, w), 1)
    eps = mk((branches * S, h, w, 4), 2)
    unet_in = mk((branches * S, h, w, 8), 3).half()
    t_dev = mk((branches * S,), 4)
    live = [s for s in range(S) if idx[s] < ns[s]]
    for s in range(S):
        if s not in live:                    # sentinels: whatever a finished / parked slot holds must come back byte for byte
            x[s] = float("nan")
            for br in range(branches):
                eps[br * S + s] = float("nan")
                unet_in[br * S + s] = float("nan")
                t_dev[br * S + s] = float("nan")
    x0, u0, t0 = bits(x), bits(unet_in), bits(t_dev)
    refs = {}
    for s in live:
        xs = x[s:s + 1].clone()
        us = torch.stack([unet_in[br * S + s] for br in range(branches)]).contiguous()
        es = torch.stack([eps[br * S + s] for br in range(branches)]).contiguous()
        g, ig = float(scal[s, 0]), float(scal[s, 1])
        ops.cfg_euler_step(es, xs, us, branches, g, ig, float(sig[s, idx[s]]), float(sig[s, idx[s] + 1]))
        refs[s] = (xs, us)
    n0 = _lib.launch_count()
    ops.cfg_euler_slots(eps, x, unet_in, t_dev, state, sig, ts, scal, branches)
    assert _lib.launch_count() - n0 == 2                                       # combine + advance
    st = state.cpu()
    for s in range(S):
        rows = [br * S + s for br in range(branches)]
        if s in live:
            assert torch.equal(bits(x[s]), bits(refs[s][0][0]))
            for k, r in enumerate(rows):
                assert torch.equal(bits(unet_in[r]), bits(refs[s][1][k]))
            assert st[s].tolist() == [idx[s] + 1, ns[s]]
            want = float(ts[s, idx[s] + 1]) if idx[s] + 1 < ns[s] else None
            for r in rows:
                assert (float(t_dev[r]) == want) if want is not None else torch.equal(bits(t_dev[r]), t0[r])
        else:
            assert torch.equal(bits(x[s]), x0[s]) and st[s].tolist() == [idx[s], ns[s]]
            for r in rows:
                assert torch.equal(bits(unet_in[r]), u0[r]) and torch.equal(bits(t_dev[r]), t0[r])

    # initialisation of a subset: x = noise * init_noise_sigma, inputs scaled by sigma_0, t_dev = first timestep; the other slots untouched
    fresh = [0, 2]
    x1, u1, t1, s1 = bits(x), bits(unet_in), bits(t_dev), state.clone()
    refs = {}
    for s in fresh:
        xs = x[s:s + 1].clone()
        us = torch.stack([unet_in[br * S + s] for br in range(branches)]).contiguous()
        ops.cfg_euler_step(None, xs, us, branches, 0.0, 0.0, 1.0, float(sig[s, 0]), float(scal[s, 2]))
        refs[s] = (xs, us)
    n0 = _lib.launch_count()
    ops.cfg_euler_slots(None, x, unet_in, t_dev, state, sig, ts, scal, branches, fresh=fresh)
    assert _lib.launch_count() - n0 == 1 and torch.equal(state, s1)
    for s in range(S):
        rows = [br * S + s for br in range(branches)]
        if s in fresh:
            assert torch.equal(bits(x[s]), bits(refs[s][0][0]))
            for k, r in enumerate(rows):
                assert torch.equal(bits(unet_in[r]), bits(refs[s][1][k])) and float(t_dev[r]) == float(ts[s, 0])
        else:
            assert torch.equal(bits(x[s]), x1[s])
            for r in rows:
                assert torch.equal(bits(unet_in[r]), u1[r]) and torch.equal(bits(t_dev[r]), t1[r])


def test_slots_kernel_rejects_bad_arguments_without_launching():
    S, h, w, M = 2, 8, 8, 4
    x = torch.zeros((S, 4, h, w), device="cuda")
    u = torch.zeros((2 * S, h, w, 8), device="cuda", dtype=torch.float16)
    eps = torch.zeros((2 * S, h, w, 4), device="cuda")
    t = torch.zeros((2 * S,), device="cuda")
    st = torch.zeros((S, 2), device="cuda", dtype=torch.int32)
    sig, ts, sc = torch.zeros((S, M + 1), device="cuda"), torch.zeros((S, M), device="cuda"), torch.zeros((S, 3), device="cuda")
    P = lambda a: C.c_void_p(a.data_ptr()) if a is not None else None     # noqa: E731
    fn = _lib.lib().seedx_cfg_euler_slots

    def call(branches=2, state=st, sigmas=sig, timesteps=ts, scalars=sc, max_steps=M, e=eps, mask=0):
        return fn(P(e), P(x), P(u), P(t), P(state), P(sigmas), P(timesteps), P(scalars), C.c_int64(S), C.c_int64(h * w), C.c_int(branches),
                  C.c_int64(max_steps), C.c_uint64(mask), None)
    n0 = _lib.launch_count()
    for kw in (dict(branches=1), dict(branches=4), dict(state=None), dict(sigmas=None), dict(timesteps=None), dict(scalars=None),
               dict(max_steps=0), dict(e=None, mask=0), dict(e=None, mask=4)):
        assert call(**kw) != 0, kw
        assert _lib.lib().seedx_last_error()
    assert _lib.launch_count() == n0
    assert call() == 0 and _lib.launch_count() == n0 + 2                       # all slots parked: launches, changes nothing
    torch.cuda.synchronize()


# ---- 2.-4. the batcher on the tiny adapter -----------------------------------------------------------------------------------------------
H = W = 256
IMG = 224


def _adapter(edit, weight_format="fp16"):
    """the tiny adapter of tests/test_sdxl_gpu.py::test_adapter_t2i_tiny_end_to_end (8-channel conv_in for the edit variant)"""
    from seedx_b200.adapter import SDXLAdapter, SDXLAdapterWithLatentImage
    from seedx_b200.resampler_xl import ResamplerXLV2
    from seedx_b200.sdxl import AutoencoderKL, EulerDiscreteScheduler, UNet2DConditionModel
    from seedx_b200.vit import VisionTransformerWithAttnPool
    vcfg = dict(width=208, layers=2, heads=2, mlp_width=520, output_dim=256, n_queries=256, patch=14)
    rcfg = dict(synth.TINY_RESAMPLER_XL, embedding_dim=256)
    ucfg = dict(synth.TINY_UNET, cross_attention_dim=256, text_embed_dim=160, in_channels=8 if edit else 4)
    vit = VisionTransformerWithAttnPool(image_size=448, patch_size=14, width=208, layers=2, heads=2, mlp_ratio=2.5, output_dim=256)
    vit.load_state_dict(synth.vit_state_dict(**vcfg))
    rx = ResamplerXLV2(normalize=False, **rcfg)
    rx.load_state_dict(synth.resampler_xl_state_dict(rcfg))
    unet, vae = UNet2DConditionModel(ucfg, weight_format=weight_format), AutoencoderKL(synth.TINY_VAE)
    unet.load_state_dict(synth.unet_state_dict(ucfg))
    vae.load_state_dict(synth.vae_state_dict(synth.TINY_VAE))
    ad = (SDXLAdapterWithLatentImage if edit else SDXLAdapter)(unet=unet, resampler=rx, vit_down=True)
    ad.init_pipe(vae=vae, scheduler=EulerDiscreteScheduler(), visual_encoder=vit, image_transform=None)
    return ad


def _requests(edit, tag, k):
    steps = [5, 3, 4, 2, 6, 3][:k]
    reqs = []
    for i, n in enumerate(steps):
        r = dict(image_embeds=synth.randn(f"{tag}_feats_{i}", (1, 64, 256)).cuda(), num_inference_steps=n, guidance_scale=7.5 - i,
                 image_guidance_scale=1.5 + 0.25 * i, seed=100 + i, input_image_size=IMG)
        if edit:
            r["latent_image"] = synth.randn(f"{tag}_il_{i}", (1, 4, H // 8, W // 8), 0.7).cuda()
        reqs.append(r)
    return reqs


def _lockstep(ad, req, slots, loops={}):
    """DenoiseLoop at batch `slots` with this request's conditioning, noise, steps and guidance in every slot"""
    from seedx_b200.sampler import DenoiseLoop
    from seedx_b200.sdxl import EulerDiscreteScheduler
    key = (id(ad), slots)
    if key not in loops:
        loops[key] = DenoiseLoop(ad.unet, EulerDiscreteScheduler(), slots, (H // 8, W // 8), ad.branches, use_graph=True)
    loop = loops[key]
    p, n, pp, npool = ad.get_image_embeds(image_embeds=req["image_embeds"], return_negative=True, image_size=IMG)
    rep = lambda t: t.expand((slots,) + tuple(t.shape[1:]))                   # noqa: E731
    tid = torch.tensor([[H, W, 0, 0, H, W]], dtype=torch.float32, device="cuda").repeat(ad.branches * slots, 1)
    if ad.branches == 2:
        loop.set_condition(torch.cat([rep(n), rep(p)]), torch.cat([rep(npool), rep(pp)]), tid)
    else:
        loop.set_condition(torch.cat([rep(p), rep(n), rep(n)]), torch.cat([rep(pp), rep(npool), rep(npool)]), tid,
                           image_latents=rep(req["latent_image"]).contiguous())
    noise = ad._noise(1, H, W, req["seed"], None)
    return loop.run(rep(noise).contiguous(), steps=req["num_inference_steps"], guidance=req["guidance_scale"],
                    image_guidance=req["image_guidance_scale"]).clone()


@pytest.mark.parametrize("weight_format", ["fp16", "fp8_e4m3_conv"])
@pytest.mark.parametrize("edit", [False, True])
def test_batcher_matches_lockstep_loop_bit_for_bit(edit, weight_format):
    from seedx_b200.serving import DenoiseBatcher
    ad = _adapter(edit, weight_format)
    S = 4
    b = DenoiseBatcher(ad, slots=S, height=H, width=W, max_steps=8, output_type="latent")
    reqs = _requests(edit, f"batcher_{int(edit)}", 6)
    # 0 and 1 at step 0, 2 at step 1, 3 and 4 at step 2 (4 waits for a free slot), 5 at step 4
    out = b.run({0: reqs[:2], 1: reqs[2:3], 2: reqs[3:5], 4: reqs[5:]})
    assert sorted(out) == list(range(6)) and b.captures == 1 and b.idle()
    assert b.slot_of[0] == 0 and b.slot_of[1] == 1 and b.slot_of[2] == 2 and b.slot_of[3] == 3
    for rid, r in enumerate(reqs):
        s = b.slot_of[rid]
        ref = _lockstep(ad, r, S)
        assert torch.equal(out[rid][0], ref[s]), (rid, s, (out[rid][0] - ref[s]).abs().max().item())

    # launches per step = the graph's kernel count (the UNet forward + combine + advance), recorded through note_replay
    rid = b.submit(**reqs[4])
    b.step()
    n0 = _lib.launch_count()
    b.step()
    assert _lib.launch_count() - n0 == b.graph_kernels
    n1 = _lib.launch_count()
    ad.unet.forward_nhwc(b.unet_in, b.t_dev, b.cond)
    assert b.graph_kernels == _lib.launch_count() - n1 + 2
    while not b.idle():
        b.step()

    # a partial checkpoint after capture: weights change in place, the next request sees them, the graph is not captured again
    sd = synth.unet_state_dict(ad.unet.cfg)
    k = next(k for k in sd if k.endswith("attn2.to_k.weight"))
    ad.unet.load_state_dict({k: sd[k] * 1.5, "conv_out.bias": sd["conv_out.bias"] + 0.05})
    rid2 = b.submit(**reqs[0])
    got = b.run()[rid2]
    assert b.captures == 1
    assert not torch.equal(got, out[0])
    assert torch.equal(got[0], _lockstep(ad, reqs[0], S)[b.slot_of[rid2]])
    assert rid2 == rid + 1


@pytest.mark.parametrize("edit", [False, True])
def test_one_slot_matches_adapter_generate(edit):
    from seedx_b200.serving import DenoiseBatcher
    ad = _adapter(edit)
    r = _requests(edit, f"generate_{int(edit)}", 1)[0]
    kw = dict(image_embeds=r["image_embeds"], seed=r["seed"], height=H, width=W, guidance_scale=r["guidance_scale"],
              num_inference_steps=r["num_inference_steps"], input_image_size=IMG)
    if edit:
        kw.update(latent_image=r["latent_image"], image_guidance_scale=r["image_guidance_scale"])
    ref_lat = ad.generate(output_type="latent", **kw)
    ref_u8 = ad.generate(output_type="uint8", **kw)
    outs = {}
    for fmt in ("latent", "uint8"):
        b = DenoiseBatcher(ad, slots=1, height=H, width=W, max_steps=10, output_type=fmt)
        rid = b.submit(**r)
        outs[fmt] = b.run()[rid]
    assert torch.equal(outs["latent"], ref_lat)
    assert outs["uint8"].dtype == torch.uint8 and torch.equal(outs["uint8"], ref_u8)


# ---- 5. full size ------------------------------------------------------------------------------------------------------------------------
class _FullSizeAdapter:
    """the adapter helpers DenoiseBatcher uses, over the SDXL UNet with synthetic weights and synthetic resampler outputs"""
    branches = 2

    def __init__(self, unet):
        from seedx_b200.sdxl import EulerDiscreteScheduler
        self.unet, self.scheduler, self.vae, self.device = unet, EulerDiscreteScheduler(), None, torch.device("cuda")
        cd, te = unet.cfg["cross_attention_dim"], unet.cfg["text_embed_dim"]
        self.neg = (synth.randn("fs_neg", (1, 64, cd)).cuda(), synth.randn("fs_negpool", (1, te)).cuda())

    def get_image_embeds(self, image_embeds=None, return_negative=True, image_size=448):
        """image_embeds [1, 65, ctx_dim]: 64 prompt tokens, then the pooled embedding in the first text_embed_dim columns"""
        return image_embeds[:, :64], self.neg[0], image_embeds[:, 64, :self.unet.cfg["text_embed_dim"]], self.neg[1]

    def _noise(self, B, h, w, seed, latents):
        return synth.randn(f"fs_noise_{seed}", (B, 4, h // 8, w // 8)).cuda()


def test_full_size_two_slots_staggered():
    from seedx_b200.sampler import DenoiseLoop
    from seedx_b200.sdxl import SDXL_UNET, EulerDiscreteScheduler, UNet2DConditionModel
    from seedx_b200.serving import DenoiseBatcher
    cfg = dict(SDXL_UNET)
    unet = UNet2DConditionModel(cfg)
    unet.load_state_dict(synth.unet_state_dict(cfg))
    ad = _FullSizeAdapter(unet)
    cd, te = cfg["cross_attention_dim"], cfg["text_embed_dim"]
    embeds = []
    for i in range(2):
        e = torch.zeros((1, 65, cd), device="cuda", dtype=torch.float16)
        e[:, :64], e[:, 64, :te] = synth.randn(f"fs_p{i}", (1, 64, cd)).cuda(), synth.randn(f"fs_pp{i}", (1, te)).cuda()
        embeds.append(e)
    reqs = [dict(image_embeds=embeds[0], num_inference_steps=3, guidance_scale=7.5, seed=0),
            dict(image_embeds=embeds[1], num_inference_steps=3, guidance_scale=5.0, seed=1)]
    b = DenoiseBatcher(ad, slots=2, height=1024, width=1024, max_steps=50, output_type="latent")
    out = b.run({0: reqs[:1], 1: reqs[1:]})
    assert b.captures == 1 and b.steps == 4
    loop = DenoiseLoop(unet, EulerDiscreteScheduler(), 2, (128, 128), 2, use_graph=True)
    tid = torch.tensor([[1024.0, 1024.0, 0.0, 0.0, 1024.0, 1024.0]], device="cuda").repeat(4, 1)
    for rid, r in enumerate(reqs):
        p, _, pp, _ = ad.get_image_embeds(image_embeds=r["image_embeds"])
        loop.set_condition(torch.cat([ad.neg[0], ad.neg[0], p, p]), torch.cat([ad.neg[1], ad.neg[1], pp, pp]), tid)
        ref = loop.run(ad._noise(1, 1024, 1024, r["seed"], None).expand(2, -1, -1, -1).contiguous(), steps=3, guidance=r["guidance_scale"])
        assert torch.equal(out[rid][0], ref[b.slot_of[rid]]), rid
