"""Host logic of `seedx_b200.serving.DenoiseBatcher` on the CPU: the batcher runs unchanged over tests/fake_ops.py plus a restatement of
seedx_cfg_euler_slots (below), with a UNet stand-in that evaluates the oracle UNet (oracle/sdxl.py) row by row, each row at its own timestep.
Checked: staggered admission into 2 slots (t2i and edit, different step counts and guidance, a slot reused) against oracle.t2i_sample /
oracle.edit_sample run alone; FIFO into the lowest free slot; parked slots left alone; the schedule tables; the requests it refuses."""
import types

import pytest
import torch

import fake_ops
from oracle import sdxl as osd
from seedx_b200 import serving, synth
from seedx_b200._lib import SeedxError
from seedx_b200.sdxl import EulerDiscreteScheduler

HW = 16                     # latent side; the pixel size is 8x
T = 16                      # conditioning tokens


def rel(a, b):
    return ((a.float() - b.float()).norm() / b.float().norm()).item()


def cfg_euler_slots(eps, x, unet_in, t_dev, state, sigmas, timesteps, scalars, branches, fresh=None):
    """restates seedx_cfg_euler_slots: per live slot (step index < step count) the cfg_euler_kernel arithmetic with that slot's sigmas and
    guidance, then index += 1 and the next timestep into its t_dev rows; eps None initialises the fresh slots"""
    S = x.shape[0]
    calls.append(("init" if eps is None else "step", sorted(fresh or ()) if eps is None else
                  [s for s in range(S) if int(state[s, 0]) < int(state[s, 1])]))
    for s in range(S):
        i, n = int(state[s, 0]), int(state[s, 1])
        g, ig, init = (float(v) for v in scalars[s])
        if eps is None:
            if s not in (fresh or ()):
                continue
            xn, sn = x[s] * init, float(sigmas[s, 0])
            t_dev[s::S] = timesteps[s, 0]
        else:
            if i >= n:
                continue
            sg, sn = float(sigmas[s, i]), float(sigmas[s, i + 1])
            e = eps.reshape(branches, S, x.shape[2], x.shape[3], 4)[:, s].permute(0, 3, 1, 2)      # [branch, 4, h, w]
            xv = x[s]
            if branches == 2:
                comb = e[0] + g * (e[1] - e[0])
            else:
                et, ei, eu = (xv - sg * e[b] for b in range(3))
                comb = (eu + g * (et - ei) + ig * (ei - eu) - xv) / (-sg)
            xn = xv + (xv - (xv - sg * comb)) / sg * (sn - sg)
            state[s, 0] = i + 1
            if i + 1 < n:
                t_dev[s::S] = timesteps[s, i + 1]
        x[s] = xn
        unet_in[s::S, ..., :4] = (xn * (sn ** 2 + 1.0) ** -0.5).permute(1, 2, 0).to(torch.float16)
    return x


calls = []
fake = types.SimpleNamespace(**{k: getattr(fake_ops, k) for k in dir(fake_ops) if not k.startswith("_")}, cfg_euler_slots=cfg_euler_slots)


class RowOracleUNet:
    """forward_nhwc / prepare_cond surface of seedx_b200.sdxl.UNet2DConditionModel; the oracle evaluates every row alone at t_dev[row]"""

    def __init__(self, sd, cfg):
        self.sd, self.cfg, self.device = sd, cfg, torch.device("cpu")
        self.forwards = 0

    def prepare_cond(self, ctx, text_embeds, time_ids):
        return dict(ctx=ctx.clone().float(), te=text_embeds.clone().float(), tid=time_ids.clone().float())

    def forward_nhwc(self, x_in, t_dev, cond):
        self.forwards += 1
        x = x_in[..., : self.cfg["in_channels"]].float().permute(0, 3, 1, 2).contiguous()
        rows = [osd.unet_forward(self.sd, self.cfg, x[r:r + 1], float(t_dev[r]), cond["ctx"][r:r + 1], cond["te"][r:r + 1],
                                 cond["tid"][r:r + 1]) for r in range(x.shape[0])]
        return torch.cat(rows).permute(0, 2, 3, 1).contiguous().float()


class FakeAdapter:
    """the adapter helpers DenoiseBatcher uses, at batch 1.  image_embeds [1, T+1, ctx_dim] carries the resampler output directly: tokens
    0..T-1 are the prompt, token T holds the pooled embedding in its first text_embed_dim columns; the negative conditioning is fixed."""

    def __init__(self, unet, branches):
        self.unet, self.branches, self.scheduler, self.vae = unet, branches, EulerDiscreteScheduler(), None
        te = unet.cfg["text_embed_dim"]
        self.neg = (synth.randn("batcher_neg", (1, T, unet.cfg["cross_attention_dim"])), synth.randn("batcher_negpool", (1, te)))

    def get_image_embeds(self, image_embeds=None, return_negative=True, image_size=448):
        te = self.unet.cfg["text_embed_dim"]
        return image_embeds[:, :T], self.neg[0], image_embeds[:, T, :te], self.neg[1]

    def _noise(self, B, h, w, seed, latents):
        return latents.float() if latents is not None else synth.randn(f"batcher_noise_{seed}", (B, 4, h // 8, w // 8))

    def _image_latents(self, latent_image, height, width):
        return latent_image.float()


def _embeds(cfg, tag):
    e = torch.zeros((1, T + 1, cfg["cross_attention_dim"]))
    e[:, :T] = synth.randn(tag + "p", (1, T, cfg["cross_attention_dim"]))
    e[:, T, :cfg["text_embed_dim"]] = synth.randn(tag + "pp", (1, cfg["text_embed_dim"]))
    return e


@pytest.fixture
def patched(monkeypatch):
    monkeypatch.setattr(serving, "ops", fake)
    calls.clear()


def _batcher(branches, slots=2, max_steps=8):
    cfg = dict(synth.TINY_UNET, in_channels=4 if branches == 2 else 8)
    unet = RowOracleUNet(synth.unet_state_dict(cfg), cfg)
    ad = FakeAdapter(unet, branches)
    return serving.DenoiseBatcher(ad, slots=slots, height=8 * HW, width=8 * HW, max_steps=max_steps, output_type="latent", use_graph=False), ad


def _reference(ad, req):
    cfg, sd = ad.unet.cfg, ad.unet.sd
    te = cfg["text_embed_dim"]
    e = req["image_embeds"]
    noise = ad._noise(1, 8 * HW, 8 * HW, req.get("seed"), req.get("latents"))
    p, pp = e[:, :T], e[:, T, :te]
    if ad.branches == 2:
        return osd.t2i_sample(sd, cfg, noise, p, pp, ad.neg[0], ad.neg[1], steps=req["num_inference_steps"], guidance=req["guidance_scale"],
                              size=8 * HW)
    return osd.edit_sample(sd, cfg, noise, req["latent_image"], p, pp, ad.neg[0], ad.neg[1], steps=req["num_inference_steps"],
                           guidance=req["guidance_scale"], image_guidance=req["image_guidance_scale"], size=8 * HW)


@pytest.mark.parametrize("branches", [2, 3])
def test_staggered_arrivals_match_requests_run_alone(patched, branches):
    b, ad = _batcher(branches)
    cfg = ad.unet.cfg
    reqs = [dict(num_inference_steps=4, guidance_scale=7.5, image_guidance_scale=1.5, seed=1),
            dict(num_inference_steps=2, guidance_scale=5.0, image_guidance_scale=2.0, seed=2),
            dict(num_inference_steps=3, guidance_scale=3.0, image_guidance_scale=1.2,
                 latents=synth.randn("batcher_lat3", (1, 4, HW, HW)))]
    for k, r in enumerate(reqs):
        r["image_embeds"] = _embeds(cfg, f"batcher_{branches}_{k}")
        if branches == 3:
            r["latent_image"] = synth.randn(f"batcher_il_{k}", (1, 4, HW, HW), 0.7)
    # request 0 at step 0; 1 and 2 arrive at step 1 while 0 is mid-walk: 1 takes slot 1, 2 waits for slot 1 to retire (after step 2)
    out = b.run({0: [reqs[0]], 1: [reqs[1], reqs[2]]})
    assert sorted(out) == [0, 1, 2]
    for rid, r in enumerate(reqs):
        e = rel(out[rid][0], _reference(ad, r)[0])
        assert e < 2e-3, (rid, e)                                        # fp16 rounding of the UNet input only
    # slot 0: request 0 (steps 0..3); slot 1: request 1 (steps 1..2), then request 2 (steps 3..5)
    assert calls[0] == ("init", [0]) and calls[2] == ("init", [1])
    assert ("init", [1]) in calls[4:] and calls.count(("init", [1])) == 2
    assert b.steps == 6 and ad.unet.forwards == 6
    assert b.idle() and int(b.state[:, 1].abs().sum()) == 0


def test_admission_order_and_parked_slots(patched):
    b, ad = _batcher(2, slots=3)
    cfg = ad.unet.cfg
    mk = lambda k, n: dict(image_embeds=_embeds(cfg, f"order_{k}"), num_inference_steps=n, seed=10 + k)   # noqa: E731
    for k, n in enumerate((3, 1, 2)):
        b.submit(**mk(k, n))
    b.step()
    assert calls[0] == ("init", [0, 1, 2]) and [r and r["rid"] for r in b.live] == [0, None, 2]     # request 1 made its only step
    # slot 1 is parked: count 0, UNet input rows zero, and neither the step nor a later admission into another slot writes its rows
    assert b.state[1].tolist() == [0, 0] and float(b.unet_in[1::3].abs().max()) == 0.0
    x1, t1 = b.x[1].clone(), b.t_dev[1::3].clone()
    b.step()                                                              # slot 2 retires
    assert torch.equal(b.x[1], x1) and torch.equal(b.t_dev[1::3], t1) and float(b.unet_in[1::3].abs().max()) == 0.0
    assert calls[-1] == ("step", [0, 2])
    b.submit(**mk(3, 2))
    b.submit(**mk(4, 2))
    b.step()                                                              # FIFO into the lowest free slots: request 3 -> 1, request 4 -> 2
    assert [r["rid"] if r else None for r in b.live] == [None, 3, 4]      # slot 0 retired after its 3rd step
    assert ("init", [1, 2]) in calls


@pytest.mark.parametrize("n", [1, 2, 30, 50, 100])
def test_table_rows_and_init_scalars(patched, n):
    b, ad = _batcher(2, slots=2, max_steps=100)
    b.submit(image_embeds=_embeds(ad.unet.cfg, "tables"), num_inference_steps=n, guidance_scale=6.0, image_guidance_scale=1.7, seed=3)
    b.submit(image_embeds=_embeds(ad.unet.cfg, "tables"), num_inference_steps=1, seed=4)
    b._admit()
    sch = EulerDiscreteScheduler().set_timesteps(n)
    assert torch.equal(b.sig[0, :n + 1], torch.tensor(sch.sigmas, dtype=torch.float32)) and float(b.sig[0, n:].abs().sum()) == 0.0
    assert torch.equal(b.ts[0, :n], torch.tensor(sch.timesteps, dtype=torch.float32)) and float(b.ts[0, n:].abs().sum()) == 0.0
    assert torch.equal(b.scal[0], torch.tensor([6.0, 1.7, sch.init_noise_sigma], dtype=torch.float32))
    assert b.state[0].tolist() == [0, n] and float(b.t_dev[0]) == sch.timesteps[0] == float(b.t_dev[2])
    assert torch.equal(b.x[0], ad._noise(1, 8 * HW, 8 * HW, 3, None)[0] * torch.tensor(sch.init_noise_sigma, dtype=torch.float32))
    # the second admission's set_timesteps(1) did not change the first slot's copy of its schedule
    assert b.ts[1, 0].item() == EulerDiscreteScheduler().set_timesteps(1).timesteps[0] and b.state[1].tolist() == [0, 1]


def test_rejections_enqueue_nothing(patched):
    b, ad = _batcher(2, max_steps=8)
    e = _embeds(ad.unet.cfg, "reject")
    bad = [dict(num_inference_steps=0), dict(num_inference_steps=9), dict(num_inference_steps=2.5), dict(num_inference_steps=True),
           dict(latent_image=torch.zeros(1, 4, HW, HW)), dict(latents=torch.zeros(1, 4, HW, HW + 8)), dict(latents=torch.zeros(2, 4, HW, HW))]
    for kw in bad:
        with pytest.raises(SeedxError):
            b.submit(e, **kw)
    with pytest.raises(SeedxError):
        b.submit(torch.cat([e, e]))
    assert not b.pending and b.next_rid == 0 and b.idle()
    assert b.submit(e, num_inference_steps=8) == 0 and len(b.pending) == 1
    with pytest.raises(SeedxError):
        serving.DenoiseBatcher(ad, slots=2, height=128, width=128, max_steps=0)
    cfg4 = synth.TINY_UNET
    with pytest.raises(SeedxError):                       # an edit adapter over a 4-channel conv_in
        serving.DenoiseBatcher(FakeAdapter(RowOracleUNet({}, cfg4), 3), slots=2, height=128, width=128)
