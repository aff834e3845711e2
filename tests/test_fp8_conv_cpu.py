"""Host logic of the opt-in FP8 (e4m3) UNet convolutions on the CPU: `UNet2DConditionModel(weight_format="fp8_e4m3_conv")` runs over
tests/fake_ops.py, extended with the FP8 projection restatements of test_fp8_unet_cpu.py and, here, plain-torch restatements of the two FP8 conv
entry points (seedx_quant_images_fp8, seedx_conv_fp8).  Checked: the weight_format switch, which convs get FP8 copies, their repacked layout and
scales, the forward against the fp16 and "fp8_e4m3" hosts, the in-place re-derivation after a partial checkpoint, and that an image's
quantisation does not depend on the rest of its batch.  The kernels themselves are checked in test_fp8_conv_gpu.py."""
import json
import types

import pytest
import torch
import torch.nn.functional as F

import fake_ops
import test_fp8_unet_cpu as fp8_unet
from seedx_b200 import sdxl as sdxl_mod
from seedx_b200 import synth
from seedx_b200._lib import SeedxError
from seedx_b200.llm import quantize_fp8_rows

E4 = torch.float8_e4m3fn


def _quant_images_fp8(x, q=None, scale=None, ws=None):
    """seedx_quant_images_fp8: llm.quantize_fp8_rows on x.view(n, -1).float()"""
    n = x.shape[0]
    q8, s = quantize_fp8_rows(x.reshape(n, -1).float())
    if q is None:
        q = torch.empty(x.shape, dtype=E4)
    if scale is None:
        scale = torch.empty((n,), dtype=torch.float32)
    q.view(n, -1).copy_(q8), scale.copy_(s)
    return q, scale


def _conv2d_nhwc(x, w, out=None, *, a_scale=None, w_scale=None, taps=3, bias=None, bias_g=None, residual=None, act=fake_ops.ACT_NONE,
                 out_dtype=torch.float16, tile_n=0, alpha=1.0, col_part=None):
    """ops.conv2d_nhwc: fp16 operands as in fake_ops; e4m3 operands (seedx_conv_fp8): the exact conv of q.float() over the channels that exist
    (w [Cout, taps*taps*roundup(C,128)]), then (acc * a_scale[image]) * w_scale[n] in fp32, then the fake_ops conv epilogue"""
    if a_scale is None:
        return fake_ops.conv2d_nhwc(x, w, out, taps=taps, bias=bias, bias_g=bias_g, residual=residual, act=act, out_dtype=out_dtype,
                                    tile_n=tile_n, alpha=alpha, col_part=col_part)
    assert x.dtype == w.dtype == E4 and w_scale is not None
    n, h, wd, c = x.shape
    cout = w.shape[0]
    cpad = w.shape[1] // (taps * taps)
    assert cpad == (c + 127) // 128 * 128
    w4 = w.double().view(cout, taps, taps, cpad)[..., :c].permute(0, 3, 1, 2)
    acc = F.conv2d(x.double().permute(0, 3, 1, 2), w4, padding=taps // 2).float()           # exact: integer-valued e4m3 sums fit in fp64
    y = alpha * ((acc * a_scale[:, None, None, None]) * w_scale[None, :, None, None])
    if bias is not None:
        y = y + bias[None, :, None, None]
    if bias_g is not None:
        y = y + bias_g[:, :, None, None]
    y = y.permute(0, 2, 3, 1)
    if act == fake_ops.ACT_SILU:
        y = F.silu(y)
    elif act == fake_ops.ACT_GELU:
        y = F.gelu(y)
    if residual is not None:
        y = y + residual.float()
    if out is None:
        out = torch.empty((n, h, wd, cout), dtype=out_dtype)
    out.copy_(y.to(out.dtype))
    fake_ops._emit_parts(out.view(-1, cout), y.reshape(-1, cout), None, col_part)
    return out


fake_ops_fp8 = types.SimpleNamespace(**vars(fp8_unet.fake_ops_fp8))
fake_ops_fp8.conv2d_nhwc, fake_ops_fp8.quant_images_fp8 = _conv2d_nhwc, _quant_images_fp8


@pytest.fixture
def patched(monkeypatch):
    monkeypatch.setattr(sdxl_mod, "ops", fake_ops_fp8)


def _unet(weight_format, sd, cfg=synth.TINY_UNET):
    m = sdxl_mod.UNet2DConditionModel(cfg, device="cpu", weight_format=weight_format)
    m.load_state_dict({k: v.clone() for k, v in sd.items()})
    return m


def _resnets(m):
    return [r for b in m.down for r in b["res"]] + [m.mid["r0"], m.mid["r1"]] + [r for b in m.up for r in b["res"]]


def test_weight_format_switch(tmp_path):
    assert "fp8_e4m3_conv" in sdxl_mod.UNET_WEIGHT_FORMATS
    assert sdxl_mod.UNet2DConditionModel(synth.TINY_UNET, device="cpu", weight_format="fp8_e4m3_conv").weight_format == "fp8_e4m3_conv"
    with pytest.raises(SeedxError):
        sdxl_mod.UNet2DConditionModel(synth.TINY_UNET, device="cpu", weight_format="fp8_conv")
    c = synth.TINY_UNET
    json.dump(dict(in_channels=4, out_channels=4, block_out_channels=list(c["block_out_channels"]), layers_per_block=c["layers_per_block"],
                   transformer_layers_per_block=list(c["transformer_layers"]), attention_head_dim=list(c["heads"]),
                   cross_attention_dim=c["cross_attention_dim"], addition_time_embed_dim=c["addition_time_embed_dim"],
                   down_block_types=["CrossAttnDownBlock2D" if a else "DownBlock2D" for a in c["down_attn"]]), open(tmp_path / "config.json", "w"))
    torch.save(synth.unet_state_dict(c), tmp_path / "diffusion_pytorch_model.bin")
    m = sdxl_mod.UNet2DConditionModel.from_pretrained(str(tmp_path), device="cpu", weight_format="fp8_e4m3_conv")
    assert m.weight_format == "fp8_e4m3_conv" and len(m.conv_fp8_slots()) == 36 and all(t.fp8_slots() for t in m.transformers())


def test_exactly_the_resnet_and_upsampler_convs_get_fp8_copies():
    sd = synth.unet_state_dict(synth.TINY_UNET)
    for fmt in ("fp16", "fp8_e4m3"):
        m = _unet(fmt, sd)
        assert m.conv_fp8_slots() == [] and all(r.fp8 is None for r in _resnets(m)) and all(b["us8"] is None for b in m.up)
    m = _unet("fp8_e4m3_conv", sd)
    slots = m.conv_fp8_slots()
    # 3 levels: down 3 x 2 resnets, mid 2, up 3 x 3 resnets, two convs each; plus the two upsamplers
    assert len(slots) == 2 * (3 * 2 + 2 + 3 * 3) + 2 == 36
    names = [n for n, _ in slots]
    assert len(set(names)) == 36 and all(n.endswith((".conv1", ".conv2", "upsamplers.0.conv")) for n in names)
    srcs = {id(c.w16) for _, c in slots}
    want = {id(r.w1) for r in _resnets(m)} | {id(r.w2) for r in _resnets(m)} | {id(b["us"][0]) for b in m.up if b["us"] is not None}
    assert srcs == want
    fp16_only = [m.conv_in[0], m.conv_out[0]] + [r.wsc for r in _resnets(m) if r.wsc is not None] + [b["ds"][0] for b in m.down if b["ds"] is not None]
    assert len(fp16_only) >= 2 + 2 + 2 and not srcs & {id(t) for t in fp16_only}
    assert all(t.fp8_slots() for t in m.transformers())           # the projections are FP8 as in "fp8_e4m3"
    for k in sd:                                                  # every checkpoint key of a copied conv is one the registry knows
        if k.endswith(".conv1.weight") or k.endswith("upsamplers.0.conv.weight"):
            assert k[: -len(".weight")] in names
    # the VAE shares _Resnet and stays fp16
    vae = sdxl_mod.AutoencoderKL(synth.TINY_VAE, device="cpu")
    vae.load_state_dict(synth.vae_state_dict(synth.TINY_VAE))
    assert all(r.fp8 is None for r in [vae.d_mid[0], vae.d_mid[2]] + [r for res, _ in vae.d_up for r in res] + [r for res, _ in vae.e_down for r in res])


def test_repacked_layout_padding_and_scales():
    sd = synth.unet_state_dict(synth.TINY_UNET)
    m = _unet("fp8_e4m3_conv", sd)
    for name, c in m.conv_fp8_slots():
        cout, cin = sd[name + ".weight"].shape[:2]
        c64, c128 = (cin + 63) // 64 * 64, (cin + 127) // 128 * 128
        assert c.cin == cin and c.q.dtype == E4 and c.q.shape == (cout, 9 * c128) and c.s.dtype == torch.float32 and c.s.shape == (cout,)
        q_ref, s_ref = quantize_fp8_rows(c.w16)
        assert torch.equal(c.s, s_ref)
        q3 = c.q.view(torch.uint8).view(cout, 9, c128)
        assert torch.equal(q3[..., :cin], q_ref.view(torch.uint8).view(cout, 9, c64)[..., :cin])
        assert int(q3[..., cin:].abs().sum()) == 0                                  # zero channel padding up to the 128-channel stage
        w = sd[name + ".weight"].float().permute(0, 2, 3, 1)                        # [Cout, kh, kw, Cin]
        deq = (q3[..., :cin].view(E4).float() * c.s[:, None, None]).view(cout, 3, 3, cin)
        assert ((deq - w.half().float()).abs() <= 2.0 ** -4 * w.half().float().abs() + c.s[:, None, None, None] * 2.0 ** -9).all()


def _inputs(B=2, hw=16):
    cfg = synth.TINY_UNET
    x = synth.randn("cpu_unet_x", (B, 4, hw, hw))
    ctx = synth.randn("cpu_unet_ctx", (B, 16, cfg["cross_attention_dim"]))
    te = synth.randn("cpu_unet_te", (B, cfg["text_embed_dim"]))
    tid = torch.tensor([[1024.0, 1024.0, 0.0, 0.0, 1024.0, 1024.0]]).repeat(B, 1)
    return x, ctx, dict(text_embeds=te, time_ids=tid)


def rel(a, b):
    return ((a.float() - b.float()).norm() / b.float().norm()).item()


def test_tiny_unet_fp8_conv_forward_tracks_the_fp16_and_fp8_hosts(patched):
    """e4m3 rounds each operand to u = 2^-4; with random signs a conv output carries a few percent of relative error, and the 36 FP8 convs sit
    on the residual path of every block, so eps moves by more than with FP8 projections alone but stays below 2u = 12.5 % of the fp16 host"""
    sd = synth.unet_state_dict(synth.TINY_UNET)
    x, ctx, added = _inputs()
    ref = _unet("fp16", sd)(x, 601.0, ctx, added_cond_kwargs=added)
    e8 = _unet("fp8_e4m3", sd)(x, 601.0, ctx, added_cond_kwargs=added)
    out = _unet("fp8_e4m3_conv", sd)(x, 601.0, ctx, added_cond_kwargs=added)
    e_16, e_8 = rel(out, ref), rel(out, e8)
    print(f"tiny UNet fp8_e4m3_conv: eps rel vs fp16 host {e_16:.3e}, vs fp8_e4m3 host {e_8:.3e}, fp8_e4m3 vs fp16 {rel(e8, ref):.3e}")
    assert 1e-4 < e_16 < 2 * 2.0 ** -4, e_16
    assert 1e-4 < e_8 < 2 * 2.0 ** -4, e_8                          # the conv path ran: different from FP8 projections alone


def test_partial_checkpoint_rederives_conv_copies_in_place(patched):
    """conv weights of a few resnets and an upsampler loaded after the model is built: every FP8 conv copy keeps its storage (captured graphs
    stay valid) and equals the copy of a model built from the merged weights"""
    sd = synth.unet_state_dict(synth.TINY_UNET)
    m = _unet("fp8_e4m3_conv", sd)
    ptrs = [(c.q.data_ptr(), c.s.data_ptr()) for _, c in m.conv_fp8_slots()]
    part = {k: synth.randn("fc8:" + k, v.shape, v[0].numel() ** -0.5)
            for k, v in sd.items() if k.endswith(("resnets.0.conv1.weight", "resnets.1.conv2.weight", "upsamplers.0.conv.weight"))}
    assert len(part) >= 10
    m.load_state_dict(part)
    assert ptrs == [(c.q.data_ptr(), c.s.data_ptr()) for _, c in m.conv_fp8_slots()]
    fresh = _unet("fp8_e4m3_conv", {**sd, **part})
    changed = 0
    for (n1, c), (n2, cf) in zip(m.conv_fp8_slots(), fresh.conv_fp8_slots()):
        assert n1 == n2 and torch.equal(c.q.view(torch.uint8), cf.q.view(torch.uint8)) and torch.equal(c.s, cf.s)
        changed += (n1 + ".weight") in part
    assert changed == len(part)
    x, ctx, added = _inputs(B=1)
    assert torch.equal(m(x, 301.0, ctx, added_cond_kwargs=added), fresh(x, 301.0, ctx, added_cond_kwargs=added))


def test_image_quantisation_does_not_depend_on_the_batch():
    g = torch.Generator().manual_seed(3)
    x = (torch.randn((8, 16, 16, 320), generator=g) * torch.logspace(-3, 2, 8)[:, None, None, None]).half()
    q8, s8 = _quant_images_fp8(x)
    for i in (0, 5, 7):
        q1, s1 = _quant_images_fp8(x[i:i + 1].contiguous())
        assert torch.equal(q1[0].view(torch.uint8), q8[i].view(torch.uint8)) and torch.equal(s1[0], s8[i])
