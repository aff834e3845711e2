"""Host logic of the opt-in FP8 (e4m3) UNet transformer projections on the CPU: `UNet2DConditionModel(weight_format="fp8_e4m3")` runs over
tests/fake_ops.py, extended here with plain-torch restatements of the two FP8 entry points (seedx_quant_rows_fp8, seedx_gemm_fp8).  Checked: the
weight_format switch, which packed matrices get FP8 copies, their scales and folded-LayerNorm column sums, the forward against the fp16 host,
and the in-place re-derivation after a partial checkpoint.  The kernels themselves are checked in test_fp8_unet_gpu.py."""
import json
import types

import pytest
import torch
import torch.nn.functional as F

import fake_ops
from seedx_b200 import sdxl as sdxl_mod
from seedx_b200 import synth
from seedx_b200._lib import SeedxError
from seedx_b200.llm import quantize_fp8_rows

FP8_KINDS = {"attn1.qkv", "attn1.to_out", "attn2.to_q", "attn2.to_out", "ff.net.0", "ff.net.2"}     # per block, plus proj_in / proj_out
FOLDED = {"attn1.qkv", "attn2.to_q", "ff.net.0"}


def _quant_rows_fp8(x, q=None, scale=None):
    """seedx_quant_rows_fp8: llm.quantize_fp8_rows on x.float()"""
    q8, s = quantize_fp8_rows(x.float())
    if q is None:
        q = torch.empty(x.shape, dtype=torch.float8_e4m3fn)
    if scale is None:
        scale = torch.empty((x.shape[0],), dtype=torch.float32)
    q.copy_(q8), scale.copy_(s)
    return q, scale


def _gemm(a, w, out=None, *, a_scale=None, w_scale=None, bias=None, residual=None, act=fake_ops.ACT_NONE, gated=False, alpha=1.0,
          out_dtype=torch.float16, ln=None, row_part=None, col_part=None, row_stats=None, **kw):
    """ops.gemm: fp16 operands as in fake_ops; e4m3 operands with the accumulator scaled as (acc * a_scale[m]) * w_scale[n] (seedx_gemm_fp8),
    then the same epilogue order"""
    if a_scale is None:
        return fake_ops.gemm(a, w, out, bias=bias, residual=residual, act=act, gated=gated, alpha=alpha, out_dtype=out_dtype, ln=ln,
                             row_part=row_part, col_part=col_part, row_stats=row_stats, **kw)
    assert a.dtype == w.dtype == torch.float8_e4m3fn and w_scale is not None and not any(v is not None and v is not False and v != 0 for v in kw.values())
    acc = (a.float() @ w.float().t()) * a_scale[:, None] * w_scale[None, :]
    if ln is not None:
        st, cs = ln
        acc = st[:, 1:2] * (acc - st[:, 0:1] * cs[None, :])
    else:
        acc = alpha * acc
    if bias is not None:
        acc = acc + bias
    if gated:
        acc = acc[:, 0::2] * F.gelu(acc[:, 1::2])
    elif act == fake_ops.ACT_GELU:
        acc = F.gelu(acc)
    if residual is not None:
        acc = acc + residual.float()
    if out is None:
        out = torch.empty(acc.shape, dtype=out_dtype)
    out.copy_(acc.to(out.dtype))
    fake_ops._emit_parts(out, acc, row_part, col_part)
    if row_stats is not None:
        fake_ops.row_finalize(row_part.view(-1, acc.shape[0], 2), row_stats[2], out=row_stats[0])
    return out


fake_ops_fp8 = types.SimpleNamespace(**{k: v for k, v in vars(fake_ops).items() if not k.startswith("__")})
fake_ops_fp8.gemm, fake_ops_fp8.quant_rows_fp8 = _gemm, _quant_rows_fp8


@pytest.fixture
def patched(monkeypatch):
    monkeypatch.setattr(sdxl_mod, "ops", fake_ops_fp8)


def _unet(weight_format, sd):
    m = sdxl_mod.UNet2DConditionModel(synth.TINY_UNET, device="cpu", weight_format=weight_format)
    m.load_state_dict({k: v.clone() for k, v in sd.items()})
    return m


def _inputs(B=2, hw=16):
    cfg = synth.TINY_UNET
    x = synth.randn("cpu_unet_x", (B, 4, hw, hw))
    ctx = synth.randn("cpu_unet_ctx", (B, 16, cfg["cross_attention_dim"]))
    te = synth.randn("cpu_unet_te", (B, cfg["text_embed_dim"]))
    tid = torch.tensor([[1024.0, 1024.0, 0.0, 0.0, 1024.0, 1024.0]]).repeat(B, 1)
    return x, ctx, dict(text_embeds=te, time_ids=tid)


def rel(a, b):
    return ((a.float() - b.float()).norm() / b.float().norm()).item()


def test_weight_format_is_validated(tmp_path):
    with pytest.raises(SeedxError):
        sdxl_mod.UNet2DConditionModel(synth.TINY_UNET, device="cpu", weight_format="fp8")
    with pytest.raises(SeedxError):
        sdxl_mod.UNet2DConditionModel(synth.TINY_UNET, device="cpu", weight_format="bf16")
    assert sdxl_mod.UNet2DConditionModel(synth.TINY_UNET, device="cpu").weight_format == "fp16"
    c = synth.TINY_UNET
    json.dump(dict(in_channels=4, out_channels=4, block_out_channels=list(c["block_out_channels"]), layers_per_block=c["layers_per_block"],
                   transformer_layers_per_block=list(c["transformer_layers"]), attention_head_dim=list(c["heads"]),
                   cross_attention_dim=c["cross_attention_dim"], addition_time_embed_dim=c["addition_time_embed_dim"],
                   down_block_types=["CrossAttnDownBlock2D" if a else "DownBlock2D" for a in c["down_attn"]]), open(tmp_path / "config.json", "w"))
    torch.save(synth.unet_state_dict(c), tmp_path / "diffusion_pytorch_model.bin")
    m = sdxl_mod.UNet2DConditionModel.from_pretrained(str(tmp_path), device="cpu", weight_format="fp8_e4m3")
    assert m.weight_format == "fp8_e4m3" and all(t.fp8_slots() for t in m.transformers())
    with pytest.raises(SeedxError):
        sdxl_mod.UNet2DConditionModel.from_pretrained(str(tmp_path), device="cpu", weight_format="e5m2")


def test_exactly_the_projection_gemms_get_fp8_copies():
    sd = synth.unet_state_dict(synth.TINY_UNET)
    assert all(not t.fp8_slots() for t in _unet("fp16", sd).transformers())
    m = _unet("fp8_e4m3", sd)
    ts = m.transformers()
    assert len(ts) == 2 * 2 + 1 + 2 * 3                                # down (2 levels with attention x 2), mid, up (2 levels x 3)
    for t in ts:
        assert set(t.fp8_w) == {"proj_in", "proj_out"}
        assert t.fp8_w["proj_in"][0] is t.w_in and t.fp8_w["proj_out"][0] is t.w_out
        for blk in t.blocks:
            f8 = blk["fp8"]
            assert set(f8) == FP8_KINDS
            # the sources are the PACKED fp16 matrices: gamma-folded, QKV-concatenated, GEGLU-interleaved
            assert f8["attn1.qkv"][0] is blk["qkv"].w and f8["attn2.to_q"][0] is blk["q2"].w and f8["ff.net.0"][0] is blk["ff1"].w
            assert f8["attn1.to_out"][0] is blk["w_o1"] and f8["attn2.to_out"][0] is blk["w_o2"] and f8["ff.net.2"][0] is blk["w_ff2"]
            # the hoisted cross-attention K/V stays fp16 only
            assert all(v[0] is not blk["w_kv2"] for v in f8.values())
        for _, (w16, q, s, cs) in t.fp8_slots():
            assert q.dtype == torch.float8_e4m3fn and q.shape == w16.shape and s.dtype == torch.float32 and s.shape == (w16.shape[0],)


def test_scales_and_folded_column_sums():
    sd = synth.unet_state_dict(synth.TINY_UNET)
    m = _unet("fp8_e4m3", sd)
    for t in m.transformers():
        for name, (w16, q, s, cs) in t.fp8_slots():
            q_ref, s_ref = quantize_fp8_rows(w16)
            assert torch.equal(q.view(torch.uint8), q_ref.view(torch.uint8)) and torch.equal(s, s_ref)
            assert ((q.float() * s[:, None] - w16.float()).abs() <= 2.0 ** -4 * w16.float().abs() + s[:, None] * 2.0 ** -9).all()
            if name in FOLDED:
                # the mean correction cancels against what the MMA sums: the dequantized FP8 rows, not the fp16 ones
                # colsum8[n] = s[n] * sum_k q[n, k], within fp32 summation error of the float64 value
                ref = s.double() * q.double().sum(1)
                assert ((cs.double() - ref).abs() <= 1e-6 * s.double() * q.double().abs().sum(1)).all()
            else:
                assert cs is None


def test_tiny_unet_fp8_forward_tracks_the_fp16_host(patched):
    """e4m3 keeps 3 mantissa bits: unit roundoff u = 2^-4 per quantised operand, two operands per product.  Rounding errors of random sign
    average over K in each dot product, so a projection's output carries about sqrt(2/3) u ~ 5 % relative error; the transformer outputs are
    added to a residual stream that the resnets and convs (fp16, unchanged) dominate, so the eps output moves by less than 2u = 12.5 %."""
    sd = synth.unet_state_dict(synth.TINY_UNET)
    x, ctx, added = _inputs()
    ref = _unet("fp16", sd)(x, 601.0, ctx, added_cond_kwargs=added)
    out = _unet("fp8_e4m3", sd)(x, 601.0, ctx, added_cond_kwargs=added)
    e = rel(out, ref)
    assert 1e-4 < e < 2 * 2.0 ** -4, e                                   # different (the FP8 path ran), within the e4m3 bound


def test_partial_checkpoint_rederives_fp8_copies_in_place(patched):
    """a partial checkpoint (to_k / to_v, as the adapter checkpoints carry, plus a folded and a plain projection) loaded after the model is
    built: every FP8 copy keeps its storage (captured graphs stay valid) and equals the copy of a model built from the merged weights"""
    sd = synth.unet_state_dict(synth.TINY_UNET)
    m = _unet("fp8_e4m3", sd)
    ptrs = [(q.data_ptr(), s.data_ptr(), None if cs is None else cs.data_ptr()) for t in m.transformers() for _, (_, q, s, cs) in t.fp8_slots()]
    part = {k: synth.randn("ft8:" + k, v.shape, v.shape[-1] ** -0.5)
            for k, v in sd.items() if k.endswith(("attn2.to_k.weight", "attn2.to_v.weight", "ff.net.2.weight", "attn1.to_q.weight"))}
    assert len(part) >= 16
    m.load_state_dict(part)
    assert ptrs == [(q.data_ptr(), s.data_ptr(), None if cs is None else cs.data_ptr()) for t in m.transformers() for _, (_, q, s, cs) in t.fp8_slots()]
    fresh = _unet("fp8_e4m3", {**sd, **part})
    for t, tf in zip(m.transformers(), fresh.transformers()):
        for (n1, (_, q, s, cs)), (n2, (_, qf, sf, csf)) in zip(t.fp8_slots(), tf.fp8_slots()):
            assert n1 == n2 and torch.equal(q.view(torch.uint8), qf.view(torch.uint8)) and torch.equal(s, sf)
            assert (cs is None) == (csf is None) and (cs is None or torch.equal(cs, csf))
    x, ctx, added = _inputs(B=1)
    assert torch.equal(m(x, 301.0, ctx, added_cond_kwargs=added), fresh(x, 301.0, ctx, added_cond_kwargs=added))
