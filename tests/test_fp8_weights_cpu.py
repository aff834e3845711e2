"""Host logic of the opt-in FP8 (e4m3) LLaMA weights on the CPU: the per-row quantiser, the in-place LoRA / plain updates of an FP8 model,
and the prefill / decode wiring of `LlamaForCausalLM(weight_format="fp8_e4m3")` through tests/fake_ops.py, extended here with plain-torch
restatements of the two FP8 entry points (seedx_gemv_fp8, seedx_dequant_fp8).  The kernels themselves are checked in test_fp8_weights_gpu.py."""
import inspect
import types

import pytest
import torch
import torch.nn.functional as F

import fake_ops
from seedx_b200 import llm as llm_mod
from seedx_b200 import synth
from seedx_b200._lib import SeedxError
from seedx_b200.llm import FP8_MAX, PROJECTIONS, quantize_fp8_rows
from seedx_b200.lora import lora_delta


def _gemv(W, x, out, *, rms_w=None, eps=1e-5, residual=None, gated=False, scale=None):
    """ops.gemv: fp16 weights as in fake_ops; FP8 weights with their row scales applied to the fp32 dot product (seedx_gemv_fp8)"""
    if scale is None:
        return fake_ops.gemv(W, x, out, rms_w=rms_w, eps=eps, residual=residual, gated=gated)
    assert W.dtype == torch.float8_e4m3fn and scale.numel() == W.shape[0]
    x2 = x.reshape(-1, W.shape[1]).float()
    if rms_w is not None:
        x2 = x2 * torch.rsqrt(x2.pow(2).mean(-1, keepdim=True) + eps) * rms_w
    r = (x2.half().float() @ W.float().t()) * scale                  # activations staged as fp16; s[n] * dot(n, b)
    if gated:
        r = r[:, 0::2] * F.silu(r[:, 1::2])                          # s[2j] * up * silu(s[2j+1] * gate)
    if residual is not None:
        r = r + residual.reshape(r.shape)
    out.reshape(r.shape).copy_(r)
    return out


def _dequant_fp8(W8, scale, out):
    out.copy_((W8.float() * scale[:, None]).half())
    return out


fake_ops_fp8 = types.SimpleNamespace(**{k: v for k, v in vars(fake_ops).items() if not k.startswith("__")})
fake_ops_fp8.gemv, fake_ops_fp8.dequant_fp8 = _gemv, _dequant_fp8


@pytest.fixture
def host(monkeypatch):
    monkeypatch.setattr(llm_mod, "ops", fake_ops_fp8)
    cfg = synth.TINY_LLAMA
    sd = synth.llama_state_dict(cfg)

    def make(weight_format, state=None, max_len=256):
        m = llm_mod.LlamaForCausalLM(cfg, max_len=max_len, device="cpu", kv_page_size=16, weight_format=weight_format)
        m.load_state_dict({k: v.clone() for k, v in (state or sd).items()})
        return m
    return dict(cfg=cfg, sd=sd, make=make)


def _weights(seed=0):
    g = torch.Generator().manual_seed(seed)
    w = torch.randn((64, 320), generator=g) * torch.logspace(-3, 3, 64)[:, None]       # row magnitudes over six decades
    w[5] = 0.0                                                                            # an all-zero row
    w[9] *= 1e4                                                                           # values far beyond 448 before scaling
    w[11, :] = 0.0
    w[11, 7] = -3.0                                                                       # a single non-zero element
    return w


def test_quantiser_scales_nan_zero_rows_and_round_trip():
    w = _weights()
    q, s = quantize_fp8_rows(w)
    assert q.dtype == torch.float8_e4m3fn and s.dtype == torch.float32 and q.shape == w.shape and s.shape == (64,)
    amax = w.abs().amax(1)
    nz = amax > 0
    assert torch.equal(s[nz], amax[nz] / FP8_MAX)                     # per-row scale = amax / 448
    assert torch.equal(s[~nz], torch.ones_like(s[~nz]))               # all-zero row: s = 1 ...
    qf = q.float()
    assert torch.equal(qf[5], torch.zeros(320))                       # ... and q = 0
    assert not torch.isnan(qf).any() and qf.abs().max() <= FP8_MAX    # rows beyond 448 before scaling: no NaN from the cast
    assert torch.equal(qf.abs().amax(1)[nz], torch.full((int(nz.sum()),), FP8_MAX))   # the row maximum maps to 448 exactly
    # every element whose scaled value is a normal e4m3 number (|w / s| >= 2^-6) round-trips within half an e4m3 ulp: 2^-4 relative
    back = qf * s[:, None]
    normal = (w / s[:, None]).abs() >= 2.0 ** -6
    assert normal.float().mean() > 0.9
    err = (back - w).abs()[normal] / w.abs()[normal]
    assert err.max() <= 2.0 ** -4 * (1 + 1e-6), err.max()


def test_weight_format_is_validated_and_reaches_every_projection(host):
    with pytest.raises(SeedxError):
        llm_mod.LlamaForCausalLM(host["cfg"], device="cpu", weight_format="fp8")
    m16, m8 = host["make"]("fp16"), host["make"]("fp8_e4m3")
    for L16, L8 in zip(m16.layers, m8.layers):
        for k in PROJECTIONS:
            assert L8[k].dtype == torch.float8_e4m3fn and L8[k].shape == L16[k].shape and L8[k + "_s"].shape == (L16[k].shape[0],)
            q, s = quantize_fp8_rows(L16[k])                          # quantised from the packed fp16 matrix
            assert torch.equal(L8[k].view(torch.uint8), q.view(torch.uint8)) and torch.equal(L8[k + "_s"], s)
            assert k + "_s" not in L16
    for a in ("embed", "lm_head"):                                     # stays fp16
        assert getattr(m8, a).dtype == torch.float16 and torch.equal(getattr(m8, a), getattr(m16, a))
    assert m8.norm.dtype == torch.float32 and m8.layers[0]["ln1"].dtype == torch.float32
    assert "llm_weight_format" in inspect.signature(__import__("seedx_b200.engine", fromlist=["x"]).SeedXEngine).parameters
    assert inspect.signature(llm_mod.LlamaForCausalLM.from_pretrained).parameters["weight_format"].default == "fp16"


def _dequantized_state_dict(m8, sd, cfg):
    """HF-named state dict whose projections are the FP8 model's s * q rounded to fp16 (exactly what prefill's dequantization produces)"""
    D, Fh = cfg["hidden"], cfg["ffn"]
    out = dict(sd)
    for i, L in enumerate(m8.layers):
        p = f"model.layers.{i}."
        deq = {k: (L[k].float() * L[k + "_s"][:, None]).half().float() for k in PROJECTIONS}
        for j, n in enumerate(("q_proj", "k_proj", "v_proj")):
            out[p + f"self_attn.{n}.weight"] = deq["wqkv"][j * D:(j + 1) * D]
        out[p + "self_attn.o_proj.weight"] = deq["wo"]
        out[p + "mlp.up_proj.weight"] = deq["wgu"].view(Fh, 2, D)[:, 0]
        out[p + "mlp.gate_proj.weight"] = deq["wgu"].view(Fh, 2, D)[:, 1]
        out[p + "mlp.down_proj.weight"] = deq["wdown"]
    return out


def test_fp8_prefill_and_greedy_loop_through_the_host(host):
    """prefill of the FP8 model = fp16 model on the dequantized weights, exactly (same fp16 operands); the decode loop applies the row scales
    after the dot product instead of rounding s*q to fp16, so its states agree to fp16 operand rounding and the greedy ids agree."""
    cfg, sd = host["cfg"], host["sd"]
    m8 = host["make"]("fp8_e4m3")
    ref = host["make"]("fp16", _dequantized_state_dict(m8, sd, cfg))
    tok = synth.SynthTokenizer(vocab=cfg["vocab"])
    ids = [tok.bos_token_id] + tok.encode("draw a cat and a dog")
    emb = sd["model.embed_tokens.weight"][torch.tensor(ids)].float()
    l8, h8 = m8.logits_all(m8.prefill(emb))
    lr, hr = ref.logits_all(ref.prefill(emb))
    assert torch.equal(l8, lr) and torch.equal(h8, hr)
    o8 = m8.generate_greedy(ids, emb, max_new_tokens=12, use_graph=False)
    orf = ref.generate_greedy(ids, emb, max_new_tokens=12, use_graph=False)
    assert o8.sequences.tolist() == orf.sequences.tolist()
    rel = ((o8.last_hidden_states - orf.last_hidden_states).norm() / orf.last_hidden_states.norm()).item()
    assert rel < 1e-3, rel


def test_update_weights_requantizes_the_touched_rows_in_place(host):
    cfg = host["cfg"]
    D, Fh = cfg["hidden"], cfg["ffn"]
    m = host["make"]("fp8_e4m3")
    before = [{k: (v.view(torch.uint8).clone() if v.dtype == torch.float8_e4m3fn else v.clone()) for k, v in L.items()} for L in m.layers]
    ptrs = [(L[k].data_ptr(), L[k + "_s"].data_ptr()) for L in m.layers for k in PROJECTIONS]
    g = torch.Generator().manual_seed(3)
    r = 4
    lora = {"model.layers.0.self_attn.q_proj": (torch.randn((r, D), generator=g) * D ** -0.5, torch.randn((D, r), generator=g) * 0.1),
            "model.layers.1.mlp.up_proj": (torch.randn((r, D), generator=g) * D ** -0.5, torch.randn((Fh, r), generator=g) * 0.1),
            "model.layers.1.mlp.down_proj": (torch.randn((r, Fh), generator=g) * Fh ** -0.5, torch.randn((D, r), generator=g) * 0.1)}
    plain = {"model.layers.0.self_attn.v_proj.weight": torch.randn((D, D), generator=g) * 0.05}
    deq = lambda q, s: q.float() * s[:, None]  # noqa: E731
    # expected: quantise the fp32 merged weight (dequantized rows + delta), or the replacement, row for row
    L0, L1 = before[0], before[1]
    u8 = lambda t: t.view(torch.float8_e4m3fn)  # noqa: E731
    exp_q = quantize_fp8_rows(deq(u8(L0["wqkv"][:D]), L0["wqkv_s"][:D]) + lora_delta(*lora["model.layers.0.self_attn.q_proj"], 2.0))
    exp_v = quantize_fp8_rows(plain["model.layers.0.self_attn.v_proj.weight"])
    exp_up = quantize_fp8_rows(deq(u8(L1["wgu"][0::2]), L1["wgu_s"][0::2]) + lora_delta(*lora["model.layers.1.mlp.up_proj"], 2.0))
    exp_dn = quantize_fp8_rows(deq(u8(L1["wdown"]), L1["wdown_s"]) + lora_delta(*lora["model.layers.1.mlp.down_proj"], 2.0))
    assert m.update_weights(plain, lora, scaling=2.0) == []
    assert ptrs == [(L[k].data_ptr(), L[k + "_s"].data_ptr()) for L in m.layers for k in PROJECTIONS]   # in place: graphs stay valid
    bits = lambda t: t.view(torch.uint8)  # noqa: E731
    A0, A1 = m.layers
    for got_q, got_s, (eq, es) in ((A0["wqkv"][:D], A0["wqkv_s"][:D], exp_q), (A0["wqkv"][2 * D:], A0["wqkv_s"][2 * D:], exp_v),
                                   (A1["wgu"][0::2], A1["wgu_s"][0::2], exp_up), (A1["wdown"], A1["wdown_s"], exp_dn)):
        assert torch.equal(bits(got_q), bits(eq)) and torch.equal(got_s, es)
    # untouched rows keep their bits: k rows of wqkv, the gate rows of wgu, and every other matrix
    assert torch.equal(bits(A0["wqkv"][D:2 * D]), L0["wqkv"][D:2 * D]) and torch.equal(A0["wqkv_s"][D:2 * D], L0["wqkv_s"][D:2 * D])
    assert torch.equal(bits(A1["wgu"][1::2]), L1["wgu"][1::2]) and torch.equal(A1["wgu_s"][1::2], L1["wgu_s"][1::2])
    for L, B, keys in ((A0, L0, ("wo", "wgu", "wdown")), (A1, L1, ("wqkv", "wo"))):
        for k in keys:
            assert torch.equal(bits(L[k]), B[k]) and torch.equal(L[k + "_s"], B[k + "_s"])
    # a shape mismatch is still refused
    with pytest.raises(SeedxError):
        m.update_weights({"model.layers.0.self_attn.o_proj.weight": torch.zeros((D, D + 1))})
