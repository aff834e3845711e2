"""Opt-in FP8 (e4m3) LLaMA weights on the device: seedx_gemv_fp8 and seedx_dequant_fp8 against float64 / bit-exact references, and
`LlamaForCausalLM(weight_format="fp8_e4m3")` end to end (prefill, CUDA-graph decode, continuous batching, LoRA after capture) against a float32
forward over the dequantized weights."""
import json
import os

import pytest
import torch
import torch.nn.functional as F

from seedx_b200 import synth

pytestmark = pytest.mark.gpu
TOL = 1e-3


def rel(a, b):
    return ((a.float().cpu() - b.float().cpu()).norm() / b.float().cpu().norm()).item()


def _fp8_matrix(N, K, seed):
    """random FP8 weight with per-row scales over four decades, plus two all-zero rows (scale 1, q = 0)"""
    from seedx_b200.llm import quantize_fp8_rows
    g = torch.Generator(device="cuda").manual_seed(seed)
    w = torch.randn((N, K), generator=g, device="cuda") * torch.logspace(-2, 2, N, device="cuda")[torch.randperm(N, device="cuda")][:, None]
    w[min(3, N - 1)] = 0.0
    w[N - 1] = 0.0
    return quantize_fp8_rows(w)


# (N, K, batches): K in {64, 192, 5120, 13824}; N with a partial last 8-row tile (7, 1202) and the 13B projection shapes
GEMV_CASES = [(7, 64, (1, 2, 4, 8)), (1202, 192, (1, 2, 4, 8)), (15360, 5120, (1, 4)), (5120, 5120, (2,)), (27648, 5120, (8,)),
              (5120, 13824, (1, 2, 4))]


@pytest.mark.parametrize("N,K,batches", GEMV_CASES)
def test_gemv_fp8_matches_float64(N, K, batches):
    """out = s * dot(q, fp16(x)) (+ residual) or the gated form, per element within 1e-3 of sum_k |s q x| of float64 (fp32 accumulation is
    ~1e-6 of that; a wrong scale or k permutation misses by orders of magnitude).  x is staged as fp16 like in the fp16 GEMV; with RMSNorm
    the reference normalises in fp32 and may round an element to the neighbouring fp16 value: 2^-11 relative, inside the bound."""
    from seedx_b200 import ops
    q, s = _fp8_matrix(N, K, N + K)
    q64, s64 = q.double(), s.double()
    g = torch.Generator(device="cuda").manual_seed(7)
    rw = torch.randn((K,), generator=g, device="cuda") * 0.1 + 1.0
    for B in batches:
        x = torch.randn((B, K), generator=g, device="cuda") * 2.0
        res = torch.randn((B, N), generator=g, device="cuda")
        xn = (x * torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + 1e-5) * rw)
        for name, kw, xs in (("plain", {}, x), ("rms", dict(rms_w=rw, eps=1e-5), xn), ("residual", dict(residual=res), x)):
            x16 = xs.half().double()
            dot = (x16 @ q64.t()) * s64                                   # [B, N]
            mag = (x16.abs() @ q64.abs().t()) * s64
            out = torch.full((B, N), float("nan"), device="cuda")
            ops.gemv(q, x, out, scale=s, **kw)
            ref = dot + (res.double() if name == "residual" else 0.0)
            bound = TOL * mag + (1e-6 * res.double().abs() if name == "residual" else 0.0)
            err = (out.double() - ref).abs()
            assert torch.isfinite(out).all() and (err <= bound).all(), (name, B, (err - bound).max().item())
            assert (out[:, [min(3, N - 1), N - 1]].double() == (ref[:, [min(3, N - 1), N - 1]])).all()     # zero rows: exactly 0 (+ residual)
        if N % 2 == 0:
            x16 = xn.half().double()
            r = (x16 @ q64.t()) * s64
            a = (x16.abs() @ q64.abs().t()) * s64
            up, gate, a_up, a_gate = r[:, 0::2], r[:, 1::2], a[:, 0::2], a[:, 1::2]
            ref = up * F.silu(gate)
            bound = TOL * (a_up * F.silu(gate).abs() + up.abs() * 1.1 * a_gate) + 1e-30   # |silu'| <= 1.1
            out = torch.full((B, N // 2), float("nan"), device="cuda")
            ops.gemv(q, x, out, scale=s, rms_w=rw, eps=1e-5, gated=True)
            err = (out.double() - ref).abs()
            assert torch.isfinite(out).all() and (err <= bound).all(), ("gated", B, (err - bound).max().item())


def test_gemv_fp8_argument_checks():
    from seedx_b200 import ops
    from seedx_b200._lib import SeedxError
    q, s = _fp8_matrix(64, 13824, 1)
    with pytest.raises(SeedxError):           # 8 slots x K = 13824 fp16 activations exceed shared memory
        ops.gemv(q, torch.zeros((8, 13824), device="cuda"), torch.zeros((8, 64), device="cuda"), scale=s)
    q, s = _fp8_matrix(64, 96, 1)
    with pytest.raises(SeedxError):           # K % 64
        ops.gemv(q, torch.zeros((1, 96), device="cuda"), torch.zeros((1, 64), device="cuda"), scale=s)
    q, s = _fp8_matrix(63, 64, 1)
    with pytest.raises(SeedxError):           # gated needs even N
        ops.gemv(q, torch.zeros((1, 64), device="cuda"), torch.zeros((1, 32), device="cuda"), scale=s, gated=True)


@pytest.mark.parametrize("N,K", [(7, 64), (1202, 192), (5120, 13824), (27648, 5120), (3, 16)])
def test_dequant_fp8_is_bit_exact(N, K):
    from seedx_b200 import ops
    q, s = _fp8_matrix(N, K, 11)
    buf = torch.full((N * K + 64,), float("nan"), device="cuda", dtype=torch.float16)
    out = buf[:N * K].view(N, K)
    ops.dequant_fp8(q, s, out)
    torch.cuda.synchronize()
    assert torch.equal(out.view(torch.int16), (q.float() * s[:, None]).half().view(torch.int16))
    assert torch.isnan(buf[N * K:]).all()                                # nothing written past the end


# ------------------------------------------------------------------------------------------------------------------------------------------
# end to end
# ------------------------------------------------------------------------------------------------------------------------------------------
def _dequantized_sd(m8, sd):
    """HF-named fp32 state dict whose projections are the FP8 model's s * q (CPU, for the oracle)"""
    D, Fh = m8.cfg["hidden"], m8.cfg["ffn"]
    out = dict(sd)
    for i, L in enumerate(m8.layers):
        p = f"model.layers.{i}."
        deq = {k: (L[k].float() * L[k + "_s"][:, None]).cpu() for k in ("wqkv", "wo", "wgu", "wdown")}
        for j, n in enumerate(("q_proj", "k_proj", "v_proj")):
            out[p + f"self_attn.{n}.weight"] = deq["wqkv"][j * D:(j + 1) * D]
        out[p + "self_attn.o_proj.weight"] = deq["wo"]
        out[p + "mlp.up_proj.weight"] = deq["wgu"].view(Fh, 2, D)[:, 0]
        out[p + "mlp.gate_proj.weight"] = deq["wgu"].view(Fh, 2, D)[:, 1]
        out[p + "mlp.down_proj.weight"] = deq["wdown"]
    return out


def _check_against_dequantized_forward(m8, m16, sd, ids, new, label):
    """prefill logits, and the decode-step hidden states and last-step logits of a CUDA-graph greedy run, vs a float32 forward over the
    dequantized weights with the generated ids teacher-forced"""
    from oracle import llm as ollm
    cfg = m8.cfg
    emb_tab = sd["model.embed_tokens.weight"]
    P = len(ids)
    emb = emb_tab[torch.tensor(ids)].float()
    logits, _ = m8.logits_all(m8.prefill(emb.cuda()))
    out = m8.generate_greedy(ids, emb.cuda(), max_new_tokens=new)          # decode steps replay the captured graph
    assert m8._graphs, "the decode loop did not run under a CUDA graph"
    seq = out.sequences[0].tolist()
    assert len(seq) == P + new
    sdq = _dequantized_sd(m8, sd)
    with torch.no_grad():
        ref_logits, ref_hid, _ = ollm.llama_forward(sdq, cfg, emb_tab[torch.tensor(seq[:-1])].float(), 0, None)
    e1 = rel(logits, ref_logits[:P])
    e2 = rel(out.last_hidden_states, ref_hid[P:P + new - 1])
    e3 = rel(m8.logits[0], ref_logits[P + new - 2])
    l16, _ = m16.logits_all(m16.prefill(emb.cuda()))
    d16 = rel(logits, l16)
    ids16 = m16.generate_greedy(ids, emb.cuda(), max_new_tokens=new).sequences[0][P:].tolist()
    print(f"{label}: FP8 vs float32 forward on the dequantized weights: prefill logits rel {e1:.3e}, decode hidden rel {e2:.3e}, "
          f"last decode-step logits rel {e3:.3e}; FP8 vs fp16 model: prefill logits rel {d16:.3e}, greedy ids "
          f"{'equal' if ids16 == seq[P:] else 'differ'}")
    assert e1 < TOL and e2 < TOL and e3 < TOL, (e1, e2, e3)


def test_tiny_llama_fp8_end_to_end():
    from seedx_b200.llm import LlamaForCausalLM
    cfg = synth.TINY_LLAMA
    sd = synth.llama_state_dict(cfg)
    m8 = LlamaForCausalLM(cfg, max_len=256, weight_format="fp8_e4m3")
    m8.load_state_dict(sd)
    m16 = LlamaForCausalLM(cfg, max_len=256)
    m16.load_state_dict(sd)
    tok = synth.SynthTokenizer(vocab=cfg["vocab"])
    ids = [tok.bos_token_id] + tok.encode("a photo of a cat sitting on a red chair")
    _check_against_dequantized_forward(m8, m16, sd, ids, 12, "tiny LLaMA")


def test_full_width_two_layers_fp8_end_to_end_and_memory():
    """hidden 5120 / 40 heads / FFN 13824 / vocab 32330, 2 layers: K = 5120 and 13824 in the GEMVs, 283 MB dequantization scratch"""
    from seedx_b200.llm import LLAMA_13B, PROJECTIONS, LlamaForCausalLM
    cfg = dict(LLAMA_13B, layers=2)
    synth.set_device("cuda")
    try:
        sd_dev = synth.llama_state_dict(cfg)
    finally:
        synth.set_device("cpu")
    sd = {k: v.cpu().float() for k, v in sd_dev.items()}
    m8 = LlamaForCausalLM(cfg, max_len=128, weight_format="fp8_e4m3")
    m8.load_state_dict(sd_dev)
    m16 = LlamaForCausalLM(cfg, max_len=128)
    m16.load_state_dict(sd_dev)
    del sd_dev
    b8 = sum(L[k].numel() * L[k].element_size() + L[k + "_s"].numel() * 4 for L in m8.layers for k in PROJECTIONS)
    b16 = sum(L[k].numel() * L[k].element_size() for L in m16.layers for k in PROJECTIONS)
    print(f"packed projections: FP8 + scales {b8 / 1e6:.1f} MB = {100 * b8 / b16:.3f} % of fp16 {b16 / 1e6:.1f} MB")
    assert b8 <= 0.501 * b16
    ids = ((synth.randn("fp8_fs_ids", (40,)).abs() * 1000).long() % 30000 + 3).tolist()
    _check_against_dequantized_forward(m8, m16, sd, ids, 6, "LLaMA 13B width x 2 layers")


def _tiny_fp8(max_len=512):
    from seedx_b200.llm import LlamaForCausalLM
    cfg = synth.TINY_LLAMA
    m = LlamaForCausalLM(cfg, max_len=max_len, weight_format="fp8_e4m3")
    m.load_state_dict(synth.llama_state_dict(cfg))
    return m, cfg


def test_continuous_batching_fp8():
    """staggered admissions on 4 slots between replays of one captured FP8 decode graph == each request decoded alone"""
    from seedx_b200.serving import ContinuousBatcher
    m, cfg = _tiny_fp8()
    sd = synth.llama_state_dict(cfg)
    tok = synth.SynthTokenizer(vocab=cfg["vocab"])
    img_ids = tok.encode("".join(["<img>"] + ["<img_{:05d}>".format(i) for i in range(64)] + ["</img>"]))
    emb_of = lambda ids: sd["model.embed_tokens.weight"][torch.tensor(ids)].float()  # noqa: E731
    base = [tok.bos_token_id] + tok.encode("describe the picture of a small boat on a lake at night")
    ids_b = base + [tok.encode("<img>")[0]]
    reqs = [(base, emb_of(base), 16), (ids_b, emb_of(ids_b), 72), (base[:9], emb_of(base[:9]), 20), (base[3:15], emb_of(base[3:15]), 9),
            (base[:6], emb_of(base[:6]), 33), (ids_b[4:], emb_of(ids_b[4:]), 70)]
    want = [m.generate_greedy(i, e.cuda(), img_ids=img_ids, max_new_tokens=n) for i, e, n in reqs]
    cb = ContinuousBatcher(m, slots=4, img_ids=img_ids, eos_id=None, use_graph=True)
    got = cb.run(arrivals={0: [reqs[0], reqs[1]], 2: [reqs[2]], 3: [reqs[3], reqs[4]], 25: [reqs[5]]})
    assert sorted(got) == list(range(len(reqs)))
    for rid, w in enumerate(want):
        assert torch.equal(got[rid].sequences, w.sequences), rid
        assert rel(got[rid].last_hidden_states, w.last_hidden_states) < 1e-3, rid
    assert cb.idle() and cb.graph is not None


def test_lora_update_after_capture_reaches_the_replayed_graph():
    """update_weights on a captured FP8 model writes q and the scales in place: the next replay of the same graph computes with the new weights
    (the merge arithmetic itself is pinned on the CPU in test_fp8_weights_cpu.py)"""
    m, cfg = _tiny_fp8()
    D, Fh = cfg["hidden"], cfg["ffn"]
    sd = synth.llama_state_dict(cfg)
    tok = synth.SynthTokenizer(vocab=cfg["vocab"])
    ids = [tok.bos_token_id] + tok.encode("a dog running on the beach")
    emb = sd["model.embed_tokens.weight"][torch.tensor(ids)].float().cuda()
    before = m.generate_greedy(ids, emb, max_new_tokens=10)
    graph = next(iter(m._graphs.values()))
    g = torch.Generator().manual_seed(5)
    lora = {f"model.layers.{i}.{n}": (torch.randn((8, din), generator=g) * din ** -0.5, torch.randn((dout, 8), generator=g) * 0.3)
            for i in range(cfg["layers"]) for n, din, dout in (("self_attn.q_proj", D, D), ("self_attn.v_proj", D, D),
                                                                 ("mlp.up_proj", D, Fh), ("mlp.down_proj", Fh, D))}
    assert m.update_weights(lora=lora, scaling=2.0) == []
    after = m.generate_greedy(ids, emb, max_new_tokens=10)
    assert next(iter(m._graphs.values())) is graph                          # the same captured graph was replayed
    eager = m.generate_greedy(ids, emb, max_new_tokens=10, use_graph=False)
    assert after.sequences.tolist() == eager.sequences.tolist()
    assert rel(after.last_hidden_states, eager.last_hidden_states) < 1e-6
    assert rel(after.last_hidden_states, before.last_hidden_states) > 1e-2   # the update changed the model


def test_from_pretrained_through_the_yaml_factory(tmp_path):
    from safetensors.torch import save_file
    from seedx_b200 import compat
    from seedx_b200._lib import SeedxError
    compat.install()
    import hydra
    from omegaconf import OmegaConf
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cfg = synth.TINY_LLAMA
    d = tmp_path / "llm"
    os.makedirs(d)
    json.dump(dict(vocab_size=cfg["vocab"], hidden_size=cfg["hidden"], num_hidden_layers=cfg["layers"], num_attention_heads=cfg["heads"],
                   intermediate_size=cfg["ffn"], rms_norm_eps=cfg["eps"]), open(d / "config.json", "w"))
    save_file({k: v.half().contiguous() for k, v in synth.llama_state_dict(cfg).items()}, str(d / "model.safetensors"))
    y = OmegaConf.load(os.path.join(root, "configs", "clm_models", "llm_seed_x.yaml"))
    y["pretrained_model_name_or_path"] = str(d)
    llm = hydra.utils.instantiate(y, weight_format="fp8_e4m3")
    assert llm.weight_format == "fp8_e4m3" and llm.layers[0]["wgu"].dtype == torch.float8_e4m3fn
    assert hydra.utils.instantiate(y).layers[0]["wgu"].dtype == torch.float16
    with pytest.raises(SeedxError):
        hydra.utils.instantiate(y, weight_format="int8")
