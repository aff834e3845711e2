"""Stage 2 host: LLaMA causal LM (prefill on the tensor-core GEMM, token loop on HBM-bound GEMV kernels) behind the
surface of the reference class ``src.models.mllm.modeling_llama_xformer.LlamaForCausalLM``
(/root/reference/src/models/mllm/modeling_llama_xformer.py:612-779): ``from_pretrained``, ``get_input_embeddings``,
and a greedy ``generate`` that reproduces what seed_x.py:184-197 consumes (sequences + last-layer hidden states).

HBM layout: weights fp16 ([q|k|v] fused, [up_j,gate_j] row-interleaved for the SwiGLU epilogue); residual stream fp32;
KV cache fp16, PAGED: per layer and tensor a pool [n_pages, 64 tokens, H*d]; every sequence slot owns a row of a device page table,
rows are appended in place (the reference re-copies the whole cache with torch.cat every step, :215-218); sampler state (sequence,
length, EOS marker) device resident.
"""
import json
import os

import torch

from . import _lib, ops, trace
from ._lib import SeedxError

LLAMA_13B = dict(vocab=32330, hidden=5120, layers=40, heads=40, ffn=13824, eps=1e-5)
WEIGHT_FORMATS = ("fp16", "fp8_e4m3")
FP8_MAX = 448.0                                # largest finite float8_e4m3fn
PROJECTIONS = ("wqkv", "wo", "wgu", "wdown")   # the packed per-layer matrices that weight_format="fp8_e4m3" stores in FP8


def quantize_fp8_rows(w):
    """Per-output-row FP8 quantisation of a weight [N, K]: s[n] = amax|w[n]| / 448 (1 for an all-zero row), q = w / s in float8_e4m3fn.
    Returns (q, s fp32 [N]) with w[n] ~= s[n] * q[n].  The clamp matters: torch's cast turns anything beyond +-448 into NaN, and w / s can
    round a hair above 448 at the row maximum."""
    w = w.float()
    s = w.abs().amax(dim=1) / FP8_MAX
    s = torch.where(s > 0, s, torch.ones_like(s))
    q = (w / s[:, None]).clamp(-FP8_MAX, FP8_MAX).to(torch.float8_e4m3fn)
    return q.contiguous(), s.contiguous()


class _Embedding:
    def __init__(self, llm):
        self.llm = llm

    def __call__(self, input_ids):
        """ids [1,P] or [P] (any device / list) -> fp32 device tensor [1,P,D] (the reference returns model-dtype rows)."""
        ids = torch.as_tensor(input_ids).reshape(-1).to(self.llm.device, torch.int32)
        out = torch.empty((1, ids.numel(), self.llm.cfg["hidden"]), device=self.llm.device, dtype=torch.float32)
        ops.embed_rows(self.llm.embed, out, ids=ids)
        return out


class KVPageAllocator:
    """Host-side free list of KV-cache pages (the device side only ever sees the page table).  Pages are handed out from the END of the
    list, so consecutive logical pages of a sequence are not physically consecutive even on a fresh pool — the indirection is always
    exercised, not just after fragmentation."""

    def __init__(self, n_pages):
        self.n_pages = n_pages
        self.free = list(range(n_pages))

    def alloc(self, n):
        if n > len(self.free):
            raise SeedxError(f"KV cache exhausted: {n} pages requested, {len(self.free)} of {self.n_pages} free")
        out = [self.free.pop() for _ in range(n)]
        return out

    def release(self, pages):
        self.free.extend(pages)

    def shuffle(self, seed=0):
        import random
        random.Random(seed).shuffle(self.free)


class GreedyOutput:
    def __init__(self, sequences, hidden, n_generated):
        self.sequences = sequences          # [1, P + n] int64 (host)
        self.last_hidden_states = hidden    # fp32 device [n - 1, D]: post-norm state of the position that consumed generated token j
        self.n_generated = n_generated


class AutoImageTokenGenerationProcessor:
    """Same constructor and ``img_ids_list`` as the reference logits processor (/root/reference/src/models/mllm/generation.py:9-31).
    The rule itself — after ``<img>`` / ``<img_k>`` force the next id of the span (score = max + 10), otherwise set the scores of
    ``<img_0..n-1>`` and ``</img>`` to 0.0 — runs inside ``logits_argmax_kernel`` on the device; ``__call__`` restates it for host tensors
    so the object still works as a plain HF ``LogitsProcessor``."""

    def __init__(self, tokenizer, num_img_gen_tokens=64):
        s = "".join(["<img>"] + ["<img_{:05d}>".format(i) for i in range(num_img_gen_tokens)] + ["</img>"])
        self.img_ids_list = tokenizer.encode(s, add_special_tokens=False)

    def __call__(self, input_ids, scores):
        for i in range(input_ids.shape[0]):
            cur = int(input_ids[i, -1])
            if cur in self.img_ids_list[:-1]:
                scores[i, ..., self.img_ids_list[self.img_ids_list.index(cur) + 1]] = scores[i, ...].max() + 10.0
            else:
                scores[i, ..., torch.tensor(self.img_ids_list[1:], dtype=torch.long)] = 0.0
        return scores


class GreedySearchOutput(dict):
    """``return_dict_in_generate=True`` result: ``.sequences`` [1, P+n] int64 and ``.hidden_states`` in the HF layout the reference
    consumes at seed_x.py:196-197 — one tuple per generation step whose LAST element is the post-norm hidden state, [1, P, D] for the
    first step and [1, 1, D] afterwards (the per-layer intermediate states are not materialised)."""

    def __getattr__(self, k):
        try:
            return self[k]
        except KeyError as e:
            raise AttributeError(k) from e


class LlamaForCausalLM:
    def __init__(self, cfg=None, max_len=2048, device="cuda", kv_page_size=64, kv_pages=None, weight_format="fp16"):
        """weight_format="fp8_e4m3" stores the four projection matrices of every layer (wqkv, wo, wgu, wdown) as float8_e4m3fn with one
        fp32 scale per output row: the token loop streams half the bytes (seedx_gemv_fp8) and prefill dequantizes each matrix into an fp16
        scratch buffer right before its GEMM.  The embedding table, lm_head and the norms stay in fp16 / fp32."""
        if weight_format not in WEIGHT_FORMATS:
            raise SeedxError(f"weight_format {weight_format!r}: expected one of {WEIGHT_FORMATS}")
        self.weight_format = weight_format
        self.cfg = dict(LLAMA_13B if cfg is None else cfg)
        self.device = torch.device(device)
        self.max_len = max_len
        if kv_page_size < 1 or kv_page_size & (kv_page_size - 1):
            raise SeedxError("kv_page_size must be a power of two")
        self.page_size, self.kv_pages = kv_page_size, kv_pages
        self.dtype = torch.float16
        self._loaded = False
        self._graphs = {}
        self._hidden = None
        self.batched_prefill = os.environ.get("SEEDX_BATCHED_PREFILL", "1") != "0"
        self.jump_forward = os.environ.get("SEEDX_JUMP_FORWARD", "1") != "0"     # forced image spans ride in the prefill pass
        self.jump_forward_mid = os.environ.get("SEEDX_JUMP_FORWARD_MID", "0") == "1"   # experimental: also spans opened mid-generation

    # ---- reference-compatible plumbing --------------------------------------------------------------------------------
    @classmethod
    def from_pretrained(cls, pretrained_model_name_or_path, low_cpu_mem_usage=True, torch_dtype=None, weight_format="fp16", **kw):
        d = pretrained_model_name_or_path
        c = json.load(open(os.path.join(d, "config.json")))
        cfg = dict(vocab=c["vocab_size"], hidden=c["hidden_size"], layers=c["num_hidden_layers"], heads=c["num_attention_heads"],
                   ffn=c["intermediate_size"], eps=c.get("rms_norm_eps", 1e-5), eos=c.get("eos_token_id", 2))
        m = cls(cfg, weight_format=weight_format)
        sd = {}
        idx = os.path.join(d, "pytorch_model.bin.index.json")
        sidx = os.path.join(d, "model.safetensors.index.json")
        if os.path.exists(sidx):
            from safetensors.torch import load_file
            for f in sorted(set(json.load(open(sidx))["weight_map"].values())):
                sd.update(load_file(os.path.join(d, f)))
        elif os.path.exists(idx):
            for f in sorted(set(json.load(open(idx))["weight_map"].values())):
                sd.update(torch.load(os.path.join(d, f), map_location="cpu"))
        elif os.path.exists(os.path.join(d, "model.safetensors")):
            from safetensors.torch import load_file
            sd = load_file(os.path.join(d, "model.safetensors"))
        else:
            sd = torch.load(os.path.join(d, "pytorch_model.bin"), map_location="cpu")
        m.load_state_dict(sd)
        return m

    def eval(self):
        return self

    def to(self, *a, **k):
        return self

    def get_input_embeddings(self):
        return _Embedding(self)

    def load_state_dict(self, sd, strict=False, device_generator=None):
        cfg, dev = self.cfg, self.device
        D, H = cfg["hidden"], cfg["heads"]
        if D // H != 128:
            raise SeedxError("the decode kernels are specialised for head_dim 128 (LLaMA)")
        h = lambda t: t.to(dev, torch.float16).contiguous()  # noqa: E731
        f = lambda t: t.float().to(dev).contiguous()  # noqa: E731
        self.embed = h(sd["model.embed_tokens.weight"])
        self.layers = []
        for i in range(cfg["layers"]):
            p = f"model.layers.{i}."
            up, gate = sd[p + "mlp.up_proj.weight"], sd[p + "mlp.gate_proj.weight"]
            self.layers.append(dict(
                ln1=f(sd[p + "input_layernorm.weight"]), ln2=f(sd[p + "post_attention_layernorm.weight"]),
                wqkv=h(torch.cat([sd[p + "self_attn.q_proj.weight"], sd[p + "self_attn.k_proj.weight"], sd[p + "self_attn.v_proj.weight"]], 0)),
                wo=h(sd[p + "self_attn.o_proj.weight"]),
                wgu=h(torch.stack([up, gate], dim=1).reshape(2 * up.shape[0], -1)),   # rows [up_0, gate_0, up_1, gate_1, ...]
                wdown=h(sd[p + "mlp.down_proj.weight"])))
            if self.weight_format == "fp8_e4m3":
                L = self.layers[-1]
                for k in PROJECTIONS:
                    L[k], L[k + "_s"] = quantize_fp8_rows(L[k])
        self._wscratch = None
        if self.weight_format == "fp8_e4m3":   # prefill: each projection is dequantized here right before its GEMM (sized for the largest)
            self._wscratch = torch.empty((max(L[k].numel() for L in self.layers for k in PROJECTIONS),), device=dev, dtype=torch.float16)
        self.norm = f(sd["model.norm.weight"])
        self.lm_head = h(sd["lm_head.weight"])
        if self.embed.shape[0] != cfg["vocab"] or self.lm_head.shape[0] != cfg["vocab"]:
            raise SeedxError(f"checkpoint vocabulary {self.embed.shape[0]} != configured vocab_size {cfg['vocab']}")
        d = D // H
        self.inv_freq = (1.0 / (10000.0 ** (torch.arange(0, d, 2).float() / d))).to(dev)   # modeling_llama_xformer.py:101
        self._alloc_state()
        self._loaded = True
        return [], []

    # ---- fine-tuned checkpoints: partial updates and LoRA adapters, folded into the packed weights in place ------------------
    @property
    def config(self):
        """the two HF config fields the reference reads through the model object (peft_models.py:63, seed_x.py)"""
        import types
        return types.SimpleNamespace(vocab_size=self.cfg["vocab"], hidden_size=self.cfg["hidden"], tie_word_embeddings=False)

    def get_output_embeddings(self):
        return self.lm_head

    def resize_token_embeddings(self, vocab_size):
        """HF ``resize_token_embeddings`` + the reference's initialisation of the new rows (peft_models.py:62-82): input rows = mean of the
        old input rows, output rows = 3 x the mean of the old output rows.  Shrinking truncates."""
        if not self._loaded:
            raise SeedxError("resize_token_embeddings: weights not loaded")
        old = self.cfg["vocab"]
        if vocab_size == old:
            return self
        def grow(w, gain):
            new = torch.empty((vocab_size, w.shape[1]), device=w.device, dtype=w.dtype)
            n = min(old, vocab_size)
            new[:n] = w[:n]
            if vocab_size > old:
                new[old:] = (w.float().mean(dim=0, keepdim=True) * gain).to(w.dtype)
            return new
        self.embed, self.lm_head = grow(self.embed, 1.0), grow(self.lm_head, 3.0)
        self.cfg["vocab"] = int(vocab_size)
        self._alloc_state(self.slots)
        return self

    def update_weights(self, plain=None, lora=None, scaling=1.0):
        """plain: {HF parameter name: tensor} replacements; lora: {HF module name: (A [r,in], B [out,r])} low-rank updates added as
        ``W += scaling * B @ A`` (fp32 arithmetic at load time, result rounded to the fp16 storage format).  The packed device tensors
        are updated IN PLACE, so captured decode graphs stay valid.  Returns the names that matched nothing."""
        from .lora import lora_delta
        if not self._loaded:
            raise SeedxError("update_weights: load the base checkpoint first")
        plain, lora = dict(plain or {}), dict(lora or {})
        dev, cfg = self.device, self.cfg
        D, Fh = cfg["hidden"], cfg["ffn"]

        def fold(dst, name, scale=None):
            """dst: a (possibly strided) view into a packed fp16 weight; name: HF module name, e.g. model.layers.0.self_attn.q_proj.
            FP8 weights: dst is the float8_e4m3fn view and `scale` the matching rows of its scale vector; the rows are dequantized, updated
            in fp32 and requantized, and both q and the scales are written in place."""
            w = plain.pop(name + ".weight", None)
            ab = lora.pop(name, None)
            if w is None and ab is None:
                return
            if w is not None:
                cur = w.to(dev).float()
            else:
                cur = dst.float() * scale[:, None] if scale is not None else dst.float()
            if tuple(cur.shape) != tuple(dst.shape):
                raise SeedxError(f"{name}.weight: shape {tuple(cur.shape)} != {tuple(dst.shape)}")
            if ab is not None:
                delta = lora_delta(ab[0].to(dev), ab[1].to(dev), scaling)
                if tuple(delta.shape) != tuple(dst.shape):
                    raise SeedxError(f"LoRA update of {name}: shape {tuple(delta.shape)} != {tuple(dst.shape)}")
                cur = cur + delta
            if scale is None:
                dst.copy_(cur.to(torch.float16))
            else:
                q, sc = quantize_fp8_rows(cur)
                dst.copy_(q)
                scale.copy_(sc)

        def setf(dst, name):
            v = plain.pop(name, None)
            if v is not None:
                if tuple(v.shape) != tuple(dst.shape):
                    raise SeedxError(f"{name}: shape {tuple(v.shape)} != {tuple(dst.shape)}")
                dst.copy_(v.to(dev).to(dst.dtype))

        for i, L in enumerate(self.layers):
            p = f"model.layers.{i}."
            sq, so, sgu, sdown = (L.get(k + "_s") for k in PROJECTIONS)      # row scales of an FP8 model (None for fp16): sliced like the rows
            for j, n in enumerate(("q_proj", "k_proj", "v_proj")):
                fold(L["wqkv"][j * D:(j + 1) * D], p + "self_attn." + n, None if sq is None else sq[j * D:(j + 1) * D])
            fold(L["wo"], p + "self_attn.o_proj", so)
            gu = L["wgu"].view(Fh, 2, D)                                   # rows [up_0, gate_0, up_1, gate_1, ...]
            sgu = None if sgu is None else sgu.view(Fh, 2)
            fold(gu[:, 0], p + "mlp.up_proj", None if sgu is None else sgu[:, 0])
            fold(gu[:, 1], p + "mlp.gate_proj", None if sgu is None else sgu[:, 1])
            fold(L["wdown"], p + "mlp.down_proj", sdown)
            setf(L["ln1"], p + "input_layernorm.weight")
            setf(L["ln2"], p + "post_attention_layernorm.weight")
        setf(self.norm, "model.norm.weight")
        for attr, name in (("embed", "model.embed_tokens"), ("lm_head", "lm_head")):
            w = plain.get(name + ".weight")
            if w is not None and w.shape[0] != getattr(self, attr).shape[0]:
                raise SeedxError(f"{name}.weight has {w.shape[0]} rows, the model {getattr(self, attr).shape[0]}: call resize_token_embeddings first")
            fold(getattr(self, attr), name)
        return [k for k in plain if "rotary_emb" not in k] + list(lora)

    def apply_peft_state_dict(self, sd, adapter="default"):
        """keys as saved from a PEFT-wrapped model (``base_model.model.…lora_A.default.weight`` …): LoRA pairs are merged with the
        scaling of ``self.peft_config`` (set by get_peft_model_with_resize_embedding), modules_to_save / plain tensors replace."""
        from .lora import split_peft_state_dict
        base, lora, saved = split_peft_state_dict(sd, adapter)
        if lora and getattr(self, "peft_config", None) is None:
            raise SeedxError("the checkpoint holds LoRA adapters but the LLM was not built with a peft_config "
                             "(use configs/clm_models/llm_seed_x_lora.yaml)")
        # alpha / r spelled out: the real peft.LoraConfig dataclass (when the package is installed) has no `.scaling` property
        sc = float(self.peft_config.lora_alpha) / float(self.peft_config.r) if lora else 1.0
        for mod, (a, _) in lora.items():
            if a.shape[0] != self.peft_config.r:
                raise SeedxError(f"{mod}: adapter rank {a.shape[0]} != peft_config.r {self.peft_config.r}")
        return self.update_weights({**base, **saved}, lora, sc)

    def _alloc_state(self, slots=1):
        cfg, dev = self.cfg, self.device
        D, L = cfg["hidden"], cfg["layers"]
        self.slots = slots
        self._graphs = {}          # captured decode graphs reference the state buffers below
        self._hidden = None
        # paged KV cache: per layer and tensor one pool fp16 [n_pages, page_size, H*d]; a sequence slot reaches its rows through its row of
        # the page table (shared by all layers).  Default pool = enough pages for every slot at max_len; `kv_pages` shrinks it (admission
        # then fails with "KV cache exhausted" instead of over-committing).
        PS = self.page_size
        self.pages_per_slot = (self.max_len + PS - 1) // PS
        n_pages = self.kv_pages if self.kv_pages is not None else slots * self.pages_per_slot
        self.kv_alloc = KVPageAllocator(n_pages)
        self.slot_pages = [[] for _ in range(slots)]
        self.page_table = torch.zeros((slots, self.pages_per_slot), device=dev, dtype=torch.int32)
        self.kcache = [torch.zeros((n_pages, PS, D), device=dev, dtype=torch.float16) for _ in range(L)]
        self.vcache = [torch.zeros((n_pages, PS, D), device=dev, dtype=torch.float16) for _ in range(L)]
        self.seq = torch.zeros((slots, self.max_len), device=dev, dtype=torch.int32)
        self.state = torch.zeros((slots, 4), device=dev, dtype=torch.int32)
        z = lambda n: torch.zeros((slots, n), device=dev, dtype=torch.float32)  # noqa: E731
        self.xa, self.xb, self.qkv1, self.att1, self.g1, self.hn1 = z(D), z(D), z(3 * D), z(D), z(cfg["ffn"]), z(D)
        self.logits = z(cfg["vocab"])

    # ---- KV pages --------------------------------------------------------------------------------------------------------------
    def reserve_kv(self, slot, n_tokens, fresh=False):
        """make sure sequence slot `slot` owns pages for positions [0, n_tokens); fresh=True first returns its old pages (new request)."""
        if n_tokens > self.max_len:
            raise SeedxError(f"sequence length {n_tokens} exceeds the KV cache ({self.max_len})")
        if fresh and self.slot_pages[slot]:
            self.kv_alloc.release(self.slot_pages[slot])
            self.slot_pages[slot] = []
        need = (n_tokens + self.page_size - 1) // self.page_size - len(self.slot_pages[slot])
        if need > 0:
            self.slot_pages[slot] += self.kv_alloc.alloc(need)
            row = torch.zeros((self.pages_per_slot,), dtype=torch.int32)
            row[:len(self.slot_pages[slot])] = torch.tensor(self.slot_pages[slot], dtype=torch.int32)
            self.page_table[slot].copy_(row)          # same device buffer: captured decode graphs keep reading it

    def kv_rows(self, li, slot, n):
        """contiguous copies [n, H*d] of the first n cached K and V rows of a slot (page gather; chunked prefill and tests)"""
        pages = torch.tensor(self.slot_pages[slot][:(n + self.page_size - 1) // self.page_size], dtype=torch.long, device=self.device)
        D = self.cfg["hidden"]
        return self.kcache[li][pages].reshape(-1, D)[:n], self.vcache[li][pages].reshape(-1, D)[:n]

    # ---- prefill: tensor-core path ---------------------------------------------------------------------------------------
    def _gemm(self, a, L, name, **kw):
        """prefill projection a @ L[name]^T.  FP8 weights are first dequantized into the shared fp16 scratch buffer; the GEMM then reads a
        B operand the previous kernel wrote, so it must not prefetch it before the PDL wait (dynamic_b)."""
        s = L.get(name + "_s")
        if s is None:
            return ops.gemm(a, L[name], **kw)
        w8 = L[name]
        w = self._wscratch[:w8.numel()].view(w8.shape)
        ops.dequant_fp8(w8, s, w)
        return ops.gemm(a, w, dynamic_b=True, **kw)

    def _gemv(self, L, name, x, out, **kw):
        """token-loop projection: seedx_gemv_f16, or seedx_gemv_fp8 with the row scales of an FP8 matrix"""
        s = L.get(name + "_s")
        if s is not None:
            kw["scale"] = s
        return ops.gemv(L[name], x, out, **kw)

    def prefill(self, x, pos0=0, slot=0):
        """x: fp32 device [P, D] input embeddings for positions pos0.. of sequence slot `slot`; fills its KV cache; returns the fp32
        residual stream [P, D]."""
        cfg = self.cfg
        D, H = cfg["hidden"], cfg["heads"]
        d = D // H
        P = x.shape[0]
        self.reserve_kv(slot, pos0 + P, fresh=(pos0 == 0))
        x = x.contiguous().clone()
        n = torch.empty((P, D), device=x.device, dtype=torch.float16)
        qkv = torch.empty((P, 3 * D), device=x.device, dtype=torch.float16)
        o = torch.empty((P, D), device=x.device, dtype=torch.float16)
        gu = torch.empty((P, cfg["ffn"]), device=x.device, dtype=torch.float16)
        q4 = qkv.view(1, P, 3, H, d)
        qv, kv, vv = (q4[:, :, i].permute(0, 2, 1, 3) for i in range(3))
        ov = o.view(1, P, H, d).permute(0, 2, 1, 3)
        for li, L in enumerate(self.layers):
            ops.layernorm(x, L["ln1"], None, cfg["eps"], out=n, rms=True)
            self._gemm(n, L, "wqkv", out=qkv)
            ops.rope_kv_prefill(qkv, pos0, H, d, self.inv_freq, self.kcache[li], self.vcache[li], page_table_row=self.page_table[slot],
                                page_size=self.page_size)
            if pos0 == 0:
                ops.attention(qv, kv, vv, ov, scale=d ** -0.5, causal=True)
            else:   # chunked prefill: keys/values come from the cache (positions 0..pos0+P-1), gathered from their pages
                kc, vc = self.kv_rows(li, slot, pos0 + P)
                ops.attention(qv, kc.view(1, pos0 + P, H, d).permute(0, 2, 1, 3), vc.view(1, pos0 + P, H, d).permute(0, 2, 1, 3), ov,
                              scale=d ** -0.5, causal=True)
            self._gemm(o, L, "wo", out=x, residual=x)
            ops.layernorm(x, L["ln2"], None, cfg["eps"], out=n, rms=True)
            self._gemm(n, L, "wgu", out=gu, act=ops.ACT_SILU, gated=True)
            self._gemm(gu, L, "wdown", out=x, residual=x)
        return x

    def prefill_batch(self, xs, slots):
        """Prefill several sequences in ONE pass over the weights: the rows of all prompts are concatenated for the four projection GEMMs of
        a layer (each fp16 weight matrix is streamed once instead of once per prompt — at P ~ 240 a single prompt's GEMMs are weight-read
        bound), while RoPE + KV append and the causal attention run per sequence on its row block.  xs: list of fp32 device [P_r, D];
        slots: the KV-cache slot of each.  Returns the list of fp32 residual streams [P_r, D] (views of one buffer)."""
        cfg = self.cfg
        D, H = cfg["hidden"], cfg["heads"]
        d = D // H
        lens = [int(x.shape[0]) for x in xs]
        for n_, slot in zip(lens, slots):
            self.reserve_kv(slot, n_, fresh=True)
        offs = [0]
        for n_ in lens:
            offs.append(offs[-1] + n_)
        T = offs[-1]
        x = torch.cat([t.reshape(-1, D) for t in xs], dim=0).contiguous()
        n = torch.empty((T, D), device=x.device, dtype=torch.float16)
        qkv = torch.empty((T, 3 * D), device=x.device, dtype=torch.float16)
        o = torch.empty((T, D), device=x.device, dtype=torch.float16)
        gu = torch.empty((T, cfg["ffn"]), device=x.device, dtype=torch.float16)
        for li, L in enumerate(self.layers):
            ops.layernorm(x, L["ln1"], None, cfg["eps"], out=n, rms=True)
            self._gemm(n, L, "wqkv", out=qkv)
            for r, slot in enumerate(slots):
                a, P = offs[r], lens[r]
                blk = qkv[a:a + P]
                ops.rope_kv_prefill(blk, 0, H, d, self.inv_freq, self.kcache[li], self.vcache[li], page_table_row=self.page_table[slot],
                                    page_size=self.page_size)
                q4 = blk.view(1, P, 3, H, d)
                qv, kv, vv = (q4[:, :, i].permute(0, 2, 1, 3) for i in range(3))
                ops.attention(qv, kv, vv, o[a:a + P].view(1, P, H, d).permute(0, 2, 1, 3), scale=d ** -0.5, causal=True)
            self._gemm(o, L, "wo", out=x, residual=x)
            ops.layernorm(x, L["ln2"], None, cfg["eps"], out=n, rms=True)
            self._gemm(n, L, "wgu", out=gu, act=ops.ACT_SILU, gated=True)
            self._gemm(gu, L, "wdown", out=x, residual=x)
        return [x[offs[r]:offs[r + 1]] for r in range(len(xs))]

    def logits_all(self, x):
        """final RMSNorm + lm_head over every row of the residual stream (parity checks; LlamaForCausalLM.forward :702-707)."""
        hn = ops.layernorm(x, self.norm, None, self.cfg["eps"], out_dtype=torch.float32, rms=True)
        h16 = ops.cast(hn, torch.float16)
        return ops.gemm(h16, self.lm_head, out_dtype=torch.float32), hn

    # ---- token loop: HBM-bound path ----------------------------------------------------------------------------------------
    def _decode_step(self, hidden, img_ids, eos_id, suppress_eos):
        """one token for every sequence slot: the weights (fp16, or FP8 + row scales) are streamed once and shared by all slots"""
        cfg = self.cfg
        H = cfg["heads"]
        d = cfg["hidden"] // H
        ops.embed_rows(self.embed, self.xa, state=self.state, seq=self.seq)
        for li, L in enumerate(self.layers):
            self._gemv(L, "wqkv", self.xa, self.qkv1, rms_w=L["ln1"], eps=cfg["eps"])
            ops.decode_attention(self.qkv1, self.state, self.inv_freq, self.kcache[li], self.vcache[li], self.att1, H, d,
                                 page_table=self.page_table, page_size=self.page_size)
            self._gemv(L, "wo", self.att1, self.xb, residual=self.xa)
            self._gemv(L, "wgu", self.xb, self.g1, rms_w=L["ln2"], eps=cfg["eps"], gated=True)
            self._gemv(L, "wdown", self.g1, self.xa, residual=self.xb)
        ops.layernorm(self.xa, self.norm, None, cfg["eps"], out=self.hn1, rms=True)
        ops.store_hidden(self.hn1, self.state, hidden)
        ops.gemv(self.lm_head, self.hn1, self.logits)
        ops.logits_argmax(self.logits, img_ids, self.seq, self.state, eos_id, suppress_eos)

    def generate_greedy_batch(self, input_ids_list, inputs_embeds_list, img_ids=None, max_new_tokens=120, eos_id=None, suppress_eos=False,
                              use_graph=True, sync_every=32, keep_prefill_hidden=False):
        """Greedy decoding of up to 8 independent requests in lock-step (HF greedy_search per request, seed_x.py:184-189):
        request r's inputs_embeds [P_r, D] feed its prefill, then its last id each step.  Returns a list of GreedyOutput."""
        if not self._loaded:
            raise SeedxError("LlamaForCausalLM: weights not loaded")
        dev = self.device
        n_req = len(input_ids_list)
        if not 1 <= n_req <= 8:
            raise SeedxError("generate_greedy_batch handles 1..8 requests per call")
        slots = 1 if n_req == 1 else 2 if n_req == 2 else 4 if n_req <= 4 else 8
        if slots != self.slots:
            self._alloc_state(slots)
        # static device state shared by every call with the same slot count, so the captured decode graph can be replayed across calls
        ikey = tuple(int(i) for i in img_ids) if img_ids is not None else None
        if getattr(self, "_img_key", "unset") != ikey:
            self._img_key = ikey
            self._img_dev = torch.tensor(list(ikey), dtype=torch.int32, device=dev) if ikey is not None else None
            self._graphs = {}
        img_dev = self._img_dev
        if getattr(self, "_hidden", None) is None or self._hidden.shape[0] != slots:
            self._hidden = torch.zeros((slots, self.max_len, self.cfg["hidden"]), device=dev, dtype=torch.float32)
            self._graphs = {}
        hidden = self._hidden
        st0, plens, pre_hidden, embs, ids_all, ahead = [], [], [], [], [], []
        for s in range(slots):
            r = min(s, n_req - 1)                       # padding slots replay the last request
            ids = torch.as_tensor(input_ids_list[r]).reshape(-1)
            P = ids.numel()
            if P + max_new_tokens > self.max_len:
                raise SeedxError("prompt + max_new_tokens exceeds the KV cache")
            plens.append(P)
            ids_all.append(ids)
            embs.append(inputs_embeds_list[r].reshape(P, -1).to(dev, torch.float32))
            # Jump-forward over a forced image span.  The reference's logits processor makes the continuation of a prompt that ends inside
            # "<img><img_00000>...<img_00063></img>" independent of the logits (generation.py:23-26: score[next id of the span] = max + 10),
            # so those tokens are known before the model runs.  All but (at least) the last generated token are appended to the prompt
            # and ride through the prefill pass as teacher-forced rows on the tensor cores — same positions, same causal attention, same
            # hidden states as feeding them one by one, but the 26 GB of weights are streamed once instead of once per forced token.
            last = int(ids[-1])
            a = []
            if self.jump_forward and ikey is not None and last in ikey[:-1]:
                a = list(ikey[ikey.index(last) + 1:])[: max(max_new_tokens - 1, 0)]
            ahead.append(a)
        over = max(len(a) for a in ahead) - min(len(a) for a in ahead)     # slots with a longer span run `over` surplus steps (dropped below)
        if any(plens[s] + max_new_tokens + over > self.max_len for s in range(slots)):
            ahead, over = [[] for _ in range(slots)], 0
        for s in range(slots):
            P, a = plens[s], ahead[s]
            self.seq[s, :P].copy_(ids_all[s].to(dev, torch.int32))
            if a:
                a_t = torch.tensor(a, dtype=torch.int32, device=dev)
                self.seq[s, P:P + len(a)].copy_(a_t)
                embs[s] = torch.cat([embs[s], self.get_input_embeddings()(a_t)[0]], dim=0)
            st0.append([P + len(a), 0, len(a), P])
        if slots > 1 and self.batched_prefill:          # one pass over the weights for all prompts
            streams = self.prefill_batch(embs, list(range(slots)))
        else:
            streams = [self.prefill(embs[s], slot=s) for s in range(slots)]
        for s in range(slots):                           # pages for the tokens the loop will append
            self.reserve_kv(s, plens[s] + max_new_tokens + over)
        for s, xs in enumerate(streams):
            P, na = plens[s], len(ahead[s])
            ops.gemv(self.lm_head, xs[P + na - 1], self.logits[s], rms_w=self.norm, eps=self.cfg["eps"])
            if na:   # post-norm states of the positions that consumed the pre-appended tokens = rows 0..na-1 of the harvest buffer
                ops.layernorm(xs[P:P + na], self.norm, None, self.cfg["eps"], out=hidden[s, :na], rms=True)
            if keep_prefill_hidden and s < n_req:      # post-norm states of the prompt positions (HF hidden_states[0][-1])
                pre_hidden.append(ops.layernorm(xs[:P], self.norm, None, self.cfg["eps"], out_dtype=torch.float32, rms=True))
        self.state.copy_(torch.tensor(st0, dtype=torch.int32))
        ops.logits_argmax(self.logits, img_dev, self.seq, self.state, eos_id, suppress_eos)
        trace.mark("llm.prefill")
        steps = max_new_tokens - 1 - min(len(a) for a in ahead)
        if steps > 0:
            g = None
            if use_graph:
                gkey = (slots, eos_id, bool(suppress_eos))
                g = self._graphs.get(gkey)
                if g is None:   # one capture per (slot count, stop rule): the step reads lengths / prompt lengths from device state
                    s_ = torch.cuda.Stream()
                    s_.wait_stream(torch.cuda.current_stream())
                    g = torch.cuda.CUDAGraph()
                    n0 = _lib.launch_count()
                    with torch.cuda.graph(g, stream=s_):
                        self._decode_step(hidden, img_dev, eos_id, suppress_eos)
                    g.n_kernels = _lib.launch_count() - n0
                    torch.cuda.current_stream().wait_stream(s_)
                    self._graphs[gkey] = g
            def run_step():
                if g is not None:
                    g.replay()
                    _lib.note_replay(g.n_kernels)
                else:
                    self._decode_step(hidden, img_dev, eos_id, suppress_eos)

            if self.jump_forward_mid and ikey is not None:
                self._decode_with_span_jumps(run_step, hidden, ikey, slots, n_req, plens, max_new_tokens, suppress_eos)
            else:
                for i in range(steps):
                    run_step()
                    if eos_id is not None and not suppress_eos and (i + 1) % sync_every == 0:
                        if bool((self.state[:n_req, 1] != 0).all().item()):
                            break
        trace.mark("llm.decode")
        st = self.state.cpu().tolist()
        seq_host = self.seq.cpu()
        outs = []
        for r in range(n_req):
            n_gen = st[r][1] if st[r][1] else st[r][2]   # stop at (and include) the first EOS, like HF greedy_search
            n_gen = min(n_gen, max_new_tokens)           # surplus lock-step tokens of a slot that jumped further ahead are dropped
            outs.append(GreedyOutput(seq_host[r, : plens[r] + n_gen].to(torch.int64).unsqueeze(0), hidden[r, : max(n_gen - 1, 0)].clone(), n_gen))
            outs[-1].prefill_hidden = pre_hidden[r] if keep_prefill_hidden else None
        return outs

    def _decode_with_span_jumps(self, run_step, hidden, ikey, slots, n_req, plens, max_new_tokens, suppress_eos):
        """EXPERIMENTAL (SEEDX_JUMP_FORWARD_MID=1, off by default): token loop that also jumps over image spans the model opens by itself
        ("... here it is: <img>" in the middle of an answer).  The decision needs the last generated id on the host, so every step pays one
        device sync; in exchange the rest of a span is computed as ONE chunked prefill over the cached keys (tensor-core GEMMs) instead of
        up to 64 weight-streaming steps.  Slots then progress unevenly: the loop runs until every request has its `max_new_tokens` (or
        EOS); a slot that is already done keeps stepping in lock-step and its surplus tokens are dropped by the caller."""
        dev = self.device
        for _ in range(4 * max_new_tokens + 16):
            st = self.state.cpu().tolist()
            gen = [st[s][2] for s in range(slots)]
            done = [(st[s][1] != 0 and not suppress_eos) or gen[s] >= max_new_tokens for s in range(slots)]
            if all(done[:n_req]):
                return
            lens = [st[s][0] for s in range(slots)]
            last = self.seq[torch.arange(slots, device=dev), torch.tensor(lens, device=dev) - 1].cpu().tolist()
            for s in range(slots):
                if done[s] or last[s] not in ikey[:-1]:
                    continue
                forced = list(ikey[ikey.index(last[s]) + 1:])[: max_new_tokens - 1 - gen[s]]      # keep one token for the step below
                L, P, a = lens[s], plens[s], len(forced)
                if a < 2 or L + a + 1 > self.max_len:
                    continue
                # consume [last, forced[:-1]] at positions L-1 .. L+a-2 in one pass; forced[-1] is consumed by the regular step
                chunk = torch.tensor([last[s]] + forced[:-1], dtype=torch.int32, device=dev)
                xs = self.prefill(self.get_input_embeddings()(chunk)[0], pos0=L - 1, slot=s)
                ops.layernorm(xs, self.norm, None, self.cfg["eps"], out=hidden[s, L - 1 - P:L - 1 - P + a], rms=True)
                self.seq[s, L:L + a].copy_(torch.tensor(forced, dtype=torch.int32, device=dev))
                self.state[s].copy_(torch.tensor([L + a, st[s][1], gen[s] + a, P], dtype=torch.int32))
                lens[s] = L + a
            for s in range(slots):
                self.reserve_kv(s, min(lens[s], self.max_len))
            run_step()
        raise SeedxError("decode loop did not terminate")

    def generate(self, input_ids=None, inputs_embeds=None, output_hidden_states=False, return_dict_in_generate=False, logits_processor=None,
                 max_new_tokens=20, do_sample=False, num_beams=1, temperature=None, top_p=None, eos_token_id="default", **kw):
        """The slice of HF ``GenerationMixin.generate`` that the reference calls (seed_x.py:184-189; transformers==4.30.2 greedy_search,
        SURVEY.md B.1): greedy decoding of ONE prompt whose first step consumes ``inputs_embeds`` [1,P,D] and later steps the embedding
        of the last id; stops at EOS or after ``max_new_tokens``.  ``temperature`` / ``top_p`` are accepted and unused because
        ``do_sample=False`` (the reference passes them the same way).  ``logits_processor``: an iterable holding at most one
        AutoImageTokenGenerationProcessor (anything exposing ``img_ids_list``); its rule runs on the device."""
        if do_sample or num_beams != 1:
            raise SeedxError("only greedy search (do_sample=False, num_beams=1) is implemented: it is the only mode the reference uses")
        if input_ids is None:
            raise SeedxError("generate() needs input_ids (the returned sequences start with them)")
        ids = torch.as_tensor(input_ids)
        if ids.dim() == 1:
            ids = ids.unsqueeze(0)
        if ids.shape[0] != 1:
            raise SeedxError("generate() decodes one prompt per call like the reference (seed_x.py:191 reads sequences[0]); "
                             "use generate_greedy_batch for lock-step decoding of several requests")
        P = ids.shape[1]
        emb = inputs_embeds if inputs_embeds is not None else self.get_input_embeddings()(ids)
        emb = emb.reshape(P, -1)
        img_ids = None
        for proc in (logits_processor or []):
            if not hasattr(proc, "img_ids_list") or img_ids is not None:
                raise SeedxError(f"unsupported logits processor {type(proc).__name__}: only one AutoImageTokenGenerationProcessor runs on the device")
            img_ids = list(proc.img_ids_list)
        eos = self.cfg.get("eos", 2) if isinstance(eos_token_id, str) else eos_token_id
        out = self.generate_greedy_batch([ids[0]], [emb], img_ids=img_ids, max_new_tokens=max_new_tokens, eos_id=eos,
                                         keep_prefill_hidden=bool(output_hidden_states), use_graph=kw.get("use_graph", True))[0]
        if not return_dict_in_generate:
            return out.sequences
        res = GreedySearchOutput(sequences=out.sequences)
        if output_hidden_states:
            steps = [(out.prefill_hidden.unsqueeze(0),)]
            steps += [(out.last_hidden_states[j].view(1, 1, -1),) for j in range(out.last_hidden_states.shape[0])]
            res["hidden_states"] = tuple(steps)
        return res

    def generate_greedy(self, input_ids, inputs_embeds, img_ids=None, max_new_tokens=120, eos_id=None, suppress_eos=False, use_graph=True,
                        sync_every=32):
        """single-request form of generate_greedy_batch"""
        return self.generate_greedy_batch([input_ids], [inputs_embeds], img_ids=img_ids, max_new_tokens=max_new_tokens, eos_id=eos_id,
                                          suppress_eos=suppress_eos, use_graph=use_graph, sync_every=sync_every)[0]
