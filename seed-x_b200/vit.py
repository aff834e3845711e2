"""Stage 1 host: Qwen ViT-bigG visual encoder with attention pooling, driven kernel-by-kernel through libseedx.so.

Mirrors the public surface of the reference class
``src.models.tokenizer.qwen_visual.VisionTransformerWithAttnPool`` (/root/reference/src/models/tokenizer/qwen_visual.py:325-459):
same constructor keywords, ``from_pretrained``, ``eval()``, ``to()``, ``__call__(x[N,3,H,W]) -> [N, n_queries, output_dim]``,
and it ingests the reference state-dict key names (SURVEY.md A.5).

Device data layout (HBM): activations are token-major [N*S, C]; the residual stream is fp32, GEMM operands fp16,
accumulation fp32.  Input-independent pieces (bicubic-resized position tables, the pooled query
projection) are computed once at load / first use.
"""
import math

import torch
import torch.nn.functional as F  # load-time only: bicubic resize of constant position tables

from . import ops
from ._lib import SeedxError


def _resize_pos(table, n_tokens):
    """Load-time constant folding of get_abs_pos (qwen_visual.py:24-40): bicubic, align_corners=False, fp32."""
    src = int(math.isqrt(table.shape[0]))
    dst = int(math.isqrt(n_tokens))
    if src == dst:
        return table.float().contiguous()
    t = table.float().reshape(1, src, src, -1).permute(0, 3, 1, 2)
    t = F.interpolate(t, size=(dst, dst), mode="bicubic", align_corners=False)
    return t.permute(0, 2, 3, 1).reshape(dst * dst, -1).contiguous()


class ResamplerWeights:
    """Packed device weights of one qwen_visual.Resampler (attn_pool / input_resampler / output_resampler)."""

    def __init__(self, sd, prefix, heads, eps, device):
        self.heads, self.eps = heads, eps
        g = lambda k: sd[prefix + k]  # noqa: E731
        self.embed_dim = g("query").shape[1]
        self.n_queries = g("query").shape[0]
        self.pos_cpu = g("pos_embed").float().cpu()
        self.pos_q = self.pos_cpu.to(device).contiguous()
        self.query = g("query").float().to(device).contiguous()
        self.kv_proj = g("kv_proj.weight").to(device, torch.float16).contiguous() if (prefix + "kv_proj.weight") in sd else None
        w = g("attn.in_proj_weight").to(device, torch.float16).contiguous()
        b = g("attn.in_proj_bias").float().to(device).contiguous()
        E = self.embed_dim
        self.wq, self.wk, self.wv = w[:E], w[E:2 * E], w[2 * E:]
        self.bq, self.bk, self.bv = b[:E].contiguous(), b[E:2 * E].contiguous(), b[2 * E:].contiguous()
        self.wo = g("attn.out_proj.weight").to(device, torch.float16).contiguous()
        self.bo = g("attn.out_proj.bias").float().to(device).contiguous()
        self.ln_q = (g("ln_q.weight").float().to(device), g("ln_q.bias").float().to(device))
        self.ln_kv = (g("ln_kv.weight").float().to(device), g("ln_kv.bias").float().to(device))
        self._q = None
        self._pos_k = {}
        self.device = device

    def q_proj(self):
        """Q = (LN_q(query) + pos) Wq^T + bq — input independent, computed once with the library kernels."""
        if self._q is None:
            _, qin = ops.layernorm(self.query, self.ln_q[0], self.ln_q[1], self.eps, add=self.pos_q)
            self._q = ops.gemm(qin, self.wq, bias=self.bq)
        return self._q

    def pos_k(self, n_kv):
        if n_kv not in self._pos_k:
            self._pos_k[n_kv] = _resize_pos(self.pos_cpu, n_kv).to(self.device)
        return self._pos_k[n_kv]

    def forward(self, x16, batch, n_kv, out_dtype=torch.float32, residual=None):
        """x16: fp16 [batch*n_kv, kv_dim] -> [batch*n_queries, E] (qwen_visual.py:136-146)."""
        E, H, Nq = self.embed_dim, self.heads, self.n_queries
        d = E // H
        kv = ops.gemm(x16, self.kv_proj, out_dtype=torch.float32) if self.kv_proj is not None else x16
        v_in, k_in = ops.layernorm(kv, self.ln_kv[0], self.ln_kv[1], self.eps, add=self.pos_k(n_kv))
        k = ops.gemm(k_in, self.wk, bias=self.bk)
        v = ops.gemm(v_in, self.wv, bias=self.bv)
        q = self.q_proj()
        o = torch.empty((batch * Nq, E), device=x16.device, dtype=torch.float16)
        ops.attention(q.view(1, Nq, H, d).permute(0, 2, 1, 3), k.view(batch, n_kv, H, d).permute(0, 2, 1, 3),
                      v.view(batch, n_kv, H, d).permute(0, 2, 1, 3), o.view(batch, Nq, H, d).permute(0, 2, 1, 3), scale=d ** -0.5)
        return ops.gemm(o, self.wo, bias=self.bo, out_dtype=out_dtype, residual=residual)


class VisionTransformerWithAttnPool:
    """Drop-in for the reference visual encoder (forward only)."""

    def __init__(self, image_size, patch_size, width, layers, heads, mlp_ratio, n_queries=256, output_dim=512,
                 patch_pos=False, **kwargs):
        if patch_pos:
            raise SeedxError("patch_pos=True is not used by any shipped config (qwen_vitg_448.yaml) and is not implemented")
        self.image_size, self.patch_size = image_size, patch_size
        self.width, self.layers, self.heads = width, layers, heads
        self.mlp_width = int(width * mlp_ratio)
        self.n_queries, self.output_dim = n_queries, output_dim
        self.eps = 1e-6
        self.device = torch.device("cuda")
        self.kpad = (3 * patch_size * patch_size + 7) // 8 * 8
        self._loaded = False
        self._pos = {}
        self.out_dtype = torch.float16

    # ---- reference-compatible plumbing -------------------------------------------------------------------------
    @classmethod
    def from_pretrained(cls, pretrained_model_path=None, **kwargs):
        model = cls(**kwargs)
        if pretrained_model_path is not None:
            model.load_state_dict(torch.load(pretrained_model_path, map_location="cpu"))
        return model

    def eval(self):
        return self

    def to(self, device=None, dtype=None, **kw):
        if dtype is not None and dtype not in (torch.float16, torch.float32):
            raise SeedxError("the engine computes with fp16 operands / fp32 accumulate only")
        if dtype is not None:
            self.out_dtype = dtype
        return self

    def load_state_dict(self, sd, strict=False):
        dev = self.device
        h = lambda t: t.to(dev, torch.float16).contiguous()  # noqa: E731
        f = lambda t: t.float().to(dev).contiguous()  # noqa: E731
        w = sd["conv1.weight"].reshape(self.width, -1)
        wp = torch.zeros((self.width, self.kpad), dtype=torch.float16, device=w.device)
        wp[:, : w.shape[1]] = w.to(torch.float16)
        self.w_patch = wp.to(dev)
        self.pos_cpu = sd["positional_embedding"].float().cpu()
        self.ln_pre = (f(sd["ln_pre.weight"]), f(sd["ln_pre.bias"]))
        self.blocks = []
        for i in range(self.layers):
            p = f"transformer.resblocks.{i}."
            self.blocks.append(dict(
                ln1=(f(sd[p + "ln_1.weight"]), f(sd[p + "ln_1.bias"])), ln2=(f(sd[p + "ln_2.weight"]), f(sd[p + "ln_2.bias"])),
                w_in=h(sd[p + "attn.in_proj.weight"]), b_in=f(sd[p + "attn.in_proj.bias"]),
                w_out=h(sd[p + "attn.out_proj.weight"]), b_out=f(sd[p + "attn.out_proj.bias"]),
                w_fc=h(sd[p + "mlp.c_fc.weight"]), b_fc=f(sd[p + "mlp.c_fc.bias"]),
                w_proj=h(sd[p + "mlp.c_proj.weight"]), b_proj=f(sd[p + "mlp.c_proj.bias"])))
        self.pool = ResamplerWeights(sd, "attn_pool.", self.output_dim // 128, self.eps, dev)
        self.ln_post = (f(sd["ln_post.weight"]), f(sd["ln_post.bias"]))
        self.proj_t = h(sd["proj"].t())  # x @ proj == gemm(x, proj^T)
        self._loaded = True
        return [], []

    # ---- forward --------------------------------------------------------------------------------------------------
    def _pos_table(self, n_tokens):
        if n_tokens not in self._pos:
            self._pos[n_tokens] = _resize_pos(self.pos_cpu, n_tokens).to(self.device)
        return self._pos[n_tokens]

    def tokens(self, x):
        """patch embed + position + ln_pre + transformer blocks -> fp32 residual stream [N*S, width]."""
        if not self._loaded:
            raise SeedxError("VisionTransformerWithAttnPool: weights not loaded")
        if not x.is_cuda:
            x = x.to(self.device, non_blocking=True)
        x = x.contiguous()
        if x.dtype not in (torch.float16, torch.float32):
            x = x.float()
        N, _, H, W = x.shape
        P, E, heads = self.patch_size, self.width, self.heads
        S = (H // P) * (W // P)
        d = E // heads
        a = ops.patchify(x, P, self.kpad)
        tok = ops.gemm(a, self.w_patch, residual=self._pos_table(S), res_row_mod=S, out_dtype=torch.float32)
        xs = ops.layernorm(tok, self.ln_pre[0], self.ln_pre[1], self.eps, out_dtype=torch.float32)
        qkv = torch.empty((N * S, 3 * E), device=x.device, dtype=torch.float16)
        att = torch.empty((N * S, E), device=x.device, dtype=torch.float16)
        hbuf = torch.empty((N * S, E), device=x.device, dtype=torch.float16)
        mbuf = torch.empty((N * S, self.mlp_width), device=x.device, dtype=torch.float16)
        qkv5 = qkv.view(N, S, heads, 3, d)
        qv, kv, vv = (qkv5[:, :, :, i].permute(0, 2, 1, 3) for i in range(3))   # [N, heads, S, d] strided views
        ov = att.view(N, S, heads, d).permute(0, 2, 1, 3)
        for blk in self.blocks:
            ops.layernorm(xs, blk["ln1"][0], blk["ln1"][1], self.eps, out=hbuf)
            ops.gemm(hbuf, blk["w_in"], out=qkv, bias=blk["b_in"])
            ops.attention(qv, kv, vv, ov, scale=d ** -0.5)
            ops.gemm(att, blk["w_out"], out=xs, bias=blk["b_out"], residual=xs)
            ops.layernorm(xs, blk["ln2"][0], blk["ln2"][1], self.eps, out=hbuf)
            ops.gemm(hbuf, blk["w_fc"], out=mbuf, bias=blk["b_fc"], act=ops.ACT_GELU)
            ops.gemm(mbuf, blk["w_proj"], out=xs, bias=blk["b_proj"], residual=xs)
        return xs, N, S

    def __call__(self, x, patch_positions=None):
        xs, N, S = self.tokens(x)
        x16 = ops.cast(xs, torch.float16)
        z = self.pool.forward(x16, N, S, out_dtype=torch.float32)
        zn = ops.layernorm(z, self.ln_post[0], self.ln_post[1], self.eps)
        out = ops.gemm(zn, self.proj_t, out_dtype=self.out_dtype)
        return out.view(N, self.n_queries, self.output_dim)

    forward = __call__
