"""Stage 3 host: SDXL UNet2DConditionModel, AutoencoderKL and EulerDiscreteScheduler stand-ins driven through libseedx.so.

The reference instantiates these three classes from diffusers==0.25.0 (src/inference/eval_*.py:97-101) and calls them at
src/models/detokenizer/pipeline_stable_diffusion_xl_t2i_edit.py:823,828,908,915-922,953,973 and (t2i) inside
StableDiffusionXLPipeline.__call__ reached from src/models/detokenizer/adapter_modules.py:156-167.  diffusers is not a
dependency of this engine: the classes below expose the constructor/loader surface the reference scripts use
(``from_pretrained(path, subfolder=...)``) and ingest diffusers state-dict key names (SURVEY.md Appendix B.2).

HBM layout: activations are NHWC fp16 ([B*H*W, C] token-major, so a feature map IS the A operand of the transformer
GEMMs); transformer residual stream fp32; sampler state (latents) fp32; all accumulation fp32.
"""
import json
import math
import os

import torch

from . import ops
from ._lib import SeedxError
from .llm import quantize_fp8_rows

SDXL_UNET = dict(in_channels=4, out_channels=4, block_out_channels=(320, 640, 1280), layers_per_block=2,
                 down_attn=(False, True, True), transformer_layers=(1, 2, 10), heads=(5, 10, 20), cross_attention_dim=2048,
                 time_embed_dim=1280, addition_time_embed_dim=256, text_embed_dim=1280, groups=32)
SDXL_VAE = dict(block_out_channels=(128, 256, 512, 512), layers_per_block=2, latent_channels=4, groups=32, scaling_factor=0.13025)
UNET_WEIGHT_FORMATS = ("fp16", "fp8_e4m3", "fp8_e4m3_conv")


def _load_weights_dir(path):
    """diffusers checkpoint directory -> state dict (safetensors preferred, then .bin)."""
    for name in ("diffusion_pytorch_model.fp16.safetensors", "diffusion_pytorch_model.safetensors"):
        f = os.path.join(path, name)
        if os.path.exists(f):
            from safetensors.torch import load_file
            return load_file(f)
    f = os.path.join(path, "diffusion_pytorch_model.bin")
    if os.path.exists(f):
        return torch.load(f, map_location="cpu")
    raise SeedxError(f"no diffusers weights found under {path}")


def _h(t, dev):
    return t.to(dev, torch.float16).contiguous()


def _f(t, dev):
    return t.float().to(dev).contiguous()


# Statistics for the next normalisation come out of the producing kernel's epilogue (seedx_gemm_args.col_part / row_part) instead of a pass over
# the tensor; SEEDX_EPI_STATS=0 restores the separate statistics kernels (A/B switch, same results up to summation order).
EPI_STATS = os.environ.get("SEEDX_EPI_STATS", "1") != "0"
ROW_TICKETS = os.environ.get("SEEDX_ROW_TICKETS", "1") != "0"     # 0: LayerNorm statistics by the row-finalize kernel instead of inside the producing GEMM


def _new_col_part(n, h, w, c, dev):
    """buffer for the column partials of an NHWC fp16 map [n,h,w,c] that a GroupNorm will read, or None when the shape is not eligible"""
    # maps of more than 256 x 256 pixels (the upper levels of the VAE) keep the statistics pass: their partials would be > 100 MB per tensor and the
    # per-(image, group) finalize, one CTA each, has too little parallelism to read them quickly (measured: 86 us vs 100 us for the pass, with slower convs)
    if not EPI_STATS or (h * w) % 32 or c % 32 or h * w > 65536:
        return None
    return torch.empty((n * h * w // 32, c, 2), device=dev, dtype=torch.float32)


def _tag(t, part):
    """attach the partials to the tensor OBJECT that travels to the consumer (a reused storage address can never inherit stale statistics)"""
    if part is not None:
        t.seedx_col_part = part
    return t


def _part(t):
    return getattr(t, "seedx_col_part", None) if t is not None else None


def pack_conv(w, dev, cin_pad_to=None):
    """[Cout, Cin, k, k] -> fp16 [Cout, k*k*Cpad], k index = (kh*k + kw)*Cpad + c, Cpad = roundup(Cin, 64)."""
    cout, cin, k, _ = w.shape
    cpad = (cin + 63) // 64 * 64
    wp = torch.zeros((cout, k, k, cpad), dtype=torch.float16, device=w.device)
    wp[..., :cin] = w.permute(0, 2, 3, 1).to(torch.float16)
    return wp.reshape(cout, k * k * cpad).to(dev).contiguous()


def conv_fp8(w16, cin, taps=3):
    """FP8 copy of a packed fp16 conv weight (pack_conv layout, Cpad = roundup(cin, 64)) for seedx_conv_fp8: (q, s) = quantize_fp8_rows(w16), the
    scale per output channel, with q repacked to [Cout, taps*taps*roundup(cin, 128)] (the conv's 128-channel stages) and zero channel padding."""
    cout = w16.shape[0]
    q, sc = quantize_fp8_rows(w16)
    c128 = (cin + 127) // 128 * 128
    q8 = torch.zeros((cout, taps * taps, c128), dtype=torch.uint8, device=w16.device)
    q8[..., :cin] = q.view(torch.uint8).view(cout, taps * taps, -1)[..., :cin]
    return q8.view(cout, taps * taps * c128).view(torch.float8_e4m3fn), sc


class _ConvFP8:
    """FP8 copy of one packed fp16 3x3 conv weight (w16 stays resident and is what checkpoints update): q e4m3 [Cout, 9*roundup(cin, 128)] and
    s fp32 [Cout], re-derived in place by requantize() so that captured graphs keep their pointers"""

    def __init__(self, w16, cin):
        self.w16, self.cin = w16, cin
        self.q, self.s = conv_fp8(w16, cin)

    def requantize(self):
        q, sc = conv_fp8(self.w16, self.cin)
        self.q.copy_(q), self.s.copy_(sc)

    def __call__(self, x, **kw):
        """the conv on fp16 NHWC x: x is quantised per image right before it (seedx_quant_images_fp8), then seedx_conv_fp8"""
        qx, sx = ops.quant_images_fp8(x)
        return ops.conv2d_nhwc(qx, self.q, a_scale=sx, w_scale=self.s, **kw)


def pad_rows(w, b, nmin=8):
    """pad a tiny output dimension up to a multiple of 8 rows (so the NHWC result keeps 16-byte pixels)."""
    n = w.shape[0]
    npad = (n + nmin - 1) // nmin * nmin
    if npad == n:
        return w, b
    wp = torch.zeros((npad,) + tuple(w.shape[1:]), dtype=w.dtype, device=w.device)
    wp[:n] = w
    bp = torch.zeros((npad,), dtype=b.dtype, device=b.device)
    bp[:n] = b
    return wp, bp


class _ParamRegistry:
    """checkpoint key -> (packed device tensor or slice of one, packing function): lets a later (partial) state dict overwrite the packed
    parameters IN PLACE (the reference loads adapter checkpoints with strict=False: only `to_k` / `to_v` (+ `conv_in`) of the UNet are present
    when full_ft is false, adapter_modules.py:20-33,59-65), so captured CUDA graphs and cached loops keep pointing at live storage."""

    def __init__(self):
        self.slots = {}
        self.folded = []          # _FoldedLinear objects: their consistency is checked once an update is complete

    def add(self, key, dest, fn, hook=None):
        """hook(value) runs after the copy (derived tensors of a folded layer)"""
        self.slots[key] = (dest, fn, hook)

    def update(self, key, value):
        dest, fn, hook = self.slots[key]
        new = fn(value)
        if new.shape != dest.shape:
            raise SeedxError(f"{key}: shape {tuple(value.shape)} does not match the loaded model")
        dest.copy_(new)
        if hook is not None:
            hook(value)

    def finish(self):
        for f in self.folded:
            f.check()


class _FoldedLinear:
    """A linear layer that follows a LayerNorm, stored with the normalisation folded in (seedx_gemm_args.ln_stats):
         LN(x) . W^T + b  =  rstd * (x . (W*gamma)^T - mean * colsum) + (W . beta + b)
    w = fp16(W * gamma) [N, K] (rows possibly interleaved / concatenated from several checkpoint tensors), colsum[n] = sum_k float(w[n, k]) —
    taken from the ROUNDED weights so that a constant row cancels exactly —, bias = W . beta + b in fp32.  gamma / beta stay referenced so that a
    later partial checkpoint (to_k / to_v only, adapter_modules.py:20-33) can re-fold the rows it replaces."""

    def __init__(self, parts, gamma, beta, dev, bias=None, pack=None):
        """parts: list of raw [n_i, K] weights concatenated along rows; pack: optional row permutation applied after concatenation"""
        self.gamma, self.beta, self.dev, self.pack = gamma, beta, dev, (pack or (lambda t: t))
        w = self.pack(torch.cat([p_.float() for p_ in parts], dim=0))
        self.N, self.K = w.shape
        self.w = torch.empty((self.N, self.K), device=dev, dtype=torch.float16)
        self.colsum = torch.empty((self.N,), device=dev, dtype=torch.float32)
        self.raw_bias = None if bias is None else _f(self.pack(bias), dev)
        self.bias = torch.empty((self.N,), device=dev, dtype=torch.float32)
        self.stale_rows = None                     # set when gamma / beta changed: rows still folded with the old values
        self._set(slice(0, self.N), w)

    def _set(self, rows, w_raw):
        w_raw = w_raw.to(self.dev, torch.float32)
        wf = (w_raw * self.gamma[None, :]).to(torch.float16)
        self.w[rows].copy_(wf)
        self.colsum[rows].copy_(wf.float().sum(dim=1))
        b = w_raw @ self.beta
        self.bias[rows].copy_(b if self.raw_bias is None else b + self.raw_bias[rows])
        if self.stale_rows is not None:
            self.stale_rows[rows] = False

    def set_rows(self, rows, w_raw):
        """replace a row range by a raw (un-folded, un-packed) checkpoint tensor; only valid for un-permuted layouts"""
        self._set(rows, w_raw)

    def set_all(self, w_raw):
        self._set(slice(0, self.N), self.pack(w_raw.float()))

    def set_bias(self, b_raw):
        new = _f(self.pack(b_raw), self.dev)
        self.bias.add_(new - self.raw_bias)
        self.raw_bias.copy_(new)

    def norm_changed(self):
        self.stale_rows = torch.ones((self.N,), dtype=torch.bool)

    def check(self):
        if self.stale_rows is not None:
            if bool(self.stale_rows.any()):
                raise SeedxError("a checkpoint that replaces a LayerNorm folded into the following projection must also carry that projection's weights")
            self.stale_rows = None

    def ln(self, stats):
        return (stats, self.colsum)


def _interleave_rows(w):
    """GEGLU / SwiGLU weight [2*inner, ...] -> rows [hidden_0, gate_0, hidden_1, gate_1, ...] (gate beside its value in one accumulator tile)"""
    inner = w.shape[0] // 2
    return torch.stack([w[:inner], w[inner:]], dim=1).reshape((2 * inner,) + tuple(w.shape[1:]))


class _Resnet:
    def __init__(self, sd, p, dev, eps, reg=None, fp8=False):
        """fp8: conv1 and conv2 run as FP8 convs (seedx_conv_fp8) on _ConvFP8 copies of the packed fp16 weights, their inputs quantised per image;
        the shortcut and everything else stay fp16.  The VAE builds its blocks with fp8=False."""
        self.eps = eps
        self._sb = {}
        self.n1 = (_f(sd[p + ".norm1.weight"], dev), _f(sd[p + ".norm1.bias"], dev))
        self.n2 = (_f(sd[p + ".norm2.weight"], dev), _f(sd[p + ".norm2.bias"], dev))
        self.w1, self.b1 = pack_conv(sd[p + ".conv1.weight"], dev), _f(sd[p + ".conv1.bias"], dev)
        self.w2, self.b2 = pack_conv(sd[p + ".conv2.weight"], dev), _f(sd[p + ".conv2.bias"], dev)
        self.fp8 = None
        if fp8:
            self.fp8 = dict(conv1=_ConvFP8(self.w1, sd[p + ".conv1.weight"].shape[1]), conv2=_ConvFP8(self.w2, sd[p + ".conv2.weight"].shape[1]))
        self.wt = self.bt = None
        if (p + ".time_emb_proj.weight") in sd:
            self.wt, self.bt = _h(sd[p + ".time_emb_proj.weight"], dev), _f(sd[p + ".time_emb_proj.bias"], dev)
        self.wsc = self.bsc = None
        if (p + ".conv_shortcut.weight") in sd:
            w = sd[p + ".conv_shortcut.weight"]
            self.wsc, self.bsc = _h(w.reshape(w.shape[0], w.shape[1]), dev), _f(sd[p + ".conv_shortcut.bias"], dev)
        if reg is not None:
            hh, ff = (lambda t: _h(t, dev)), (lambda t: _f(t, dev))
            for nm, pair in (("norm1", self.n1), ("norm2", self.n2)):
                reg.add(f"{p}.{nm}.weight", pair[0], ff), reg.add(f"{p}.{nm}.bias", pair[1], ff)
            for nm, w_, b_ in (("conv1", self.w1, self.b1), ("conv2", self.w2, self.b2)):
                reg.add(f"{p}.{nm}.weight", w_, lambda t: pack_conv(t, dev)), reg.add(f"{p}.{nm}.bias", b_, ff)
            if self.wt is not None:
                reg.add(p + ".time_emb_proj.weight", self.wt, hh), reg.add(p + ".time_emb_proj.bias", self.bt, ff)
            if self.wsc is not None:
                reg.add(p + ".conv_shortcut.weight", self.wsc, lambda t: _h(t.reshape(t.shape[0], t.shape[1]), dev))
                reg.add(p + ".conv_shortcut.bias", self.bsc, ff)

    def _scaled(self, alpha):
        """biases of the convs that write the scaled stream, multiplied by alpha once (the GEMM epilogue computes alpha*acc + bias)"""
        if alpha not in self._sb:
            self._sb[alpha] = tuple(None if b is None else (b * alpha).contiguous() for b in (self.b1, self.b2, self.bsc))
        return self._sb[alpha]

    def __call__(self, x, skip, semb, groups, ws, alpha=1.0):
        """ResnetBlock2D on NHWC fp16; `skip` (optional) is channel-concatenated behind x (UNet up blocks).
        alpha != 1 (VAE `force_upcast` mode, AutoencoderKL.stream_scale): x, the conv1 output and the result are alpha * their true
        values.  GroupNorm is scale invariant once eps is scaled by alpha^2, so the normalised operands of both convs are unchanged and
        only the conv epilogues carry the factor — exact in fp32, and the stored fp16 stream stays 1/alpha below the overflow limit."""
        n, h, w, _ = x.shape
        raw = None
        if skip is not None:
            raw = torch.empty((n, h, w, x.shape[3] + skip.shape[3]), device=x.device, dtype=torch.float16)
        b1, b2, bsc = (self.b1, self.b2, self.bsc) if alpha == 1.0 else self._scaled(alpha)
        eps = self.eps * alpha * alpha
        a = ops.groupnorm_nhwc(x, self.n1[0], self.n1[1], eps, x2=skip, silu=True, groups=groups, raw_out=raw, stats_ws=ws,
                               part1=_part(x), part2=_part(skip))
        tb = ops.gemm(semb, self.wt, bias=self.bt, out_dtype=torch.float32) if self.wt is not None else None
        if tb is not None and alpha != 1.0:
            raise SeedxError("scaled-stream ResnetBlock2D with a time embedding is not used by any model")
        cout = self.w1.shape[0]
        p1 = _new_col_part(n, h, w, cout, x.device)            # norm2 statistics: emitted by conv1's epilogue
        conv1 = self.fp8["conv1"] if self.fp8 else (lambda x, **kw: ops.conv2d_nhwc(x, self.w1, **kw))
        conv2 = self.fp8["conv2"] if self.fp8 else (lambda x, **kw: ops.conv2d_nhwc(x, self.w2, **kw))
        a = conv1(a, bias=b1, bias_g=tb, alpha=alpha, col_part=p1)
        a = ops.groupnorm_nhwc(a, self.n2[0], self.n2[1], eps, silu=True, groups=groups, stats_ws=ws, part1=p1)
        xin = raw if raw is not None else x
        if self.wsc is not None:
            sc = ops.gemm(xin.view(n * h * w, xin.shape[3]), self.wsc, bias=bsc).view(n, h, w, -1)     # linear in the scaled input
        else:
            sc = xin
        p2 = _new_col_part(n, h, w, cout, x.device)            # statistics of the block output for whichever GroupNorm reads it next
        return _tag(conv2(a, bias=b2, residual=sc, alpha=alpha, col_part=p2), p2)


class _Transformer:
    # dtype of the residual stream of the transformer blocks.  fp16 matches the reference (which runs the whole UNet in fp16) and
    # halves the HBM traffic of the residual epilogues and LayerNorm reads; fp32 is available for parity experiments.
    stream_dtype = torch.float16

    def __init__(self, sd, p, dev, depth, heads, reg=None, fp8=False):
        """fp8: every projection GEMM of the block runs as e4m3 x e4m3 (seedx_gemm_fp8) on per-row FP8 copies of the packed fp16 weights;
        the fp16 weights stay resident (they are what the registry and the folding update) and the copies are re-derived from them in place
        (requantize_fp8) whenever a checkpoint changes weights."""
        self.heads = heads
        self.fp8 = fp8
        self.norm = (_f(sd[p + ".norm.weight"], dev), _f(sd[p + ".norm.bias"], dev))
        self.w_in, self.b_in = _h(sd[p + ".proj_in.weight"], dev), _f(sd[p + ".proj_in.bias"], dev)
        self.w_out, self.b_out = _h(sd[p + ".proj_out.weight"], dev), _f(sd[p + ".proj_out.bias"], dev)
        hh, ff = (lambda t: _h(t, dev)), (lambda t: _f(t, dev))
        if reg is not None:
            reg.add(p + ".norm.weight", self.norm[0], ff), reg.add(p + ".norm.bias", self.norm[1], ff)
            reg.add(p + ".proj_in.weight", self.w_in, hh), reg.add(p + ".proj_in.bias", self.b_in, ff)
            reg.add(p + ".proj_out.weight", self.w_out, hh), reg.add(p + ".proj_out.bias", self.b_out, ff)
        self.blocks = []
        for k in range(depth):
            b = f"{p}.transformer_blocks.{k}"
            g = lambda s: sd[f"{b}.{s}"]  # noqa: E731
            n1 = (_f(g("norm1.weight"), dev), _f(g("norm1.bias"), dev))
            n2 = (_f(g("norm2.weight"), dev), _f(g("norm2.bias"), dev))
            n3 = (_f(g("norm3.weight"), dev), _f(g("norm3.bias"), dev))
            # the three projections that read a LayerNorm output carry it folded in (no normalised copy of the stream is ever written):
            # fused QKV (norm1), cross-attention q (norm2), GEGLU projection with [hidden_j, gate_j] interleaved rows (norm3)
            qkv = _FoldedLinear([g("attn1.to_q.weight"), g("attn1.to_k.weight"), g("attn1.to_v.weight")], n1[0], n1[1], dev)
            q2 = _FoldedLinear([g("attn2.to_q.weight")], n2[0], n2[1], dev)
            ff1 = _FoldedLinear([g("ff.net.0.proj.weight")], n3[0], n3[1], dev, bias=g("ff.net.0.proj.bias"), pack=_interleave_rows)
            self.blocks.append(dict(
                n1=n1, n2=n2, n3=n3, qkv=qkv, q2=q2, ff1=ff1,
                w_o1=_h(g("attn1.to_out.0.weight"), dev), b_o1=_f(g("attn1.to_out.0.bias"), dev),
                w_kv2=_h(torch.cat([g("attn2.to_k.weight"), g("attn2.to_v.weight")], dim=0), dev),
                w_o2=_h(g("attn2.to_out.0.weight"), dev), b_o2=_f(g("attn2.to_out.0.bias"), dev),
                w_ff2=_h(g("ff.net.2.weight"), dev), b_ff2=_f(g("ff.net.2.bias"), dev)))
            if reg is not None:
                blk = self.blocks[-1]
                c = blk["w_o1"].shape[0]
                reg.folded += [qkv, q2, ff1]
                for i, (nm, fl) in enumerate((("n1", qkv), ("n2", q2), ("n3", ff1))):
                    reg.add(f"{b}.norm{i + 1}.weight", blk[nm][0], ff, hook=lambda v, fl=fl: fl.norm_changed())
                    reg.add(f"{b}.norm{i + 1}.bias", blk[nm][1], ff, hook=lambda v, fl=fl: fl.norm_changed())
                keep = lambda dest: (lambda t: dest)        # the hook writes the folded rows; the registry's own copy is then a no-op  # noqa: E731
                for i, nm in enumerate(("to_q", "to_k", "to_v")):
                    rows = slice(i * c, (i + 1) * c)
                    reg.add(f"{b}.attn1.{nm}.weight", qkv.w[rows], keep(qkv.w[rows]), hook=lambda v, rows=rows, fl=qkv: fl.set_rows(rows, v))
                reg.add(f"{b}.attn2.to_q.weight", q2.w, keep(q2.w), hook=lambda v, fl=q2: fl.set_all(v))
                reg.add(f"{b}.attn2.to_k.weight", blk["w_kv2"][:c], hh), reg.add(f"{b}.attn2.to_v.weight", blk["w_kv2"][c:], hh)
                for a_, wn, bn in (("attn1", "w_o1", "b_o1"), ("attn2", "w_o2", "b_o2")):
                    reg.add(f"{b}.{a_}.to_out.0.weight", blk[wn], hh), reg.add(f"{b}.{a_}.to_out.0.bias", blk[bn], ff)
                reg.add(f"{b}.ff.net.0.proj.weight", ff1.w, keep(ff1.w), hook=lambda v, fl=ff1: fl.set_all(v))
                reg.add(f"{b}.ff.net.0.proj.bias", ff1.raw_bias, keep(ff1.raw_bias), hook=lambda v, fl=ff1: fl.set_bias(v))
                reg.add(f"{b}.ff.net.2.weight", blk["w_ff2"], hh), reg.add(f"{b}.ff.net.2.bias", blk["b_ff2"], ff)
        # FP8 copies: name -> (packed fp16 source, q float8_e4m3fn, s fp32 per output row, colsum8 of a folded projection or None)
        self.fp8_w = {}
        if fp8:
            for name, w16, folded in (("proj_in", self.w_in, False), ("proj_out", self.w_out, False)):
                self.fp8_w[name] = self._fp8_copy(w16, folded)
            for blk in self.blocks:
                blk["fp8"] = {name: self._fp8_copy(w16, folded) for name, w16, folded in (
                    ("attn1.qkv", blk["qkv"].w, True), ("attn1.to_out", blk["w_o1"], False), ("attn2.to_q", blk["q2"].w, True),
                    ("attn2.to_out", blk["w_o2"], False), ("ff.net.0", blk["ff1"].w, True), ("ff.net.2", blk["w_ff2"], False))}

    @staticmethod
    def _fp8_rows(w16):
        """(q, s, colsum8) of a packed fp16 weight.  colsum8[n] = s[n] * sum_k float(q[n, k]): the folded LayerNorm's mean correction must cancel
        against the weights the MMA actually sums, the dequantized FP8 ones (as _FoldedLinear takes its colsum from the ROUNDED fp16 weights)."""
        q, sc = quantize_fp8_rows(w16)
        return q, sc, q.float().sum(dim=1) * sc

    def _fp8_copy(self, w16, folded):
        q, sc, cs = self._fp8_rows(w16)
        return (w16, q, sc, cs if folded else None)

    def fp8_slots(self):
        """every FP8 copy of this transformer: (name, (fp16 source, q, s, colsum8 or None))"""
        out = list(self.fp8_w.items())
        for blk in self.blocks:
            out += list(blk.get("fp8", {}).items())
        return out

    def requantize_fp8(self):
        """re-derive every FP8 copy from its fp16 source, writing q, s and colsum8 in place (captured graphs keep their pointers)"""
        for _, (w16, q, sc, cs) in self.fp8_slots():
            nq, ns, ncs = self._fp8_rows(w16)
            q.copy_(nq), sc.copy_(ns)
            if cs is not None:
                cs.copy_(ncs)

    def context_kv(self, ctx16):
        """cross-attention K/V of every block for a step-invariant context [B*T, ctx_dim] (hoisted out of the sampler loop)."""
        return [ops.gemm(ctx16, blk["w_kv2"]) for blk in self.blocks]

    def _row_tickets(self, slabs, device):
        """persistent ticket counters of the in-epilogue row finalize: the kernel that takes a slab's last ticket resets it, so one zeroed buffer
        per block and slab count serves every call of this block (no fill kernel per transformer in the forward)"""
        key = (str(device), slabs)
        tk = self.__dict__.setdefault("_tickets", {})
        if key not in tk:
            tk[key] = torch.zeros((slabs,), device=device, dtype=torch.int32)
        return tk[key]

    def __call__(self, x, kv, n_ctx, groups, ws):
        n, h, w, c = x.shape
        S, M, H = h * w, n * h * w, self.heads
        d = c // H
        scale = d ** -0.5
        hn = ops.groupnorm_nhwc(x, self.norm[0], self.norm[1], 1e-6, silu=False, groups=groups, stats_ws=ws, part1=_part(x))
        if self.stream_dtype != torch.float16:
            raise SeedxError("the folded LayerNorm path reads the residual stream as the fp16 GEMM operand: _Transformer.stream_dtype must be float16")
        # LayerNorm statistics of the residual stream: row partials written by the epilogue of every GEMM that stores the stream (one (sum, sumsq)
        # pair per 32-column chunk), reduced to (mean, rstd) per row by a finalize kernel that reads c/32 * 8 bytes per row instead of the row;
        # shapes that cannot use them fall back to the row-statistics kernel over the stream itself
        rp = torch.empty((c // 32, M, 2), device=x.device, dtype=torch.float32) if (EPI_STATS and M % 32 == 0 and c % 32 == 0) else None
        stats = torch.empty((M, 2), device=x.device, dtype=torch.float32)
        # the epilogue warp that delivers a 32-row slab's last partial also reduces the slab to (mean, rstd): no statistics launch at all
        rs = (stats, self._row_tickets(M // 32, x.device), 1e-5) if (rp is not None and ROW_TICKETS) else None

        def ln_of(fl):
            if rp is None:
                ops.row_stats(hs, 1e-5, out=stats)
            elif rs is None:
                ops.row_finalize(rp, 1e-5, out=stats)
            return (stats, fl.colsum)
        if self.fp8:
            # every projection input is quantised per row right before its GEMM, into one scratch operand (the GEMM that reads it has finished
            # before the next quantisation writes: each kernel waits for its predecessor)
            a8 = torch.empty((M * 4 * c,), device=x.device, dtype=torch.float8_e4m3fn)
            a8s = torch.empty((M,), device=x.device, dtype=torch.float32)

        def proj(a, w16, w8, ln_fl=None, **kw):
            """a . w^T through the fp16 GEMM, or through the FP8 GEMM on the quantised a and w8 = (fp16 source, q, s, colsum8)"""
            if not self.fp8:
                return ops.gemm(a, w16, ln=None if ln_fl is None else ln_of(ln_fl), **kw)
            qa = a8[: a.shape[0] * a.shape[1]].view(a.shape[0], a.shape[1])
            ops.quant_rows_fp8(a, q=qa, scale=a8s)
            ln = None
            if ln_fl is not None:
                ln = (ln_of(ln_fl)[0], w8[3])
            return ops.gemm(qa, w8[1], ln=ln, a_scale=a8s, w_scale=w8[2], **kw)
        f8 = self.fp8_w
        hs = proj(hn.view(M, c), self.w_in, f8.get("proj_in"), bias=self.b_in, out_dtype=torch.float16, row_part=rp, row_stats=rs)
        qkv = torch.empty((M, 3 * c), device=x.device, dtype=torch.float16)
        obuf = torch.empty((M, c), device=x.device, dtype=torch.float16)
        qbuf = torch.empty((M, c), device=x.device, dtype=torch.float16)
        fbuf = torch.empty((M, 4 * c), device=x.device, dtype=torch.float16)
        q5 = qkv.view(n, S, 3, H, d)
        q1, k1, v1 = (q5[:, :, i].permute(0, 2, 1, 3) for i in range(3))
        ov = obuf.view(n, S, H, d).permute(0, 2, 1, 3)
        q2 = qbuf.view(n, S, H, d).permute(0, 2, 1, 3)
        for blk, kvb in zip(self.blocks, kv):
            b8 = blk.get("fp8", {})
            # norm1 -> fused QKV, norm2 -> cross-attention q, norm3 -> GEGLU: the normalisation happens in the projection's epilogue
            proj(hs, blk["qkv"].w, b8.get("attn1.qkv"), blk["qkv"], out=qkv, bias=blk["qkv"].bias)
            ops.attention(q1, k1, v1, ov, scale=scale)
            proj(obuf, blk["w_o1"], b8.get("attn1.to_out"), out=hs, bias=blk["b_o1"], residual=hs, row_part=rp, row_stats=rs)
            proj(hs, blk["q2"].w, b8.get("attn2.to_q"), blk["q2"], out=qbuf, bias=blk["q2"].bias)
            kv5 = kvb.view(n, n_ctx, 2, H, d)
            ops.attention(q2, kv5[:, :, 0].permute(0, 2, 1, 3), kv5[:, :, 1].permute(0, 2, 1, 3), ov, scale=scale)
            proj(obuf, blk["w_o2"], b8.get("attn2.to_out"), out=hs, bias=blk["b_o2"], residual=hs, row_part=rp, row_stats=rs)
            proj(hs, blk["ff1"].w, b8.get("ff.net.0"), blk["ff1"], out=fbuf, bias=blk["ff1"].bias, act=ops.ACT_GELU, gated=True)
            proj(fbuf, blk["w_ff2"], b8.get("ff.net.2"), out=hs, bias=blk["b_ff2"], residual=hs, row_part=rp, row_stats=rs)
        po = _new_col_part(n, h, w, c, x.device)
        return _tag(proj(hs, self.w_out, f8.get("proj_out"), bias=self.b_out, residual=x.view(M, c), col_part=po).view(n, h, w, c), po)


# diffusers name of the block above: src/inference/eval_img2edit_seed_x_edit.py:8 imports it (and never instantiates it)
Transformer2DModel = _Transformer


def _conv_s2(x, w, b, pad_before):
    """3x3 stride-2 conv = patch gather + GEMM (UNet Downsample2D pad 1; VAE encoder asymmetric pad (0,1))."""
    n, h, wd, c = x.shape
    ho, wo = h // 2, wd // 2
    a = ops.im2col_nhwc(x, 3, 2, pad_before, ho, wo)
    part = _new_col_part(n, ho, wo, w.shape[0], x.device)
    return _tag(ops.gemm(a, w, bias=b, col_part=part).view(n, ho, wo, -1), part)


def pack_conv_dense(w, dev):
    """[Cout, Cin, k, k] -> fp16 [Cout, k*k*Cin] matching seedx_im2col_nhwc's column order."""
    cout, cin, k, _ = w.shape
    return w.permute(0, 2, 3, 1).reshape(cout, k * k * cin).to(dev, torch.float16).contiguous()


class UNet2DConditionModel:
    """SDXL UNet (forward only). ``cfg`` follows SDXL_UNET; in_channels 8 = the edit variant (adapter_modules.py:183-198)."""

    def __init__(self, cfg=None, device="cuda", weight_format="fp16"):
        """weight_format="fp8_e4m3": the projection GEMMs of every transformer block (proj_in, fused QKV, attn1.to_out, attn2.to_q,
        attn2.to_out, GEGLU ff.net.0, ff.net.2, proj_out) run as e4m3 x e4m3 with per-row scales on both operands; everything else (convs,
        attention, the hoisted cross-attention K/V, embeddings) stays fp16.  The fp16 weights stay resident beside the FP8 copies.
        weight_format="fp8_e4m3_conv": all of that, and conv1 / conv2 of every ResnetBlock2D plus both upsampler convs run as FP8 convs with
        one scale per image and per output channel (36 convs at SDXL size); conv_in, conv_out, the 1x1 shortcuts and the stride-2
        downsamplers stay fp16."""
        if weight_format not in UNET_WEIGHT_FORMATS:
            raise SeedxError(f"weight_format {weight_format!r}: expected one of {UNET_WEIGHT_FORMATS}")
        self.weight_format = weight_format
        self.cfg = dict(SDXL_UNET if cfg is None else cfg)
        self.device = torch.device(device)
        self.dtype = torch.float16
        self._loaded = False
        self._reg = _ParamRegistry()

    @classmethod
    def from_pretrained(cls, path, subfolder=None, **kw):
        d = os.path.join(path, subfolder) if subfolder else path
        cfg = dict(SDXL_UNET)
        cj = os.path.join(d, "config.json")
        if os.path.exists(cj):
            c = json.load(open(cj))
            cfg.update(in_channels=c.get("in_channels", 4), out_channels=c.get("out_channels", 4),
                       block_out_channels=tuple(c["block_out_channels"]), layers_per_block=c["layers_per_block"],
                       transformer_layers=tuple(c["transformer_layers_per_block"]), heads=tuple(c["attention_head_dim"]),
                       cross_attention_dim=c["cross_attention_dim"], addition_time_embed_dim=c["addition_time_embed_dim"],
                       down_attn=tuple("CrossAttn" in t for t in c["down_block_types"]))
        m = cls(cfg, device=kw.get("device", "cuda"), weight_format=kw.get("weight_format", "fp16"))
        m.load_state_dict(_load_weights_dir(d))
        return m

    def to(self, *a, **k):
        return self

    def eval(self):
        return self

    def transformers(self):
        return [t for b in self.down for t in b["att"]] + [self.mid["att"]] + [t for b in self.up for t in b["att"]]

    def conv_fp8_slots(self):
        """every FP8 conv copy: (checkpoint prefix of the conv, _ConvFP8); empty unless weight_format="fp8_e4m3_conv" """
        if not self._loaded:
            return []
        out = []
        res = [(f"down_blocks.{i}.resnets.{j}", r) for i, b in enumerate(self.down) for j, r in enumerate(b["res"])]
        res += [("mid_block.resnets.0", self.mid["r0"]), ("mid_block.resnets.1", self.mid["r1"])]
        res += [(f"up_blocks.{i}.resnets.{j}", r) for i, b in enumerate(self.up) for j, r in enumerate(b["res"])]
        for p, r in res:
            out += [(f"{p}.{k}", c) for k, c in (r.fp8 or {}).items()]
        out += [(f"up_blocks.{i}.upsamplers.0.conv", b["us8"]) for i, b in enumerate(self.up) if b.get("us8") is not None]
        return out

    def state_shape_in_channels(self):
        return self.cfg["in_channels"]

    def update_state_dict(self, sd):
        """overwrite the packed parameters named in `sd` in place (a partial checkpoint, `load_state_dict(..., strict=False)` in the
        reference: adapter_modules.py:59-65).  Returns the keys this model does not have (the 'unexpected' list)."""
        unexpected = []
        for k, v in sd.items():
            if k not in self._reg.slots:
                unexpected.append(k)
                continue
            if k == "conv_in.weight":
                if v.shape[1] > 8:
                    raise SeedxError("conv_in with more than 8 input channels is not supported")
                self.cfg["in_channels"] = v.shape[1]
        # LayerNorm parameters first: the projections folded with them are re-folded with the new values as their own keys arrive
        for k in sorted((k for k in sd if k in self._reg.slots), key=lambda k: (0 if ".norm" in k else 1)):
            self._reg.update(k, sd[k])
        self._reg.finish()
        if self.weight_format in ("fp8_e4m3", "fp8_e4m3_conv"):
            for t in self.transformers():
                t.requantize_fp8()
        for _, c in self.conv_fp8_slots():
            c.requantize()
        return unexpected

    def load_state_dict(self, sd, strict=False):
        if self._loaded:
            # a second checkpoint on top of the loaded base model (possibly partial): in place, storage pointers unchanged
            return [k for k in self._reg.slots if k not in sd], self.update_state_dict(sd)
        cfg, dev = self.cfg, self.device
        boc = cfg["block_out_channels"]
        nb = len(boc)
        reg = self._reg = _ParamRegistry()
        fp8 = self.weight_format in ("fp8_e4m3", "fp8_e4m3_conv")
        conv8 = self.weight_format == "fp8_e4m3_conv"
        cin = sd["conv_in.weight"].shape[1]
        self.cfg["in_channels"] = cin
        # widths the checkpoint itself fixes (diffusers: time_embed_dim = 4*block_out_channels[0], projection_class_embeddings_input_dim)
        self.cfg["time_embed_dim"] = sd["time_embedding.linear_1.weight"].shape[0]
        self.cfg["text_embed_dim"] = sd["add_embedding.linear_1.weight"].shape[1] - 6 * cfg["addition_time_embed_dim"]
        if cin > 8:
            raise SeedxError("conv_in with more than 8 input channels is not supported")
        hh, ff = (lambda t: _h(t, dev)), (lambda t: _f(t, dev))
        self.conv_in = (pack_conv(sd["conv_in.weight"], dev), _f(sd["conv_in.bias"], dev))
        reg.add("conv_in.weight", self.conv_in[0], lambda t: pack_conv(t, dev)), reg.add("conv_in.bias", self.conv_in[1], ff)

        def lin(p):
            w, b = _h(sd[p + ".weight"], dev), _f(sd[p + ".bias"], dev)
            reg.add(p + ".weight", w, hh), reg.add(p + ".bias", b, ff)
            return w, b
        self.t1, self.t2 = lin("time_embedding.linear_1"), lin("time_embedding.linear_2")
        self.a1, self.a2 = lin("add_embedding.linear_1"), lin("add_embedding.linear_2")
        self.down, self.up = [], []
        for i in range(nb):
            blk = dict(res=[], att=[], ds=None)
            for j in range(cfg["layers_per_block"]):
                blk["res"].append(_Resnet(sd, f"down_blocks.{i}.resnets.{j}", dev, 1e-5, reg, conv8))
                if cfg["down_attn"][i]:
                    blk["att"].append(_Transformer(sd, f"down_blocks.{i}.attentions.{j}", dev, cfg["transformer_layers"][i], cfg["heads"][i], reg, fp8))
            if i < nb - 1:
                p = f"down_blocks.{i}.downsamplers.0.conv"
                blk["ds"] = (pack_conv_dense(sd[p + ".weight"], dev), _f(sd[p + ".bias"], dev))
                reg.add(p + ".weight", blk["ds"][0], lambda t: pack_conv_dense(t, dev)), reg.add(p + ".bias", blk["ds"][1], ff)
            self.down.append(blk)
        self.mid = dict(r0=_Resnet(sd, "mid_block.resnets.0", dev, 1e-5, reg, conv8),
                        att=_Transformer(sd, "mid_block.attentions.0", dev, cfg["transformer_layers"][-1], cfg["heads"][-1], reg, fp8),
                        r1=_Resnet(sd, "mid_block.resnets.1", dev, 1e-5, reg, conv8))
        for i in range(nb):
            r = nb - 1 - i
            blk = dict(res=[], att=[], us=None, us8=None)
            for j in range(cfg["layers_per_block"] + 1):
                blk["res"].append(_Resnet(sd, f"up_blocks.{i}.resnets.{j}", dev, 1e-5, reg, conv8))
                if cfg["down_attn"][r]:
                    blk["att"].append(_Transformer(sd, f"up_blocks.{i}.attentions.{j}", dev, cfg["transformer_layers"][r], cfg["heads"][r], reg, fp8))
            if i < nb - 1:
                p = f"up_blocks.{i}.upsamplers.0.conv"
                blk["us"] = (pack_conv(sd[p + ".weight"], dev), _f(sd[p + ".bias"], dev))
                reg.add(p + ".weight", blk["us"][0], lambda t: pack_conv(t, dev)), reg.add(p + ".bias", blk["us"][1], ff)
                if conv8:
                    blk["us8"] = _ConvFP8(blk["us"][0], sd[p + ".weight"].shape[1])
            self.up.append(blk)
        self.norm_out = (_f(sd["conv_norm_out.weight"], dev), _f(sd["conv_norm_out.bias"], dev))
        self.conv_out = (pack_conv(sd["conv_out.weight"], dev), _f(sd["conv_out.bias"], dev))
        reg.add("conv_norm_out.weight", self.norm_out[0], ff), reg.add("conv_norm_out.bias", self.norm_out[1], ff)
        reg.add("conv_out.weight", self.conv_out[0], lambda t: pack_conv(t, dev)), reg.add("conv_out.bias", self.conv_out[1], ff)
        self._loaded = True
        return [], []

    # ---- step-invariant conditioning ---------------------------------------------------------------------------
    def prepare_cond(self, ctx, text_embeds, time_ids):
        """ctx [Be,T,ctx_dim], text_embeds [Be,1280], time_ids [Be,6] (any float dtype, device tensors).  Returns the
        hoisted cross-attention K/V of every transformer block and the 'text_time' additive embedding."""
        cfg = self.cfg
        Be, T, cd = ctx.shape
        ctx16 = ops.unary_f16(ctx.reshape(Be * T, cd).contiguous())
        kv = dict(n_ctx=T, down=[[a.context_kv(ctx16) for a in b["att"]] for b in self.down], mid=self.mid["att"].context_kv(ctx16),
                  up=[[a.context_kv(ctx16) for a in b["att"]] for b in self.up])
        td = cfg["addition_time_embed_dim"]
        te = cfg["text_embed_dim"]
        aug_in = torch.empty((Be, te + 6 * td), device=self.device, dtype=torch.float16)
        ops.unary_f16(text_embeds.reshape(Be, te).contiguous(), out=aug_in[:, :te])
        tid = time_ids.reshape(-1).float().contiguous()
        tid_emb = torch.empty((Be * 6, td), device=self.device, dtype=torch.float16)
        ops.timestep_embedding(tid, td, tid_emb)                       # row b*6+i = Timesteps(td)(time_ids[b, i])
        ops.unary_f16(tid_emb.view(Be, 6 * td), out=aug_in[:, te:])    # flatten(1) and concatenate behind text_embeds
        a = ops.gemm(aug_in, self.a1[0], bias=self.a1[1], act=ops.ACT_SILU)
        kv["aug"] = ops.gemm(a, self.a2[0], bias=self.a2[1], out_dtype=torch.float32)
        return kv

    # ---- forward ---------------------------------------------------------------------------------------------------
    def forward_nhwc(self, x_in, t_dev, cond):
        """x_in: fp16 NHWC [Be,H,W,8] (scaled latents in channels 0..3, image latents / zeros in 4..7);
        t_dev: fp32 device tensor [Be] holding the timestep; cond: prepare_cond(...) -> eps fp32 [Be,H,W,4]."""
        if not self._loaded:
            raise SeedxError("UNet2DConditionModel: weights not loaded")
        cfg = self.cfg
        G = cfg["groups"]
        Be = x_in.shape[0]
        nb = len(cfg["block_out_channels"])
        ws = ops.groupnorm_ws(Be, G, self.device)
        T = cond["n_ctx"]
        temb_in = torch.empty((Be, cfg["block_out_channels"][0]), device=self.device, dtype=torch.float16)
        ops.timestep_embedding(t_dev, cfg["block_out_channels"][0], temb_in)
        e1 = ops.gemm(temb_in, self.t1[0], bias=self.t1[1], act=ops.ACT_SILU)
        emb = ops.gemm(e1, self.t2[0], bias=self.t2[1], residual=cond["aug"], out_dtype=torch.float32)
        semb = ops.unary_f16(emb, act=ops.ACT_SILU)

        pin = _new_col_part(Be, x_in.shape[1], x_in.shape[2], self.conv_in[0].shape[0], self.device)
        h = _tag(ops.conv2d_nhwc(x_in, self.conv_in[0], bias=self.conv_in[1], col_part=pin), pin)
        skips = [h]
        for i, blk in enumerate(self.down):
            for j, res in enumerate(blk["res"]):
                h = res(h, None, semb, G, ws)
                if blk["att"]:
                    h = blk["att"][j](h, cond["down"][i][j], T, G, ws)
                skips.append(h)
            if blk["ds"] is not None:
                h = _conv_s2(h, blk["ds"][0], blk["ds"][1], 1)
                skips.append(h)
        h = self.mid["r0"](h, None, semb, G, ws)
        h = self.mid["att"](h, cond["mid"], T, G, ws)
        h = self.mid["r1"](h, None, semb, G, ws)
        for i, blk in enumerate(self.up):
            for j, res in enumerate(blk["res"]):
                h = res(h, skips.pop(), semb, G, ws)
                if blk["att"]:
                    h = blk["att"][j](h, cond["up"][i][j], T, G, ws)
            if blk["us"] is not None:
                up = ops.upsample2x_nhwc(h)
                pu = _new_col_part(up.shape[0], up.shape[1], up.shape[2], blk["us"][0].shape[0], self.device)
                if blk["us8"] is not None:
                    h = _tag(blk["us8"](up, bias=blk["us"][1], col_part=pu), pu)
                else:
                    h = _tag(ops.conv2d_nhwc(up, blk["us"][0], bias=blk["us"][1], col_part=pu), pu)
        a = ops.groupnorm_nhwc(h, self.norm_out[0], self.norm_out[1], 1e-5, silu=True, groups=G, stats_ws=ws, part1=_part(h))
        return ops.conv2d_nhwc(a, self.conv_out[0], bias=self.conv_out[1], out_dtype=torch.float32, tile_n=64)

    def __call__(self, sample, timestep, encoder_hidden_states, added_cond_kwargs=None, **kw):
        """diffusers-style call on NCHW tensors (used by parity tests): returns eps NCHW fp32."""
        Be = sample.shape[0]
        cond = self.prepare_cond(encoder_hidden_states.to(self.device), added_cond_kwargs["text_embeds"].to(self.device),
                                 added_cond_kwargs["time_ids"].to(self.device))
        x_in = ops.nchw_to_nhwc_f16(sample.to(self.device).float().contiguous(), 8)
        t = torch.full((Be,), float(timestep), device=self.device, dtype=torch.float32)
        eps = self.forward_nhwc(x_in, t, cond)
        return ops.nhwc_to_nchw_f32(eps, self.cfg["out_channels"])


# ------------------------------------------------------------------------------------------------------------------
# VAE
# ------------------------------------------------------------------------------------------------------------------
class _VaeAttention:
    def __init__(self, sd, p, dev):
        self.norm = (_f(sd[p + ".group_norm.weight"], dev), _f(sd[p + ".group_norm.bias"], dev))
        self.wq, self.bq = _h(sd[p + ".to_q.weight"], dev), _f(sd[p + ".to_q.bias"], dev)
        self.wk, self.bk = _h(sd[p + ".to_k.weight"], dev), _f(sd[p + ".to_k.bias"], dev)
        self.wv, self.bv = _h(sd[p + ".to_v.weight"], dev), _f(sd[p + ".to_v.bias"], dev)
        self.wo, self.bo = _h(sd[p + ".to_out.0.weight"], dev), _f(sd[p + ".to_out.0.bias"], dev)

    def __call__(self, x, groups, ws, alpha=1.0):
        """single-head attention over H*W tokens, head dim = C (512): scores are materialised per image (C > 160).
        alpha: scale of the residual stream x (see _Resnet.__call__); q/k/v come from the scale-invariant GroupNorm output."""
        n, h, w, c = x.shape
        S = h * w
        hn = ops.groupnorm_nhwc(x, self.norm[0], self.norm[1], 1e-6 * alpha * alpha, silu=False, groups=groups, stats_ws=ws, part1=_part(x)).view(n, S, c)
        q = ops.gemm(hn.view(n * S, c), self.wq, bias=self.bq).view(n, S, c)
        k = ops.gemm(hn.view(n * S, c), self.wk, bias=self.bk).view(n, S, c)
        out = torch.empty((n, S, c), device=x.device, dtype=torch.float16)
        scores = torch.empty((S, S), device=x.device, dtype=torch.float32)   # fp32 scores: no fp16 overflow on real VAE weights
        probs = torch.empty((S, S), device=x.device, dtype=torch.float16)
        scale = c ** -0.5
        for i in range(n):
            vt = ops.gemm(self.wv, hn[i], bias_m=self.bv, dynamic_b=True)       # V^T [c, S]: K-major operand of P.V
            ops.gemm(q[i], k[i], out=scores, alpha=scale, dynamic_b=True)
            ops.softmax_rows(scores, 1.0, out=probs)
            ops.gemm(probs, vt, out=out[i], dynamic_b=True)
        xr = x.view(n * S, c)
        bo = self.bo if alpha == 1.0 else (self.bo * alpha)
        po = _new_col_part(n, h, w, c, x.device)
        return _tag(ops.gemm(out.view(n * S, c), self.wo, bias=bo, residual=xr, alpha=alpha, col_part=po).view(n, h, w, c), po)


class AutoencoderKL:
    """SDXL VAE (encode -> latent mode, decode).

    Precision: the reference up-casts the VAE to fp32 when its config says `force_upcast` (pipeline_stable_diffusion_xl_t2i_edit.py:569-586,
    965-975) because the activations of the stock stabilityai SDXL VAE exceed the fp16 range (NaN / black images); the `sdxl-vae-fp16-fix`
    checkpoint sets force_upcast=false.  This engine keeps fp16 tensor-core operands with fp32 accumulation in both cases and honours
    `force_upcast` by storing the un-normalised activations — the residual stream and the conv1 outputs, everything a GroupNorm reads —
    multiplied by `stream_scale` = 2^-7: GroupNorm is invariant to that factor (its eps is scaled by stream_scale^2), the normalised conv /
    attention operands are unchanged, and only epilogue constants (alpha, biases) carry it, which is exact in fp32.  Activations up to
    65504 * 128 = 8.4e6 are then representable; fp16 keeps 11 mantissa bits (bf16 would keep 8).  With force_upcast=false the stream is
    stored unscaled (stream_scale = 1), identical to round 1."""

    UPCAST_STREAM_SCALE = 2.0 ** -7

    def __init__(self, cfg=None, device="cuda"):
        self.cfg = dict(SDXL_VAE if cfg is None else cfg)
        self.cfg.setdefault("force_upcast", False)
        self.device = torch.device(device)
        self.dtype = torch.float16
        self._loaded = False

    @property
    def stream_scale(self):
        env = os.environ.get("SEEDX_VAE_STREAM_SCALE")
        if env:
            return float(env)
        return self.UPCAST_STREAM_SCALE if self.cfg.get("force_upcast") else 1.0

    class _Config:
        pass

    @property
    def config(self):
        c = AutoencoderKL._Config()
        c.scaling_factor = self.cfg["scaling_factor"]
        # False towards the caller: the pipeline's `upcast_vae()` branch (pipeline...edit.py:965-975) would cast modules this class does not
        # have; the range problem it exists for is handled inside (cfg["force_upcast"] -> stream_scale)
        c.force_upcast = False
        c.block_out_channels = list(self.cfg["block_out_channels"])
        return c

    @classmethod
    def from_pretrained(cls, path, subfolder=None, **kw):
        d = os.path.join(path, subfolder) if subfolder else path
        cfg = dict(SDXL_VAE)
        cj = os.path.join(d, "config.json")
        if os.path.exists(cj):
            c = json.load(open(cj))
            cfg.update(block_out_channels=tuple(c["block_out_channels"]), layers_per_block=c["layers_per_block"],
                       latent_channels=c["latent_channels"], scaling_factor=c.get("scaling_factor", 0.13025),
                       force_upcast=bool(c.get("force_upcast", True)))      # diffusers' AutoencoderKL default is True
        m = cls(cfg, device=kw.get("device", "cuda"))
        m.load_state_dict(_load_weights_dir(d))
        return m

    def to(self, *a, **k):
        return self

    def eval(self):
        return self

    def load_state_dict(self, sd, strict=False):
        cfg, dev = self.cfg, self.device
        boc = cfg["block_out_channels"]
        rev = list(reversed(boc))
        cv = lambda p: (pack_conv(sd[p + ".weight"], dev), _f(sd[p + ".bias"], dev))  # noqa: E731
        self.has_decoder = "decoder.conv_in.weight" in sd
        self.has_encoder = "encoder.conv_in.weight" in sd
        if self.has_decoder:
            w, b = pad_rows(sd["post_quant_conv.weight"].reshape(cfg["latent_channels"], -1), sd["post_quant_conv.bias"])
            wq = torch.zeros((w.shape[0], 8), dtype=w.dtype, device=w.device)
            wq[:, : w.shape[1]] = w
            self.post_quant = (_h(wq, dev), _f(b, dev))
            self.d_conv_in = cv("decoder.conv_in")
            self.d_mid = (_Resnet(sd, "decoder.mid_block.resnets.0", dev, 1e-6), _VaeAttention(sd, "decoder.mid_block.attentions.0", dev),
                          _Resnet(sd, "decoder.mid_block.resnets.1", dev, 1e-6))
            self.d_up = []
            for i in range(len(rev)):
                res = [_Resnet(sd, f"decoder.up_blocks.{i}.resnets.{j}", dev, 1e-6) for j in range(cfg["layers_per_block"] + 1)]
                us = cv(f"decoder.up_blocks.{i}.upsamplers.0.conv") if i < len(rev) - 1 else None
                self.d_up.append((res, us))
            self.d_norm_out = (_f(sd["decoder.conv_norm_out.weight"], dev), _f(sd["decoder.conv_norm_out.bias"], dev))
            self.d_conv_out = cv("decoder.conv_out")
        if self.has_encoder:
            w = sd["encoder.conv_in.weight"]
            self.e_conv_in = cv("encoder.conv_in")
            self.e_down = []
            for i in range(len(boc)):
                res = [_Resnet(sd, f"encoder.down_blocks.{i}.resnets.{j}", dev, 1e-6) for j in range(cfg["layers_per_block"])]
                ds = None
                if i < len(boc) - 1:
                    p = f"encoder.down_blocks.{i}.downsamplers.0.conv"
                    ds = (pack_conv_dense(sd[p + ".weight"], dev), _f(sd[p + ".bias"], dev))
                self.e_down.append((res, ds))
            self.e_mid = (_Resnet(sd, "encoder.mid_block.resnets.0", dev, 1e-6), _VaeAttention(sd, "encoder.mid_block.attentions.0", dev),
                          _Resnet(sd, "encoder.mid_block.resnets.1", dev, 1e-6))
            self.e_norm_out = (_f(sd["encoder.conv_norm_out.weight"], dev), _f(sd["encoder.conv_norm_out.bias"], dev))
            wco, bco = pad_rows(sd["encoder.conv_out.weight"], sd["encoder.conv_out.bias"])
            self.e_conv_out = (pack_conv(wco, dev), _f(bco, dev))
            L2 = 2 * cfg["latent_channels"]
            wq, bq = pad_rows(sd["quant_conv.weight"].reshape(L2, L2), sd["quant_conv.bias"])
            self.quant = (_h(wq, dev), _f(bq, dev))
        self._loaded = True
        return [], []

    def decode_nhwc(self, latents, scale=1.0):
        """latents: fp32 NCHW [B,4,h,w]; z = latents * scale (pass 1/scaling_factor) -> fp32 NHWC image [B,8h,8w,3] in ~[-1,1]."""
        if not (self._loaded and self.has_decoder):
            raise SeedxError("AutoencoderKL: decoder weights not loaded")
        G = self.cfg["groups"]
        B, _, h, w = latents.shape
        al = self.stream_scale
        sb = (lambda b: b) if al == 1.0 else (lambda b: b * al)       # bias of a conv that writes the scaled stream
        ws = ops.groupnorm_ws(B, G, self.device)
        z = ops.nchw_to_nhwc_f16(latents.to(self.device).float().contiguous(), 8, scale=scale)
        x = ops.gemm(z.view(B * h * w, 8), self.post_quant[0], bias=self.post_quant[1]).view(B, h, w, -1)
        pc = _new_col_part(B, h, w, self.d_conv_in[0].shape[0], self.device)
        x = _tag(ops.conv2d_nhwc(x, self.d_conv_in[0], bias=sb(self.d_conv_in[1]), alpha=al, col_part=pc), pc)
        x = self.d_mid[0](x, None, None, G, ws, al)
        x = self.d_mid[1](x, G, ws, al)
        x = self.d_mid[2](x, None, None, G, ws, al)
        for res, us in self.d_up:
            for r in res:
                x = r(x, None, None, G, ws, al)
            if us is not None:
                up = ops.upsample2x_nhwc(x)
                pu = _new_col_part(up.shape[0], up.shape[1], up.shape[2], us[0].shape[0], self.device)
                x = _tag(ops.conv2d_nhwc(up, us[0], bias=sb(us[1]), col_part=pu), pu)     # linear in the scaled stream
        a = ops.groupnorm_nhwc(x, self.d_norm_out[0], self.d_norm_out[1], 1e-6 * al * al, silu=True, groups=G, stats_ws=ws, part1=_part(x))
        return ops.conv2d_nhwc(a, self.d_conv_out[0], bias=self.d_conv_out[1], tile_n=64, out_dtype=torch.float32)

    def decode(self, latents, scale=1.0):
        """-> NCHW fp32 image (diffusers AutoencoderKL.decode(...).sample layout)."""
        return ops.nhwc_to_nchw_f32(self.decode_nhwc(latents, scale), 3)

    def encode_mode(self, image):
        """image NCHW fp32 in [-1,1] -> latent_dist.mode() NCHW fp32 [B,4,H/8,W/8] (NOT multiplied by scaling_factor,
        as at pipeline_stable_diffusion_xl_t2i_edit.py:523)."""
        if not (self._loaded and self.has_encoder):
            raise SeedxError("AutoencoderKL: encoder weights not loaded")
        G = self.cfg["groups"]
        B = image.shape[0]
        al = self.stream_scale
        sb = (lambda b: b) if al == 1.0 else (lambda b: b * al)
        ws = ops.groupnorm_ws(B, G, self.device)
        x = ops.nchw_to_nhwc_f16(image.to(self.device).float().contiguous(), 8)
        pc = _new_col_part(B, x.shape[1], x.shape[2], self.e_conv_in[0].shape[0], self.device)
        x = _tag(ops.conv2d_nhwc(x, self.e_conv_in[0], bias=sb(self.e_conv_in[1]), alpha=al, col_part=pc), pc)
        for res, ds in self.e_down:
            for r in res:
                x = r(x, None, None, G, ws, al)
            if ds is not None:
                x = _conv_s2(x, ds[0], sb(ds[1]), 0)
        x = self.e_mid[0](x, None, None, G, ws, al)
        x = self.e_mid[1](x, G, ws, al)
        x = self.e_mid[2](x, None, None, G, ws, al)
        a = ops.groupnorm_nhwc(x, self.e_norm_out[0], self.e_norm_out[1], 1e-6 * al * al, silu=True, groups=G, stats_ws=ws, part1=_part(x))
        m = ops.conv2d_nhwc(a, self.e_conv_out[0], bias=self.e_conv_out[1], tile_n=64)
        n, h, w, c = m.shape
        mo = ops.gemm(m.view(n * h * w, c), self.quant[0], bias=self.quant[1], out_dtype=torch.float32).view(n, h, w, -1)
        return ops.nhwc_to_nchw_f32(mo, self.cfg["latent_channels"])


# ------------------------------------------------------------------------------------------------------------------
# scheduler (host-side constants only; the per-step arithmetic runs in seedx_cfg_euler_step)
# ------------------------------------------------------------------------------------------------------------------
class EulerDiscreteScheduler:
    """SDXL scheduler_config defaults: scaled_linear betas .00085-.012, 1000 train steps, 'leading' spacing, offset 1."""

    def __init__(self, num_train_timesteps=1000, beta_start=0.00085, beta_end=0.012, steps_offset=1, **kw):
        self.num_train, self.steps_offset = num_train_timesteps, steps_offset
        betas = [(beta_start ** 0.5 + (beta_end ** 0.5 - beta_start ** 0.5) * i / (num_train_timesteps - 1)) ** 2
                 for i in range(num_train_timesteps)]
        ac, s = 1.0, []
        for b in betas:
            ac *= (1.0 - b)
            s.append(math.sqrt((1.0 - ac) / ac))
        self._sig = s
        self.order = 1
        self.sigmas = None

    @classmethod
    def from_pretrained(cls, path, subfolder=None, **kw):
        d = os.path.join(path, subfolder) if subfolder else path
        cj = os.path.join(d, "scheduler_config.json")
        if os.path.exists(cj):
            c = json.load(open(cj))
            cls.check_config(c)
            return cls(c.get("num_train_timesteps", 1000), c.get("beta_start", 0.00085), c.get("beta_end", 0.012), c.get("steps_offset", 1))
        return cls()

    # what the sampler implements = the SDXL-base scheduler_config.json the reference loads (eval_*.py:97); anything else would sample with
    # the wrong sigmas / init_noise_sigma without an error, so it is refused instead
    SUPPORTED = dict(beta_schedule="scaled_linear", timestep_spacing="leading", prediction_type="epsilon", interpolation_type="linear",
                     use_karras_sigmas=False, rescale_betas_zero_snr=False, timestep_type="discrete")

    @classmethod
    def check_config(cls, c):
        for k, want in cls.SUPPORTED.items():
            if k in c and c[k] is not None and c[k] != want:
                raise SeedxError(f"EulerDiscreteScheduler: {k}={c[k]!r} is not implemented (only {want!r}, the SDXL-base scheduler config)")
        if c.get("trained_betas") is not None:
            raise SeedxError("EulerDiscreteScheduler: trained_betas is not implemented")

    def set_timesteps(self, n, device=None):
        ratio = self.num_train // n
        ts = [float(i * ratio + self.steps_offset) for i in range(n)][::-1]
        sig = []
        for t in ts:
            lo = min(int(math.floor(t)), self.num_train - 1)
            hi = min(lo + 1, self.num_train - 1)
            w = t - lo
            sig.append(self._sig[lo] * (1 - w) + self._sig[hi] * w)
        self.timesteps = ts
        self.sigmas = sig + [0.0]
        self.init_noise_sigma = math.sqrt(max(sig) ** 2 + 1.0)
        return self
