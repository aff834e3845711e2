"""TEST DOUBLE — not product code.  Plain-torch CPU restatements of the `seedx_b200.ops` entry points that `seedx_b200.llm.LlamaForCausalLM`
calls, with the semantics documented in include/seedx.h (fp16 storage / operand rounding where the kernels round, fp32 accumulation).

Purpose: the HOST logic of the stage-2 engine — paged KV bookkeeping, lock-step batching, jump-forward over forced image spans, the
HF-style `generate` surface — can then run in the `-m "not gpu"` suite against the reference goldens, without a GPU and without the
library.  The product never imports this module (it lives under tests/); on a GPU the same host code runs over libseedx.so and is checked by
tests/test_llm_gpu.py.
"""
import torch
import torch.nn.functional as F

ACT_NONE, ACT_GELU, ACT_SILU = 0, 1, 2


def _f16(t):
    return t.to(torch.float16).float()


def cast(x, dtype):
    return x.to(dtype)


def unary_f16(x, out=None, act=ACT_NONE):
    v = x.float()
    v = F.silu(v) if act == ACT_SILU else F.gelu(v) if act == ACT_GELU else v
    if out is None:
        out = torch.empty(x.shape, dtype=torch.float16)
    out.copy_(v.to(torch.float16))
    return out


def scatter_rows(src, idx, dst, src_idx=None):
    rows = src[: idx.numel()] if src_idx is None else src[src_idx.long()]       # without src_idx, row r of src goes to idx[r]
    dst[idx.long()] = rows.float()
    return dst


def patchify(x, patch, kpad):
    """NCHW image -> fp16 [N*S, kpad] rows of flattened (c, ph, pw) patches, zero padded from 3*patch^2 to kpad (the patch-embed GEMM's A)"""
    cols = F.unfold(x.float(), kernel_size=patch, stride=patch).transpose(1, 2).reshape(-1, 3 * patch * patch)
    out = torch.zeros((cols.shape[0], kpad), dtype=torch.float16)
    out[:, : cols.shape[1]] = cols.to(torch.float16)
    return out


def gemm(a, w, out=None, *, bias=None, bias_m=None, bias_g=None, bias_g_rows=0, residual=None, res_row_mod=0, act=ACT_NONE, gated=False, alpha=1.0,
         out_dtype=torch.float16, ln=None, dynamic_b=False, row_part=None, col_part=None, row_stats=None, **kw):
    assert a.dtype == torch.float16 and w.dtype == torch.float16 and a.dim() == 2 and not any(v is not None and v is not False and v != 0 for v in kw.values())
    if residual is not None and res_row_mod:                     # residual row = output row % res_row_mod (position tables)
        residual = residual.repeat(-(-a.shape[0] // res_row_mod), 1)[: a.shape[0]]
    acc = alpha * (a.float() @ w.float().t())
    if ln is not None:                                           # folded LayerNorm: rstd * (acc - mean * colsum)
        st, cs = ln[0], ln[1]
        if len(ln) == 3:                                         # statistics from the producer's row partials [K/32, M, 2]
            tot = st.view(-1, a.shape[0], 2).sum(0)
            mean = tot[:, 0] / a.shape[1]
            st = torch.stack([mean, torch.rsqrt((tot[:, 1] / a.shape[1] - mean * mean).clamp_min(0) + ln[2])], dim=1)
        acc = st[:, 1:2] * (acc - st[:, 0:1] * cs[None, :])
    if bias is not None:
        acc = acc + bias
    if bias_m is not None:                                       # one bias per output ROW (transposed products)
        acc = acc + bias_m[:, None]
    if bias_g is not None:                                       # one additive row per group of bias_g_rows output rows
        acc = acc + bias_g.repeat_interleave(bias_g_rows, dim=0)[: a.shape[0]]
    if gated:                                                    # interleaved rows [value_j, gate_j]; ACT_NONE gates with the plain product
        g = acc[:, 1::2]
        acc = acc[:, 0::2] * (F.silu(g) if act == ACT_SILU else F.gelu(g) if act == ACT_GELU else g)
    elif act == ACT_SILU:
        acc = F.silu(acc)
    elif act == ACT_GELU:
        acc = F.gelu(acc)
    if residual is not None:
        acc = acc + residual.float()
    if out is None:
        out = torch.empty(acc.shape, dtype=out_dtype)
    out.copy_(acc.to(out.dtype))
    _emit_parts(out, acc, row_part, col_part)
    if row_stats is not None:
        row_finalize(row_part.view(-1, acc.shape[0], 2), row_stats[2], out=row_stats[0])
        assert int(row_stats[1].abs().sum()) == 0            # tickets: zero before, zero after
    return out


def _emit_parts(out, acc, row_part, col_part):
    """epilogue statistics of seedx_gemm_f16: row partials from the fp32 values, column partials from the stored fp16 values"""
    M, N = acc.shape
    if row_part is not None:
        v = acc.float().view(M, N // 32, 32)
        row_part.view(N // 32, M, 2).copy_(torch.stack([v.sum(-1), (v * v).sum(-1)], dim=-1).permute(1, 0, 2))
    if col_part is not None:
        v = out.reshape(M, N).float().view(M // 32, 32, N)
        col_part.view(M // 32, N, 2).copy_(torch.stack([v.sum(1), (v * v).sum(1)], dim=-1))


def row_finalize(row_part, eps, out=None):
    tot = row_part.sum(0)
    cols = 32 * row_part.shape[0]
    mean = tot[:, 0] / cols
    st = torch.stack([mean, torch.rsqrt((tot[:, 1] / cols - mean * mean).clamp_min(0) + eps)], dim=1)
    if out is not None:
        out.copy_(st)
        return out
    return st


def row_stats(x, eps, out=None):
    xf = x.float()
    st = torch.stack([xf.mean(-1), torch.rsqrt(xf.var(-1, unbiased=False) + eps)], dim=1)
    if out is not None:
        out.copy_(st)
        return out
    return st


def layernorm(x, gamma, beta, eps, out=None, *, out_dtype=torch.float16, rms=False, add=None, out2=None):
    x2 = x.reshape(-1, x.shape[-1]).float()
    if rms:
        y = x2 * torch.rsqrt(x2.pow(2).mean(-1, keepdim=True) + eps) * gamma
    else:
        y = F.layer_norm(x2, (x2.shape[-1],), gamma, beta, eps)
    if out is None:
        out = torch.empty(x2.shape, dtype=out_dtype)
    out.reshape(-1, x2.shape[-1]).copy_(y.to(out.dtype))
    if add is not None:                                          # second output y + add[row % add_rows]
        y2 = y + add.repeat(-(-x2.shape[0] // add.shape[0]), 1)[: x2.shape[0]]
        out2 = torch.empty(x2.shape, dtype=out.dtype) if out2 is None else out2
        out2.copy_(y2.to(out2.dtype))
        return out, out2
    return out


def attention(q, k, v, out, *, scale, causal=False):
    """[batch, head, seq, d] fp16 views; fp32 softmax; causal = bottom-right aligned like the kernels (query i sees keys <= i + Sk - Sq)"""
    Sq, Sk = q.shape[2], k.shape[2]
    q = q.expand(k.shape[0], -1, -1, -1)                         # shared queries (attention pooling): q batch 1
    s = torch.einsum("bhqd,bhkd->bhqk", q.float(), k.float()) * scale
    if causal:
        mask = torch.arange(Sk)[None, :] > (torch.arange(Sq)[:, None] + (Sk - Sq))
        s = s.masked_fill(mask, float("-inf"))
    o = torch.einsum("bhqk,bhkd->bhqd", s.softmax(-1), v.float())
    out.copy_(o.to(out.dtype))
    return out


def _rows(pt_row, page_size, positions):
    p = torch.as_tensor(positions, dtype=torch.long)
    return pt_row.long()[p // page_size] * page_size + p % page_size


def _rope(x, pos, inv_freq):
    """x [..., H, d]; rotate-half RoPE at integer positions pos [...]"""
    d = x.shape[-1]
    ang = pos.float()[..., None] * inv_freq                      # [..., d/2]
    c, s = ang.cos()[..., None, :], ang.sin()[..., None, :]
    x0, x1 = x[..., : d // 2], x[..., d // 2:]
    return torch.cat([x0 * c - x1 * s, x1 * c + x0 * s], dim=-1)


def rope_kv_prefill(qkv, pos0, heads, head_dim, inv_freq, kcache, vcache, page_table_row=None, page_size=0):
    T, D = qkv.shape[0], heads * head_dim
    pos = torch.arange(pos0, pos0 + T)
    q = _rope(qkv[:, :D].float().view(T, heads, head_dim), pos, inv_freq).reshape(T, D).half()
    k = _rope(qkv[:, D:2 * D].float().view(T, heads, head_dim), pos, inv_freq).reshape(T, D).half()
    qkv[:, :D] = q
    qkv[:, D:2 * D] = k
    assert page_table_row is not None
    rows = _rows(page_table_row, page_size, pos)
    kcache.view(-1, D)[rows] = k
    vcache.view(-1, D)[rows] = qkv[:, 2 * D:]


def embed_rows(table, out, *, ids=None, state=None, seq=None):
    if ids is None:
        ids = torch.stack([seq[b, state[b, 0] - 1] for b in range(state.shape[0])])
    out.reshape(-1, out.shape[-1]).copy_(table[ids.long()].float())
    return out


def gemv(W, x, out, *, rms_w=None, eps=1e-5, residual=None, gated=False):
    x2 = x.reshape(-1, W.shape[1]).float()
    if rms_w is not None:
        x2 = x2 * torch.rsqrt(x2.pow(2).mean(-1, keepdim=True) + eps) * rms_w
    r = _f16(x2) @ W.float().t()                                 # activations are staged as fp16
    if gated:
        r = r[:, 0::2] * F.silu(r[:, 1::2])
    if residual is not None:
        r = r + residual.reshape(r.shape)
    out.reshape(r.shape).copy_(r)
    return out


def decode_attention(qkv, state, inv_freq, kcache, vcache, out, heads, head_dim, page_table=None, page_size=0):
    B, D = qkv.shape[0], heads * head_dim
    assert page_table is not None
    for b in range(B):
        pos = int(state[b, 0]) - 1
        p = torch.tensor(pos)
        q = _rope(qkv[b, :D].view(heads, head_dim), p, inv_freq)
        k = _rope(qkv[b, D:2 * D].view(heads, head_dim), p, inv_freq)
        row = _rows(page_table[b], page_size, [pos])
        kcache.view(-1, D)[row] = k.reshape(1, D).half()
        vcache.view(-1, D)[row] = qkv[b, 2 * D:].reshape(1, D).half()
        rows = _rows(page_table[b], page_size, list(range(pos + 1)))
        K = kcache.view(-1, D)[rows].float().view(pos + 1, heads, head_dim)
        V = vcache.view(-1, D)[rows].float().view(pos + 1, heads, head_dim)
        s = torch.einsum("hd,thd->ht", q, K) * head_dim ** -0.5
        out[b] = torch.einsum("ht,thd->hd", s.softmax(-1), V).reshape(D)
    return out


def store_hidden(x, state, hidden):
    for b in range(hidden.shape[0]):
        row = int(state[b, 0]) - int(state[b, 3]) - 1
        if 0 <= row < hidden.shape[1]:
            hidden[b, row] = x[b]


def logits_argmax(logits, img_ids, seq, state, eos_id, suppress_eos):
    """generation.py:19-31 + greedy argmax + append (restates logits_argmax_kernel; lowest index wins ties)"""
    ids = img_ids.tolist() if img_ids is not None else []
    for b in range(logits.shape[0]):
        n = int(state[b, 0])
        last = int(seq[b, n - 1])
        if last in ids[:-1]:
            nxt = ids[ids.index(last) + 1]
        else:
            if ids:
                logits[b, torch.tensor(ids[1:])] = 0.0
            if suppress_eos and eos_id is not None and 0 <= eos_id < logits.shape[1]:
                logits[b, eos_id] = float("-inf")
            nxt = int(torch.argmax(logits[b]))
        if n < seq.shape[1] and int(state[b, 1]) == 0:              # parked slots (EOS produced / retired by the host) stop moving
            seq[b, n] = nxt
            state[b, 0] = n + 1
            state[b, 2] += 1
            if eos_id is not None and nxt == eos_id and not suppress_eos and int(state[b, 1]) == 0:
                state[b, 1] = state[b, 2]


def nchw_to_nhwc_f16(x, cpad, scale=1.0, out=None):
    """fp32 NCHW [B,C,H,W] -> fp16 NHWC [B,H,W,cpad] (channels C..cpad-1 zero), values scaled"""
    B, C, H, W = x.shape
    if out is None:
        out = torch.zeros((B, H, W, cpad), dtype=torch.float16)
    out[..., :C] = (x.float() * scale).permute(0, 2, 3, 1).to(torch.float16)
    return out


def cfg_euler_step(eps, x, unet_in, branches, guidance, image_guidance, sigma, sigma_next, init_sigma=1.0):
    """restates cfg_euler_kernel: classifier-free-guidance combine (2-way, or 3-way in sigma space: pipeline_stable_diffusion_xl_t2i_edit.py:
    928-950) + Euler step (EulerDiscreteScheduler.step) + scale_model_input for the next step written into channels 0..3 of every branch"""
    B = x.shape[0]
    if eps is None:
        xn = x * init_sigma
    else:
        e = eps.reshape(branches, B, x.shape[2], x.shape[3], 4).permute(0, 1, 4, 2, 3)          # [branch, B, 4, h, w]
        if branches == 2:
            comb = e[0] + guidance * (e[1] - e[0])
        else:
            et, ei, eu = (x - sigma * e[i] for i in range(3))
            c = eu + guidance * (et - ei) + image_guidance * (ei - eu)
            comb = (c - x) / (-sigma)
        x0 = x - sigma * comb
        xn = x + (x - x0) / sigma * (sigma_next - sigma)
    x.copy_(xn)
    s = (xn * (sigma_next ** 2 + 1.0) ** -0.5).permute(0, 2, 3, 1).to(torch.float16)
    for br in range(branches):
        unet_in[br * B:(br + 1) * B, ..., :4] = s
    return x


def avgpool_tokens(x, k):
    n, t, c = x.shape
    return x.float().view(n, t // k, k, c).mean(2).to(x.dtype)


def add_bcast_f16(a, b, out=None):
    a2 = a.reshape(-1, a.shape[-1]).float()
    r = (a2 + b.repeat(a2.shape[0] // b.shape[0], 1)).to(torch.float16)
    if out is None:
        return r
    out.copy_(r)
    return out


# ---- stage 3 (NHWC fp16 feature maps) ---------------------------------------------------------------------------------------------------
def conv2d_nhwc(x, w, out=None, *, taps=3, bias=None, bias_g=None, residual=None, act=ACT_NONE, out_dtype=torch.float16, tile_n=0, alpha=1.0, col_part=None):
    """stride-1 'same' conv; w packed [Cout, taps*taps*Cpad] with k = (kh*taps + kw)*Cpad + c, Cpad = roundup(Cin, 64); bias_g fp32 [N, Cout] per image"""
    n, h, wd, c = x.shape
    cout = w.shape[0]
    cpad = w.shape[1] // (taps * taps)
    w4 = w.float().view(cout, taps, taps, cpad)[..., :c].permute(0, 3, 1, 2)                 # [Cout, Cin, kh, kw]
    y = alpha * F.conv2d(x.float().permute(0, 3, 1, 2), w4, padding=taps // 2)       # epilogue order of seedx_gemm_f16: alpha*acc, then the biases
    if bias is not None:
        y = y + bias[None, :, None, None]
    if bias_g is not None:
        y = y + bias_g[:, :, None, None]
    y = y.permute(0, 2, 3, 1)
    if act == ACT_SILU:
        y = F.silu(y)
    elif act == ACT_GELU:
        y = F.gelu(y)
    if residual is not None:
        y = y + residual.float()
    if out is None:
        out = torch.empty((n, h, wd, cout), dtype=out_dtype)
    out.copy_(y.to(out.dtype))
    _emit_parts(out.view(-1, cout), y.reshape(-1, cout), None, col_part)
    return out


def groupnorm_ws(n, groups, device):
    return torch.empty((1,), dtype=torch.float64)


def groupnorm_nhwc(x1, gamma, beta, eps, *, x2=None, silu=False, groups=32, out=None, raw_out=None, stats_ws=None, part1=None, part2=None):
    x = torch.cat([x1, x2], dim=3) if x2 is not None else x1
    if raw_out is not None:
        raw_out.copy_(x)
    n, h, w, C = x.shape
    if part1 is not None and (x2 is None or part2 is not None) and (h * w) % 32 == 0:
        # statistics from the producers' column partials (seedx_groupnorm_nhwc_from_partials), not from the tensor
        parts = torch.cat([part1.view(-1, x1.shape[3], 2)] + ([part2.view(-1, x2.shape[3], 2)] if x2 is not None else []), dim=1)   # [n*hw/32, C, 2]
        tot = parts.view(n, h * w // 32, groups, C // groups, 2).double().sum(dim=(1, 3))                                                # [n, groups, 2]
        cnt = h * w * (C // groups)
        mean = tot[..., 0] / cnt
        rstd = torch.rsqrt((tot[..., 1] / cnt - mean * mean).clamp_min(0) + eps)
        cpg = C // groups
        xf = x.float().view(n, h * w, groups, cpg)
        y = ((xf - mean[:, None, :, None].float()) * rstd[:, None, :, None].float()).view(n, h, w, C) * gamma + beta
        y = y.permute(0, 3, 1, 2)
    else:
        y = F.group_norm(x.float().permute(0, 3, 1, 2), groups, gamma, beta, eps)
    if silu:
        y = F.silu(y)
    y = y.permute(0, 2, 3, 1).to(torch.float16)
    if out is None:
        return y.contiguous()
    out.copy_(y)
    return out


def im2col_nhwc(x, k, stride, pad_before, ho, wo):
    """rows = output pixels, columns ordered (kh, kw, c); zero fill outside the image"""
    n, h, w, c = x.shape
    pad_after_h = max((ho - 1) * stride + k - pad_before - h, 0)
    pad_after_w = max((wo - 1) * stride + k - pad_before - w, 0)
    xp = F.pad(x.float().permute(0, 3, 1, 2), (pad_before, pad_after_w, pad_before, pad_after_h))
    cols = F.unfold(xp, kernel_size=k, stride=stride)                                         # [n, c*k*k, ho*wo], (c, kh, kw) order
    cols = cols.view(n, c, k * k, ho * wo).permute(0, 3, 2, 1).reshape(n * ho * wo, k * k * c)
    return cols.to(torch.float16)


def upsample2x_nhwc(x):
    return x.repeat_interleave(2, dim=1).repeat_interleave(2, dim=2).contiguous()


def timestep_embedding(t, dim, out):
    half = dim // 2
    f = torch.exp(-9.210340371976184 * torch.arange(half, dtype=torch.float32) / half)
    a = t.float().reshape(-1, 1) * f
    out[:, :half] = torch.cos(a).to(torch.float16)
    out[:, half:dim] = torch.sin(a).to(torch.float16)
    return out


def softmax_rows(x, scale, out=None):
    y = (x.float() * scale).softmax(-1).to(torch.float16)
    if out is None:
        return y
    out.copy_(y)
    return out


def nhwc_to_nchw_f32(x, c, scale=1.0):
    return (x[..., :c].float() * scale).permute(0, 3, 1, 2).contiguous()


def image_to_u8(x):
    v = (x[..., :3].float() * 0.5 + 0.5).clamp(0, 1)
    return torch.round(v * 255.0).to(torch.uint8)
