"""Parity of the non-GEMM kernels against torch fp32 references of the same op (CUDA path through the C ABI)."""
import pytest
import torch
import torch.nn.functional as F
from fp16_ulp import ulp16

pytestmark = pytest.mark.gpu


def rel(a, b):
    return ((a.float() - b.float()).norm() / b.float().norm().clamp_min(1e-12)).item()


def mk(shape, seed, scale=1.0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).cuda()


@pytest.mark.parametrize("B,H,Sq,Sk,D,causal", [
    (2, 16, 1024, 1024, 104, False),   # ViT MHSA
    (2, 2, 256, 256, 104, False),
    (3, 32, 256, 1024, 128, False),    # attn_pool (shared queries)
    (2, 32, 64, 256, 160, False),      # input resampler
    (1, 40, 174, 174, 128, True),      # LLaMA prefill (causal, ragged)
    (1, 4, 370, 370, 128, True),
    (4, 40, 241, 241, 128, True),      # LLaMA prefill of 4 equal-length prompts as one batched call
    (2, 10, 4096, 4096, 64, False),    # UNet self-attention 64x64
    (8, 20, 1024, 1024, 64, False),    # UNet self-attention 32x32 at batch: enough items for the two-tile kernel
    (5, 16, 1024, 1024, 104, False),   # ViT MHSA, 5 views: two-tile kernel, padded head dim
    (2, 20, 1024, 64, 64, False),      # UNet cross-attention: the 64 context tokens are one 64-key wgmma tile
    (8, 10, 4096, 64, 64, False),      # ... at the 64x64 level, bench batch
    (3, 5, 640, 48, 64, False),        # 64-key tile with 16 masked keys, ragged query tiles
    (2, 4, 256, 64, 40, False),        # head dim padded to 64 by TMA zero fill
    (2, 16, 64, 128, 64, False),       # perceiver
    (2, 16, 1, 65, 64, False),         # AttentionPool2d (single query)
    (1, 3, 77, 33, 72, False),
    (2, 8, 64, 16, 64, False),         # the smallest problem of the wgmma kernel: one 64-row half tile, 16 keys of a 64-key tile
    (1, 4, 300, 300, 104, True),       # causal, head dim 104 (two 64-column TMA chunks), ragged query and key tiles
    (2, 3, 1000, 1000, 128, True),     # causal over eight 128-key tiles, ragged last query tile
    (1, 2, 1000, 129, 64, False),      # 128-key tiles with one valid key in the last
    (3, 2, 200, 65, 128, False),       # 65 keys: first size past the 64-key tile
    (1, 1, 64, 4096, 8, False),        # head dim 8 zero-filled to 64
    (2, 6, 4096, 64, 120, False),      # head dim 120, 64-key tile
    (1, 5, 640, 640, 64, True),        # causal at the UNet head dim
    (4, 4, 512, 300, 96, False),       # head dim 96
])
@pytest.mark.parametrize("impl", ["wgmma", "mma_sync"])
def test_attention(B, H, Sq, Sk, D, causal, impl):
    from seedx_b200 import ops
    from seedx_b200._lib import lib
    lib().seedx_attention_set_impl({"wgmma": 0, "mma_sync": 1}[impl])
    shared_q = (Sq == 256 and Sk == 1024)
    q = mk((1 if shared_q else B, Sq, H, D), 1).half()
    k = mk((B, Sk, H, D), 2).half()
    v = mk((B, Sk, H, D), 3).half()
    o = torch.empty((B, Sq, H, D), device="cuda", dtype=torch.float16)
    scale = D ** -0.5
    ops.attention(q.permute(0, 2, 1, 3), k.permute(0, 2, 1, 3), v.permute(0, 2, 1, 3), o.permute(0, 2, 1, 3), scale=scale, causal=causal)
    qf = q.float().expand(B, -1, -1, -1).permute(0, 2, 1, 3)
    used = lib().seedx_attention_last_impl()
    lib().seedx_attention_set_impl(0)
    ref = F.scaled_dot_product_attention(qf, k.float().permute(0, 2, 1, 3), v.float().permute(0, 2, 1, 3), is_causal=causal, scale=scale)
    assert rel(o.permute(0, 2, 1, 3), ref) < 2e-3
    if impl == "wgmma" and Sq >= 64 and Sk >= 16 and D <= 128:
        assert used == 2, "the wgmma kernel should have handled this shape, got %d" % used
    if impl == "mma_sync":
        assert used == 1


@pytest.mark.parametrize("growth", [0.0, 1.5, 6.0])
def test_attention_one_pass_softmax_redo(growth):
    """Keys whose magnitude rises with their index push later key tiles above the running maximum of the online softmax: a little, and by far
    more than 2^8 (fp16 P would be inf if a tile were exponentiated against a stale maximum)."""
    from seedx_b200 import ops
    from seedx_b200._lib import lib
    B, H, S, D = 8, 20, 1024, 64
    q = mk((B, S, H, D), 11).half()
    ramp = (1.0 + growth * torch.arange(S, device="cuda").float() / S).view(1, S, 1, 1)
    k = (mk((B, S, H, D), 12) * ramp).half()
    v = mk((B, S, H, D), 13).half()
    o = torch.empty((B, S, H, D), device="cuda", dtype=torch.float16)
    ops.attention(q.permute(0, 2, 1, 3), k.permute(0, 2, 1, 3), v.permute(0, 2, 1, 3), o.permute(0, 2, 1, 3), scale=D ** -0.5)
    assert lib().seedx_attention_last_impl() == 2
    ref = F.scaled_dot_product_attention(q.float().permute(0, 2, 1, 3), k.float().permute(0, 2, 1, 3), v.float().permute(0, 2, 1, 3), scale=D ** -0.5)
    assert torch.isfinite(o).all()
    assert rel(o.permute(0, 2, 1, 3), ref) < 2e-3


def test_attention_strided_qkv():
    """ViT layout: packed [N,S,heads,3,d] projection output read in place."""
    from seedx_b200 import ops
    N, S, Hh, d = 2, 320, 4, 104
    qkv = mk((N, S, Hh, 3, d), 5).half()
    o = torch.empty((N, S, Hh, d), device="cuda", dtype=torch.float16)
    q, k, v = (qkv[:, :, :, i].permute(0, 2, 1, 3) for i in range(3))
    ops.attention(q, k, v, o.permute(0, 2, 1, 3), scale=d ** -0.5)
    ref = F.scaled_dot_product_attention(q.float(), k.float(), v.float(), scale=d ** -0.5)
    assert rel(o.permute(0, 2, 1, 3), ref) < 2e-3


# seedx_layernorm picks its kernel from the shape (norm.cu, LN_VEC_DISPATCH): rows >= 64 and cols <= 2048 -> the warp-persistent rows kernel
# (NV 4/8/12/16 for cols <= 512/1024/1536/2048); otherwise one warp per row (TPR 32, NV 2/4/8/16 for cols <= 256/512/1024/2048) or one CTA
# per row (TPR 256, NV 4/8 for cols <= 4096/8192).  Unaligned rows or cols % 4 != 0 take the scalar kernel (test_layernorm_scalar_and_mixed_dtypes).
@pytest.mark.parametrize("rows,cols", [
    (2048, 1664),   # rows kernel, NV 16 (ViT width)
    (5, 208),       # TPR 32, NV 2
    (300, 4096),    # TPR 256, NV 4
    (174, 5120),    # TPR 256, NV 8 (LLaMA prefill)
    (64, 1024),     # rows kernel, NV 8
    (7, 8192),      # TPR 256, NV 8 at the widest vectorised row
    (128, 320),     # rows kernel, NV 4
    (96, 1280),     # rows kernel, NV 12
    (33, 320),      # TPR 32, NV 4
    (7, 1024),      # TPR 32, NV 8
    (8, 1664),      # TPR 32, NV 16
])
def test_layernorm_rmsnorm(rows, cols):
    from seedx_b200 import ops
    x = mk((rows, cols), 1, 3.0) + 0.5
    g, b = mk((cols,), 2) + 1.0, mk((cols,), 3)
    ref = F.layer_norm(x, (cols,), g, b, 1e-6)
    assert rel(ops.layernorm(x, g, b, 1e-6, out_dtype=torch.float32), ref) < 1e-5
    assert rel(ops.layernorm(x.half(), g, b, 1e-6, out_dtype=torch.float16), F.layer_norm(x.half().float(), (cols,), g, b, 1e-6)) < 1e-3
    add = mk((rows if rows < 64 else 64, cols), 4) if rows % 64 == 0 or rows < 64 else None
    if add is not None:
        y, y2 = ops.layernorm(x, g, b, 1e-6, out_dtype=torch.float32, add=add)
        assert rel(y, ref) < 1e-5
        assert rel(y2, ref + add.repeat(rows // add.shape[0], 1)) < 1e-5
    rms = x * torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + 1e-5) * g
    assert rel(ops.layernorm(x, g, None, 1e-5, out_dtype=torch.float32, rms=True), rms) < 1e-5


def _ln64(x, g, eps, rms):
    """float64 normalised row times gamma (the bias is added by the caller)"""
    x = x.double()
    if rms:
        return x * torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + eps) * g.double()
    return (x - x.mean(-1, keepdim=True)) * torch.rsqrt(x.var(-1, unbiased=False, keepdim=True) + eps) * g.double()


# fp32 outputs: max |y - ref| / max |ref|.  The statistics are fp32 sums over the row (two passes), rstd one rsqrtf, then (x - mean) rstd g + b
# in fp32, so the error is a few fp32 ulps of the row's scale.
LN_F32_TOL = 6e-7        # worst measured 1.6e-7 on an H100 80GB HBM3 (SXM, 700 W power limit)


@pytest.mark.parametrize("rows,cols,tin,tout,pad,add_rows", [
    (64, 1280, torch.float32, torch.float32, 2, 0),     # scalar: row stride 1282 floats is not a multiple of 4
    (9, 640, torch.float16, torch.float16, 6, 4),       # scalar: row stride 646 halves, add_rows 4 does not divide 9
    (70, 1001, torch.float16, torch.float16, 0, 64),    # scalar: cols % 4 != 0, add_rows 64 does not divide 70
    (3, 1001, torch.float32, torch.float16, 0, 0),      # scalar, fp32 -> fp16
    (5, 1001, torch.float16, torch.float32, 0, 2),      # scalar, fp16 -> fp32
    (100, 1280, torch.float16, torch.float32, 0, 64),   # rows kernel NV 12, fp16 -> fp32, add_rows 64 does not divide 100
    (200, 320, torch.float32, torch.float16, 0, 0),     # rows kernel NV 4, fp32 -> fp16
    (10, 2048, torch.float32, torch.float16, 0, 4),     # TPR 32 NV 16, fp32 -> fp16, add_rows 4 does not divide 10
    (6, 5120, torch.float16, torch.float32, 0, 4),      # TPR 256 NV 8 (LLaMA final norm), fp16 -> fp32, add_rows 4 does not divide 6
])
def test_layernorm_scalar_and_mixed_dtypes(rows, cols, tin, tout, pad, add_rows, record_property):
    """LayerNorm and RMSNorm through the calls the shape-only cases above do not make: strided and unaligned rows, cols % 4 != 0, mixed input
    and output dtypes, and the second output y + add[row % add_rows] with add_rows not dividing rows, all against float64.
    fp16 outputs must be within 1 fp16 ulp of the float64 result: they are rounded once from an fp32 value within half an ulp plus its fp32
    error, and that error, bounded here by (|x_hat g| + |b| + |add|) 2^-19, only matters where y cancels to within a few thousandths of 0."""
    from seedx_b200 import ops
    g = torch.Generator(device="cpu").manual_seed(rows * cols)
    full = (torch.randn((rows, cols + pad), generator=g) * 3 + 0.5).to(tin)
    x = full.cuda()[:, :cols]
    gam, bet = torch.randn(cols, generator=g) + 1.0, torch.randn(cols, generator=g)
    add = torch.randn((add_rows, cols), generator=g) if add_rows else None
    worst_f32 = worst_ulps = 0.0
    for rms in (False, True):
        xg = _ln64(full[:, :cols], gam, 1e-6, rms)
        b = torch.zeros(cols, dtype=torch.float64) if rms else bet.double()
        refs = [(xg + b, xg.abs() + b.abs())]
        if add_rows:
            a = add.double().repeat(rows // add_rows + 1, 1)[:rows]
            refs.append((xg + b + a, xg.abs() + b.abs() + a.abs()))
        got = ops.layernorm(x, gam.cuda(), None if rms else bet.cuda(), 1e-6, out_dtype=tout, rms=rms, add=add.cuda() if add_rows else None)
        for y, (r, mag) in zip(got if add_rows else (got,), refs):
            assert y.dtype == tout
            d = (y.cpu().double() - r).abs()
            assert torch.isfinite(y).all()
            if tout == torch.float16:
                worst_ulps = max(worst_ulps, (d / ulp16(r)).max().item())
                assert (d <= ulp16(r) + mag * 2.0 ** -19).all(), (d / ulp16(r)).max().item()
            else:
                worst_f32 = max(worst_f32, (d.max() / r.abs().max()).item())
                assert (d <= LN_F32_TOL * r.abs().max()).all(), (d.max() / r.abs().max()).item()
    record_property("fp16_out_ulps", worst_ulps)
    record_property("fp32_out_err", worst_f32)


@pytest.mark.parametrize("n,h,w,c1,c2,silu", [(2, 32, 32, 320, 0, True), (2, 16, 16, 1280, 640, True), (1, 64, 64, 640, 320, False),
                                              (3, 8, 8, 128, 0, True), (1, 128, 128, 320, 0, True)])
def test_groupnorm(n, h, w, c1, c2, silu):
    from seedx_b200 import ops
    x1 = (mk((n, h, w, c1), 1, 2.0) + 0.3).half()
    x2 = (mk((n, h, w, c2), 2, 0.5) - 1.0).half() if c2 else None
    C = c1 + c2
    g, b = mk((C,), 3) + 1.0, mk((C,), 4)
    xc = torch.cat([x1, x2], dim=3) if c2 else x1
    ref = F.group_norm(xc.float().permute(0, 3, 1, 2), 32, g, b, 1e-5)
    if silu:
        ref = F.silu(ref)
    ref = ref.permute(0, 2, 3, 1)
    raw = torch.empty_like(xc) if c2 else None
    out = ops.groupnorm_nhwc(x1, g, b, 1e-5, x2=x2, silu=silu, raw_out=raw)
    assert rel(out, ref) < 2e-3
    if c2:
        assert torch.equal(raw, xc)


@pytest.mark.parametrize("n,h,w,c1,c2", [(2, 32, 32, 320, 0), (2, 16, 16, 1280, 640), (1, 64, 64, 640, 320), (3, 8, 8, 128, 0), (8, 32, 32, 1280, 1280)])
def test_groupnorm_from_epilogue_partials(n, h, w, c1, c2):
    """GroupNorm whose statistics come from the column partials emitted by the producing conv / GEMM epilogues (no pass over the tensor): the 3x3 conv
    that produces x1 (and a 1x1 GEMM that produces the skip x2) write col_part; the finalize over the partials is bit-reproducible and the result
    matches torch GroupNorm(+SiLU) of the stored fp16 tensors, including groups that straddle the x1 | x2 boundary (C/32 = 60 channels per group)"""
    from seedx_b200 import ops
    xin = mk((n, h, w, 64), 21).half()
    w1 = mk((c1, 9 * 64), 22, (9 * 64) ** -0.5).half()
    p1 = torch.empty((n * h * w // 32, c1, 2), device="cuda")
    x1 = ops.conv2d_nhwc(xin, w1, bias=mk((c1,), 23), col_part=p1)
    x2 = p2 = None
    if c2:
        w2 = mk((c2, 64), 24, 0.2).half()
        p2 = torch.empty((n * h * w // 32, c2, 2), device="cuda")
        x2 = ops.gemm(xin.view(-1, 64), w2, bias=mk((c2,), 25) - 0.5, col_part=p2).view(n, h, w, c2)
    C = c1 + c2
    g, b = mk((C,), 3) + 1.0, mk((C,), 4)
    xc = torch.cat([x1, x2], dim=3) if c2 else x1
    ref = F.silu(F.group_norm(xc.float().permute(0, 3, 1, 2), 32, g, b, 1e-5)).permute(0, 2, 3, 1)
    out = ops.groupnorm_nhwc(x1, g, b, 1e-5, x2=x2, silu=True, part1=p1, part2=p2).clone()
    assert rel(out, ref) < 2e-3
    plain = ops.groupnorm_nhwc(x1, g, b, 1e-5, x2=x2, silu=True)          # statistics pass over the tensor
    assert rel(out, plain) < 1e-3
    for _ in range(2):
        assert torch.equal(ops.groupnorm_nhwc(x1, g, b, 1e-5, x2=x2, silu=True, part1=p1, part2=p2), out)


def test_patchify_cast_pool():
    from seedx_b200 import ops
    x = mk((2, 3, 56, 42), 1)
    p = ops.patchify(x, 14, 592)
    ref = F.unfold(x, kernel_size=14, stride=14).transpose(1, 2).reshape(-1, 588)
    assert torch.equal(p[:, :588], ref.half()) and (p[:, 588:] == 0).all()
    assert torch.equal(ops.cast(x, torch.float16), x.half())
    t = mk((3, 256, 128), 2).half()
    assert rel(ops.avgpool_tokens(t, 4), F.avg_pool1d(t.float().transpose(1, 2), 4, 4).transpose(1, 2)) < 1e-3


def test_groupnorm_is_bitwise_reproducible():
    """The statistics are reduced in a fixed order (no floating-point atomics): repeated calls give identical bits, also when the
    allocator hands back recycled, dirty scratch memory."""
    from seedx_b200 import ops
    x = mk((2, 64, 64, 320), 11).half()
    g, b = mk((320,), 12), mk((320,), 13)
    a = ops.groupnorm_nhwc(x, g, b, 1e-5, silu=True).clone()
    junk = [torch.full((1 << 20,), float(i + 3), device="cuda") for i in range(32)]
    del junk
    for _ in range(3):
        assert torch.equal(ops.groupnorm_nhwc(x, g, b, 1e-5, silu=True), a)
    ref = F.silu(F.group_norm(x.float().permute(0, 3, 1, 2), 32, g, b, 1e-5)).permute(0, 2, 3, 1)
    assert rel(a, ref) < 2e-3


def test_programmatic_dependent_launch_does_not_change_results():
    """Every kernel waits (griddepcontrol.wait) before its first dependent access: a chain of dependent launches gives the same bits with
    the programmatic-stream-serialization attribute on and off."""
    from seedx_b200 import ops
    from seedx_b200._lib import lib
    x = mk((1024, 1280), 21).half()
    w1, w2 = mk((2560, 1280), 22, 0.03).half(), mk((1280, 1280), 23, 0.03).half()
    gam, bet = mk((1280,), 24), mk((1280,), 25)

    def chain():
        h = x.clone()
        for _ in range(6):
            n = ops.layernorm(h, gam, bet, 1e-5)
            u = ops.gemm(n, w1, act=ops.ACT_GELU, gated=True)
            ops.gemm(u, w2, out=h, residual=h)
        return h.clone()

    try:
        lib().seedx_set_pdl(1)
        a = chain()
        lib().seedx_set_pdl(0)
        b = chain()
    finally:
        lib().seedx_set_pdl(1)
    assert torch.isfinite(a.float()).all()
    assert torch.equal(a, b)
