"""FP8 (e4m3) UNet transformer projections on the GPU: seedx_quant_rows_fp8 bit for bit against llm.quantize_fp8_rows, seedx_gemm_fp8 bit for
bit on an integer grid (every FP8 tile width, ragged shapes, every epilogue the UNet uses, TMA / vector / scalar stores), its rejections, and
`UNet2DConditionModel(weight_format="fp8_e4m3")` against the fp16 UNet and, at tiny size, against its CPU restatement (test_fp8_unet_cpu.py),
under the CUDA graph and after a partial checkpoint.

Why the GEMM is exact: the e4m3 operands are integers (every one exactly representable in e4m3) and the scales are powers of two, so
(acc * a_scale) * b_scale only moves the exponent.  The FP8 wgmma does NOT accumulate in full fp32: measured on an H100, integer sums past about
2^13 lose their low bits (K = 5120 with |q| <= 16 differed; K <= 1296 did not), as reported for FP8 tensor cores of this generation.  So the
operand range shrinks with K: |q| <= sqrt(4096 / K) (at least 1), which keeps every partial sum within 2^12 in the worst case up to K = 4096
and, for random signs, far below it at K = 5120.  Biases and residuals on a 1/64 grid keep the linear epilogue exact: an fp32 output
equals the float64 reference bit for bit, an fp16 output equals it rounded once.  Outputs are views cut out of NaN-sentinel buffers and every
input gap holds NaN (e4m3 0x7F in the operands), as in test_gemm_exact_gpu.py, whose helpers this file uses."""
import ctypes as C

import pytest
import torch

from fp16_ulp import ulp16
from seedx_b200 import synth
from seedx_b200.llm import quantize_fp8_rows
from test_gemm_exact_gpu import (F16, F32, U32, OutBuf, act_ref_and_bound, assert_exact, check_col_part, check_ln_epilogue, grid, last_config, lib,
                                 nan_tail, padded, r32, stats_from_parts, to_out)

pytestmark = pytest.mark.gpu
E4 = torch.float8_e4m3fn
FP8_TILES = [64, 128, 160, 192, 224, 256]


def rel(a, b):
    return ((a.float().cpu() - b.float().cpu()).norm() / b.float().cpu().norm()).item()


def padded8(vals, ld):
    """device e4m3 copy of vals [R, C] (exact e4m3 values) with row stride ld; every gap byte, and one row after the end, is NaN (0x7F)"""
    R, Cc = vals.shape
    buf = torch.full((R * ld + ld,), 0x7F, dtype=torch.uint8, device="cuda").view(E4)
    view = buf.as_strided((R, Cc), (ld, 1), 0)
    q = vals.to(E4)
    assert torch.equal(q.double(), vals), "operand not exactly representable in e4m3"
    view.copy_(q.cuda())
    return view


def pow2_scales(n, seed):
    g = torch.Generator().manual_seed(seed)
    return nan_tail(torch.pow(2.0, torch.randint(-6, 4, (n,), generator=g).double()))


def fp8_lim(K):
    return max(1, min(16, int((4096 / K) ** 0.5)))


def fp8_operands(M, N, K, seed):
    lim = fp8_lim(K)
    a64, w64 = grid((M, K), seed, 1, lim), grid((N, K), seed + 1, 1, lim)     # integers |q| <= lim
    a, w = padded8(a64, K + 16), padded8(w64, K + 32)
    sa, sw = pow2_scales(M, seed + 2), pow2_scales(N, seed + 3)
    acc = (a64.cuda() * sa.double()[:, None]) @ (w64.cuda() * sw.double()[:, None]).t()       # exact
    return a, w, sa, sw, acc


# ---------------------------------------------------------------------------------------------------------------------------------------------
# quantiser
# ---------------------------------------------------------------------------------------------------------------------------------------------
def _quant_rows():
    g = torch.Generator().manual_seed(7)
    x = torch.randn((70, 1000), generator=g) * torch.logspace(-4, 2, 70)[:, None]
    x[3] = 0.0                                                          # all-zero row: scale 1, q = 0
    x[4, :] = 0.0
    x[4, 17] = -1e-6                                                    # a single fp16-subnormal-sized value
    x[5, ::3] = 65504.0                                                 # the fp16 extremes
    x[5, 1::3] = -65504.0
    x[6] = torch.linspace(-1, 1, 1000) * 2.0 ** -6                      # with 448 below: x / s in e4m3's subnormal range (< 2^-6)
    x[6, 0] = 448.0
    x[7, 999] = 1e4                                                      # the row maximum in the tail past the last 16-byte vector
    return x.half()


@pytest.mark.parametrize("cols,ldx", [(1000, 1000), (1000, 1048), (37, 40), (5120, 5120), (640, 656), (16, 16)])
def test_quant_rows_fp8_bit_exact(cols, ldx):
    from seedx_b200 import ops
    x16 = _quant_rows()
    x16 = torch.cat([x16] * (1 + cols // 1000), dim=1)[:, :cols].contiguous() if cols != 1000 else x16
    buf = torch.full((x16.shape[0], ldx), float("nan"), dtype=F16, device="cuda")    # NaN in the row gaps
    x = buf[:, :cols]
    x.copy_(x16.cuda())
    q, s = ops.quant_rows_fp8(x)
    q_ref, s_ref = quantize_fp8_rows(x16.float())
    torch.cuda.synchronize()
    assert torch.equal(s.cpu(), s_ref)
    assert torch.equal(q.cpu().view(torch.uint8), q_ref.view(torch.uint8))
    assert float(s[3]) == 1.0 and not bool(torch.isnan(q.float()).any())


# ---------------------------------------------------------------------------------------------------------------------------------------------
# GEMM: tiles and edges
# ---------------------------------------------------------------------------------------------------------------------------------------------
FP8_SHAPES = [
    (1, 24, 16),         # one row; N below one 32-column chunk; one stage only 16 deep (the rest is TMA zero fill)
    (127, 200, 144),     # one m-block one row short; ragged last chunk (200 = 6 x 32 + 8); K = 128 + 16
    (129, 330, 1296),    # the second m-block holds one row; 11 stages, the last 16 deep
    (300, 1000, 5120),   # ff.net.2's K at C = 1280
    (8192, 264, 1280),   # the UNet's M at 32x32 latents x 8 samples; the last tile narrower than one chunk for several widths
]


@pytest.mark.parametrize("M,N,K", FP8_SHAPES)
@pytest.mark.parametrize("tile_n", FP8_TILES)
@pytest.mark.parametrize("dt", [F32, F16], ids=["f32", "f16"])
def test_gemm_fp8_exact_tiles_and_edges(M, N, K, tile_n, dt):
    from seedx_b200 import ops
    a, w, sa, sw, acc = fp8_operands(M, N, K, seed=M + N + K)
    bias = nan_tail(grid((N,), 5, 64, 64, nonzero=True))
    ob = OutBuf((M, N), dt, (N + 7) // 8 * 8 + 8)
    ops.gemm(a, w, out=ob.view, bias=bias, a_scale=sa, w_scale=sw, tile_n=tile_n)
    cfg = last_config()
    torch.cuda.synchronize()
    ob.check_outside()
    assert_exact(ob.view, to_out(acc + bias.double(), dt), f"M={M} N={N} K={K} tile={tile_n}")
    assert (cfg["tile"], cfg["cluster"], cfg["stream_k"]) == (tile_n, 1, 0)


def test_gemm_fp8_auto_tile_is_single_cta_data_parallel():
    """auto mode (tile_n = 0) with cluster pairs and stream-K forced for fp16: the FP8 GEMM still runs one CTA per tile, data-parallel"""
    from seedx_b200 import ops
    M, N, K = 8192, 1280, 5120
    a, w, sa, sw, acc = fp8_operands(M, N, K, seed=3)
    lib().seedx_gemm_set_cluster(2)
    lib().seedx_gemm_set_stream_k(2)
    try:
        out = ops.gemm(a, w, a_scale=sa, w_scale=sw, out_dtype=F32)
        cfg = last_config()
    finally:
        lib().seedx_gemm_set_cluster(1)
        lib().seedx_gemm_set_stream_k(1)
    assert cfg["tile"] in (128, 160, 192, 224, 256) and cfg["cluster"] == 1 and cfg["stream_k"] == 0
    assert_exact(out, acc.float(), "auto tile")


# ---------------------------------------------------------------------------------------------------------------------------------------------
# GEMM: the epilogues the UNet runs, through every store path
# ---------------------------------------------------------------------------------------------------------------------------------------------
@pytest.fixture
def store_mode():
    yield lambda s: lib().seedx_gemm_set_tma_epilogue(0 if s == "vector" else 1)
    lib().seedx_gemm_set_tma_epilogue(1)


@pytest.mark.parametrize("store", ["tma", "vector", "scalar"])
@pytest.mark.parametrize("tile_n", [128, 256])
@pytest.mark.parametrize("case", ["bias_residual", "gated_plain", "alpha"])
def test_gemm_fp8_exact_epilogues(case, tile_n, store, store_mode):
    """bias + fp16 residual (attn1.to_out, attn2.to_out, ff.net.2, proj_out), the gated product with ACT_NONE (exact: one fp32 rounding, restated),
    alpha; fp16 output.  TMA: 16-byte aligned rows; vector: the TMA epilogue switched off; scalar: rows that do not start 16-byte aligned"""
    from seedx_b200 import ops
    M, N, K = 300, 392, 1296
    gated = case == "gated_plain"
    n_out = N // 2 if gated else N
    a, w, sa, sw, acc = fp8_operands(M, N, K, seed=17)
    bias = nan_tail(grid((N,), 6, 64, 64, nonzero=True))
    aligned = store != "scalar"
    ob = OutBuf((M, n_out), F16, (n_out + 7) // 8 * 8 + (8 if aligned else 9))
    kw = dict(bias=bias, a_scale=sa, w_scale=sw, tile_n=tile_n)
    x = r32(acc + bias.double())                                     # fma(acc, alpha, bias): the exact sum rounded once
    if case == "bias_residual":
        r64 = grid((M, n_out), 8, 64, 64)
        kw["residual"] = padded(r64, (n_out + 7) // 8 * 8 + (16 if aligned else 17), F16)
        want = r32(x + r64.cuda())
    elif gated:
        kw["gated"] = True
        want = r32(x[:, 0::2] * x[:, 1::2])
    else:
        kw["alpha"] = 0.5
        want = 0.5 * acc + bias.double()
    store_mode(store)
    ops.gemm(a, w, out=ob.view, **kw)
    cfg = last_config()
    torch.cuda.synchronize()
    ob.check_outside()
    assert_exact(ob.view, want.float().half(), f"{case} {store}")
    tma_ok = store == "tma" and not gated
    assert (cfg["tile"], cfg["cluster"], cfg["tma"]) == (tile_n, 1, int(tma_ok))
    assert cfg["vec"] == int(aligned)


def test_gemm_fp8_geglu_bounds():
    """GEGLU (ff.net.0): x[2j] * gelu(x[2j+1]) on the exact scaled accumulator, bounded elementwise like test_gemm_activation_bounds"""
    from seedx_b200 import ops
    M, N, K = 300, 640, 256
    a64, w64 = grid((M, K), 23, 1, 4), grid((N, K), 24, 1, 4)
    a, w = padded8(a64, K + 16), padded8(w64, K + 32)
    # fixed scales 2^-3, 2^-3: acc on a 2^-6 grid, so acc + bias (1/64 grid) is exact in fp32; pre-activations over about [-16, 16]
    sa, sw = nan_tail(torch.full((M,), 2.0 ** -3)), nan_tail(torch.full((N,), 2.0 ** -3))
    acc = (a64 @ w64.t()).cuda() * 2.0 ** -6
    bias = nan_tail(grid((N,), 9, 64, 64, nonzero=True))
    out = ops.gemm(a, w, bias=bias, act=1, gated=True, a_scale=sa, w_scale=sw, tile_n=128)
    x = acc + bias.double()
    g, bnd_g = act_ref_and_bound(x[:, 1::2], 1)
    v = x[:, 0::2]
    y = v * g
    bound = v.abs() * bnd_g + U32 * y.abs() + ulp16(y)
    err = (out.double() - y).abs()
    assert float((err / bound.clamp_min(1e-30)).max()) <= 1.0


def test_gemm_fp8_folded_layernorm_and_statistics():
    """the folded LayerNorm in both forms, with the statistics an FP8 producer writes (residual + row_part + row_stats, as attn1.to_out,
    attn2.to_out and ff.net.2 do), and col_part (proj_out), each against float64"""
    from seedx_b200 import ops
    M, K, N, eps = 256, 1024, 384, 1e-5
    # --- producer: FP8 GEMM with an fp16 residual, row partials and the in-epilogue row finalize
    a0, w0, sa0, sw0, acc0 = fp8_operands(M, K, 512, seed=41)
    b0 = nan_tail(grid((K,), 42, 8, 64, nonzero=True))
    r0 = grid((M, K), 43, 64, 64)
    res = padded(r0, K + 16, F16)
    rp = torch.full((K // 32, M, 2), float("nan"), device="cuda")
    st_epi = torch.full((M, 2), float("nan"), device="cuda")
    tickets = torch.zeros((M // 32,), device="cuda", dtype=torch.int32)
    xp = ops.gemm(a0, w0, bias=b0, residual=res, a_scale=sa0, w_scale=sw0, row_part=rp, row_stats=(st_epi, tickets, eps))
    assert last_config()["tma"] == 1 and int(tickets.abs().sum()) == 0
    xpre = r32(r32(acc0 + b0.double()) + r0.cuda())
    assert torch.equal(xp, xpre.float().half())
    v = xpre.view(M, K // 32, 32)
    e1 = (rp[..., 0].t().double() - v.sum(-1)).abs()
    assert bool((e1 <= 31 * U32 * v.abs().sum(-1)).all())
    mean, rstd, dmean, drstd = stats_from_parts(rp, K, eps)
    assert bool(((st_epi[:, 0].double() - mean).abs() <= dmean).all()) and bool(((st_epi[:, 1].double() - rstd).abs() <= drstd).all())
    # --- consumers: grid operands (exact scaled accumulator) with the producer's statistics; colsum8 of the dequantized weights
    qa, w8, sa, sw, acc = fp8_operands(M, N, K, seed=44)          # K = 1024: |q| <= 2
    w64 = w8.double()
    colsum8 = nan_tail(w64.sum(1) * sw.double())
    bias = nan_tail(grid((N,), 46, 64, 64, nonzero=True))
    assert torch.equal(r32(acc), acc), "scaled accumulator not exact in fp32"
    zero = torch.zeros(M, dtype=torch.float64, device="cuda")
    for ln, st, dm, dr in (((st_epi, colsum8), st_epi, zero, zero), ((rp, colsum8, eps), None, dmean, drstd)):
        out = OutBuf((M, N), F32, N + 8)
        ops.gemm(qa, w8, out=out.view, bias=bias, ln=ln, a_scale=sa, w_scale=sw)
        torch.cuda.synchronize()
        out.check_outside()
        m_, r_ = (st[:, 0].double(), st[:, 1].double()) if st is not None else (mean, rstd)
        check_ln_epilogue(out.view, acc, m_, r_, dm, dr, colsum8, bias)
    # --- col_part of an FP8 GEMM's fp16 output (the GroupNorm that reads proj_out's result)
    cp = torch.full((M // 32, N, 2), float("nan"), device="cuda")
    y = ops.gemm(qa, w8, bias=bias, a_scale=sa, w_scale=sw, col_part=cp)
    assert last_config()["tma"] == 1
    check_col_part(cp, y)


# ---------------------------------------------------------------------------------------------------------------------------------------------
# rejections
# ---------------------------------------------------------------------------------------------------------------------------------------------
def _args(a, w, out, **kw):
    from seedx_b200._lib import GemmArgs
    g = GemmArgs()
    g.A, g.B, g.D = a.data_ptr(), w.data_ptr(), out.data_ptr()
    g.M, g.N, g.K, g.batch = a.shape[0], w.shape[0], a.shape[1], 1
    g.lda, g.ldb, g.ldd = a.stride(0), w.stride(0), out.stride(0)
    g.alpha, g.out_dtype = 1.0, 1
    for k, v in kw.items():
        setattr(g, k, v)
    return g


@pytest.mark.parametrize("case", ["conv", "batch2", "no_a_scale", "no_b_scale", "tile96", "tile240"])
def test_gemm_fp8_rejections_launch_nothing(case):
    a = torch.zeros((256, 128), dtype=torch.uint8, device="cuda")
    w = torch.zeros((128, 128), dtype=torch.uint8, device="cuda")
    out = torch.zeros((256, 128), dtype=F16, device="cuda")
    sa, sw = torch.ones(256, device="cuda"), torch.ones(128, device="cuda")
    kw = dict(conv=dict(conv_taps_h=3, conv_taps_w=3, conv_n=1, conv_h=16, conv_w=16, conv_c=128), batch2=dict(batch=2, strideA=256 * 128,
              strideD=256 * 128), tile96=dict(tile_n=96), tile240=dict(tile_n=240)).get(case, {})
    g = _args(a, w, out, **{k: v for k, v in kw.items()})
    pa = None if case == "no_a_scale" else C.c_void_p(sa.data_ptr())
    pb = None if case == "no_b_scale" else C.c_void_p(sw.data_ptr())
    torch.cuda.synchronize()
    n0 = lib().seedx_launch_count()
    rc = lib().seedx_gemm_fp8(C.byref(g), pa, pb, None)
    assert rc != 0 and b"seedx_gemm_fp8" in lib().seedx_last_error()
    assert lib().seedx_launch_count() == n0
    torch.cuda.synchronize()
    assert int(out.abs().sum()) == 0


# ---------------------------------------------------------------------------------------------------------------------------------------------
# UNet
# ---------------------------------------------------------------------------------------------------------------------------------------------
def _tiny_inputs(B, in_ch=4, hw=32):
    cfg = synth.TINY_UNET
    x = synth.randn("g8_x", (B, in_ch, hw, hw))
    ctx = synth.randn("g8_ctx", (B, 16, cfg["cross_attention_dim"]))
    te = synth.randn("g8_te", (B, cfg["text_embed_dim"]))
    tid = torch.tensor([[1024.0, 1024.0, 0.0, 0.0, 1024.0, 1024.0]]).repeat(B, 1)
    return x.cuda(), ctx.cuda(), dict(text_embeds=te.cuda(), time_ids=tid.cuda())


def test_tiny_unet_fp8_matches_the_cpu_restatement_and_tracks_fp16():
    """the tiny UNet in FP8 on the device against the same host over the CPU restatements of the two FP8 entry points (test_fp8_unet_cpu.py),
    and against the fp16 UNet on the device"""
    import test_fp8_unet_cpu as hostfp8
    from seedx_b200 import sdxl as sdxl_mod
    from seedx_b200.sdxl import UNet2DConditionModel
    cfg = synth.TINY_UNET
    sd = synth.unet_state_dict(cfg)
    x, ctx, added = _tiny_inputs(2)
    m16, m8 = UNet2DConditionModel(cfg), UNet2DConditionModel(cfg, weight_format="fp8_e4m3")
    m16.load_state_dict(sd), m8.load_state_dict(sd)
    e16, e8 = m16(x, 601.0, ctx, added_cond_kwargs=added), m8(x, 601.0, ctx, added_cond_kwargs=added)
    real_ops = sdxl_mod.ops
    sdxl_mod.ops = hostfp8.fake_ops_fp8
    try:
        mc = UNet2DConditionModel(cfg, device="cpu", weight_format="fp8_e4m3")
        mc.load_state_dict(sd)
        ec = mc(x.cpu(), 601.0, ctx.cpu(), added_cond_kwargs={k: v.cpu() for k, v in added.items()})
    finally:
        sdxl_mod.ops = real_ops
    e_host, e_16 = rel(e8, ec), rel(e8, e16)
    print(f"tiny UNet FP8: eps rel vs CPU restatement {e_host:.3e}, vs fp16 UNet {e_16:.3e}")
    # measured on an H100 80GB HBM3 (700 W): 0.024 vs the restatement (whose fp32 sums are exact where the FP8 MMA's are not, and whose fp16
    # activations round differently, moving later quantisation points by one e4m3 step), 0.026 vs fp16; bounds ~3x
    assert e_host < 0.08 and 1e-4 < e_16 < 0.08, (e_host, e_16)


@pytest.mark.parametrize("graph", [True])
def test_fp8_t2i_walk_under_the_cuda_graph(graph):
    """4 Euler steps of the 2-way CFG loop with the FP8 UNet replayed as a CUDA graph: latents near the fp16 walk, a second request through the
    same graph bitwise repeatable, and a partial checkpoint loaded after capture (attn2.to_k / to_v, ff.net.2) replays exactly what a freshly
    built FP8 UNet with the merged weights computes"""
    from seedx_b200.sampler import DenoiseLoop
    from seedx_b200.sdxl import EulerDiscreteScheduler, UNet2DConditionModel
    cfg = synth.TINY_UNET
    sd = synth.unet_state_dict(cfg)
    B, hw, steps = 1, 32, 4
    noise = synth.randn("g8_noise", (B, 4, hw, hw)).cuda()
    p, n = synth.randn("g8_p", (B, 16, cfg["cross_attention_dim"])), synth.randn("g8_n", (B, 16, cfg["cross_attention_dim"]))
    pp, npool = synth.randn("g8_pp", (B, cfg["text_embed_dim"])), synth.randn("g8_np", (B, cfg["text_embed_dim"]))
    tid = torch.tensor([[1024.0, 1024.0, 0.0, 0.0, 1024.0, 1024.0]]).repeat(2 * B, 1).cuda()

    def walk(unet):
        loop = DenoiseLoop(unet, EulerDiscreteScheduler(), B, (hw, hw), 2, use_graph=graph)
        loop.set_condition(torch.cat([n, p]).cuda(), torch.cat([npool, pp]).cuda(), tid)
        return loop, loop.run(noise, steps=steps, guidance=7.5).clone()
    u16, u8 = UNet2DConditionModel(cfg), UNet2DConditionModel(cfg, weight_format="fp8_e4m3")
    u16.load_state_dict(sd), u8.load_state_dict(sd)
    _, lat16 = walk(u16)
    loop8, lat8 = walk(u8)
    assert loop8.graph is not None
    e = rel(lat8, lat16)
    print(f"tiny t2i walk, FP8 vs fp16 UNet: latents rel = {e:.3e}")
    # measured on an H100 80GB HBM3 (700 W): 0.064; bound ~3x
    assert 1e-5 < e < 0.2, e
    assert torch.equal(loop8.run(noise, steps=steps, guidance=7.5), lat8)
    part = {k: synth.randn("g8ft:" + k, v.shape, v.shape[-1] ** -0.5)
            for k, v in sd.items() if k.endswith(("attn2.to_k.weight", "attn2.to_v.weight", "ff.net.2.weight"))}
    g0 = loop8.graph
    u8.load_state_dict(part)
    loop8.set_condition(torch.cat([n, p]).cuda(), torch.cat([npool, pp]).cuda(), tid)          # the hoisted K/V of the new to_k / to_v
    got = loop8.run(noise, steps=steps, guidance=7.5).clone()
    assert loop8.graph is g0
    fresh = UNet2DConditionModel(cfg, weight_format="fp8_e4m3")
    fresh.load_state_dict({**sd, **part})
    _, want = walk(fresh)
    assert torch.equal(got, want)


def test_fp8_edit_loop_runs():
    """the 3-branch edit loop (8-channel conv_in) with the FP8 UNet under the CUDA graph"""
    from seedx_b200.sampler import DenoiseLoop
    from seedx_b200.sdxl import EulerDiscreteScheduler, UNet2DConditionModel
    cfg = dict(synth.TINY_UNET, in_channels=8)
    sd = synth.unet_state_dict(cfg)
    B, hw = 1, 32
    u16, u8 = UNet2DConditionModel(cfg), UNet2DConditionModel(cfg, weight_format="fp8_e4m3")
    u16.load_state_dict(sd), u8.load_state_dict(sd)
    noise = synth.randn("g8e_noise", (B, 4, hw, hw)).cuda()
    il = synth.randn("g8e_il", (B, 4, hw, hw), 0.7).cuda()
    p, n = synth.randn("g8e_p", (B, 16, cfg["cross_attention_dim"])), synth.randn("g8e_n", (B, 16, cfg["cross_attention_dim"]))
    pp, npool = synth.randn("g8e_pp", (B, cfg["text_embed_dim"])), synth.randn("g8e_np", (B, cfg["text_embed_dim"]))
    tid = torch.tensor([[1024.0, 1024.0, 0.0, 0.0, 1024.0, 1024.0]]).repeat(3 * B, 1).cuda()
    lats = []
    for u in (u16, u8):
        loop = DenoiseLoop(u, EulerDiscreteScheduler(), B, (hw, hw), 3, use_graph=True)
        loop.set_condition(torch.cat([p, n, n]).cuda(), torch.cat([pp, npool, npool]).cuda(), tid, image_latents=il)
        lats.append(loop.run(noise, steps=4, guidance=7.5, image_guidance=1.5).clone())
    e = rel(lats[1], lats[0])
    print(f"tiny edit walk, FP8 vs fp16 UNet: latents rel = {e:.3e}")
    assert torch.isfinite(lats[1]).all() and e < 0.2, e        # measured on an H100 80GB HBM3 (700 W): 0.068; bound ~3x


def test_engine_passes_the_unet_weight_format():
    from seedx_b200.engine import SeedXEngine
    small = dict(vit_cfg=dict(width=208, layers=2, heads=2, mlp_width=520, output_dim=256, n_queries=256, patch=14), llm_cfg=synth.TINY_LLAMA,
                 unet_cfg=dict(synth.TINY_UNET, cross_attention_dim=256, text_embed_dim=160), vae_cfg=synth.TINY_VAE,
                 rxl_cfg=dict(synth.TINY_RESAMPLER_XL, embedding_dim=256, output1_dim=96, output2_dim=160))
    for edit in (False, True):
        eng = SeedXEngine(**small, edit=edit, unet_weight_format="fp8_e4m3")
        u = eng.adapter.unet
        assert u.weight_format == "fp8_e4m3" and all(t.fp8_slots() for t in u.transformers())
        del eng
        torch.cuda.empty_cache()


# ---------------------------------------------------------------------------------------------------------------------------------------------
# full size
# ---------------------------------------------------------------------------------------------------------------------------------------------
def test_unet_full_size_fp8_sample_forward():
    """one SDXL UNet sample-forward at BASELINE dimensions in FP8 against the fp16 UNet on the same weights (and the fp16 UNet against the CPU
    oracle is test_fullsize_oracle_gpu.py).  e4m3 rounds each operand to 2^-4; a few percent on eps is FP8 itself, more than 10 % would be a
    scale or permutation bug."""
    from seedx_b200.sdxl import SDXL_UNET, UNet2DConditionModel
    cfg = dict(SDXL_UNET)
    synth.set_device("cuda")
    try:
        sd = synth.unet_state_dict(cfg)
    finally:
        synth.set_device("cpu")
    x = synth.randn("fs8_x", (1, 4, 128, 128)).cuda()
    ctx = synth.randn("fs8_ctx", (1, 64, 2048)).cuda()
    added = dict(text_embeds=synth.randn("fs8_te", (1, 1280)).cuda(), time_ids=torch.tensor([[1024.0, 1024.0, 0.0, 0.0, 1024.0, 1024.0]]).cuda())
    m = UNet2DConditionModel(cfg)
    m.load_state_dict(sd)
    e16 = m(x, 601.0, ctx, added_cond_kwargs=added).cpu()
    del m
    torch.cuda.empty_cache()
    m8 = UNet2DConditionModel(cfg, weight_format="fp8_e4m3")
    m8.load_state_dict(sd)
    del sd
    e8 = m8(x, 601.0, ctx, added_cond_kwargs=added).cpu()
    e = rel(e8, e16)
    print(f"full-size UNet sample-forward, FP8 vs fp16: eps rel = {e:.3e}")
    assert torch.isfinite(e8).all() and e < 0.10, e       # measured on an H100 80GB HBM3 (700 W): 0.043; bound ~2.3x
