"""FP8 (e4m3) UNet convolutions on the GPU: seedx_quant_images_fp8 bit for bit against llm.quantize_fp8_rows, seedx_conv_fp8 bit for bit on an
integer grid (every FP8 conv tile width, image sizes 8x8 to 128x128, partial 128-channel chunks, ragged Cout, every epilogue the UNet uses through
the TMA / vector / scalar stores), its rejections, its accuracy on random data at the 14 UNet conv shapes, and
`UNet2DConditionModel(weight_format="fp8_e4m3_conv")` against the fp16 UNet and, at tiny size, its CPU restatement (test_fp8_conv_cpu.py), under
the CUDA graph and after a partial checkpoint.

Why the conv is exact: the e4m3 operands are integers with |q| <= 7 and the scales are powers of two.  A 128-element k-block sum is then below
128 * 49 = 6272 < 2^13, which the FP8 MMA keeps exactly (test_fp8_unet_gpu.py: integer sums past about 2^13 lose low bits), and the promoted
fp32 accumulator holds every whole sum exactly while it stays below 2^24.  The long-K cases use non-negative operands, so their sums grow to
about 2^20 at K = 23 040: without the promotion they would lose bits.  With the scales and biases chosen on grids that keep the linear epilogue
exact, an fp32 output equals the float64 reference bit for bit and an fp16 output equals it rounded once.  Outputs sit in NaN-sentinel buffers
and every input gap holds NaN, as in test_gemm_exact_gpu.py, whose helpers this file uses."""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

from seedx_b200 import synth
from seedx_b200.llm import quantize_fp8_rows
from test_gemm_exact_gpu import F16, F32, assert_exact, check_col_part, contiguous_out, grid, last_config, lib, nan_tail, r32, ref_conv, ref_epilogue

pytestmark = pytest.mark.gpu
E4 = torch.float8_e4m3fn
CONV8_TILES = [64, 128, 160]


def rel(a, b):
    return ((a.float().cpu() - b.float().cpu()).norm() / b.float().cpu().norm()).item()


# ---------------------------------------------------------------------------------------------------------------------------------------------
# quantiser
# ---------------------------------------------------------------------------------------------------------------------------------------------
def _images(n, h, w, c, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn((n, h, w, c), generator=g) * torch.logspace(-3, 2, n)[:, None, None, None]
    if n > 1:
        x[1] = 0.0                                                       # an all-zero image: scale 1, q = 0
    x[-1].view(-1)[::7] = 65504.0                                        # the fp16 extremes: clamped, no NaN
    x[-1].view(-1)[3::7] = -65504.0
    if n > 1:
        x[0].view(-1)[-1] = 1e4                                          # the maximum in the very last element
    return x.half()


@pytest.mark.parametrize("n,h,w,c", [(1, 8, 8, 64), (3, 8, 8, 64), (8, 8, 8, 64), (8, 16, 16, 320), (3, 24, 24, 320), (1, 128, 128, 960),
                                     (3, 128, 128, 960), (8, 32, 32, 1280)])
def test_quant_images_fp8_bit_exact(n, h, w, c):
    """per_image 4096 (half a chunk), 81 920 (10 chunks), 184 320 (22.5 chunks), 15.7 M (1920 chunks); a NaN tail after q keeps its bits"""
    from seedx_b200 import ops
    x16 = _images(n, h, w, c, seed=n * 1000 + c)
    x = x16.cuda()
    qbuf = torch.full((x.numel() + 64,), 0x7F, dtype=torch.uint8, device="cuda")
    q = qbuf[: x.numel()].view(E4).view(x.shape)
    s = nan_tail(torch.zeros(n))
    torch.cuda.synchronize()
    n0 = lib().seedx_launch_count()
    ops.quant_images_fp8(x, q=q, scale=s)
    assert lib().seedx_launch_count() - n0 == 2
    torch.cuda.synchronize()
    q_ref, s_ref = quantize_fp8_rows(x16.view(n, -1).float())
    assert torch.equal(s.cpu(), s_ref)
    assert torch.equal(q.view(torch.uint8).view(n, -1).cpu(), q_ref.view(torch.uint8))
    assert bool((qbuf[x.numel():] == 0x7F).all()) and not bool(torch.isnan(q.float()).any())
    if n > 1:
        assert float(s[1]) == 1.0


def test_quant_images_fp8_image_alone_equals_in_batch():
    from seedx_b200 import ops
    x = _images(8, 32, 32, 640, seed=5).cuda()
    q8, s8 = ops.quant_images_fp8(x)
    for i in (0, 4, 7):
        q1, s1 = ops.quant_images_fp8(x[i:i + 1].contiguous())
        assert torch.equal(q1[0].view(torch.uint8), q8[i].view(torch.uint8)) and torch.equal(s1[0], s8[i])


# ---------------------------------------------------------------------------------------------------------------------------------------------
# conv: exact on the integer grid
# ---------------------------------------------------------------------------------------------------------------------------------------------
def conv8_operands(n, h, w, c, cout, seed, positive):
    """integer image |q| <= 7 (0..7 when positive) and packed weights [cout, 3, 3, roundup(c, 128)] whose padded channel columns hold finite
    non-zero values (7): only the TMA zero fill of the image's missing channels cancels them"""
    c128 = (c + 127) // 128 * 128
    lim = 7
    x64 = grid((n, h, w, c), seed, 1, lim)
    w64 = grid((cout, 3, 3, c128), seed + 1, 1, lim)
    if positive:
        x64, w64 = x64.abs(), w64.abs()
    w64[..., c:] = 7.0
    x8 = x64.to(E4).cuda()
    w8 = w64.reshape(cout, -1).to(E4).cuda()
    assert torch.equal(x8.double().cpu(), x64) and torch.equal(w8.double().cpu(), w64.reshape(cout, -1))
    return x64, w64, x8, w8


def pow2(n, lo, hi, seed):
    g = torch.Generator().manual_seed(seed)
    return nan_tail(torch.pow(2.0, torch.randint(lo, hi + 1, (n,), generator=g).double()))


def run_conv8(n, h, w, c, cout, tile, dt, *, residual=True, col_part=True, bias_g=True, positive=False, seed=0):
    """one seedx_conv_fp8 on grid operands with bias, per-image bias_g, fp16/fp32 residual and col_part; returns (output, float64 want, cfg, part)"""
    from seedx_b200 import ops
    x64, w64, x8, w8 = conv8_operands(n, h, w, c, cout, seed, positive)
    if positive:      # sums up to ~2^20: scales in [1/4, 1] and biases on a 1/16 grid keep every fp32 value exact
        sa, sw, den = pow2(n, -2, 0, seed + 2), pow2(cout, -2, 0, seed + 3), 16
    else:             # sums up to ~2^14: scales down to 2^-12 combined, biases on a 1/64 grid
        sa, sw, den = pow2(n, -6, -3, seed + 2), pow2(cout, -6, -3, seed + 3), 64
    M = n * h * w
    bias = nan_tail(grid((cout,), seed + 4, den, 64, nonzero=True))
    temb = nan_tail(grid((n, cout), seed + 5, den, 64, nonzero=True)) if bias_g else None
    res = grid((n, h, w, cout), seed + 6, den, 64).to(dt).cuda() if residual else None
    part = torch.full((M // 32, cout, 2), float("nan"), device="cuda") if col_part else None
    ob = contiguous_out((n, h, w, cout), dt)
    ops.conv2d_nhwc(x8, w8, out=ob.view, bias=bias, bias_g=temb, residual=res, tile_n=tile, col_part=part, a_scale=sa, w_scale=sw)
    cfg = last_config()
    torch.cuda.synchronize()
    ob.check_outside()
    acc = ref_conv(x64, w64, 3)                                         # exact integer sums
    acc = acc * sa.double().repeat_interleave(h * w)[:, None] * sw.double()[None, :]
    x = ref_epilogue(acc, bias=bias, bias_g=temb, bias_g_rows=h * w)
    if res is not None:
        x = r32(x + res.double().reshape(M, cout))
    want = (x.float() if dt == F32 else x.float().half()).view(n, h, w, cout)
    return ob, want, cfg, part


CONV8_CASES = [
    # n, h,   w,   c,    cout, tile, out, positive
    (8, 8, 8, 64, 320, 64, F16, False),        # two 8x8 images per 128-row tile; C = 64: half a 128-channel chunk
    (3, 8, 8, 320, 200, 128, F16, False),      # the second tile holds one image and a zero-filled half; C = 320 (2.5 chunks); Cout ragged
    (2, 16, 16, 320, 640, 160, F16, False),    # 640 / 160; 16x16: a tile spans 8 image rows
    (1, 32, 32, 640, 600, 160, F32, False),    # 600 = 3 x 160 + 120: ragged last tile
    (2, 64, 64, 960, 320, 128, F16, False),    # 960 = 7.5 chunks
    (1, 128, 128, 320, 320, 160, F16, False),  # 128-wide rows: one image row per tile
    (1, 32, 32, 1280, 1280, 64, F32, True),    # K = 11 520, non-negative: whole sums ~2^19
    (1, 16, 16, 2560, 1280, 160, F32, True),   # K = 23 040: whole sums ~2^20
    (2, 8, 16, 1920, 640, 128, F32, True),     # K = 17 280, 8x16 images: two per tile
]


@pytest.mark.parametrize("n,h,w,c,cout,tile,dt,positive", CONV8_CASES)
def test_conv_fp8_exact(n, h, w, c, cout, tile, dt, positive):
    M = n * h * w
    stats = M % 32 == 0 and cout % 32 == 0 and dt == F16
    ob, want, cfg, part = run_conv8(n, h, w, c, cout, tile, dt, col_part=stats, positive=positive, seed=c + cout + n)
    assert_exact(ob.view, want, f"conv8 n={n} {h}x{w} C={c} Cout={cout} tile={tile}")
    es = 4 if dt == F32 else 2
    tma = int(tile % 32 == 0 and cout * es % 16 == 0)
    assert (cfg["tile"], cfg["cluster"], cfg["stream_k"], cfg["tma"], cfg["vec"]) == (tile, 1, 0, tma, int(cout % (16 // es) == 0))
    if part is not None:
        check_col_part(part, ob.view.reshape(M, cout))


@pytest.fixture
def store_mode():
    yield lambda s: lib().seedx_gemm_set_tma_epilogue(0 if s == "vector" else 1)
    lib().seedx_gemm_set_tma_epilogue(1)


@pytest.mark.parametrize("store", ["tma", "vector", "scalar"])
@pytest.mark.parametrize("tile", CONV8_TILES)
@pytest.mark.parametrize("dt", [F16, F32], ids=["f16", "f32"])
def test_conv_fp8_exact_epilogues(store, tile, dt, store_mode):
    """bias + per-image bias_g (ResnetBlock2D conv1: the time embedding), fp16 / fp32 residual (conv2), col_part (the next GroupNorm's
    statistics) through each store path.  TMA: 16-byte rows; vector: the TMA epilogue switched off; scalar: Cout = 38 (rows of 76 / 152 bytes)"""
    cout = 38 if store == "scalar" else 320
    stats = store == "tma" and dt == F16
    store_mode(store)
    ob, want, cfg, part = run_conv8(2, 16, 16, 320, cout, tile, dt, col_part=stats, seed=tile + cout)
    assert_exact(ob.view, want, f"{store} tile={tile}")
    tma = int(store == "tma" and tile % 32 == 0)
    vec = int(store != "scalar")
    assert (cfg["tile"], cfg["cluster"], cfg["stream_k"], cfg["tma"], cfg["vec"]) == (tile, 1, 0, tma, vec)
    if part is not None:
        check_col_part(part, ob.view.reshape(-1, cout))


def test_conv_fp8_auto_tile():
    """auto mode picks an instantiated width even with cluster pairs and stream-K forced for fp16"""
    lib().seedx_gemm_set_cluster(2)
    lib().seedx_gemm_set_stream_k(2)
    try:
        ob, want, cfg, _ = run_conv8(2, 32, 32, 640, 1280, 0, F32, col_part=False, positive=True, seed=77)
    finally:
        lib().seedx_gemm_set_cluster(1)
        lib().seedx_gemm_set_stream_k(1)
    assert cfg["tile"] in CONV8_TILES and cfg["cluster"] == 1 and cfg["stream_k"] == 0
    assert_exact(ob.view, want, "auto tile")


# ---------------------------------------------------------------------------------------------------------------------------------------------
# rejections
# ---------------------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", ["not_conv", "batch2", "no_a_scale", "no_b_scale", "c_not_16", "k_mismatch", "k_fp16_layout", "tile96",
                                  "tile192", "width48", "height_ragged"])
def test_conv_fp8_rejections_launch_nothing(case):
    from seedx_b200._lib import GemmArgs
    n, h, w, c, cout = 2, 16, 16, 320, 256
    geo = dict(width48=(16, 48), height_ragged=(12, 16)).get(case, (h, w))
    h, w = geo
    c = 24 if case == "c_not_16" else c
    K = 9 * ((c + 127) // 128 * 128)
    K = {"k_mismatch": K + 128, "k_fp16_layout": 9 * ((c + 63) // 64 * 64)}.get(case, K)
    x = torch.zeros((n * h * w * c,), dtype=torch.uint8, device="cuda")
    wt = torch.zeros((cout, K), dtype=torch.uint8, device="cuda")
    out = torch.zeros((n * h * w, cout), dtype=F16, device="cuda")
    sa, sw = torch.ones(n, device="cuda"), torch.ones(cout, device="cuda")
    g = GemmArgs()
    g.A, g.B, g.D = x.data_ptr(), wt.data_ptr(), out.data_ptr()
    g.M, g.N, g.K, g.batch = n * h * w, cout, K, 1
    g.lda, g.ldb, g.ldd = c, K, cout
    g.alpha, g.out_dtype = 1.0, 1
    g.conv_taps_h = g.conv_taps_w = 0 if case == "not_conv" else 3
    g.conv_n, g.conv_h, g.conv_w, g.conv_c = n, h, w, c
    g.tile_n = dict(tile96=96, tile192=192).get(case, 0)
    if case == "batch2":
        g.batch, g.strideA, g.strideD = 2, n * h * w * c, n * h * w * cout
    pa = None if case == "no_a_scale" else C.c_void_p(sa.data_ptr())
    pb = None if case == "no_b_scale" else C.c_void_p(sw.data_ptr())
    torch.cuda.synchronize()
    n0 = lib().seedx_launch_count()
    rc = lib().seedx_conv_fp8(C.byref(g), pa, pb, None)
    assert rc != 0 and lib().seedx_last_error()
    assert lib().seedx_launch_count() == n0
    torch.cuda.synchronize()
    assert int(out.abs().sum()) == 0


# ---------------------------------------------------------------------------------------------------------------------------------------------
# accuracy on random data at the UNet's conv shapes
# ---------------------------------------------------------------------------------------------------------------------------------------------
# (h = w, C_in, C_out) of the 36 FP8 convs of the SDXL UNet at 128 x 128 latents: 14 distinct shapes
UNET_CONVS = [(128, 320, 320), (64, 320, 640), (64, 640, 640), (32, 640, 1280), (32, 1280, 1280), (32, 2560, 1280), (32, 1920, 1280),
              (64, 1280, 1280), (64, 1920, 640), (64, 1280, 640), (64, 960, 640), (128, 640, 640), (128, 960, 320), (128, 640, 320)]


def _random_conv_operands(n, hw, c, cout, seed):
    """GroupNorm+SiLU-like activations and conv weights of fan-in scale, quantised the way the UNet quantises them"""
    from seedx_b200 import ops
    from seedx_b200.sdxl import conv_fp8, pack_conv
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = F.silu(torch.randn((n, hw, hw, c), device="cuda", generator=g)).half()
    w = torch.randn((cout, c, 3, 3), device="cuda", generator=g) * (9 * c) ** -0.5
    qx, sx = ops.quant_images_fp8(x)
    qw, sw = conv_fp8(pack_conv(w, "cuda"), c)
    return qx, sx, qw, sw


def _deq_conv64(qx, sx, qw, sw, c):
    cout = qw.shape[0]
    c128 = qw.shape[1] // 9
    xd = qx.double() * sx.double()[:, None, None, None]
    wd = (qw.double() * sw.double()[:, None]).view(cout, 3, 3, c128)[..., :c].permute(0, 3, 1, 2)
    return F.conv2d(xd.permute(0, 3, 1, 2), wd, padding=1).permute(0, 2, 3, 1)


@pytest.mark.parametrize("hw,c,cout", UNET_CONVS)
def test_conv_fp8_random_accuracy_at_unet_shapes(hw, c, cout):
    """fp32 output against a float64 conv of the same dequantized operands: what is left is the MMA's error inside each 128-element block (the
    promoted fp32 sum of the blocks adds little).  Relative (Frobenius) error measured on an H100 80GB HBM3 (700 W): 1.30e-4 to 1.43e-4 over the
    14 shapes, independent of K from 3456 to 23 040; bound 4.5e-4 (~3x).  The unpromoted seedx_gemm_fp8 on the same operands:
    test_unpromoted_gemm_error_at_conv_k."""
    from seedx_b200 import ops
    n = 2
    qx, sx, qw, sw = _random_conv_operands(n, hw, c, cout, seed=hw + c + cout)
    out = ops.conv2d_nhwc(qx, qw, a_scale=sx, w_scale=sw, out_dtype=F32)
    ref = _deq_conv64(qx, sx, qw, sw, c)
    e = ((out.double() - ref).norm() / ref.norm()).item()
    print(f"FP8 conv {hw}x{hw} {c}->{cout} (K = {9 * ((c + 127) // 128 * 128)}): fp32 output rel err vs float64 {e:.2e}")
    assert e < 4.5e-4, e


@pytest.mark.parametrize("hw,c,cout", [(32, 1280, 1280), (32, 2560, 1280)])
def test_unpromoted_gemm_error_at_conv_k(hw, c, cout):
    """for comparison only (no bound): the same operands through seedx_gemm_fp8 (no promotion) on an explicit im2col, K = 11 520 and 23 040,
    against the same float64 reference as the promoted conv.  Measured on an H100 80GB HBM3 (700 W): 2.65e-3 (K = 11 520) and 3.98e-3
    (K = 23 040) unpromoted, 1.40e-4 and 1.41e-4 promoted"""
    from seedx_b200 import ops
    n = 2
    qx, sx, qw, sw = _random_conv_operands(n, hw, c, cout, seed=hw + c + cout)
    c128 = qw.shape[1] // 9
    xp = F.pad(qx.view(torch.uint8), (0, c128 - c, 1, 1, 1, 1))                   # zero pixels around, zero channels up to 128
    cols = torch.stack([xp[:, kh:kh + hw, kw:kw + hw, :] for kh in range(3) for kw in range(3)], dim=3)    # [n, hw, hw, 9, c128]
    a = cols.reshape(n * hw * hw, 9 * c128).contiguous().view(E4)
    a_scale = sx.repeat_interleave(hw * hw).contiguous()
    ref = _deq_conv64(qx, sx, qw, sw, c).reshape(n * hw * hw, cout)
    e_gemm = ((ops.gemm(a, qw, a_scale=a_scale, w_scale=sw, out_dtype=F32).double() - ref).norm() / ref.norm()).item()
    e_conv = ((ops.conv2d_nhwc(qx, qw, a_scale=sx, w_scale=sw, out_dtype=F32).double().reshape(-1, cout) - ref).norm() / ref.norm()).item()
    print(f"K = {9 * c128}: rel err vs float64, unpromoted seedx_gemm_fp8 {e_gemm:.2e}, promoted seedx_conv_fp8 {e_conv:.2e}")
    assert e_gemm == e_gemm and e_conv == e_conv


# ---------------------------------------------------------------------------------------------------------------------------------------------
# UNet
# ---------------------------------------------------------------------------------------------------------------------------------------------
def _tiny_inputs(B, in_ch=4, hw=32):
    cfg = synth.TINY_UNET
    x = synth.randn("gc8_x", (B, in_ch, hw, hw))
    ctx = synth.randn("gc8_ctx", (B, 16, cfg["cross_attention_dim"]))
    te = synth.randn("gc8_te", (B, cfg["text_embed_dim"]))
    tid = torch.tensor([[1024.0, 1024.0, 0.0, 0.0, 1024.0, 1024.0]]).repeat(B, 1)
    return x.cuda(), ctx.cuda(), dict(text_embeds=te.cuda(), time_ids=tid.cuda())


def test_tiny_unet_fp8_conv_matches_the_cpu_restatement_and_tracks_fp16():
    import test_fp8_conv_cpu as hostc
    from seedx_b200 import sdxl as sdxl_mod
    from seedx_b200.sdxl import UNet2DConditionModel
    cfg = synth.TINY_UNET
    sd = synth.unet_state_dict(cfg)
    x, ctx, added = _tiny_inputs(2)
    m16, m8 = UNet2DConditionModel(cfg), UNet2DConditionModel(cfg, weight_format="fp8_e4m3_conv")
    m16.load_state_dict(sd), m8.load_state_dict(sd)
    assert len(m8.conv_fp8_slots()) == 36
    e16, e8 = m16(x, 601.0, ctx, added_cond_kwargs=added), m8(x, 601.0, ctx, added_cond_kwargs=added)
    real_ops = sdxl_mod.ops
    sdxl_mod.ops = hostc.fake_ops_fp8
    try:
        mc = UNet2DConditionModel(cfg, device="cpu", weight_format="fp8_e4m3_conv")
        mc.load_state_dict(sd)
        ec = mc(x.cpu(), 601.0, ctx.cpu(), added_cond_kwargs={k: v.cpu() for k, v in added.items()})
    finally:
        sdxl_mod.ops = real_ops
    e_host, e_16 = rel(e8, ec), rel(e8, e16)
    print(f"tiny UNet fp8_e4m3_conv: eps rel vs CPU restatement {e_host:.3e}, vs fp16 UNet {e_16:.3e}")
    # measured on an H100 80GB HBM3 (700 W): 0.041 vs the restatement (exact fp64 sums; fp16 activations that round differently move later
    # quantisation points by one e4m3 step), 0.045 vs fp16; bounds ~3x
    assert e_host < 0.12 and 1e-4 < e_16 < 0.135, (e_host, e_16)


def test_fp8_conv_t2i_walk_under_the_cuda_graph():
    """4 Euler steps of the 2-way CFG loop replayed as a CUDA graph: latents near the fp16 walk, a second run bitwise repeatable, and conv
    weights loaded after capture replay exactly what a freshly built model with the merged weights computes"""
    from seedx_b200.sampler import DenoiseLoop
    from seedx_b200.sdxl import EulerDiscreteScheduler, UNet2DConditionModel
    cfg = synth.TINY_UNET
    sd = synth.unet_state_dict(cfg)
    B, hw, steps = 1, 32, 4
    noise = synth.randn("gc8_noise", (B, 4, hw, hw)).cuda()
    p, n = synth.randn("gc8_p", (B, 16, cfg["cross_attention_dim"])), synth.randn("gc8_n", (B, 16, cfg["cross_attention_dim"]))
    pp, npool = synth.randn("gc8_pp", (B, cfg["text_embed_dim"])), synth.randn("gc8_np", (B, cfg["text_embed_dim"]))
    tid = torch.tensor([[1024.0, 1024.0, 0.0, 0.0, 1024.0, 1024.0]]).repeat(2 * B, 1).cuda()

    def walk(unet):
        loop = DenoiseLoop(unet, EulerDiscreteScheduler(), B, (hw, hw), 2, use_graph=True)
        loop.set_condition(torch.cat([n, p]).cuda(), torch.cat([npool, pp]).cuda(), tid)
        return loop, loop.run(noise, steps=steps, guidance=7.5).clone()
    u16, u8 = UNet2DConditionModel(cfg), UNet2DConditionModel(cfg, weight_format="fp8_e4m3_conv")
    u16.load_state_dict(sd), u8.load_state_dict(sd)
    _, lat16 = walk(u16)
    loop8, lat8 = walk(u8)
    assert loop8.graph is not None
    e = rel(lat8, lat16)
    print(f"tiny t2i walk, fp8_e4m3_conv vs fp16 UNet: latents rel = {e:.3e}")
    # measured on an H100 80GB HBM3 (700 W): 0.110 (fp8_e4m3 alone: 0.064); bound ~3x
    assert 1e-5 < e < 0.33, e
    assert torch.equal(loop8.run(noise, steps=steps, guidance=7.5), lat8)
    part = {k: synth.randn("gc8ft:" + k, v.shape, v[0].numel() ** -0.5)
            for k, v in sd.items() if k.endswith(("resnets.0.conv1.weight", "resnets.1.conv2.weight", "upsamplers.0.conv.weight"))}
    g0 = loop8.graph
    u8.load_state_dict(part)
    got = loop8.run(noise, steps=steps, guidance=7.5).clone()
    assert loop8.graph is g0
    fresh = UNet2DConditionModel(cfg, weight_format="fp8_e4m3_conv")
    fresh.load_state_dict({**sd, **part})
    _, want = walk(fresh)
    assert torch.equal(got, want)


def test_fp8_conv_edit_loop_runs():
    """the 3-branch edit loop (8-channel conv_in, which stays fp16) with the fp8_e4m3_conv UNet under the CUDA graph"""
    from seedx_b200.sampler import DenoiseLoop
    from seedx_b200.sdxl import EulerDiscreteScheduler, UNet2DConditionModel
    cfg = dict(synth.TINY_UNET, in_channels=8)
    sd = synth.unet_state_dict(cfg)
    B, hw = 1, 32
    u16, u8 = UNet2DConditionModel(cfg), UNet2DConditionModel(cfg, weight_format="fp8_e4m3_conv")
    u16.load_state_dict(sd), u8.load_state_dict(sd)
    noise = synth.randn("gc8e_noise", (B, 4, hw, hw)).cuda()
    il = synth.randn("gc8e_il", (B, 4, hw, hw), 0.7).cuda()
    p, n = synth.randn("gc8e_p", (B, 16, cfg["cross_attention_dim"])), synth.randn("gc8e_n", (B, 16, cfg["cross_attention_dim"]))
    pp, npool = synth.randn("gc8e_pp", (B, cfg["text_embed_dim"])), synth.randn("gc8e_np", (B, cfg["text_embed_dim"]))
    tid = torch.tensor([[1024.0, 1024.0, 0.0, 0.0, 1024.0, 1024.0]]).repeat(3 * B, 1).cuda()
    lats = []
    for u in (u16, u8):
        loop = DenoiseLoop(u, EulerDiscreteScheduler(), B, (hw, hw), 3, use_graph=True)
        loop.set_condition(torch.cat([p, n, n]).cuda(), torch.cat([pp, npool, npool]).cuda(), tid, image_latents=il)
        lats.append(loop.run(noise, steps=4, guidance=7.5, image_guidance=1.5).clone())
    e = rel(lats[1], lats[0])
    print(f"tiny edit walk, fp8_e4m3_conv vs fp16 UNet: latents rel = {e:.3e}")
    assert torch.isfinite(lats[1]).all() and e < 0.33, e       # measured on an H100 80GB HBM3 (700 W): 0.111; bound ~3x


def test_engine_passes_the_conv_weight_format():
    from seedx_b200.engine import SeedXEngine
    small = dict(vit_cfg=dict(width=208, layers=2, heads=2, mlp_width=520, output_dim=256, n_queries=256, patch=14), llm_cfg=synth.TINY_LLAMA,
                 unet_cfg=dict(synth.TINY_UNET, cross_attention_dim=256, text_embed_dim=160), vae_cfg=synth.TINY_VAE,
                 rxl_cfg=dict(synth.TINY_RESAMPLER_XL, embedding_dim=256, output1_dim=96, output2_dim=160))
    for edit in (False, True):
        eng = SeedXEngine(**small, edit=edit, unet_weight_format="fp8_e4m3_conv")
        u = eng.adapter.unet
        assert u.weight_format == "fp8_e4m3_conv" and len(u.conv_fp8_slots()) == 36 and all(t.fp8_slots() for t in u.transformers())
        del eng
        torch.cuda.empty_cache()


def test_unet_full_size_fp8_conv_sample_forward():
    """one SDXL UNet sample-forward at full size with fp8_e4m3_conv against the fp16 UNet on the same weights (fp8_e4m3 alone: 0.043 in
    test_fp8_unet_gpu.py)"""
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
    m8 = UNet2DConditionModel(cfg, weight_format="fp8_e4m3_conv")
    m8.load_state_dict(sd)
    del sd
    assert len(m8.conv_fp8_slots()) == 36
    e8 = m8(x, 601.0, ctx, added_cond_kwargs=added).cpu()
    e = rel(e8, e16)
    print(f"full-size UNet sample-forward, fp8_e4m3_conv vs fp16: eps rel = {e:.3e}")
    assert torch.isfinite(e8).all() and e < 0.16, e       # measured on an H100 80GB HBM3 (700 W): 0.055; bound ~3x
