"""Bit-exact tests of the wgmma GEMM / implicit-GEMM conv (seedx_gemm_f16) on an integer grid, with sentinel-filled outputs and NaN-filled gaps.

Why exact: the operands are fp16 values on a coarse grid (a = i/16, w = j/256 with |i|, |j| <= 16), so every product and every partial sum is an
integer multiple of 2^-12.  While |sum| < 2^24 grid units (K * max|a| * max|w| * 2^12 = 23 040 * 256 < 2^24 even in the worst case) the fp32
accumulation is exact in any order: split over k-blocks, cluster halves or stream-K partials.  The float64 reference on the device is exact too.
Biases, residuals and alpha in {0.5, 0.25} stay on the grid, so the linear epilogue is exact as well: an fp32 output must equal the reference
bit for bit, and an fp16 output must equal the reference rounded once to fp16.  The only epilogue step that rounds on the grid is the gated
product x[2j] * x[2j+1] (and a residual added to it); the reference rounds it to fp32 exactly where the kernel does, once.

Every output is a view cut out of a larger buffer filled with a NaN sentinel bit pattern (a column gap ldd > n_out, rows after M, gaps between
batches): every element outside the view must keep its bits.  Every input gap (A's lda gap and batch gap, B's ldb gap, the residual's ldr gap,
the tails behind the bias vectors) holds NaN, so a read past K, N, n_out or M would carry NaN into an output that must be exact.

seedx_gemm_last_config reports what each launch ran (tile width, cluster size, stream-K, TMA epilogue, vector stores, stages); every case
asserts that it ran the path it is named after.  Non-exact epilogues (GELU, SiLU, folded LayerNorm, output statistics) are bounded elementwise
against float64, with each bound derived below next to its constant.
"""
import ctypes as C
import math
import os
import re

import pytest
import torch
import torch.nn.functional as F

import fake_ops
from fp16_ulp import ulp16

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F16, F32 = torch.float16, torch.float32
SENT16, SENT32 = 0x7E5A, 0x7FC5A5A5          # quiet NaNs with a payload no arithmetic produces
U32 = 2.0 ** -24                              # unit roundoff of fp32
TILES = [64, 96, 128, 144, 160, 192, 208, 224, 240, 256]
SK_TILES = [128, 160, 192, 224, 256]          # the widths with stream-K kernels (cluster pairs, multiple of 32, >= 128)


# ---------------------------------------------------------------------------------------------------------------------------------------------
# helpers
# ---------------------------------------------------------------------------------------------------------------------------------------------
def lib():
    from seedx_b200._lib import lib as _l
    return _l()


def last_config():
    v = (C.c_int32 * 6)()
    lib().seedx_gemm_last_config(v)
    return dict(zip(("tile", "cluster", "stream_k", "tma", "vec", "stages"), list(v)))


@pytest.fixture(params=["single_cta", "cluster2"])
def cluster_mode(request):
    """every case with the 2-CTA cluster (TMA multicast of B) forced off and forced on wherever it is legal"""
    lib().seedx_gemm_set_cluster(0 if request.param == "single_cta" else 2)
    yield request.param
    lib().seedx_gemm_set_cluster(1)


@pytest.fixture
def store_mode():
    """seedx_gemm_set_tma_epilogue for the duration of a test, default restored afterwards"""
    yield lambda s: lib().seedx_gemm_set_tma_epilogue(0 if s == "vector" else 1)
    lib().seedx_gemm_set_tma_epilogue(1)


@pytest.fixture
def stream_k():
    yield lambda mode: lib().seedx_gemm_set_stream_k(mode)
    lib().seedx_gemm_set_stream_k(1)


def grid(shape, seed, den, lim=16, nonzero=False):
    """float64 values i / den with integer |i| <= lim (seeded, on the CPU)"""
    g = torch.Generator().manual_seed(seed)
    i = torch.randint(-lim, lim + 1, shape, generator=g)
    if nonzero:
        i = torch.where(i == 0, torch.full_like(i, lim), i)
    return i.double() / den


def r32(t):
    """round a float64 tensor to fp32 once (an fp32 operation of the kernel on exact operands)"""
    return t.float().double()


def padded(vals, ld, dtype, batch_gap=0):
    """device copy of vals [R, C] or [B, R, C] with row stride ld (> C) and batch stride R * ld + batch_gap; every gap element, and one row
    after the end, is NaN"""
    v = vals if vals.dim() == 3 else vals[None]
    B, R, Cc = v.shape
    bs = R * ld + batch_gap
    buf = torch.full((B * bs + ld,), float("nan"), dtype=dtype, device="cuda")
    view = buf.as_strided((B, R, Cc), (bs, ld, 1), 0)
    view.copy_(v.to(dtype))
    return view if vals.dim() == 3 else view[0]


def nan_tail(v):
    """contiguous fp32 vector followed by NaN: a read past its end shows"""
    buf = torch.full((v.numel() + 16,), float("nan"), dtype=F32, device="cuda")
    buf[: v.numel()] = v.reshape(-1).float().cuda()
    return buf[: v.numel()].view(v.shape)


def sentinel(numel, dtype):
    if dtype == F16:
        return torch.full((numel,), SENT16, dtype=torch.int16, device="cuda").view(F16)
    return torch.full((numel,), SENT32, dtype=torch.int32, device="cuda").view(F32)


class OutBuf:
    """output view [M, n_out] or [B, M, n_out] (row stride ldd, batch stride strideD) cut out of a sentinel-filled buffer with elements before
    the view, a column gap, rows after M, a gap between batches and a tail"""

    def __init__(self, shape, dtype, ldd, strideD=None, lead=8):
        B, M, n = (1, *shape) if len(shape) == 2 else shape
        strideD = strideD if strideD is not None else (M + 3) * ldd
        numel = lead + (B - 1) * strideD + (M + 2) * ldd + 64
        self.buf = sentinel(numel, dtype)
        st = (strideD, ldd, 1)[-len(shape):]
        self.view = self.buf.as_strided(shape, st, lead)
        self.mask = torch.zeros(numel, dtype=torch.bool, device="cuda")
        self.mask.as_strided(shape, st, lead).fill_(True)

    def check_outside(self):
        bits = self.buf.view(torch.int16 if self.buf.dtype == F16 else torch.int32)
        s = SENT16 if self.buf.dtype == F16 else SENT32
        bad = int((bits[~self.mask] != s).sum())
        assert bad == 0, f"{bad} elements outside the output view were overwritten"


def contiguous_out(shape, dtype, lead=8):
    """contiguous output (conv entry point) inside a sentinel buffer: elements before and after it must keep their bits"""
    n = math.prod(shape)
    ob = OutBuf((1, n), dtype, n, lead=lead)
    ob.view = ob.view.view(shape)
    return ob


def round8(n):
    return (n + 7) // 8 * 8


def expect(cfg, *, tile, cluster, tma, vec):
    got = (cfg["tile"], cfg["cluster"], cfg["tma"], cfg["vec"])
    assert got == (tile, cluster, tma, vec), f"ran (tile, cluster, tma, vec) = {got}, expected {(tile, cluster, tma, vec)}"


def exp_cluster(mode, M, tile):
    return 2 if (mode == "cluster2" and (M + 127) // 128 >= 2 and tile % 32 == 0) else 1


def assert_exact(out, want, what=""):
    if not torch.equal(out, want):
        d = (out.double() - want.double()).abs()
        d[torch.isnan(d)] = float("inf")
        idx = int(d.reshape(-1).argmax())
        raise AssertionError(f"{what}: {int((d != 0).sum())} of {d.numel()} elements differ; worst at flat index {idx}: "
                             f"got {out.reshape(-1)[idx].item()!r}, want {want.reshape(-1)[idx].item()!r}")


def ref_epilogue(acc, *, alpha=1.0, bias=None, bias_m=None, bias_g=None, bias_g_rows=0, gated=False, residual=None, res_row_mod=0):
    """float64 epilogue of seedx_gemm_f16 (include/seedx.h) from the exact accumulator; fp32 rounding only where the grid does not keep it
    exact (the gated product, a residual added to it)"""
    M = acc.shape[-2]
    x = acc * alpha
    if bias is not None:
        x = x + bias.double()
    if bias_m is not None:
        x = x + bias_m.double()[:, None]
    if bias_g is not None:
        x = x + bias_g.double().repeat_interleave(bias_g_rows, 0)[:M]
    assert torch.equal(r32(x), x), "the test's operands left the grid: the linear epilogue is not exact in fp32"
    if gated:
        x = r32(x[..., 0::2] * x[..., 1::2])
    if residual is not None:
        r = residual.double()
        if res_row_mod:
            r = r.repeat(-(-M // res_row_mod), 1)[:M]
        x = r32(x + r)
    return x


def to_out(x64, dtype):
    return x64.float() if dtype == F32 else x64.float().half()


# ---------------------------------------------------------------------------------------------------------------------------------------------
# GEMM driver: build grid operands in NaN-gapped storage, run, check sentinels, compare bit for bit, run the CPU test double on the same inputs
# ---------------------------------------------------------------------------------------------------------------------------------------------
def run_gemm(M, N, K, *, tile_n, out_dtype, store="tma", B=1, b_batched=False, bias=False, bias_m=False, bias_g_rows=0, res=None,
             res_batched=False, inplace=False, res_row_mod=0, alpha=1.0, dynamic_b=False, gated=False, act=0, seed=0, a_den=16, w_den=256,
             fake=True, set_store=None):
    from seedx_b200 import ops
    n_out = N // 2 if gated else N
    batched = B > 1
    a64 = grid((B, M, K) if batched else (M, K), seed, a_den)
    w64 = grid((B, N, K) if b_batched else (N, K), seed + 1, w_den)
    a = padded(a64, K + 8, F16, batch_gap=24)
    w = padded(w64, K + 16, F16, batch_gap=40)
    kw = dict(alpha=alpha, act=act, gated=gated, tile_n=tile_n, dynamic_b=dynamic_b)
    refkw = dict(alpha=alpha, gated=gated, res_row_mod=res_row_mod)
    if bias:
        refkw["bias"] = kw["bias"] = nan_tail(grid((N,), seed + 2, 64, 64, nonzero=True))
    if bias_m:
        refkw["bias_m"] = kw["bias_m"] = nan_tail(grid((M,), seed + 3, 64, 64, nonzero=True))
    if bias_g_rows:
        refkw["bias_g"] = kw["bias_g"] = nan_tail(grid((-(-M // bias_g_rows), N), seed + 4, 64, 64, nonzero=True))
        kw["bias_g_rows"] = refkw["bias_g_rows"] = bias_g_rows
    aligned = store != "scalar"
    ldd = round8(n_out) + (8 if aligned else 9)
    ob = OutBuf((B, M, n_out) if batched else (M, n_out), out_dtype, ldd)
    if res is not None:
        rrows = res_row_mod or M
        r64 = grid((B, rrows, n_out) if (batched and res_batched) else (rrows, n_out), seed + 5, 64, 64)
        if inplace:
            assert res == out_dtype and not res_row_mod
            ob.view.copy_(r64.to(res).cuda())
            kw["residual"] = ob.view
        else:
            kw["residual"] = padded(r64, round8(n_out) + (16 if aligned else 17), res, batch_gap=8)
        kw["res_row_mod"] = res_row_mod
        refkw["residual"] = kw["residual"].clone() if inplace else kw["residual"]
    acc = a.double() @ w.double().transpose(-1, -2)          # DGEMM: exact on the grid
    want = to_out(ref_epilogue(acc, **refkw), out_dtype)
    if set_store is not None:
        set_store(store)
    ops.gemm(a, w, out=ob.view, **kw)
    cfg = last_config()
    torch.cuda.synchronize()
    ob.check_outside()
    if act == 0:
        assert_exact(ob.view, want, f"M={M} N={N} K={K} tile={tile_n} {out_dtype} {store}")
    if fake and act == 0 and not batched:
        cpu = lambda t: t.cpu() if isinstance(t, torch.Tensor) else t                     # noqa: E731
        fk = {k: cpu(v) for k, v in kw.items() if k not in ("tile_n",)}
        if inplace:
            fk["residual"] = refkw["residual"].cpu()
        got = fake_ops.gemm(a.cpu(), w.cpu(), out=torch.empty((M, n_out), dtype=out_dtype), **fk)
        assert_exact(got, want.cpu(), "CPU test double")
    return ob.view, cfg, acc, (a, w, kw)


def expected_tma(store, tile, N, gated, res, out_dtype, res_row_mod):
    n_out_bytes = (N // 2 if gated else N) * (4 if out_dtype == F32 else 2)
    if store != "tma" or tile % 32 or N % 2 or n_out_bytes % 16:      # rows must end on a 16-byte boundary (test_gemm_tma_store_...)
        return 0
    if res is not None and (gated or res != out_dtype or res_row_mod % 32):
        return 0
    return 1


# ---------------------------------------------------------------------------------------------------------------------------------------------
# 1. tiles and edges: all 10 tile widths, single CTA and cluster pairs, fp16 and fp32 outputs
# ---------------------------------------------------------------------------------------------------------------------------------------------
EDGE_SHAPES = [
    (1, 24, 8),         # one row; N below one 32-column chunk; one k-block only 8 deep (the rest is TMA zero fill)
    (2, 72, 56),        # ragged last 32-column chunk (72 = 2 x 32 + 8); one k-block 56 deep
    (127, 200, 72),     # one m-block one row short; K = 64 + 8
    (129, 330, 4104),   # the second m-block holds one row; 65 k-blocks, the last 8 deep
    (300, 1000, 136),   # three m-blocks: in cluster pairs the second CTA of the last pair lies wholly past M
    (300, 264, 23040),  # the UNet's longest K (9 x 2560); the last tile has 8 columns (< one chunk) for tiles 64/128/256, 24 for 240
    (3, 32330, 256),    # lm_head: rows of 32330 fp16 or fp32 are not 16-byte aligned -> direct scalar stores
]


@pytest.mark.gpu
@pytest.mark.parametrize("M,N,K", EDGE_SHAPES)
@pytest.mark.parametrize("tile_n", TILES)
def test_gemm_exact_tiles_and_edges(M, N, K, tile_n, cluster_mode):
    from seedx_b200 import ops
    aligned_rows = N % 8 == 0                     # (every N here is either a multiple of 8 or not even of 4)
    for i, dt in enumerate((F16, F32)):
        a, w = padded(grid((M, K), 10 + i, 16), K + 8, F16), padded(grid((N, K), 20 + i, 256), K + 8, F16)
        ob = OutBuf((M, N), dt, N + 8)            # ldd = N + 8 keeps the rows' 16-byte alignment what a contiguous output would have
        ops.gemm(a, w, out=ob.view, tile_n=tile_n)
        cfg = last_config()
        want = to_out(a.double() @ w.double().t(), dt)
        torch.cuda.synchronize()
        ob.check_outside()
        assert_exact(ob.view, want, f"{dt}")
        tma = int(tile_n % 32 == 0 and aligned_rows)
        expect(cfg, tile=tile_n, cluster=exp_cluster(cluster_mode, M, tile_n), tma=tma, vec=int(aligned_rows))
        assert torch.equal(fake_ops.gemm(a.cpu(), w.cpu(), out_dtype=dt), want.cpu())


# ---------------------------------------------------------------------------------------------------------------------------------------------
# 2. epilogue terms through every store path (TMA; direct 16-byte vector stores; direct scalar stores, forced by an unaligned ldd), with
#    sentinel outputs and NaN gaps everywhere
# ---------------------------------------------------------------------------------------------------------------------------------------------
EPILOGUES = {
    "bias_n_f16": (F16, dict(bias=True)),
    "bias_m_f32": (F32, dict(bias_m=True)),
    "bias_g64_f32": (F32, dict(bias_g_rows=64)),                            # groups of 64 rows: every value fetches its own element
    "bias_g128_f16": (F16, dict(bias=True, bias_g_rows=128)),               # 128-row groups: folded into the staged bias vector
    "bias_g256_f32": (F32, dict(bias_g_rows=256)),                          # two tiles per group, staged vector
    "res_f16": (F16, dict(bias=True, res=F16)),
    "res_f32": (F32, dict(res=F32)),
    "res_f16_into_f32": (F32, dict(res=F16)),                               # mixed dtypes: never the TMA epilogue
    "inplace_f16": (F16, dict(bias=True, res=F16, inplace=True)),           # out=r, residual=r
    "inplace_f32": (F32, dict(bias_m=True, res=F32, inplace=True)),
    "res_mod32_f16": (F16, dict(res=F16, res_row_mod=32)),                  # row-modulo residual, TMA-eligible
    "res_mod77_f32": (F32, dict(res=F32, res_row_mod=77)),                  # not a multiple of 32: direct stores only
    "alpha_half_f16": (F16, dict(alpha=0.5, bias=True, bias_m=True)),
    "alpha_quarter_f32": (F32, dict(alpha=0.25, res=F32, bias_g_rows=128)),
    "dynamic_b_f16": (F16, dict(bias=True, dynamic_b=True)),                # B read after the dependency wait only
    "gated_f16": (F16, dict(gated=True, bias=True)),                        # ACT_NONE gating: x[2j] * x[2j+1]
    "gated_f32": (F32, dict(gated=True, bias_m=True)),
    "gated_res_f16": (F16, dict(gated=True, bias=True, res=F16)),           # gated + residual: never TMA
}


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(EPILOGUES))
@pytest.mark.parametrize("store", ["tma", "vector", "scalar"])
@pytest.mark.parametrize("tile_n", [128, 240])
def test_gemm_exact_epilogues(case, store, tile_n, cluster_mode, store_mode):
    dt, opt = EPILOGUES[case]
    M, N, K = 300, 392, 200          # 3 m-blocks, ragged last tile and chunk, last k-block 8 deep
    _, cfg, _, _ = run_gemm(M, N, K, tile_n=tile_n, out_dtype=dt, store=store, set_store=store_mode, seed=10 * list(EPILOGUES).index(case), **opt)
    tma = expected_tma(store, tile_n, N, opt.get("gated", False), opt.get("res"), dt, opt.get("res_row_mod", 0))
    expect(cfg, tile=tile_n, cluster=exp_cluster(cluster_mode, M, tile_n), tma=tma, vec=int(store != "scalar"))


# ---------------------------------------------------------------------------------------------------------------------------------------------
# 3. batched: strideA with a NaN gap, batched or shared B, batched or shared residual, strideD gap with sentinels
# ---------------------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("variant", ["batched_b_batched_res", "shared_b_shared_res", "batched_b_no_res"])
@pytest.mark.parametrize("dt", [F16, F32], ids=["f16", "f32"])
@pytest.mark.parametrize("store", ["tma", "vector", "scalar"])
def test_gemm_exact_batched(variant, dt, store, cluster_mode, store_mode):
    B, M, N, K, tile = 3, 200, 136, 104, 128
    res = None if variant.endswith("no_res") else dt
    _, cfg, _, _ = run_gemm(M, N, K, B=B, tile_n=tile, out_dtype=dt, store=store, set_store=store_mode, b_batched=variant.startswith("batched_b"),
                            res=res, res_batched=variant.endswith("batched_res"), bias=True, seed=7)
    expect(cfg, tile=tile, cluster=exp_cluster(cluster_mode, M, tile), tma=expected_tma(store, tile, N, False, res, dt, 0),
           vec=int(store != "scalar"))


@pytest.mark.gpu
@pytest.mark.parametrize("N,gated,dt", [(196, False, F16), (392, True, F16), (200, True, F16), (330, False, F32), (394, True, F32)],
                         ids=["f16_n196", "f16_gated_n196", "f16_gated_n100", "f32_n330", "f32_gated_n197"])
def test_gemm_tma_store_row_end_not_16_byte_aligned(N, gated, dt, cluster_mode, store_mode):
    """Regression: an output view whose rows start 16-byte aligned (ldd * size % 16 == 0) but END inside a 16-byte granule (n_out * size % 16
    != 0) used to take the TMA epilogue, and the TMA store of the last column chunk wrote the rest of the granule into the ldd gap: 4 fp16
    columns past n_out = 196 on every row.  Such views now take the direct stores and leave the gap alone."""
    M, K, tile = 300, 200, 128
    _, cfg, _, _ = run_gemm(M, N, K, tile_n=tile, out_dtype=dt, store="tma", set_store=store_mode, gated=gated, bias=True, seed=17)
    expect(cfg, tile=tile, cluster=exp_cluster(cluster_mode, M, tile), tma=0, vec=1)


# ---------------------------------------------------------------------------------------------------------------------------------------------
# 4. stream-K with cluster pairs: forced for every stream-K width, ragged M, N and K; equal to the data-parallel result and to the reference
# ---------------------------------------------------------------------------------------------------------------------------------------------
SK_EPILOGUES = {
    "f32_bias": (F32, dict(bias=True)),
    "f16_inplace_res": (F16, dict(bias=True, res=F16, inplace=True)),   # TMA residual
    "f16_gated": (F16, dict(gated=True, bias_m=True)),
    "f32_scalar_res": (F32, dict(res=F32, store="scalar")),            # direct scalar stores
}


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(SK_EPILOGUES))
@pytest.mark.parametrize("tile_n", SK_TILES)
def test_gemm_exact_stream_k(case, tile_n, stream_k, store_mode):
    """M = 6000: 47 m-blocks (the last pair's second CTA past M, the last block 112 rows); N = 1000: a ragged last tile; K = 1032: 17 k-blocks,
    the last 8 deep.  24 pair rows x 4..8 column blocks = 96..192 tiles for at most 66 clusters: every cluster starts inside a tile"""
    dt, opt = SK_EPILOGUES[case]
    opt = dict(opt)
    store = opt.pop("store", "tma")
    lib().seedx_gemm_set_cluster(2)
    try:
        stream_k(0)
        dp, cfg_dp, _, _ = run_gemm(6000, 1000, 1032, tile_n=tile_n, out_dtype=dt, store=store, set_store=store_mode, seed=3, fake=False, **opt)
        assert (cfg_dp["cluster"], cfg_dp["stream_k"]) == (2, 0)
        dp = dp.clone()
        stream_k(2)
        sk, cfg_sk, _, _ = run_gemm(6000, 1000, 1032, tile_n=tile_n, out_dtype=dt, store=store, set_store=store_mode, seed=3, fake=False, **opt)
        assert (cfg_sk["tile"], cfg_sk["cluster"], cfg_sk["stream_k"]) == (tile_n, 2, 1), cfg_sk
        assert cfg_sk["tma"] == cfg_dp["tma"] == expected_tma(store, tile_n, 1000, opt.get("gated", False), opt.get("res"), dt, 0)
        assert torch.equal(sk, dp)
    finally:
        lib().seedx_gemm_set_cluster(1)


# ---------------------------------------------------------------------------------------------------------------------------------------------
# 5. implicit-GEMM conv
# ---------------------------------------------------------------------------------------------------------------------------------------------
def conv_operands(n, h, w, c, cout, taps, seed):
    """grid image and packed weights [cout, taps*taps*Cpad]; the padded weight columns C..Cpad hold non-zero finite values, which only the
    TMA zero fill of the image's missing channels cancels (a read of the neighbouring pixel's channels would not)"""
    cpad = (c + 63) // 64 * 64
    x64 = grid((n, h, w, c), seed, 16)
    w64 = grid((cout, taps, taps, cpad), seed + 1, 256)
    w64[..., c:] = grid((cout, taps, taps, cpad - c), seed + 2, 256, nonzero=True)
    return x64, w64


def ref_conv(x64, w64, taps):
    """sum over the taps of shifted float64 matmuls: exact on the grid"""
    n, h, w, c = x64.shape
    cout = w64.shape[0]
    p = taps // 2
    xp = F.pad(x64.cuda(), (0, 0, p, p, p, p))
    acc = torch.zeros((n * h * w, cout), dtype=torch.float64, device="cuda")
    wd = w64.cuda()
    for kh in range(taps):
        for kw in range(taps):
            acc += xp[:, kh:kh + h, kw:kw + w, :].reshape(-1, c) @ wd[:, kh, kw, :c].t()
    return acc


CONVS = [
    # n, h,  w,   c,    cout, taps, tile, out, residual, col_part
    (3, 8, 8, 8, 24, 3, 64, F16, True, False),          # a tile holds two 8x8 images: the second tile is half past the last image; h*w = 64: per-element bias_g
    (2, 16, 32, 72, 320, 3, 128, F16, True, True),      # a tile spans 4 image rows; C = 72 straddles two channel chunks; staged bias_g (h*w = 512)
    (1, 8, 64, 200, 640, 3, 256, F32, True, False),     # a tile spans 2 rows; C = 200: 56 padded weight columns in the last chunk
    (1, 4, 256, 320, 320, 1, 160, F16, False, True),    # 1x1; rows cut into 128-pixel segments; a 160-wide tile leaves a ragged last tile
    (2, 16, 32, 1280, 4, 3, 64, F32, False, False),     # UNet conv_out: N = 4, fp32, tile 64
    (1, 8, 64, 72, 3, 3, 64, F32, False, False),        # VAE conv_out: N = 3 (odd: no TMA epilogue), fp32, tile 64
    (1, 4, 256, 1280, 640, 3, 224, F16, True, True),    # C = 1280 (K = 11 520), 256-wide rows, a 192-column last tile
    (3, 8, 8, 320, 320, 3, 96, F16, True, False),       # 96-wide tiles (three wgmma column groups) over multi-image tiles
]


def run_conv(n, h, w, c, cout, taps, tile, dt, residual, col_part, *, seed=0, act=0):
    from seedx_b200 import ops
    x64, w64 = conv_operands(n, h, w, c, cout, taps, seed)
    x = x64.half().cuda()
    wp = w64.reshape(cout, -1).half().cuda()
    M = n * h * w
    bias = nan_tail(grid((cout,), seed + 3, 64, 64, nonzero=True))
    temb = nan_tail(grid((n, cout), seed + 4, 64, 64, nonzero=True))
    res = grid((n, h, w, cout), seed + 5, 64, 64).to(dt).cuda() if residual else None
    part = torch.full((M // 32, cout, 2), float("nan"), device="cuda") if col_part else None
    ob = contiguous_out((n, h, w, cout), dt)
    ops.conv2d_nhwc(x, wp, out=ob.view, taps=taps, bias=bias, bias_g=temb, residual=res, act=act, tile_n=tile, col_part=part)
    cfg = last_config()
    torch.cuda.synchronize()
    ob.check_outside()
    acc = ref_conv(x64, w64, taps)
    x_pre = ref_epilogue(acc, bias=bias, bias_g=temb, bias_g_rows=h * w)
    return ob, x_pre, res, part, cfg, (x, wp, bias, temb)


def check_col_part(part, out, record=None):
    """col_part [M/32, N, 2] = (sum, sum of squares) over each 32-row slab of the STORED values, summed in row order in fp32: a sum of 32 terms
    is within 31 u sum|v| of the exact sum (32 u for the fused squares).  Worst measured on an H100 80GB HBM3 (700 W): 0.23 of the bound"""
    v = out.double().reshape(-1, 32, out.shape[-1])
    s1, s2 = v.sum(1), (v * v).sum(1)
    b1, b2 = 31 * U32 * v.abs().sum(1), 32 * U32 * (v * v).sum(1)
    e1, e2 = (part[..., 0].double() - s1).abs(), (part[..., 1].double() - s2).abs()
    assert bool((e1 <= b1).all()) and bool((e2 <= b2).all())
    return max(float((e1 / b1.clamp_min(1e-300)).max()), float((e2 / b2.clamp_min(1e-300)).max()))


@pytest.mark.gpu
@pytest.mark.parametrize("n,h,w,c,cout,taps,tile,dt,residual,col_part", CONVS)
def test_conv_exact(n, h, w, c, cout, taps, tile, dt, residual, col_part, cluster_mode, record_property):
    ob, x_pre, res, part, cfg, ins = run_conv(n, h, w, c, cout, taps, tile, dt, residual, col_part, seed=c + cout)
    M = n * h * w
    x = x_pre if res is None else r32(x_pre + res.double().reshape(M, cout))
    want = to_out(x, dt).view(n, h, w, cout)
    assert_exact(ob.view, want, "conv")
    tma = int(tile % 32 == 0 and cout % 2 == 0 and cout * (4 if dt == F32 else 2) % 16 == 0)
    vec = int(cout % (4 if dt == F32 else 8) == 0)
    expect(cfg, tile=tile, cluster=exp_cluster(cluster_mode, M, tile), tma=tma, vec=vec)
    if part is not None:
        record_property("col_part_err_over_bound", check_col_part(part, ob.view.reshape(M, cout)))
    xc, wc, bc, tc = (t.cpu() for t in ins)
    got = fake_ops.conv2d_nhwc(xc, wc, taps=taps, bias=bc, bias_g=tc, residual=None if res is None else res.cpu(), out_dtype=dt)
    assert_exact(got, want.cpu(), "CPU test double")


@pytest.mark.gpu
@pytest.mark.parametrize("tile", SK_TILES)
def test_conv_exact_stream_k(tile, stream_k):
    """3x3 conv of a 2 x 64 x 64 x 320 image to 640 channels (45 k-blocks) with per-image bias, fp16 residual and column statistics: 32 pair rows x
    3..5 column blocks for at most 66 clusters, forced to stream-K; equal to the data-parallel result and to the reference"""
    lib().seedx_gemm_set_cluster(2)
    try:
        outs = []
        for mode in (0, 2):
            stream_k(mode)
            ob, x_pre, res, part, cfg, _ = run_conv(2, 64, 64, 320, 640, 3, tile, F16, True, True, seed=5)
            assert (cfg["tile"], cfg["cluster"], cfg["stream_k"], cfg["tma"]) == (tile, 2, mode // 2, 1), cfg
            want = to_out(r32(x_pre + res.double().reshape(-1, 640)), F16).view(ob.view.shape)
            assert_exact(ob.view, want, f"stream_k={mode}")
            check_col_part(part, ob.view.reshape(-1, 640))
            outs.append((ob.view.clone(), part.clone()))
        assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])
    finally:
        lib().seedx_gemm_set_cluster(1)


# ---------------------------------------------------------------------------------------------------------------------------------------------
# 6. non-exact epilogues: elementwise bounds against float64 of the exact pre-activation
# ---------------------------------------------------------------------------------------------------------------------------------------------
# Instruction errors (PTX ISA): ex2.approx.ftz.f32 is within 2 ulp (relative 2^-22) and rcp.approx.ftz.f32 within 1 ulp (2^-23) of the exact
# result over the ranges used here.
E_EX2, E_RCP = 2.0 ** -22, 2.0 ** -23

# gelu_erf_fast (common.cuh): y = max(x, 0) - 0.5 |x| 2^-q(t), t = |x|/sqrt(2), q a degree-5 polynomial; the exact GELU is
# max(x, 0) - 0.5 |x| erfc(t).  So |y - gelu(x)| <= 0.5 |x| (|2^-q - erfc| + 2^-q E_EX2 + 2^-q ln2 |dq|) + u |y|.  The Horner evaluation of q
# rounds five times (|dq| <= 6 u q), and q 2^-q <= 1/(e ln2), so the last term is <= 0.5 |x| * 6 u / e; the rounding of t adds the same order.
# Dense float64 evaluation of the polynomial (test_activation_bounds_cover_the_implementation) gives max |2^-q - erfc| = 8.6e-7, hence
#   |y - gelu(x)| <= |x| (0.5 * 8.6e-7 + 0.5 E_EX2 + 3 u / e + u) + u |y| <= 6.2e-7 |x|;  stated with slack:
GELU_REL_X = 8e-7
# silu (common.cuh): y = x * rcp(1 + ex2(-fl(log2e) * x)).  fl(log2e) and the product each move the exponent by u |x log2e|, i.e. e by u |x|
# relatively; then ex2 (E_EX2), the add (u), rcp (E_RCP) and the final product (u):  |y - silu(x)| <= |y| (2 u |x| + E_EX2 + E_RCP + 2 u).
SILU_REL = lambda x: 2 * U32 * x.abs() + E_EX2 + E_RCP + 2 * U32          # noqa: E731
SILU_SLACK = 1.25
# Worst measured on an H100 80GB HBM3 (700 W): 0.58 of the bound (GEMM, fp16 gated GELU, the fp16 ulp included), 0.50 (conv).


def gelu64(x):
    return 0.5 * x * (1 + torch.special.erf(x / math.sqrt(2)))


def act_ref_and_bound(x, act):
    """float64 activation of the exact pre-activation x and the elementwise bound of the kernel's fp32 value"""
    if act == 1:
        y = gelu64(x)
        return y, GELU_REL_X * x.abs()
    y = x * torch.sigmoid(x)
    return y, SILU_SLACK * SILU_REL(x) * y.abs()


def gelu_fast_coefficients():
    src = open(os.path.join(ROOT, "seed-x_b200", "csrc", "common.cuh")).read()
    body = re.search(r"float gelu_erf_fast\(float x\) \{(.*?)\n\}", src, re.S).group(1)
    lits = [float(v) for v in re.findall(r"(-?\d+\.\d*(?:e-?\d+)?)f", body)]
    return lits[0], lits[1:6]        # 1/sqrt(2), then the Horner coefficients from the highest degree down


def test_activation_bounds_cover_the_implementation():
    """the GELU bound above, re-derived from the polynomial in common.cuh evaluated in float64 over t in [0, 8] (step 1e-5)"""
    s, (c5, c4, c3, c2, c1) = gelu_fast_coefficients()
    assert abs(s - 0.5 ** 0.5) < 1e-12
    t = torch.arange(0, 8, 1e-5, dtype=torch.float64)
    q = ((((c5 * t + c4) * t + c3) * t + c2) * t + c1) * t
    poly = float((torch.exp2(-q) - torch.special.erfc(t)).abs().max())
    derived = 0.5 * poly + 0.5 * E_EX2 + 3 * U32 / math.e + 2 * U32
    assert poly < 1e-6 and derived <= GELU_REL_X, (poly, derived)


@pytest.mark.gpu
@pytest.mark.parametrize("act", [1, 2], ids=["gelu", "silu"])
@pytest.mark.parametrize("gated", [False, True], ids=["plain", "gated"])
@pytest.mark.parametrize("dt", [F16, F32], ids=["f16", "f32"])
@pytest.mark.parametrize("store", ["tma", "scalar"])
def test_gemm_activation_bounds(act, gated, dt, store, store_mode, record_property):
    """operands on a wider grid (a = i/4, w = j/64): pre-activations over about [-16, 16], the whole curved part of both activations"""
    M, N, K = 300, 392, 200
    out, cfg, acc, (a, w, kw) = run_gemm(M, N, K, tile_n=128, out_dtype=dt, store=store, set_store=store_mode, act=act, gated=gated, bias=True,
                                         seed=11, a_den=4, w_den=64, fake=False)
    assert cfg["tma"] == expected_tma(store, 128, N, gated, None, dt, 0)
    x = acc + kw["bias"].double()                                  # the exact pre-activation
    if gated:
        g, bnd_g = act_ref_and_bound(x[:, 1::2], act)
        v = x[:, 0::2]
        y = v * g
        bound = v.abs() * bnd_g + U32 * y.abs()
    else:
        y, bound = act_ref_and_bound(x, act)
    err = (out.double() - y).abs()
    if dt == F16:
        bound = bound + ulp16(y)
    err[torch.isnan(err)] = float("inf")
    ratio = float((err / bound.clamp_min(1e-30)).max())
    record_property("worst_err", float(err.max()))
    record_property("worst_err_over_bound", ratio)
    assert ratio <= 1.0
    # the CPU test double on the same inputs: fp32 torch activations, within the same bound
    fk = fake_ops.gemm(a.cpu(), w.cpu(), bias=kw["bias"].cpu(), act=act, gated=gated, out_dtype=dt)
    ferr = (fk.double() - y.cpu()).abs()
    assert bool((ferr <= bound.cpu()).all())


@pytest.mark.gpu
@pytest.mark.parametrize("act", [1, 2], ids=["gelu", "silu"])
def test_conv_activation_bounds(act, record_property):
    ob, x_pre, _, _, cfg, ins = run_conv(2, 16, 32, 72, 320, 3, 128, F16, False, False, seed=9, act=act)
    y, bound = act_ref_and_bound(x_pre, act)
    y = y.view(ob.view.shape)
    bound = bound.view(ob.view.shape) + ulp16(y)
    err = (ob.view.double() - y).abs()
    err[torch.isnan(err)] = float("inf")
    ratio = float((err / bound).max())
    record_property("worst_err_over_bound", ratio)
    assert ratio <= 1.0
    xc, wc, bc, tc = (t.cpu() for t in ins)
    fk = fake_ops.conv2d_nhwc(xc, wc, taps=3, bias=bc, bias_g=tc, act=act, out_dtype=F16)
    assert bool(((fk.double() - y.cpu()).abs() <= bound.cpu()).all())


def stats_from_parts(parts, cols, eps):
    """float64 (mean, rstd) from row partials [P, M, 2] and the bound of the fp32 version the kernels form (partials added in chunk order:
    |d s| <= P u sum|s_k|; mean = s1 / cols exact for a power-of-two cols; var = s2/cols - mean^2 rounds twice; rsqrtf is within 2 ulp)"""
    p = parts.double()
    P = p.shape[0]
    s1, s2 = p[..., 0].sum(0), p[..., 1].sum(0)
    mean = s1 / cols
    var = (s2 / cols - mean * mean).clamp_min(0)
    rstd = torch.rsqrt(var + eps)
    dmean = P * U32 * p[..., 0].abs().sum(0) / cols
    dvar = P * U32 * s2 / cols + 2 * mean.abs() * dmean + 2 * U32 * (s2 / cols + mean * mean) + U32 * (var + eps)
    drstd = rstd * (0.5 * dvar / (var + eps) + 2.0 ** -22 + U32)
    return mean, rstd, 1.01 * dmean + 1e-30, 1.01 * drstd


def check_ln_epilogue(out, acc, mean, rstd, dmean, drstd, colsum, bias, slack=1.01):
    """out = rstd * acc + (bias - rstd * mean * colsum) in three fp32 roundings (-mean*rstd, the inner fma, the outer fma):
    |out - x| <= u (2 |mean rstd colsum| + |bias| + |x|) (x1.01), plus what the statistics' own error moves x by"""
    cs, b = colsum.double()[None, :], bias.double()[None, :]
    m, r = mean[:, None], rstd[:, None]
    x = r * (acc - m * cs) + b
    bound = slack * U32 * (2 * (m * r * cs).abs() + b.abs() + x.abs()) + (acc - m * cs).abs() * drstd[:, None] + r * cs.abs() * dmean[:, None]
    err = (out.double() - x).abs()
    err[torch.isnan(err)] = float("inf")
    ratio = float((err / bound.clamp_min(1e-30)).max())
    assert ratio <= 1.0, ratio
    return ratio, float(err.max())


# Worst measured on an H100 80GB HBM3 (700 W): rstd of seedx_row_stats 1.7e-7 relative (bound 1.4e-6); epilogue-formed statistics 0.12 of
# their bound; the (parts, colsum, eps) epilogue 0.42 of its bound; the (stats, colsum) epilogue 1.7e-6 absolute, within its bound.
@pytest.mark.gpu
def test_gemm_folded_layernorm_bounds(cluster_mode, record_property):
    """Folded LayerNorm, both forms.  (stats, colsum): the statistics of seedx_row_stats against float64 first, then the epilogue against
    float64 rstd*(acc - mean*colsum) + bias formed from the kernel's OWN statistics, so a statistics error and an epilogue error show apart.
    (parts, colsum, eps): a producing GEMM writes row_part and row_stats; both against float64 of the values, then the consumer's epilogue
    against float64 statistics of those partials."""
    from seedx_b200 import ops
    M, K, N, eps = 256, 1024, 384, 1e-5
    x64 = grid((M, K), 31, 16) + grid((M, 1), 32, 4)             # rows with a mean away from zero: the cancellation in acc - mean*colsum
    x = x64.half().cuda()
    wf = grid((N, K), 33, 256).half().cuda()
    colsum = (wf.double().sum(1)).float()                         # exact on the grid
    bias = grid((N,), 34, 64, 64, nonzero=True).float().cuda()
    acc = x.double() @ wf.double().t()
    # --- seedx_row_stats: two-pass fp32.  mean: the grid sum is exact and cols is a power of two -> exact.  rstd: the squared deviations round
    # once each and are summed 64 per lane, then over 5 shuffle levels: |d q| <= (cols/32 + 6) u q; then /cols, + eps and rsqrtf (2 ulp)
    st = ops.row_stats(x, eps)
    xd = x.double()
    mean64, var64 = xd.mean(1), xd.var(1, unbiased=False)
    rstd64 = torch.rsqrt(var64 + eps)
    assert torch.equal(st[:, 0].double(), mean64)
    rel_r = ((st[:, 1].double() - rstd64) / rstd64).abs().max().item()
    bound_r = 0.5 * (K / 32 + 6) * U32 + 2.0 ** -22 + 2 * U32
    record_property("row_stats_rstd_rel", rel_r)
    assert rel_r <= bound_r
    out = OutBuf((M, N), F32, N + 8)
    ops.gemm(x, wf, out=out.view, bias=bias, ln=(st, colsum))
    torch.cuda.synchronize()
    out.check_outside()
    zero = torch.zeros(M, dtype=torch.float64, device="cuda")
    ratio1, err1 = check_ln_epilogue(out.view, acc, st[:, 0].double(), st[:, 1].double(), zero, zero, colsum, bias)
    record_property("ln_stats_epilogue_err", err1)
    # --- producer GEMM with row_part and row_stats (fp16 output, TMA epilogue), then the consumer with ln=(parts, colsum, eps)
    a0, w0 = grid((M, 512), 35, 16).half().cuda(), grid((K, 512), 36, 256).half().cuda()
    b0 = grid((K,), 37, 8, 64, nonzero=True).float().cuda()                 # shifts the row means
    rp = torch.full((K // 32, M, 2), float("nan"), device="cuda")
    st_epi = torch.full((M, 2), float("nan"), device="cuda")
    tickets = torch.zeros((M // 32,), device="cuda", dtype=torch.int32)
    xp = ops.gemm(a0, w0, bias=b0, row_part=rp, row_stats=(st_epi, tickets, eps))
    assert last_config()["tma"] == 1 and int(tickets.abs().sum()) == 0
    xpre = a0.double() @ w0.double().t() + b0.double()                     # exact: the fp32 values the partials are summed from
    assert torch.equal(xp, xpre.float().half())
    v = xpre.view(M, K // 32, 32)
    e1 = (rp[..., 0].t().double() - v.sum(-1)).abs()
    e2 = (rp[..., 1].t().double() - (v * v).sum(-1)).abs()
    assert bool((e1 <= 31 * U32 * v.abs().sum(-1)).all()) and bool((e2 <= 32 * U32 * (v * v).sum(-1)).all())
    mean, rstd, dmean, drstd = stats_from_parts(rp, K, eps)
    em, er = (st_epi[:, 0].double() - mean).abs(), (st_epi[:, 1].double() - rstd).abs()
    record_property("row_stats_from_parts_err_over_bound", max(float((em / dmean).max()), float((er / drstd).max())))
    assert bool((em <= dmean).all()) and bool((er <= drstd).all())
    out2 = OutBuf((M, N), F32, N + 8)
    ops.gemm(xp, wf, out=out2.view, bias=bias, ln=(rp, colsum, eps))
    torch.cuda.synchronize()
    out2.check_outside()
    acc2 = xp.double() @ wf.double().t()
    ratio2, err2 = check_ln_epilogue(out2.view, acc2, mean, rstd, dmean, drstd, colsum, bias)
    record_property("ln_parts_epilogue_err_over_bound", ratio2)
    # the CPU test double (fp32 torch: acc - mean*colsum, * rstd, + bias: four roundings, each within u of |x| + |bias| + |mean rstd colsum|)
    fk = fake_ops.gemm(x.cpu(), wf.cpu(), bias=bias.cpu(), ln=(st.cpu(), colsum.cpu()), out_dtype=F32)
    check_ln_epilogue(fk, acc.cpu(), st[:, 0].double().cpu(), st[:, 1].double().cpu(), zero.cpu(), zero.cpu(), colsum.cpu(), bias.cpu(), slack=2.02)
