"""Thin Python wrappers over the C ABI (include/seedx.h).

Tensors are torch CUDA tensors used purely as device-memory handles: every wrapper passes raw pointers,
sizes and the current CUDA stream to libseedx.so; no torch compute op runs in here.
"""
import ctypes as C

import torch

from . import _lib
from ._lib import ACT_GELU, ACT_NONE, ACT_SILU, F16, F32, GemmArgs, check, lib  # noqa: F401


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def _dt(t):
    if t.dtype == torch.float16:
        return F16
    if t.dtype == torch.float32:
        return F32
    raise TypeError(f"unsupported dtype {t.dtype}")


def _require_cuda(*ts):
    for t in ts:
        if t is not None and not t.is_cuda:
            raise _lib.SeedxError("seedx ops need CUDA tensors: there is no CPU fallback path")


_workspace = {}


def _ensure_workspace(device):
    """stream-K fix-up workspace of seedx_gemm_f16 (include/seedx.h: seedx_gemm_set_workspace), one per process: 16 KB of flags (zero) + room for
    one fp32 partial tile per CTA (132 x 128 x 256 x 4 B = 17.3 MB).  Allocated on the first GEMM — before any CUDA-graph capture, which
    always follows an eager warm-up pass."""
    key = torch.device(device).index if torch.device(device).index is not None else torch.cuda.current_device()
    if key not in _workspace:
        if not hasattr(lib(), "seedx_gemm_set_workspace"):       # an older build of the library loaded through SEEDX_LIB (tools/ab_gemm.py)
            _workspace[key] = None
            return None
        buf = torch.zeros((24 * 1024 * 1024 + 16384,), device=device, dtype=torch.uint8)
        check(lib().seedx_gemm_set_workspace(C.c_void_p(buf.data_ptr()), C.c_int64(buf.numel())), "seedx_gemm_set_workspace")
        _workspace[key] = buf
    return _workspace[key]


def gemm(a, w, out=None, *, bias=None, bias_m=None, bias_g=None, bias_g_rows=0, residual=None, res_row_mod=0,
         act=ACT_NONE, gated=False, alpha=1.0, out_dtype=torch.float16, tile_n=0, ln=None, dynamic_b=False, row_part=None, col_part=None,
         row_stats=None, a_scale=None, w_scale=None):
    """out[b,m,n] = epi(alpha * a[b,m,:] . w[(b,)n,:]).

    a: fp16 [M,K] or [B,M,K] (last dim contiguous); w: fp16 [N,K] or [B,N,K]; returns/updates out [.., M, N_out].
    ln = (row_stats fp32 [M,2], colsum fp32 [N]): LayerNorm of `a` folded into the epilogue (w = gamma-scaled weights, bias = W.beta + b);
         (row partials fp32 [K/32, M, 2], colsum, eps): the same with the statistics formed from the partial sums the producer of `a` emitted.
    row_stats = (stats fp32 [M,2], tickets int32 [M/32] zeroed, eps): with row_part, (mean, rstd) per row of the output written by this launch itself.
    row_part / col_part: fp32 outputs [N/32, M, 2] / [M/32, N, 2] receiving partial (sum, sum of squares) of the stored output per row chunk /
         per 32-row slab and column, for the LayerNorm / GroupNorm that reads this output next (see stats_buffers()).
    dynamic_b: w is an activation written by the kernel launched just before (default: weights, prefetched before the PDL wait).
    a, w float8_e4m3fn (2-D only) with a_scale fp32 [M] and w_scale fp32 [N] (row m of the true a = a_scale[m] * a[m], likewise w): seedx_gemm_fp8,
         whose epilogue scales the accumulator by a_scale[m] * w_scale[n] and then runs as above.
    """
    _require_cuda(a, w, out, bias, residual, a_scale, w_scale)
    _ensure_workspace(a.device)
    fp8 = a.dtype == torch.float8_e4m3fn
    if fp8:
        if w.dtype != torch.float8_e4m3fn or a_scale is None or w_scale is None:
            raise _lib.SeedxError("an FP8 gemm needs float8_e4m3fn a and w and both a_scale and w_scale")
        for t, n in ((a_scale, a.shape[-2]), (w_scale, w.shape[-2])):
            assert t.dtype == torch.float32 and t.is_contiguous() and t.numel() == n
    else:
        assert a.dtype == torch.float16 and w.dtype == torch.float16 and a_scale is None and w_scale is None
    assert a.stride(-1) == 1 and w.stride(-1) == 1
    batched = a.dim() == 3
    B = a.shape[0] if batched else 1
    M, K = a.shape[-2], a.shape[-1]
    N = w.shape[-2]
    assert w.shape[-1] == K, (a.shape, w.shape)
    n_out = N // 2 if gated else N
    if out is None:
        shape = (B, M, n_out) if batched else (M, n_out)
        out = torch.empty(shape, device=a.device, dtype=out_dtype)
    assert out.stride(-1) == 1 and out.shape[-1] == n_out and out.shape[-2] == M
    g = GemmArgs()
    g.A, g.B, g.D = a.data_ptr(), w.data_ptr(), out.data_ptr()
    g.M, g.N, g.K, g.batch = M, N, K, B
    g.lda, g.ldb, g.ldd = a.stride(-2), w.stride(-2), out.stride(-2)
    g.strideA = a.stride(0) if batched else 0
    g.strideB = w.stride(0) if (w.dim() == 3) else 0
    g.strideD = out.stride(0) if batched else 0
    g.alpha = alpha
    for name, t in (("bias_n", bias), ("bias_m", bias_m), ("bias_g", bias_g)):
        if t is not None:
            assert t.dtype == torch.float32 and t.is_contiguous()
            setattr(g, name, t.data_ptr())
    g.bias_g_rows = bias_g_rows
    if residual is not None:
        assert residual.stride(-1) == 1
        g.residual = residual.data_ptr()
        g.residual_dtype = _dt(residual)
        g.ldr = residual.stride(-2)
        g.strideR = residual.stride(0) if (batched and residual.dim() == 3) else 0
        g.res_row_mod = res_row_mod
    g.act, g.gated, g.out_dtype = act, int(gated), _dt(out)
    g.tile_n = tile_n
    if ln is not None:
        st, cs = ln[0], ln[1]
        assert st.dtype == torch.float32 and st.is_contiguous() and cs.dtype == torch.float32 and cs.is_contiguous() and cs.numel() == N
        if len(ln) == 3:
            assert st.numel() == 2 * M * (K // 32) and K % 32 == 0
            g.ln_parts, g.ln_eps = K // 32, float(ln[2])
        else:
            assert st.numel() == 2 * M
        g.ln_stats, g.ln_colsum = st.data_ptr(), cs.data_ptr()
    _set_parts(g, row_part, col_part, M, n_out)
    if row_stats is not None:          # (stats fp32 [M, 2], tickets int32 [M/32] (zero), eps): the last epilogue warp of a 32-row slab finalizes it
        st, tk, eps = row_stats
        assert row_part is not None and st.dtype == torch.float32 and st.numel() == 2 * M and tk.dtype == torch.int32 and tk.numel() >= M // 32
        g.row_stats_out, g.row_tickets, g.row_eps = st.data_ptr(), tk.data_ptr(), float(eps)
    g.b_dynamic = int(dynamic_b)
    if fp8:
        check(lib().seedx_gemm_fp8(C.byref(g), _ptr(a_scale), _ptr(w_scale), _stream()), "seedx_gemm_fp8")
    else:
        check(lib().seedx_gemm_f16(C.byref(g), _stream()), "seedx_gemm_f16")
    return out


def quant_rows_fp8(x, q=None, scale=None):
    """Per-row FP8 quantisation of fp16 x [rows, cols] (row-strided view): scale[r] = amax|x[r]| / 448 (1 for a zero row), q = e4m3(x / scale)
    -> (q float8_e4m3fn [rows, cols], scale fp32 [rows]); bit-identical to llm.quantize_fp8_rows(x.float()).  A default q is a view of a buffer
    whose rows are padded to 16 bytes (the A operand of an FP8 gemm)."""
    _require_cuda(x, q, scale)
    assert x.dtype == torch.float16 and x.dim() == 2 and x.stride(1) == 1
    rows, cols = x.shape
    if q is None:
        q = torch.empty((rows, (cols + 15) // 16 * 16), device=x.device, dtype=torch.float8_e4m3fn)[:, :cols]
    if scale is None:
        scale = torch.empty((rows,), device=x.device, dtype=torch.float32)
    assert q.dtype == torch.float8_e4m3fn and q.shape == x.shape and q.stride(1) == 1
    assert scale.dtype == torch.float32 and scale.is_contiguous() and scale.numel() == rows
    check(lib().seedx_quant_rows_fp8(_ptr(x), _i64(x.stride(0)), _i64(rows), _i64(cols), _ptr(q), _i64(q.stride(0)), _ptr(scale), _stream()),
          "seedx_quant_rows_fp8")
    return q, scale


def quant_images_fp8(x, q=None, scale=None, ws=None):
    """Per-image FP8 quantisation of a contiguous fp16 tensor x [n, ...] (an NHWC map): scale[i] = amax|x[i]| / 448 (1 for an all-zero image),
    q = e4m3(x / scale[i]) -> (q float8_e4m3fn shaped like x, scale fp32 [n]); bit-identical to llm.quantize_fp8_rows(x.view(n, -1).float()).
    The A operand of an FP8 conv2d_nhwc.  ws: scratch of the per-chunk maxima (quant_images_fp8_ws(...), a few KB), allocated per call
    when not given."""
    _require_cuda(x, q, scale)
    assert x.dtype == torch.float16 and x.is_contiguous()
    n = x.shape[0]
    per_image = x.numel() // n
    if q is None:
        q = torch.empty(x.shape, device=x.device, dtype=torch.float8_e4m3fn)
    if scale is None:
        scale = torch.empty((n,), device=x.device, dtype=torch.float32)
    assert q.dtype == torch.float8_e4m3fn and q.is_contiguous() and q.numel() == x.numel()
    assert scale.dtype == torch.float32 and scale.is_contiguous() and scale.numel() == n
    if ws is None:
        ws = quant_images_fp8_ws(n, per_image, x.device)
    assert ws.numel() * ws.element_size() >= lib().seedx_quant_images_fp8_ws_bytes(_i64(n), _i64(per_image))
    check(lib().seedx_quant_images_fp8(_ptr(x), _i64(n), _i64(per_image), _ptr(q), _ptr(scale), _ptr(ws), _stream()), "seedx_quant_images_fp8")
    return q, scale


def quant_images_fp8_ws(n, per_image, device):
    """scratch for quant_images_fp8 of n images of per_image values: one fp32 maximum per 8192-value chunk"""
    nbytes = int(lib().seedx_quant_images_fp8_ws_bytes(_i64(n), _i64(per_image)))
    return torch.empty(((nbytes + 3) // 4,), device=device, dtype=torch.float32)


def row_finalize(row_part, eps, out=None):
    """(mean, rstd) per row from the row partials [cols/32, rows, 2] a producing GEMM emitted (gemm(..., row_part=...)) -> fp32 [rows, 2]"""
    _require_cuda(row_part, out)
    assert row_part.dtype == torch.float32 and row_part.is_contiguous() and row_part.dim() == 3 and row_part.shape[2] == 2
    nparts, rows = row_part.shape[0], row_part.shape[1]
    if out is None:
        out = torch.empty((rows, 2), device=row_part.device, dtype=torch.float32)
    check(lib().seedx_row_stats_from_partials(_ptr(row_part), C.c_int(nparts), C.c_int64(rows), C.c_int64(32 * nparts), C.c_float(eps), _ptr(out), _stream()),
          "seedx_row_stats_from_partials")
    return out


def _set_parts(g, row_part, col_part, M, N):
    if row_part is not None:
        assert row_part.dtype == torch.float32 and row_part.is_contiguous() and row_part.numel() == 2 * M * (N // 32) and N % 32 == 0
        g.row_part = row_part.data_ptr()
    if col_part is not None:
        assert col_part.dtype == torch.float32 and col_part.is_contiguous() and col_part.numel() == 2 * N * (M // 32) and M % 32 == 0
        g.col_part = col_part.data_ptr()


def row_stats(x, eps, out=None):
    """(mean, rstd) per row of an fp16 matrix [rows, cols] -> fp32 [rows, 2] (LayerNorm statistics for gemm(..., ln=...))."""
    _require_cuda(x, out)
    assert x.dtype == torch.float16 and x.dim() == 2 and x.stride(1) == 1
    if out is None:
        out = torch.empty((x.shape[0], 2), device=x.device, dtype=torch.float32)
    check(lib().seedx_row_stats(_ptr(x), _dt(x), C.c_int64(x.stride(0)), C.c_int64(x.shape[0]), C.c_int64(x.shape[1]), C.c_float(eps), _ptr(out),
                                _stream()), "seedx_row_stats")
    return out


def conv2d_nhwc(x, w, out=None, *, taps=3, bias=None, bias_g=None, residual=None, act=ACT_NONE,
                out_dtype=torch.float16, tile_n=0, alpha=1.0, col_part=None, a_scale=None, w_scale=None):
    """Stride-1 'same' convolution as an implicit GEMM.  x: fp16 NHWC [N,H,W,C]; w: fp16 [Cout, taps*taps*roundup(C,64)]
    (k = (kh*taps+kw)*Cpad + c); out: NHWC [N,H,W,Cout].  bias_g: fp32 [N, Cout] added per image.
    x, w float8_e4m3fn with a_scale fp32 [N] (image i of the true x = a_scale[i] * x[i]) and w_scale fp32 [Cout], w [Cout, taps*taps*roundup(C,128)]:
    seedx_conv_fp8, whose epilogue scales the accumulator by a_scale[image] * w_scale[n] and then runs as above."""
    _require_cuda(x, w, out, bias, residual, a_scale, w_scale)
    _ensure_workspace(x.device)
    fp8 = x.dtype == torch.float8_e4m3fn
    if fp8:
        if w.dtype != torch.float8_e4m3fn or a_scale is None or w_scale is None:
            raise _lib.SeedxError("an FP8 conv needs float8_e4m3fn x and w and both a_scale and w_scale")
        for t, n_ in ((a_scale, x.shape[0]), (w_scale, w.shape[0])):
            assert t.dtype == torch.float32 and t.is_contiguous() and t.numel() == n_
    else:
        assert x.dtype == torch.float16 and a_scale is None and w_scale is None
    assert x.is_contiguous() and w.is_contiguous()
    n, h, wd, c = x.shape
    cout, K = w.shape
    if out is None:
        out = torch.empty((n, h, wd, cout), device=x.device, dtype=out_dtype)
    assert out.is_contiguous()
    g = GemmArgs()
    g.A, g.B, g.D = x.data_ptr(), w.data_ptr(), out.data_ptr()
    g.M, g.N, g.K, g.batch = n * h * wd, cout, K, 1
    g.lda, g.ldb, g.ldd = c, K, cout
    g.alpha = alpha
    if bias is not None:
        assert bias.dtype == torch.float32
        g.bias_n = bias.data_ptr()
    if bias_g is not None:
        assert bias_g.dtype == torch.float32 and bias_g.is_contiguous()
        g.bias_g = bias_g.data_ptr()
        g.bias_g_rows = h * wd
    if residual is not None:
        assert residual.is_contiguous()
        g.residual = residual.data_ptr()
        g.residual_dtype = _dt(residual)
        g.ldr = cout
    g.act, g.out_dtype = act, _dt(out)
    g.conv_taps_h = g.conv_taps_w = taps
    g.conv_n, g.conv_h, g.conv_w, g.conv_c = n, h, wd, c
    g.tile_n = tile_n
    _set_parts(g, None, col_part, n * h * wd, cout)
    if fp8:
        check(lib().seedx_conv_fp8(C.byref(g), _ptr(a_scale), _ptr(w_scale), _stream()), "seedx_conv_fp8")
    else:
        check(lib().seedx_gemm_f16(C.byref(g), _stream()), "seedx_gemm_f16(conv)")
    return out


class AttnArgs(C.Structure):
    _fields_ = [
        ("q", C.c_void_p), ("k", C.c_void_p), ("v", C.c_void_p), ("o", C.c_void_p),
        ("q_sb", C.c_int64), ("q_sh", C.c_int64), ("q_ss", C.c_int64),
        ("k_sb", C.c_int64), ("k_sh", C.c_int64), ("k_ss", C.c_int64),
        ("v_sb", C.c_int64), ("v_sh", C.c_int64), ("v_ss", C.c_int64),
        ("o_sb", C.c_int64), ("o_sh", C.c_int64), ("o_ss", C.c_int64),
        ("batch", C.c_int32), ("heads", C.c_int32), ("sq", C.c_int32), ("sk", C.c_int32), ("d", C.c_int32),
        ("scale", C.c_float), ("causal", C.c_int32),
    ]


def attention(q, k, v, out, *, scale, causal=False):
    """q/k/v/out: fp16 4-D views indexed [batch, head, seq, d] (any strides with d contiguous; q batch stride may be 0)."""
    _require_cuda(q, k, v, out)
    for t in (q, k, v, out):
        assert t.dtype == torch.float16 and t.dim() == 4 and t.stride(3) == 1
    B, H, Sq, D = out.shape
    Sk = k.shape[2]
    a = AttnArgs()
    a.q, a.k, a.v, a.o = q.data_ptr(), k.data_ptr(), v.data_ptr(), out.data_ptr()
    a.q_sb, a.q_sh, a.q_ss = (q.stride(0) if q.shape[0] > 1 or B == 1 else 0), q.stride(1), q.stride(2)
    if q.shape[0] == 1 and B > 1:
        a.q_sb = 0
    a.k_sb, a.k_sh, a.k_ss = k.stride(0), k.stride(1), k.stride(2)
    a.v_sb, a.v_sh, a.v_ss = v.stride(0), v.stride(1), v.stride(2)
    a.o_sb, a.o_sh, a.o_ss = out.stride(0), out.stride(1), out.stride(2)
    a.batch, a.heads, a.sq, a.sk, a.d = B, H, Sq, Sk, D
    a.scale, a.causal = float(scale), int(causal)
    check(lib().seedx_attention_f16(C.byref(a), _stream()), "seedx_attention_f16")
    return out


def layernorm(x, gamma, beta, eps, out=None, *, out_dtype=torch.float16, rms=False, add=None, out2=None):
    """LayerNorm / RMSNorm over the last dim of a 2-D (rows, cols) view; optional out2 = y + add[row % add_rows]."""
    _require_cuda(x, out)
    x2 = x.reshape(-1, x.shape[-1])
    assert x2.stride(1) == 1
    rows, cols = x2.shape
    if out is None:
        out = torch.empty((rows, cols), device=x.device, dtype=out_dtype)
    o2 = out.reshape(-1, cols)
    assert o2.stride(1) == 1
    if add is not None:
        assert add.dtype == torch.float32 and add.is_contiguous() and add.shape[-1] == cols
        if out2 is None:
            out2 = torch.empty_like(o2)
        assert out2.stride(-2) == o2.stride(0) and out2.dtype == out.dtype
    fn = lib().seedx_layernorm
    check(fn(_ptr(x2), _dt(x2), C.c_int64(x2.stride(0)), _ptr(gamma), _ptr(beta), _ptr(o2), _dt(o2), C.c_int64(o2.stride(0)),
             _ptr(out2), _ptr(add), C.c_int64(add.shape[0] if add is not None else 0), C.c_int64(rows), C.c_int64(cols),
             C.c_float(eps), C.c_int(int(rms)), _stream()), "seedx_layernorm")
    return (out, out2) if add is not None else out


def groupnorm_ws(n, groups, device):
    """Scratch for groupnorm_nhwc (final fp64 statistics + per-CTA partials + tickets); reusable across layers of one batch size."""
    nbytes = lib().seedx_groupnorm_ws_bytes(C.c_int64(n), C.c_int(groups))
    return torch.empty(((nbytes + 7) // 8,), device=device, dtype=torch.float64)


def groupnorm_nhwc(x1, gamma, beta, eps, *, x2=None, silu=False, groups=32, out=None, raw_out=None, stats_ws=None, part1=None, part2=None):
    """GroupNorm(+SiLU) over NHWC fp16 [N,H,W,C1] (optionally channel-concatenated with x2 [N,H,W,C2]).
    part1 (and part2 when x2 is given): the col_part statistics the kernels that produced x1 / x2 emitted — the statistics pass over the tensor
    is then replaced by a finalize over the partials."""
    _require_cuda(x1, x2, out)
    assert x1.dtype == torch.float16 and x1.is_contiguous()
    n, h, w, c1 = x1.shape
    c2 = 0
    if x2 is not None:
        assert x2.dtype == torch.float16 and x2.is_contiguous() and x2.shape[:3] == x1.shape[:3]
        c2 = x2.shape[3]
    if out is None:
        out = torch.empty((n, h, w, c1 + c2), device=x1.device, dtype=torch.float16)
    if stats_ws is None:
        stats_ws = groupnorm_ws(n, groups, x1.device)
    assert stats_ws.numel() * stats_ws.element_size() >= lib().seedx_groupnorm_ws_bytes(C.c_int64(n), C.c_int(groups))
    if part1 is not None and (x2 is None or part2 is not None) and (h * w) % 32 == 0:
        assert part1.dtype == torch.float32 and part1.numel() == 2 * c1 * (n * h * w // 32)
        assert part2 is None or (part2.dtype == torch.float32 and part2.numel() == 2 * c2 * (n * h * w // 32))
        check(lib().seedx_groupnorm_nhwc_from_partials(_ptr(x1), C.c_int64(c1), _ptr(part1), _ptr(x2), C.c_int64(c2), _ptr(part2), C.c_int64(n),
                                                       C.c_int64(h * w), C.c_int(groups), _ptr(gamma), _ptr(beta), C.c_float(eps), C.c_int(int(silu)),
                                                       _ptr(out), _ptr(raw_out), _ptr(stats_ws), _stream()), "seedx_groupnorm_nhwc_from_partials")
        return out
    check(lib().seedx_groupnorm_nhwc(_ptr(x1), C.c_int64(c1), _ptr(x2), C.c_int64(c2), C.c_int64(n), C.c_int64(h * w), C.c_int(groups),
                                     _ptr(gamma), _ptr(beta), C.c_float(eps), C.c_int(int(silu)), _ptr(out), _ptr(raw_out), _ptr(stats_ws),
                                     _stream()), "seedx_groupnorm_nhwc")
    return out


def patchify(x, patch, kpad):
    _require_cuda(x)
    assert x.is_contiguous() and x.dim() == 4
    n, c, h, w = x.shape
    out = torch.empty((n * (h // patch) * (w // patch), kpad), device=x.device, dtype=torch.float16)
    check(lib().seedx_patchify(_ptr(x), _dt(x), C.c_int64(n), C.c_int64(c), C.c_int64(h), C.c_int64(w), C.c_int64(patch), _ptr(out),
                               C.c_int64(kpad), _stream()), "seedx_patchify")
    return out


def cast(x, dtype, out=None):
    _require_cuda(x)
    assert x.is_contiguous()
    if out is None:
        out = torch.empty(x.shape, device=x.device, dtype=dtype)
    check(lib().seedx_cast(_ptr(x), _dt(x), _ptr(out), _dt(out), C.c_int64(x.numel()), _stream()), "seedx_cast")
    return out


def avgpool_tokens(x, k):
    _require_cuda(x)
    assert x.is_contiguous() and x.dim() == 3
    n, t, c = x.shape
    out = torch.empty((n, t // k, c), device=x.device, dtype=x.dtype)
    check(lib().seedx_avgpool_tokens(_ptr(x), _dt(x), C.c_int64(n), C.c_int64(t), C.c_int64(c), C.c_int64(k), _ptr(out), _stream()),
          "seedx_avgpool_tokens")
    return out


def _i64(v):
    return C.c_int64(int(v))


def im2col_nhwc(x, k, stride, pad_before, ho, wo):
    _require_cuda(x)
    assert x.dtype == torch.float16 and x.is_contiguous()
    n, h, w, c = x.shape
    out = torch.empty((n * ho * wo, k * k * c), device=x.device, dtype=torch.float16)
    check(lib().seedx_im2col_nhwc(_ptr(x), _i64(n), _i64(h), _i64(w), _i64(c), C.c_int(k), C.c_int(stride), C.c_int(pad_before), _i64(ho),
                                  _i64(wo), _ptr(out), _stream()), "seedx_im2col_nhwc")
    return out


def upsample2x_nhwc(x):
    _require_cuda(x)
    assert x.dtype == torch.float16 and x.is_contiguous()
    n, h, w, c = x.shape
    out = torch.empty((n, 2 * h, 2 * w, c), device=x.device, dtype=torch.float16)
    check(lib().seedx_upsample2x_nhwc(_ptr(x), _i64(n), _i64(h), _i64(w), _i64(c), _ptr(out), _stream()), "seedx_upsample2x_nhwc")
    return out


def timestep_embedding(t, dim, out):
    """t: fp32 [count]; out: fp16 2-D view [count, >=dim] (row stride arbitrary) receiving [cos|sin]."""
    _require_cuda(t, out)
    assert t.dtype == torch.float32 and t.is_contiguous() and out.dtype == torch.float16 and out.stride(-1) == 1
    check(lib().seedx_timestep_embedding(_ptr(t), _i64(t.numel()), C.c_int(dim), _ptr(out), _i64(out.stride(0)), _stream()),
          "seedx_timestep_embedding")
    return out


def unary_f16(x, out=None, act=ACT_NONE):
    """fp16 out[r,c] = act(x[r,c]) over 2-D (possibly row-strided) views."""
    _require_cuda(x, out)
    assert x.dim() == 2 and x.stride(1) == 1
    if out is None:
        out = torch.empty(x.shape, device=x.device, dtype=torch.float16)
    assert out.dtype == torch.float16 and out.stride(1) == 1 and out.shape == x.shape
    check(lib().seedx_unary_f16(_ptr(x), _dt(x), _i64(x.shape[0]), _i64(x.shape[1]), _i64(x.stride(0)), _ptr(out), _i64(out.stride(0)),
                                C.c_int(act), _stream()), "seedx_unary_f16")
    return out


def softmax_rows(x, scale, out=None):
    _require_cuda(x, out)
    assert x.dim() == 2 and x.stride(1) == 1
    if out is None:
        out = torch.empty(x.shape, device=x.device, dtype=torch.float16)
    check(lib().seedx_softmax_rows(_ptr(x), _dt(x), _i64(x.stride(0)), _i64(x.shape[0]), _i64(x.shape[1]), C.c_float(scale), _ptr(out),
                                   _i64(out.stride(0)), _stream()), "seedx_softmax_rows")
    return out


def nchw_to_nhwc_f16(x, cpad, scale=1.0, out=None):
    _require_cuda(x, out)
    assert x.dtype == torch.float32 and x.is_contiguous() and x.dim() == 4
    n, c, h, w = x.shape
    if out is None:
        out = torch.empty((n, h, w, cpad), device=x.device, dtype=torch.float16)
    check(lib().seedx_nchw_to_nhwc_f16(_ptr(x), _i64(n), _i64(c), _i64(h * w), _i64(cpad), C.c_float(scale), _ptr(out), _stream()),
          "seedx_nchw_to_nhwc_f16")
    return out


def nhwc_to_nchw_f32(x, c, scale=1.0):
    _require_cuda(x)
    assert x.is_contiguous() and x.dim() == 4
    n, h, w, ldc = x.shape
    out = torch.empty((n, c, h, w), device=x.device, dtype=torch.float32)
    check(lib().seedx_nhwc_to_nchw_f32(_ptr(x), _dt(x), _i64(n), _i64(c), _i64(h * w), _i64(ldc), C.c_float(scale), _ptr(out), _stream()),
          "seedx_nhwc_to_nchw_f32")
    return out


def image_to_u8(x):
    """x: NHWC [n,h,w,>=3] fp16/fp32 in [-1,1] -> uint8 [n,h,w,3]."""
    _require_cuda(x)
    assert x.is_contiguous() and x.dim() == 4
    n, h, w, ldc = x.shape
    out = torch.empty((n, h, w, 3), device=x.device, dtype=torch.uint8)
    check(lib().seedx_image_to_u8(_ptr(x), _dt(x), _i64(n * h * w), _i64(ldc), _ptr(out), _stream()), "seedx_image_to_u8")
    return out


def cfg_euler_step(eps, x, unet_in, branches, guidance, image_guidance, sigma, sigma_next, init_sigma=1.0):
    _require_cuda(eps, x, unet_in)
    assert x.dtype == torch.float32 and x.is_contiguous() and unet_in.dtype == torch.float16 and unet_in.is_contiguous()
    B, c, h, w = x.shape
    assert c == 4 and unet_in.shape == (branches * B, h, w, 8)
    if eps is not None:
        assert eps.dtype == torch.float32 and eps.is_contiguous() and eps.numel() == branches * B * h * w * 4
    check(lib().seedx_cfg_euler_step(_ptr(eps), _ptr(x), _ptr(unet_in), _i64(B), _i64(h * w), C.c_int(branches), C.c_float(guidance),
                                     C.c_float(image_guidance), C.c_float(sigma), C.c_float(sigma_next), C.c_float(init_sigma), _stream()),
          "seedx_cfg_euler_step")
    return x


def cfg_euler_slots(eps, x, unet_in, t_dev, state, sigmas, timesteps, scalars, branches, fresh=None):
    """seedx_cfg_euler_slots: one CFG + Euler step of every live slot (eps given), or the initialisation of the slots listed in `fresh`
    (eps None).  x fp32 [S,4,h,w], unet_in fp16 [branches*S,h,w,8], t_dev fp32 [branches*S], state int32 [S,2] (step index, step count),
    sigmas fp32 [S,max_steps+1], timesteps fp32 [S,max_steps], scalars fp32 [S,3] (guidance, image guidance, init_noise_sigma)."""
    _require_cuda(eps, x, unet_in, t_dev, state, sigmas, timesteps, scalars)
    assert x.dtype == torch.float32 and x.is_contiguous() and unet_in.dtype == torch.float16 and unet_in.is_contiguous()
    S, c, h, w = x.shape
    assert c == 4 and unet_in.shape == (branches * S, h, w, 8) and t_dev.dtype == torch.float32 and t_dev.numel() == branches * S
    M = timesteps.shape[1]
    assert state.dtype == torch.int32 and state.shape == (S, 2) and state.is_contiguous()
    for t, shape in ((sigmas, (S, M + 1)), (timesteps, (S, M)), (scalars, (S, 3))):
        assert t.dtype == torch.float32 and t.is_contiguous() and t.shape == shape
    if eps is not None:
        assert eps.dtype == torch.float32 and eps.is_contiguous() and eps.numel() == branches * S * h * w * 4
    mask = 0
    for s in fresh or ():
        mask |= 1 << int(s)
    check(lib().seedx_cfg_euler_slots(_ptr(eps), _ptr(x), _ptr(unet_in), _ptr(t_dev), _ptr(state), _ptr(sigmas), _ptr(timesteps), _ptr(scalars),
                                      _i64(S), _i64(h * w), C.c_int(branches), _i64(M), C.c_uint64(mask), _stream()),
          "seedx_cfg_euler_slots")
    return x


def gemv(W, x, out, *, rms_w=None, eps=1e-5, residual=None, gated=False, scale=None):
    """out[b] fp32 = epi(W[N,K] . (rmsnorm(x[b])*rms_w | x[b])); x fp32 [K] or [B,K] with B in {1,2,4,8} (weights streamed once).
    W fp16, or float8_e4m3fn with scale = fp32 [N] (weight row n = scale[n] * W[n]; seedx_gemv_fp8)."""
    _require_cuda(W, x, out, scale)
    fp8 = W.dtype == torch.float8_e4m3fn
    assert (W.dtype == torch.float16 and scale is None) or (fp8 and scale is not None)
    assert W.is_contiguous() and x.dtype == torch.float32 and out.dtype == torch.float32
    N, K = W.shape
    x2 = x.reshape(-1, K)
    o2 = out.reshape(x2.shape[0], -1)
    r2 = residual.reshape(x2.shape[0], -1) if residual is not None else None
    assert x2.stride(1) == 1 and o2.stride(1) == 1
    tail = (_ptr(x2), _i64(x2.stride(0)), _ptr(rms_w), C.c_float(eps), _ptr(r2), _i64(r2.stride(0) if r2 is not None else 0),
            _ptr(o2), _i64(o2.stride(0)), _i64(N), _i64(K), C.c_int(x2.shape[0]), C.c_int(int(gated)), _stream())
    if fp8:
        assert scale.dtype == torch.float32 and scale.is_contiguous() and scale.numel() == N
        check(lib().seedx_gemv_fp8(_ptr(W), _ptr(scale), *tail), "seedx_gemv_fp8")
    else:
        check(lib().seedx_gemv_f16(_ptr(W), *tail), "seedx_gemv_f16")
    return out


def dequant_fp8(W8, scale, out):
    """fp16 out[n, k] = (half)(float(W8[n, k]) * scale[n]); W8 float8_e4m3fn [N, K], scale fp32 [N], out fp16 with W8's shape (all contiguous).
    A GEMM that reads `out` right after this call must pass dynamic_b=True."""
    _require_cuda(W8, scale, out)
    assert W8.dtype == torch.float8_e4m3fn and W8.is_contiguous() and W8.dim() == 2
    assert scale.dtype == torch.float32 and scale.is_contiguous() and scale.numel() == W8.shape[0]
    assert out.dtype == torch.float16 and out.is_contiguous() and out.shape == W8.shape
    check(lib().seedx_dequant_fp8(_ptr(W8), _ptr(scale), _ptr(out), _i64(W8.shape[0]), _i64(W8.shape[1]), _stream()), "seedx_dequant_fp8")
    return out


def decode_attention(qkv, state, inv_freq, kcache, vcache, out, heads, head_dim, page_table=None, page_size=0):
    """qkv fp32 [B, 3*H*d]; state int32 [B,4]; out fp32 [B, H*d].  Contiguous caches: kcache/vcache fp16 [B, max_len, H*d].  Paged:
    kcache/vcache = page pools fp16 [n_pages, page_size, H*d] and page_table int32 [B, pages_per_seq]."""
    B = qkv.shape[0]
    if page_table is not None:
        assert page_table.dtype == torch.int32 and page_table.is_contiguous() and page_table.shape[0] == B and kcache.shape[1] == page_size
        check(lib().seedx_decode_attention_paged(_ptr(qkv), _ptr(state), _ptr(inv_freq), _ptr(kcache), _ptr(vcache), _ptr(page_table),
                                                 _i64(page_table.stride(0)), _i64(page_size), _ptr(out), C.c_int(B), C.c_int(heads),
                                                 C.c_int(head_dim), C.c_float(head_dim ** -0.5), _stream()), "seedx_decode_attention_paged")
        return out
    check(lib().seedx_decode_attention(_ptr(qkv), _ptr(state), _ptr(inv_freq), _ptr(kcache), _ptr(vcache), _i64(kcache.stride(0)), _ptr(out),
                                       C.c_int(B), C.c_int(heads), C.c_int(head_dim), C.c_float(head_dim ** -0.5), _stream()),
          "seedx_decode_attention")
    return out


def rope_kv_prefill(qkv, pos0, heads, head_dim, inv_freq, kcache, vcache, page_table_row=None, page_size=0):
    assert qkv.dtype == torch.float16 and qkv.is_contiguous()
    if page_table_row is not None:
        assert page_table_row.dtype == torch.int32 and page_table_row.is_contiguous() and kcache.shape[1] == page_size
        check(lib().seedx_rope_kv_prefill_paged(_ptr(qkv), _i64(qkv.shape[0]), _i64(pos0), C.c_int(heads), C.c_int(head_dim), _ptr(inv_freq),
                                                _ptr(kcache), _ptr(vcache), _ptr(page_table_row), _i64(page_size), _stream()),
              "seedx_rope_kv_prefill_paged")
        return
    check(lib().seedx_rope_kv_prefill(_ptr(qkv), _i64(qkv.shape[0]), _i64(pos0), C.c_int(heads), C.c_int(head_dim), _ptr(inv_freq), _ptr(kcache),
                                      _ptr(vcache), _stream()), "seedx_rope_kv_prefill")


def embed_rows(table, out, *, ids=None, state=None, seq=None):
    n, dim = out.reshape(-1, out.shape[-1]).shape
    assert table.dtype == torch.float16 and out.dtype == torch.float32 and out.is_contiguous()
    if ids is not None:
        assert ids.dtype == torch.int32 and ids.numel() == n
    check(lib().seedx_embed_rows(_ptr(table), _ptr(ids), _ptr(state), _ptr(seq), _i64(seq.stride(0) if seq is not None else 0), _i64(n), _i64(dim),
                                 _ptr(out), _stream()), "seedx_embed_rows")
    return out


def scatter_rows(src, idx, dst, src_idx=None):
    assert idx.dtype == torch.int32 and dst.dtype == torch.float32 and src.is_contiguous() and dst.is_contiguous()
    if src_idx is not None:
        assert src_idx.dtype == torch.int32 and src_idx.numel() == idx.numel()
    check(lib().seedx_scatter_rows(_ptr(src), _dt(src), _ptr(src_idx), _ptr(idx), _i64(idx.numel()), _i64(dst.shape[-1]), _ptr(dst), _stream()),
          "seedx_scatter_rows")
    return dst


def store_hidden(x, state, hidden):
    """hidden fp32 [B, max_rows, D]; x fp32 [B, D]"""
    B, R, D = hidden.shape
    check(lib().seedx_store_hidden(_ptr(x), _ptr(state), C.c_int(B), _i64(R), _i64(D), _ptr(hidden), _stream()), "seedx_store_hidden")


def logits_argmax(logits, img_ids, seq, state, eos_id, suppress_eos):
    """logits fp32 [B, V]; seq int32 [B, max_len]; state int32 [B, 4]"""
    B, V = logits.shape
    check(lib().seedx_logits_argmax(_ptr(logits), _i64(V), _ptr(img_ids), C.c_int(0 if img_ids is None else img_ids.numel()), _ptr(seq),
                                    _ptr(state), C.c_int(B), C.c_int(eos_id if eos_id is not None else -1), C.c_int(int(suppress_eos)),
                                    _i64(seq.shape[1]), _stream()), "seedx_logits_argmax")


def add_bcast_f16(a, b, out=None):
    """fp16 out[r,:] = a[r,:] + b[r % b_rows,:] (b fp32)."""
    _require_cuda(a, b, out)
    assert a.is_contiguous() and b.dtype == torch.float32 and b.is_contiguous()
    a2 = a.reshape(-1, a.shape[-1])
    if out is None:
        out = torch.empty(a2.shape, device=a.device, dtype=torch.float16)
    check(lib().seedx_add_bcast_f16(_ptr(a2), _dt(a2), _ptr(b), _i64(a2.shape[0]), _i64(a2.shape[1]), _i64(b.shape[0]), _ptr(out), _stream()),
          "seedx_add_bcast_f16")
    return out
