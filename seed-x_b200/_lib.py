"""ctypes binding of libseedx.so (the C ABI declared in include/seedx.h).

The product path has no fallback: if the shared library is missing or a call fails, an exception is raised.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("SEEDX_LIB") or os.path.join(_HERE, "lib", "libseedx.so")     # SEEDX_LIB: A/B builds of the kernel library (tools/)

F16, F32 = 1, 2
ACT_NONE, ACT_GELU, ACT_SILU = 0, 1, 2


class SeedxError(RuntimeError):
    pass


class GemmArgs(C.Structure):
    _fields_ = [
        ("A", C.c_void_p), ("B", C.c_void_p), ("D", C.c_void_p),
        ("M", C.c_int64), ("N", C.c_int64), ("K", C.c_int64),
        ("batch", C.c_int64),
        ("lda", C.c_int64), ("ldb", C.c_int64), ("ldd", C.c_int64),
        ("strideA", C.c_int64), ("strideB", C.c_int64), ("strideD", C.c_int64),
        ("alpha", C.c_float),
        ("bias_n", C.c_void_p), ("bias_m", C.c_void_p), ("bias_g", C.c_void_p),
        ("bias_g_rows", C.c_int64),
        ("residual", C.c_void_p),
        ("residual_dtype", C.c_int32),
        ("ldr", C.c_int64), ("strideR", C.c_int64), ("res_row_mod", C.c_int64),
        ("act", C.c_int32), ("gated", C.c_int32), ("out_dtype", C.c_int32),
        ("conv_taps_h", C.c_int32), ("conv_taps_w", C.c_int32),
        ("conv_n", C.c_int64), ("conv_h", C.c_int64), ("conv_w", C.c_int64), ("conv_c", C.c_int64),
        ("tile_n", C.c_int32),
        ("ln_stats", C.c_void_p), ("ln_colsum", C.c_void_p), ("b_dynamic", C.c_int32),
        ("ln_parts", C.c_int32), ("ln_eps", C.c_float), ("row_part", C.c_void_p), ("col_part", C.c_void_p),
        ("row_stats_out", C.c_void_p), ("row_tickets", C.c_void_p), ("row_eps", C.c_float),
    ]


_lib = None


def lib():
    """Load libseedx.so once; raise loudly when it has not been built (python -c 'import __graft_entry__ as g; g.build()')."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise SeedxError(f"{LIB_PATH} not found: build it with __graft_entry__.build(); there is no fallback path")
        _lib = C.CDLL(LIB_PATH)
        _lib.seedx_last_error.restype = C.c_char_p
        _lib.seedx_launch_count.restype = C.c_int64
        _lib.seedx_groupnorm_ws_bytes.restype = C.c_int64
        _lib.seedx_quant_images_fp8_ws_bytes.restype = C.c_int64
        _lib.seedx_abi_version.restype = C.c_int
        if "SEEDX_GEMM_CLUSTER" in os.environ:      # experiment switch: 0 = single-CTA tiles, 1 = auto, 2 = CTA pairs whenever legal
            _lib.seedx_gemm_set_cluster(int(os.environ["SEEDX_GEMM_CLUSTER"]))
        if "SEEDX_GEMM_STREAM_K" in os.environ:      # 0 = data-parallel tiles only, 1 = auto (default), 2 = stream-K wherever legal
            _lib.seedx_gemm_set_stream_k(int(os.environ["SEEDX_GEMM_STREAM_K"]))
        if "SEEDX_GEMM_TMA_EPI" in os.environ:
            _lib.seedx_gemm_set_tma_epilogue(int(os.environ["SEEDX_GEMM_TMA_EPI"]))
    return _lib


def check(rc, what):
    if rc != 0:
        raise SeedxError(f"{what} failed (rc={rc}): {lib().seedx_last_error().decode()}")


_replayed = 0


def note_replay(kernels):
    """A captured CUDA graph holding `kernels` library launches was replayed once (they do not pass through the C entry points again)."""
    global _replayed
    _replayed += int(kernels)


def launch_count():
    """Library kernels launched by this process: direct launches (counted inside libseedx.so) + kernels executed by graph replays."""
    return int(lib().seedx_launch_count()) + _replayed
