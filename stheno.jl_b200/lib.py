"""ctypes binding of libstheno_b200.so -- the same symbols the Julia shim `ccall`s
(julia/SthenoB200.jl).  There is NO fallback: if the library is missing or the device is not an
H100 (sm_90) the product path raises."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libstheno_b200.so")

SB_OK, SB_ERR_INVALID, SB_ERR_CUDA, SB_ERR_NOT_POSDEF, SB_ERR_UNSUPPORTED, SB_ERR_NCCL, SB_ERR_NOMEM = 0, -1, -2, -3, -4, -5, -6
K_SE, K_MATERN12, K_MATERN32, K_MATERN52, K_WHITE, K_CONST = range(6)


class sb_array(C.Structure):
    _fields_ = [("data", C.c_void_p), ("n", C.c_int64), ("dim", C.c_int32), ("reserved", C.c_int32)]


class sb_term(C.Structure):
    _fields_ = [("kernel", C.c_int32), ("zl", C.c_int32), ("zr", C.c_int32), ("sl", C.c_int32),
                ("sr", C.c_int32), ("reserved", C.c_int32), ("coeff", C.c_double), ("param", C.c_double)]


class sb_block(C.Structure):
    _fields_ = [("row0", C.c_int64), ("nrows", C.c_int64), ("col0", C.c_int64), ("ncols", C.c_int64),
                ("term0", C.c_int32), ("nterms", C.c_int32)]


class sb_covspec(C.Structure):
    _fields_ = [("nrows", C.c_int64), ("ncols", C.c_int64), ("symmetric", C.c_int32),
                ("narrays", C.c_int32), ("arrays", C.POINTER(sb_array)), ("nterms", C.c_int32),
                ("terms", C.POINTER(sb_term)), ("nblocks", C.c_int32), ("blocks", C.POINTER(sb_block))]


class sb_noise(C.Structure):
    _fields_ = [("sigma2", C.c_double), ("diag", C.c_void_p), ("dense", C.c_void_p)]


class sb_timings(C.Structure):
    _fields_ = [("assemble_ms", C.c_double), ("panel_ms", C.c_double), ("trailing_ms", C.c_double),
                ("solve_ms", C.c_double), ("predict_ms", C.c_double), ("comm_ms", C.c_double),
                ("total_ms", C.c_double), ("trailing_flops", C.c_double),
                ("trailing_kernel_ms", C.c_double), ("trailing_launches", C.c_int64),
                ("kernel_launches", C.c_int64), ("trailing_int8_ops", C.c_double),
                ("panel_chain_ms", C.c_double)]

    def asdict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


EXPORTS = [
    "sb_abi_version", "sb_last_error", "sb_ctx_create", "sb_nccl_unique_id", "sb_ctx_create_dist",
    "sb_ctx_destroy", "sb_ctx_timings", "sb_ctx_set_option", "sb_ctx_mark", "sb_ctx_elapsed_ms", "sb_owner_of_block",
    "sb_owned_trailing_tiles", "sb_row_chunk", "sb_cov_dense", "sb_cov_diag", "sb_factor_create",
    "sb_factor_destroy", "sb_factor_logdet", "sb_logpdf", "sb_factor_set_data", "sb_factor_alpha",
    "sb_factor_set_alpha", "sb_predict", "sb_predict_cov", "sb_predict_factor", "sb_factor_append", "sb_rand",
    "sb_factor_get_L",
    "sb_vfe_create", "sb_vfe_predict", "sb_vfe_predict_cov", "sb_vfe_destroy",
    "sb_factor_export_size", "sb_factor_export", "sb_factor_import", "sb_logpdf_grad", "sb_vfe_grad",
]

_lib = None


class SthenoB200Error(RuntimeError):
    def __init__(self, status, msg):
        super().__init__(f"libstheno_b200 status {status}: {msg}")
        self.status = status


class PosDefException(SthenoB200Error):
    """Mirror of LinearAlgebra.PosDefException(info) thrown by `cholesky` in the reference."""

    def __init__(self, info, msg):
        super().__init__(SB_ERR_NOT_POSDEF, msg)
        self.info = info


def load():
    """dlopen the in-tree library; raise loudly if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f"{LIB_PATH} not found: build it with stheno.jl_b200/csrc/build.sh "
            "(or __graft_entry__.build()).  There is no CPU fallback.")
    lib = C.CDLL(LIB_PATH, mode=C.RTLD_GLOBAL)
    vp, i32, i64 = C.c_void_p, C.c_int32, C.c_int64
    P = C.POINTER
    lib.sb_abi_version.restype = i32
    lib.sb_last_error.restype = C.c_char_p
    sigs = {
        "sb_ctx_create": [i32, P(vp)],
        "sb_nccl_unique_id": [vp],
        "sb_ctx_create_dist": [i32, i32, i32, vp, P(vp)],
        "sb_ctx_destroy": [vp],
        "sb_ctx_timings": [vp, P(sb_timings), i32],
        "sb_ctx_set_option": [vp, C.c_char_p, i64],
        "sb_ctx_mark": [vp, i32],
        "sb_ctx_elapsed_ms": [vp, i32, i32, P(C.c_double)],
        "sb_cov_dense": [vp, P(sb_covspec), vp],
        "sb_cov_diag": [vp, P(sb_covspec), vp],
        "sb_factor_create": [vp, P(sb_covspec), P(sb_noise), P(vp), P(i64)],
        "sb_factor_destroy": [vp],
        "sb_factor_logdet": [vp, vp, P(C.c_double)],
        "sb_logpdf": [vp, vp, vp, i32, P(C.c_double)],
        "sb_factor_set_data": [vp, vp, vp],
        "sb_factor_alpha": [vp, vp, vp],
        "sb_factor_set_alpha": [vp, vp, vp],
        "sb_predict": [vp, vp, P(sb_covspec), P(sb_covspec), vp, vp],
        "sb_predict_cov": [vp, vp, P(sb_covspec), P(sb_covspec), vp],
        "sb_predict_factor": [vp, vp, P(sb_covspec), P(sb_covspec), P(sb_noise), P(vp), P(i64)],
        "sb_factor_append": [vp, vp, P(sb_covspec), P(sb_covspec), P(sb_noise), P(vp), P(i64)],
        "sb_rand": [vp, vp, vp, i32, vp],
        "sb_factor_get_L": [vp, vp, vp],
        "sb_logpdf_grad": [vp, vp, P(sb_covspec), vp, vp],
        "sb_factor_export_size": [vp, vp, P(i64)],
        "sb_factor_export": [vp, vp, vp, i64],
        "sb_factor_import": [vp, vp, i64, P(vp)],
        "sb_vfe_create": [vp, P(sb_covspec), P(sb_noise), P(sb_covspec), P(sb_covspec), P(sb_noise), vp,
                          P(vp), P(C.c_double), P(i64)],
        "sb_vfe_grad": [vp, vp, P(sb_covspec), P(sb_covspec), P(sb_covspec), P(sb_noise), vp,
                        vp, vp, vp, vp, vp],
        "sb_vfe_predict": [vp, vp, P(sb_covspec), P(sb_covspec), vp, vp],
        "sb_vfe_predict_cov": [vp, vp, P(sb_covspec), P(sb_covspec), vp],
        "sb_vfe_destroy": [vp],
    }
    for name, args in sigs.items():
        fn = getattr(lib, name)
        fn.argtypes = args
        fn.restype = i32
    lib.sb_owner_of_block.argtypes, lib.sb_owner_of_block.restype = [i64, i32], i32
    lib.sb_owned_trailing_tiles.argtypes, lib.sb_owned_trailing_tiles.restype = [i64, i64, i32, i32], i64
    lib.sb_row_chunk.argtypes, lib.sb_row_chunk.restype = [i64, i32, i32, P(i64), P(i64)], i32
    if lib.sb_abi_version() != 1:
        raise ImportError("libstheno_b200 ABI version mismatch")
    _lib = lib
    return lib


def check(status, info=None):
    if status == SB_OK:
        return
    msg = load().sb_last_error().decode()
    if status == SB_ERR_NOT_POSDEF:
        raise PosDefException(int(info.value) if info is not None else -1, msg)
    if status == SB_ERR_UNSUPPORTED:
        raise NotImplementedError(msg)
    raise SthenoB200Error(status, msg)


def ptr(a):
    """Raw address of a numpy array / torch CUDA tensor / int address / None."""
    if a is None:
        return None
    if isinstance(a, np.ndarray):
        return a.ctypes.data
    if isinstance(a, int):
        return a
    if hasattr(a, "data_ptr"):
        return a.data_ptr()
    raise TypeError(type(a))


class Context:
    """One CUDA device + stream (+ NCCL communicator when world > 1)."""

    def __init__(self, device=0, rank=0, world=1, nccl_id: bytes | None = None):
        lib = load()
        h = C.c_void_p()
        if world > 1:
            buf = C.create_string_buffer(nccl_id, 128)
            check(lib.sb_ctx_create_dist(device, rank, world, C.cast(buf, C.c_void_p), C.byref(h)))
        else:
            check(lib.sb_ctx_create(device, C.byref(h)))
        self.h, self.device, self.rank, self.world = h, device, rank, world

    def timings(self, reset=False):
        t = sb_timings()
        check(load().sb_ctx_timings(self.h, C.byref(t), 1 if reset else 0))
        return t.asdict()

    def set_option(self, key: str, value: int):
        """"trailing": 0 = fp64 DMMA, 1 = int8 Ozaki (wgmma) trailing update; "fine_timing": 0/1."""
        check(load().sb_ctx_set_option(self.h, key.encode(), int(value)))

    def mark(self, slot):
        check(load().sb_ctx_mark(self.h, slot))

    def elapsed_ms(self, a, b):
        v = C.c_double()
        check(load().sb_ctx_elapsed_ms(self.h, a, b, C.byref(v)))
        return v.value

    def close(self):
        if self.h:
            load().sb_ctx_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def nccl_unique_id() -> bytes:
    buf = C.create_string_buffer(128)
    check(load().sb_nccl_unique_id(C.cast(buf, C.c_void_p)))
    return buf.raw


_default_ctx = None


def default_context() -> Context:
    global _default_ctx
    if _default_ctx is None:
        _default_ctx = Context(int(os.environ.get("SB_DEVICE", "0")))
    return _default_ctx


def set_default_context(ctx: Context):
    global _default_ctx
    _default_ctx = ctx
