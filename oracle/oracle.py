"""ctypes/numpy front-end for the CPU oracle (oracle/oracle.c) and, when present, the reference's
own host code compiled unmodified into oracle/_ref/.

TEST INFRASTRUCTURE ONLY: imported by tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
--impl reference legs.  The product path (fault-tolerant-sgemm-on-nvidia-gpus_b200/, libftsgemm.so)
never imports this module.

Conventions follow the reference kernels (kernel/ft_sgemm/include_code_gen/ft_sgemm_huge.cuh:11):
A is M x K column-major (ld = M), B is N x K column-major (ld = N), C is M x N column-major (ld = M),
C = alpha * A * B^T + beta * C.  numpy arrays are passed as flat float32 buffers in that layout; the
helpers `colmajor(a2d)` / `as2d(buf, rows, cols)` convert to/from ordinary 2-D arrays.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
_F = C.POINTER(C.c_float)
_I = C.POINTER(C.c_int)


def build(verbose: bool = False) -> None:
    """Compile liboracle.so (always) and oracle/_ref/* (only where /root/reference exists)."""
    out = subprocess.run(["make", "-C", str(HERE), "all"], capture_output=True, text=True)
    if verbose or out.returncode != 0:
        print(out.stdout, out.stderr)
    if out.returncode != 0:
        raise RuntimeError("oracle build failed")


def _load(path: Path):
    if not path.exists():
        return None
    return C.CDLL(str(path))


_lib = None
_ref_utils = None
_ref_kernels = None


def lib():
    global _lib
    if _lib is None:
        p = HERE / "liboracle.so"
        if not p.exists():
            build()
        _lib = C.CDLL(str(p))
        _lib.oracle_sgemm_nt.argtypes = [C.c_int, C.c_int, C.c_int, C.c_float, _F, C.c_int, _F, C.c_int,
                                         C.c_float, _F, C.c_int]
        _lib.oracle_sgemm_nt_rows.argtypes = [C.c_int, C.c_int, C.c_int, C.c_float, _F, C.c_int, _F,
                                              C.c_int, C.c_float, _F, C.c_int, _I, C.c_int, _F]
        _lib.oracle_cpu_gemm_rowmajor.argtypes = [C.c_float, C.c_float, _F, _F, C.c_int, _F]
        _lib.oracle_verify_matrix.argtypes = [_F, _F, C.c_int, C.c_int]
        _lib.oracle_verify_matrix.restype = C.c_long
        _lib.oracle_make_inputs.argtypes = [C.c_int, _F, _F, _F]
        _lib.oracle_fill_matrix.argtypes = [_F, C.c_int]
        _lib.oracle_seed.argtypes = [C.c_uint]
        _lib.oracle_error_metrics.argtypes = [_F, _F, C.c_long, C.POINTER(C.c_double),
                                              C.POINTER(C.c_double), C.POINTER(C.c_double)]
        _lib.oracle_abft_sgemm_nt.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_float, _F, C.c_int,
                                              _F, C.c_int, C.c_float, _F, C.c_int, C.POINTER(C.c_long)]
        _lib.oracle_abft_sgemm_nt.restype = C.c_long
        _lib.oracle_abft_num_checks.argtypes = [C.c_int] * 4
        _lib.oracle_abft_num_checks.restype = C.c_int
        _lib.oracle_num_threads.restype = C.c_int
    return _lib


def ref_utils():
    """The reference's utils.cu compiled in place (None on machines without oracle/_ref)."""
    global _ref_utils
    if _ref_utils is None:
        _ref_utils = _load(HERE / "_ref" / "libref_utils.so")
        if _ref_utils is not None:
            _ref_utils.ref_generate_random_matrix.argtypes = [_F, C.c_int]
            _ref_utils.ref_cpu_gemm.argtypes = [C.c_float, C.c_float, _F, _F, C.c_int, _F]
            _ref_utils.ref_verify_matrix.argtypes = [_F, _F, C.c_int, C.c_int]
            _ref_utils.ref_verify_matrix.restype = C.c_int
            _ref_utils.ref_srand.argtypes = [C.c_uint]
    return _ref_utils


def ref_kernels():
    """The reference's generated kernels under the CPU thread shim (None if not built)."""
    global _ref_kernels
    if _ref_kernels is None:
        _ref_kernels = _load(HERE / "_ref" / "libref_kernels_cpu.so")
        if _ref_kernels is not None:
            _ref_kernels.ref_kernel_run.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, _F, _F, _F,
                                                    C.c_float, C.c_float]
            _ref_kernels.ref_kernel_run.restype = C.c_int
    return _ref_kernels


def _p(a: np.ndarray):
    assert a.dtype == np.float32 and a.flags["C_CONTIGUOUS"]
    return a.ctypes.data_as(_F)


def colmajor(a2d: np.ndarray) -> np.ndarray:
    """2-D array -> flat column-major float32 buffer."""
    return np.ascontiguousarray(np.asarray(a2d, dtype=np.float32).T).reshape(-1)


def as2d(buf: np.ndarray, rows: int, cols: int) -> np.ndarray:
    """flat column-major buffer -> (rows, cols) view."""
    return buf.reshape(cols, rows).T


def make_inputs(n: int):
    """Reference inputs for END = n (sgemm.cu:12,52-56): flat buffers A, B (n*n) and C = 0."""
    A = np.empty(n * n, np.float32)
    B = np.empty(n * n, np.float32)
    Cm = np.empty(n * n, np.float32)
    lib().oracle_make_inputs(n, _p(A), _p(B), _p(Cm))
    return A, B, Cm


def ref_make_inputs(n: int):
    """Same, through the reference's own generate_random_matrix (needs oracle/_ref)."""
    r = ref_utils()
    assert r is not None
    A = np.empty(n * n, np.float32)
    B = np.empty(n * n, np.float32)
    Cm = np.empty(n * n, np.float32)
    r.ref_srand(10)
    r.ref_generate_random_matrix(_p(A), n)
    r.ref_generate_random_matrix(_p(B), n)
    r.ref_generate_random_matrix(_p(Cm), n)
    Cm[:] = 0
    return A, B, Cm


def sgemm_nt(M, N, K, alpha, A, B, beta, Cbuf, lda=None, ldb=None, ldc=None) -> np.ndarray:
    """In-place C = alpha*A*B^T + beta*C on flat column-major buffers; returns Cbuf."""
    lib().oracle_sgemm_nt(M, N, K, alpha, _p(A), lda or M, _p(B), ldb or N, beta, _p(Cbuf), ldc or M)
    return Cbuf


def sgemm_nt_rows(M, N, K, alpha, A, B, beta, Cin, rows) -> np.ndarray:
    rows = np.ascontiguousarray(rows, dtype=np.int32)
    out = np.empty((len(rows), N), np.float32)
    lib().oracle_sgemm_nt_rows(M, N, K, alpha, _p(A), M, _p(B), N, beta,
                               _p(Cin) if Cin is not None else None, M,
                               rows.ctypes.data_as(_I), len(rows), _p(out))
    return out


def verify_matrix(ref: np.ndarray, x: np.ndarray, m: int, n: int) -> int:
    """-1 if x passes the reference's 1 %/0.01 rule against ref, else first failing linear index."""
    return int(lib().oracle_verify_matrix(_p(ref), _p(x), m, n))


def error_metrics(ref: np.ndarray, x: np.ndarray):
    a, b, c = C.c_double(), C.c_double(), C.c_double()
    lib().oracle_error_metrics(_p(ref), _p(x), ref.size, C.byref(a), C.byref(b), C.byref(c))
    return {"max_abs": a.value, "rel_fro": b.value, "max_abs_over_refmax": c.value}


class AbftCfg(C.Structure):
    _fields_ = [("ms", C.c_int), ("ns", C.c_int), ("ks", C.c_int), ("check_div", C.c_int),
                ("check_off", C.c_int), ("tau", C.c_float), ("inject_mag", C.c_float),
                ("use_col_residual", C.c_int)]


# code_gen/main.py:8-16  name -> (ms, ns, ks, mr, nr); ids per sgemm.cu:235
VARIANTS = {
    "small": (16, 16, 16, 2, 2), "medium": (32, 32, 8, 4, 4), "large": (64, 64, 8, 8, 8),
    "tall": (128, 32, 8, 8, 4), "wide": (32, 128, 8, 4, 8), "huge": (128, 128, 8, 8, 8),
}


def abft_sgemm_nt(variant: str, M, N, K, alpha, A, B, beta, Cbuf, inject=10000.0, tau=9500.0):
    ms, ns, ks, mr, nr = VARIANTS[variant]
    cfg = AbftCfg(ms, ns, ks, 20, 8, tau, inject, 1 if mr < nr else 0)
    nchk = C.c_long()
    ncorr = lib().oracle_abft_sgemm_nt(C.byref(cfg), M, N, K, alpha, _p(A), M, _p(B), N, beta, _p(Cbuf), M,
                                       C.byref(nchk))
    return int(ncorr), int(nchk.value)


def abft_num_checks(K: int, ks: int = 8) -> int:
    return int(lib().oracle_abft_num_checks(K, ks, 20, 8))


def num_threads() -> int:
    return int(lib().oracle_num_threads())


# ----------------------------------------------------------------------------------------------
# TF32 model of the kernel (used only to explain/bound the kernel's deviation from the fp32
# oracle; the parity target remains oracle_sgemm_nt).  wgmma with TF32 inputs consumes fp32 bit patterns
# and ignores the 13 low mantissa bits.
# ----------------------------------------------------------------------------------------------
def tf32_trunc(x: np.ndarray) -> np.ndarray:
    return (np.asarray(x, np.float32).view(np.uint32) & np.uint32(0xFFFFE000)).view(np.float32)


def tf32_rna(x: np.ndarray) -> np.ndarray:
    u = np.asarray(x, np.float32).view(np.uint32).astype(np.uint64)
    u = (u + np.uint64(0x1000)) & np.uint64(0xFFFFE000)
    return u.astype(np.uint32).view(np.float32)


def sgemm_nt_tf32_model(M, N, K, alpha, A, B, beta, Cin, rounding="trunc") -> np.ndarray:
    """float64-accumulated product of TF32-rounded operands (flat col-major in/out)."""
    f = tf32_trunc if rounding == "trunc" else tf32_rna
    A2 = as2d(f(A), M, K).astype(np.float64)
    B2 = as2d(f(B), N, K).astype(np.float64)
    P = A2 @ B2.T
    out = alpha * P + beta * as2d(Cin, M, N).astype(np.float64)
    return colmajor(out.astype(np.float32))
