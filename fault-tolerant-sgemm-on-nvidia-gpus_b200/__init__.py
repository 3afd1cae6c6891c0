"""Host-side mirror of the reference's ft_sgemm interface over the C ABI of libftsgemm.so (include/ftsgemm.h).

The reference (shixun404/Fault-Tolerant-SGEMM-on-NVIDIA-GPUs) has no Python API; its operator surface is
  * the kernel contract  k(M, N, K, A, B, C, alpha, beta)  selected by a kernel id
    (kernel/ft_sgemm/sgemm.cu:110-199, ids/names at :235-237, tiles at code_gen/main.py:8-16),
  * baseline_ft_sgemm(...)  (kernel/ft_sgemm/include/baseline_ft_sgemm.cuh:1),
  * verify_matrix(...)      (utils/utils.cu:61-77),
  * the CLI  ft_sgemm START END GAP ST_KERNEL END_KERNEL  (sgemm.cu:13-19).
This module mirrors exactly those, binding the shared library with ctypes (plain pointers and sizes; torch is only
used by callers to own device memory).  There is NO CPU fallback: if the library or an sm_90 device is missing,
every call raises.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
from pathlib import Path

HERE = Path(__file__).resolve().parent
LIB_PATH = HERE / "libftsgemm.so"
CLI_PATH = HERE / "ft_sgemm"

MAX_FAULTS = 8
MAX_EVENTS = 16

# kernel ids (include/ftsgemm.h; reference sgemm.cu:235-237)
ID_CUBLAS, ID_CUBLAS_TF32, ID_ABFT_BASELINE, ID_ABFT_BASELINE_TF32 = 0, 7, 10, 30
ID_SGEMM_AUTO, ID_ABFT_AUTO = 20, 40  # per-shape choice among the wgmma variants (select_kernel)
SGEMM_IDS = {"small": 1, "medium": 2, "large": 3, "tall": 4, "wide": 5, "huge": 6, "giant": 21, "pair128": 22}
ABFT_IDS = {"small": 11, "medium": 12, "large": 13, "tall": 14, "wide": 15, "huge": 16, "giant": 31, "pair128": 32}

# operand layouts of run_ex (include/ftsgemm.h): MN-major A(m,k) at A[m + k*lda], B(n,k) at B[n + k*ldb] (the reference's);
# K-major A(m,k) at A[k + m*lda], B(n,k) at B[k + n*ldb]
LAYOUT_MN_MAJOR, LAYOUT_K_MAJOR = 0, 1

# bias of run_bias (include/ftsgemm.h): ROW adds bias[m] to row m of C (length M), COL adds bias[n] to column n (length N)
BIAS_NONE, BIAS_ROW, BIAS_COL = 0, 1, 2

# activation of run_act (include/ftsgemm.h): C = act(z) with z the run_bias value; RELU is torch.relu, GELU torch's exact
# (erf) gelu.  ACTIVATIONS maps the names matmul and linear take.
ACT_NONE, ACT_RELU, ACT_GELU = 0, 1, 2
ACTIVATIONS = {None: ACT_NONE, "relu": ACT_RELU, "gelu": ACT_GELU}


class FtsgemmError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"ftsgemm error {code}: {msg}")
        self.code = code


class KernelInfo(C.Structure):
    _fields_ = [("id", C.c_int), ("name", C.c_char * 24), ("fault_tolerant", C.c_int), ("engine", C.c_int),
                ("ref_tile_m", C.c_int), ("ref_tile_n", C.c_int), ("ref_tile_k", C.c_int),
                ("tile_m", C.c_int), ("tile_n", C.c_int), ("tile_k", C.c_int)]


class Fault(C.Structure):
    _fields_ = [("row", C.c_int), ("col", C.c_int), ("mode", C.c_int), ("add_value", C.c_float),
                ("xor_mask", C.c_uint32)]


class Opts(C.Structure):
    _fields_ = [("struct_size", C.c_uint32), ("stream", C.c_void_p), ("inject_mode", C.c_int),
                ("selftest_value", C.c_float), ("selftest_row", C.c_int), ("selftest_col", C.c_int),
                ("n_faults", C.c_int), ("faults", Fault * MAX_FAULTS), ("tau_abs", C.c_float),
                ("tau_rel", C.c_float), ("detect_only", C.c_int), ("reuse_b_checksums", C.c_int),
                ("baseline_host_sync", C.c_int), ("precision", C.c_int), ("check_segments", C.c_int),
                ("no_recompute", C.c_int), ("protect_epilogue", C.c_int)]


class Event(C.Structure):
    _fields_ = [("row", C.c_int), ("col", C.c_int), ("residual", C.c_float), ("corrected_value", C.c_float),
                ("status", C.c_int)]


class Stats(C.Structure):
    _fields_ = [("tiles", C.c_ulonglong), ("rows_checked", C.c_ulonglong), ("detected", C.c_ulonglong),
                ("corrected", C.c_ulonglong), ("uncorrectable", C.c_ulonglong), ("checksum_faults", C.c_ulonglong),
                ("max_abs_residual", C.c_float), ("max_rel_residual", C.c_float), ("n_events", C.c_int),
                ("events", Event * MAX_EVENTS), ("recomputed", C.c_ulonglong),
                ("epilogue_faults", C.c_ulonglong)]

    def as_dict(self):
        return {"tiles": self.tiles, "rows_checked": self.rows_checked, "detected": self.detected,
                "corrected": self.corrected, "uncorrectable": self.uncorrectable, "recomputed": self.recomputed, "epilogue_faults": self.epilogue_faults,
                "checksum_faults": self.checksum_faults, "max_abs_residual": self.max_abs_residual,
                "max_rel_residual": self.max_rel_residual,
                "events": [{"row": e.row, "col": e.col, "residual": e.residual,
                            "corrected_value": e.corrected_value, "status": e.status}
                           for e in list(self.events)[:self.n_events]]}


# every symbol include/ftsgemm.h declares (checked by tests/test_abi.py without a GPU)
EXPORTED_SYMBOLS = [
    "ftsgemm_create", "ftsgemm_destroy", "ftsgemm_abi_version", "ftsgemm_error_string", "ftsgemm_last_cuda_error",
    "ftsgemm_default_opts", "ftsgemm_kernel_table", "ftsgemm_kernel_lookup", "ftsgemm_run", "ftsgemm_run_ex", "ftsgemm_run_bias", "ftsgemm_get_stats",
    "ftsgemm_run_host", "ftsgemm_baseline", "ftsgemm_verify", "ftsgemm_debug_set", "ftsgemm_debug_schedule",
    "ftsgemm_verify_bad_count", "ftsgemm_debug_trace", "ftsgemm_stats_device", "ftsgemm_select_kernel", "ftsgemm_launch_count", "ftsgemm_peer_export", "ftsgemm_peer_connect",
    "ftsgemm_peer_verdict", "ftsgemm_run_batched", "ftsgemm_debug_schedule_batched", "ftsgemm_run_act",
    "ftsgemm_run_batched_act", "ftsgemm_run_out", "ftsgemm_run_batched_out", "ftsgemm_run_typed", "ftsgemm_run_batched_typed",
    "ftsgemm_run_batched_mixed",
]

# element types of run_typed / run_batched_typed / run_batched_mixed (include/ftsgemm.h: FTSGEMM_TYPE_*)
TYPE_F32, TYPE_BF16 = 0, 1

_lib = None


def build(force: bool = False, verbose: bool = False) -> None:
    from importlib import util
    spec = util.spec_from_file_location("_ftsgemm_build", HERE / "build.py")
    mod = util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    mod.build(force=force, verbose=verbose)


def lib():
    """Load libftsgemm.so (raises if it has not been built: the product path never falls back to the CPU)."""
    global _lib
    if _lib is None:
        path = Path(os.environ.get("FTSGEMM_LIB", str(LIB_PATH)))  # override only for A/B experiments
        if not path.exists():
            raise FtsgemmError(-4, f"{path} not built (run __graft_entry__.build())")
        L = C.CDLL(str(path))
        vp, ip, fp = C.c_void_p, C.c_int, C.c_float
        L.ftsgemm_create.argtypes = [C.POINTER(vp)]
        L.ftsgemm_destroy.argtypes = [vp]
        L.ftsgemm_error_string.argtypes = [ip]
        L.ftsgemm_error_string.restype = C.c_char_p
        L.ftsgemm_last_cuda_error.argtypes = [vp]
        L.ftsgemm_default_opts.argtypes = [C.POINTER(Opts)]
        L.ftsgemm_default_opts.restype = None
        L.ftsgemm_kernel_table.argtypes = [C.POINTER(KernelInfo), ip]
        L.ftsgemm_kernel_lookup.argtypes = [ip, C.POINTER(KernelInfo)]
        L.ftsgemm_run.argtypes = [vp, ip, ip, ip, ip, vp, vp, vp, fp, fp, C.POINTER(Opts)]
        L.ftsgemm_run_ex.argtypes = [vp, ip, ip, ip, ip, vp, ip, ip, vp, ip, ip, vp, ip, fp, fp, C.POINTER(Opts)]
        L.ftsgemm_run_bias.argtypes = [vp, ip, ip, ip, ip, vp, ip, ip, vp, ip, ip, vp, ip, fp, fp, vp, ip, C.POINTER(Opts)]
        L.ftsgemm_run_act.argtypes = [vp, ip, ip, ip, ip, vp, ip, ip, vp, ip, ip, vp, ip, fp, fp, vp, ip, ip, vp,
                                      C.POINTER(Opts)]
        ll = C.c_longlong
        L.ftsgemm_run_batched.argtypes = [vp, ip, ip, ip, ip, vp, ip, ip, ll, vp, ip, ip, ll, vp, ip, ll, ip, fp, fp, vp, ip,
                                          C.POINTER(Opts)]
        L.ftsgemm_run_batched_act.argtypes = [vp, ip, ip, ip, ip, vp, ip, ip, ll, vp, ip, ip, ll, vp, ip, ll, ip, fp, fp, vp, ip,
                                              ll, ip, vp, C.POINTER(Opts)]
        L.ftsgemm_run_out.argtypes = [vp, ip, ip, ip, ip, vp, ip, ip, vp, ip, ip, vp, ip, vp, fp, fp, vp, ip, ip, vp,
                                      C.POINTER(Opts)]
        L.ftsgemm_run_batched_out.argtypes = [vp, ip, ip, ip, ip, vp, ip, ip, ll, vp, ip, ip, ll, vp, ip, ll, vp, ip, fp, fp,
                                              vp, ip, ll, ip, vp, C.POINTER(Opts)]
        L.ftsgemm_run_typed.argtypes = [vp, ip, ip, ip, ip, vp, ip, ip, vp, ip, ip, ip, vp, ip, vp, fp, fp, vp, ip, ip, vp,
                                        C.POINTER(Opts)]
        L.ftsgemm_run_batched_typed.argtypes = [vp, ip, ip, ip, ip, vp, ip, ip, ll, vp, ip, ip, ll, ip, vp, ip, ll, vp, ip, fp,
                                                fp, vp, ip, ll, ip, vp, C.POINTER(Opts)]
        L.ftsgemm_run_batched_mixed.argtypes = [vp, ip, ip, ip, ip, vp, ip, ip, ll, vp, ip, ip, ll, ip, vp, ip, ll, vp, ip, ip,
                                                fp, fp, vp, ip, ll, ip, vp, C.POINTER(Opts)]
        L.ftsgemm_get_stats.argtypes = [vp, C.POINTER(Stats)]
        L.ftsgemm_run_host.argtypes = [vp, ip, ip, ip, ip, vp, vp, vp, fp, fp, C.POINTER(Opts)]
        L.ftsgemm_stats_device.argtypes = [vp, vp, vp]
        L.ftsgemm_select_kernel.argtypes = [ip, ip, ip, ip]
        L.ftsgemm_peer_export.argtypes = [vp, vp]
        L.ftsgemm_peer_connect.argtypes = [vp, ip, ip, vp]
        L.ftsgemm_peer_verdict.argtypes = [vp, C.POINTER(C.c_double), C.POINTER(C.c_double), ip]
        L.ftsgemm_launch_count.argtypes = [vp]
        L.ftsgemm_launch_count.restype = C.c_ulonglong
        L.ftsgemm_baseline.argtypes = [vp, ip, ip, ip, vp, vp, vp, fp, fp, ip, C.POINTER(Opts), vp]
        L.ftsgemm_verify.argtypes = [vp, vp, vp, ip, ip, C.POINTER(C.c_longlong), C.POINTER(C.c_double), vp]
        L.ftsgemm_debug_set.argtypes = [C.c_char_p, C.c_longlong]
        L.ftsgemm_verify_bad_count.argtypes = [vp]
        L.ftsgemm_verify_bad_count.restype = C.c_longlong
        L.ftsgemm_debug_schedule.argtypes = [ip, ip, ip, ip, ip, C.POINTER(C.c_int), C.POINTER(C.c_int), ip]
        L.ftsgemm_debug_schedule_batched.argtypes = [ip, ip, ip, ip, ip, ip, C.POINTER(C.c_int), C.POINTER(C.c_int), ip]
        L.ftsgemm_debug_trace.argtypes = [vp, C.POINTER(C.c_ulonglong), ip]
        _lib = L
    return _lib


def _check(code: int):
    if code != 0:
        raise FtsgemmError(code, lib().ftsgemm_error_string(code).decode())


def kernel_table():
    """The kernel-variant table (reference: sgemm.cu:235-237 + code_gen/main.py:8-16)."""
    n = lib().ftsgemm_kernel_table(None, 0)
    arr = (KernelInfo * n)()
    lib().ftsgemm_kernel_table(arr, n)
    return [{"id": k.id, "name": k.name.decode(), "fault_tolerant": bool(k.fault_tolerant), "engine": k.engine,
             "ref_tile": (k.ref_tile_m, k.ref_tile_n, k.ref_tile_k), "tile": (k.tile_m, k.tile_n, k.tile_k)}
            for k in arr]


def select_kernel(M: int, N: int, K: int, fault_tolerant: bool) -> int:
    """The concrete kernel id the AUTO ids (20 / 40) resolve to for this shape."""
    r = lib().ftsgemm_select_kernel(M, N, K, 1 if fault_tolerant else 0)
    if r < 0:
        _check(r)
    return r


def default_opts() -> Opts:
    o = Opts()
    lib().ftsgemm_default_opts(C.byref(o))
    return o


def make_opts(stream=None, selftest=None, faults=None, tau_abs=0.0, tau_rel=0.0, detect_only=False,
              reuse_b_checksums=False, baseline_host_sync=True, no_recompute=False, precision=0, check_segments=0,
              protect_epilogue=False) -> Opts:
    """selftest: None | (value, tile_row, tile_col)  -> the reference's always-on injector (ft_sgemm_huge.cuh:324-327)
    faults: list of dicts {row, col, add=float} or {row, col, xor=int}; with xor, where="epilogue_tmem" | "epilogue_value"
    places the upset after the accumulator check (ftsgemm_fault.mode 2 / 3)
    protect_epilogue: False / 0 = unprotected store pass; True / 1 = checked store pass; 2 = every chunk verified before it
    is written and repaired whatever beta is (include/ftsgemm.h: ftsgemm_opts.protect_epilogue)"""
    o = default_opts()
    o.stream = stream
    if selftest is not None:
        o.inject_mode = 1
        o.selftest_value, o.selftest_row, o.selftest_col = float(selftest[0]), int(selftest[1]), int(selftest[2])
    if faults:
        assert selftest is None and len(faults) <= MAX_FAULTS
        o.inject_mode = 2
        o.n_faults = len(faults)
        for i, f in enumerate(faults):
            o.faults[i].row, o.faults[i].col = int(f["row"]), int(f["col"])
            if "xor" in f:
                o.faults[i].mode, o.faults[i].xor_mask = {"acc": 1, "epilogue_tmem": 2, "epilogue_value": 3}[f.get("where", "acc")], int(f["xor"]) & 0xFFFFFFFF
            else:
                o.faults[i].mode, o.faults[i].add_value = 0, float(f["add"])
    o.tau_abs, o.tau_rel = float(tau_abs), float(tau_rel)
    o.detect_only = int(detect_only)
    o.reuse_b_checksums = int(reuse_b_checksums)
    o.baseline_host_sync = int(baseline_host_sync)
    o.no_recompute = int(no_recompute)
    o.precision = int(precision)  # 0 = single-pass TF32, 1 = 3xTF32 (FP32-grade)
    o.check_segments = int(check_segments)  # > 1: intra-K checking (K-segments verified one after the other)
    o.protect_epilogue = int(protect_epilogue)
    return o


def debug_schedule(kernel_id: int, M: int, N: int, K: int, num_sms: int = 132):
    """Work decomposition of one launch, enumerated on the host (no GPU needed): (header dict, list of segment dicts)."""
    hdr = (C.c_int * 8)()
    n = lib().ftsgemm_debug_schedule(kernel_id, M, N, K, num_sms, hdr, None, 0)
    if n < 0:
        _check(n)
    rows = (C.c_int * (9 * max(n, 1)))()
    lib().ftsgemm_debug_schedule(kernel_id, M, N, K, num_sms, hdr, rows, n)
    keys = ("unit", "tile", "is_chk", "m_blk", "n_blk", "kb_begin", "kb_end", "kind", "slice")
    segs = [dict(zip(keys, rows[9 * i:9 * i + 9])) for i in range(n)]
    return dict(zip(("units", "num_tiles", "n_chk_tiles", "sk_tiles", "num_kb", "cta_group", "sk_slices", "chk_slices"), hdr)), segs


def debug_schedule_batched(kernel_id: int, M: int, N: int, K: int, batch: int, num_sms: int = 132):
    """debug_schedule for a strided batch of `batch` entries: every segment dict carries its entry as well."""
    hdr = (C.c_int * 8)()
    n = lib().ftsgemm_debug_schedule_batched(kernel_id, M, N, K, batch, num_sms, hdr, None, 0)
    if n < 0:
        _check(n)
    rows = (C.c_int * (10 * max(n, 1)))()
    lib().ftsgemm_debug_schedule_batched(kernel_id, M, N, K, batch, num_sms, hdr, rows, n)
    keys = ("unit", "tile", "is_chk", "m_blk", "n_blk", "kb_begin", "kb_end", "kind", "slice", "batch")
    segs = [dict(zip(keys, rows[10 * i:10 * i + 10])) for i in range(n)]
    return dict(zip(("units", "num_tiles", "n_chk_tiles", "sk_tiles", "num_kb", "cta_group", "sk_slices", "chk_slices"), hdr)), segs


def debug_set(key: str, value: int) -> None:
    _check(lib().ftsgemm_debug_set(key.encode(), int(value)))


def _pad4(n: int) -> int:
    return (n + 3) // 4 * 4


def _pad8(n: int) -> int:
    """_pad4 for BF16 operands: 16-byte rows are 8 elements."""
    return (n + 7) // 8 * 8


def _view(shape, stride, ptr: int, ld4: bool, elems16: int = 4):
    """("row", ld) or ("col", ld) of a 2-D matrix the library can read in place, None if it cannot: it needs a unit
    stride, a leading stride of at least the row length, a 16-byte aligned base and -- for A and B (ld4) -- 16-byte rows
    (ld a multiple of elems16: 4 FP32 or 8 BF16 elements)."""
    R, Cn = shape
    s0, s1 = stride
    pad = _pad8 if elems16 == 8 else _pad4
    if ptr % 16:
        return None
    if s1 == 1 or Cn == 1:  # row-major (a one-column matrix is both)
        ld = s0 if R > 1 else pad(Cn)
        if ld >= Cn and (not ld4 or ld % elems16 == 0):
            return ("row", ld)
    if s0 == 1 or R == 1:  # column-major
        ld = s1 if Cn > 1 else pad(R)
        if ld >= R and (not ld4 or ld % elems16 == 0):
            return ("col", ld)
    return None


def matmul_plan(a_shape, a_stride, b_shape, b_stride, out_stride, a_ptr: int = 0, b_ptr: int = 0, out_ptr: int = 0,
                bias_stride=None, bias_ptr: int = 0, bf16: bool = False, out_bf16: bool = False) -> dict:
    """run_ex arguments for out = a @ b with a: (M, K), b: (K, N), out: (M, N), from shapes, element strides and addresses.

    Column-major out: C = out, kernel A = a, kernel B = b^T.  Row-major out: C = out^T = b^T a^T (swap = True), so the
    kernel's M and N are N and M, kernel A = b^T and kernel B = a; for x @ W.T with row-major x, W and out both kernel
    operands are then K-major and no transpose runs.  copy_a / copy_b / copy_out mark matrices that cannot be read in
    place (see _view); the arguments returned describe the copies matmul makes of them: a as row-major and b as
    column-major with the row length padded to a multiple of 4 (both K-major for the kernel), out as a contiguous
    row-major matrix.  bias_stride (the element stride of a length-N bias, None without a bias) gives bias_mode: a bias
    over out's columns is one per kernel column (BIAS_COL), or per kernel row (BIAS_ROW) when swapped; copy_bias marks a
    bias without unit stride or with a base that is not 4-byte aligned.  bf16: a and b are BF16 (run_typed), whose 16-byte
    rows are 8 elements: leading strides and the copies' padded rows are multiples of 8.  out_bf16: out is BF16 too
    (run_batched_mixed), written in place only with a leading stride that is a multiple of 8, and its copy is row-major
    with rows padded to a multiple of 8 elements."""
    M, K = a_shape
    K2, N = b_shape
    if K != K2:
        raise ValueError(f"inner dimensions differ: {tuple(a_shape)} @ {tuple(b_shape)}")
    e16, pad = (8, _pad8) if bf16 else (4, _pad4)
    va = _view(a_shape, a_stride, a_ptr, True, e16)
    vb = _view(b_shape, b_stride, b_ptr, True, e16)
    vo = _view((M, N), out_stride, out_ptr, True, 8) if out_bf16 else _view((M, N), out_stride, out_ptr, False)
    copies = {"copy_a": va is None, "copy_b": vb is None, "copy_out": vo is None}
    va = va or ("row", pad(K))
    vb = vb or ("col", pad(K))
    vo = vo or ("row", _pad8(N) if out_bf16 else N)
    a_kmajor, b_kmajor = va[0] == "row", vb[0] == "col"  # a(m, k) along k / b(k, n) along k
    lay = {True: LAYOUT_K_MAJOR, False: LAYOUT_MN_MAJOR}
    if vo[0] == "col":
        args = {"M": M, "N": N, "K": K, "layout_a": lay[a_kmajor], "lda": va[1], "layout_b": lay[b_kmajor], "ldb": vb[1],
                "ldc": vo[1], "swap": False}
    else:
        args = {"M": N, "N": M, "K": K, "layout_a": lay[b_kmajor], "lda": vb[1], "layout_b": lay[a_kmajor], "ldb": va[1],
                "ldc": vo[1], "swap": True}
    args.update(copies)
    args["bias_mode"] = BIAS_NONE if bias_stride is None else (BIAS_ROW if args["swap"] else BIAS_COL)
    args["copy_bias"] = bias_stride is not None and ((bias_stride != 1 and N > 1) or bias_ptr % 4 != 0)
    return args


def bmm_plan(a_shape, a_stride, b_shape, b_stride, out_stride, a_ptr: int = 0, b_ptr: int = 0, out_ptr: int = 0,
             bias_stride=None, bias_ptr: int = 0, bias_entry_stride=None, bf16: bool = False, out_bf16: bool = False) -> dict:
    """run_batched arguments for out = a @ b with a: (Bt, M, K), b: (Bt, K, N), out: (Bt, M, N), from shapes, element strides
    and addresses.  Each matrix is mapped as in matmul_plan (layouts, lds, swap, bias_mode); stride_a / stride_b / stride_c
    are the batch strides of the kernel's A, B and C (b's and a's when swapped).  With more than one entry a tensor is also
    marked for copying when its batch stride is not a positive multiple of 4 floats (an expanded operand has stride 0), and
    out when its entries would overlap; the arguments returned then describe the dense copies bmm makes (a row-major and b
    column-major with rows padded to a multiple of 4, out contiguous row-major).

    bias_entry_stride is the entry stride of a (Bt, N) bias, one bias per entry (None: a (N,) bias shared by all entries).
    stride_bias is the entry stride run_batched_act takes: 0 for a shared bias, an expanded one (entry stride 0) or a single
    entry.  copy_bias also marks a per-entry bias with a negative entry stride; the copy bmm makes of a per-entry bias is
    (Bt, N) contiguous (stride_bias = N), of a shared one (N,).  bf16: a and b are BF16 (run_batched_typed): their rows,
    batch strides and copies' padded rows are multiples of 8 elements (16 bytes) instead of 4.  out_bf16: the same for out
    (run_batched_mixed): its rows and batch stride are multiples of 8 elements or it is copied, the copy (Bt, M, pad8(N))."""
    Bt, M, K = a_shape
    Bt2, K2, N = b_shape
    if Bt != Bt2:
        raise ValueError(f"batch sizes differ: {tuple(a_shape)} @ {tuple(b_shape)}")
    mp = matmul_plan((M, K), tuple(a_stride[1:]), (K2, N), tuple(b_stride[1:]), tuple(out_stride[1:]), a_ptr, b_ptr, out_ptr,
                     bias_stride, bias_ptr, bf16, out_bf16)
    sa, sb, so = a_stride[0], b_stride[0], out_stride[0]
    e16, pad = (8, _pad8) if bf16 else (4, _pad4)
    if Bt > 1:
        def bad(st, e=4):
            return st <= 0 or st % e != 0
        mp["copy_a"] = mp["copy_a"] or bad(sa, e16)
        mp["copy_b"] = mp["copy_b"] or bad(sb, e16)
        mp["copy_out"] = mp["copy_out"] or bad(so, 8 if out_bf16 else 4) or so < mp["ldc"] * mp["N"]
    if mp["copy_a"] or mp["copy_b"] or mp["copy_out"]:
        # the copies: a (Bt, M, pad4(K)) row-major, b as (Bt, N, pad4(K)) transposed, out (Bt, M, N) contiguous (pad8: BF16;
        # a BF16 out: (Bt, M, pad8(N)))
        on = _pad8(N) if out_bf16 else N
        a_st = (M * pad(K), pad(K), 1) if mp["copy_a"] else tuple(a_stride)
        b_st = (N * pad(K), 1, pad(K)) if mp["copy_b"] else tuple(b_stride)
        o_st = (M * on, on, 1) if mp["copy_out"] else tuple(out_stride)
        copies = {k: mp[k] for k in ("copy_a", "copy_b", "copy_out", "copy_bias")}
        mp = matmul_plan((M, K), a_st[1:], (K, N), b_st[1:], o_st[1:], 0 if copies["copy_a"] else a_ptr,
                         0 if copies["copy_b"] else b_ptr, 0 if copies["copy_out"] else out_ptr, bias_stride, bias_ptr, bf16,
                         out_bf16)
        mp.update(copies)
        sa, sb, so = a_st[0], b_st[0], o_st[0]
    mp["batch"] = Bt
    mp["stride_a"], mp["stride_b"] = (sb, sa) if mp["swap"] else (sa, sb)
    mp["stride_c"] = so
    mp["stride_bias"] = 0
    if bias_entry_stride is not None and Bt > 1 and bias_entry_stride != 0:
        mp["copy_bias"] = mp["copy_bias"] or bias_entry_stride < 0
        mp["stride_bias"] = N if mp["copy_bias"] else bias_entry_stride
    return mp


def linear_plan(x_shape, x_stride, w_shape) -> dict:
    """Shapes of linear(x, weight) with x: (..., K), weight: (N, K): the product runs on x flattened to (M, K); view is
    (M, K) element strides of that flattening when x's leading dimensions collapse into one stride (a view, no copy),
    None when x has to be copied first."""
    *lead, K = x_shape
    N, K2 = w_shape
    if K != K2:
        raise ValueError(f"x has {K} features, weight expects {K2}")
    M = 1
    for d in lead:
        M *= d
    # the leading dimensions of size > 1 must nest: stride[i] = stride[i+1] * shape[i+1]
    dims = [(d, s) for d, s in zip(lead, x_stride[:-1]) if d > 1]
    view = None
    if all(dims[i][1] == dims[i + 1][1] * dims[i + 1][0] for i in range(len(dims) - 1)):
        view = (dims[-1][1] if dims else max(K, 1), x_stride[-1])
    return {"M": M, "K": K, "N": N, "out_shape": (*lead, N), "view": view}


def _ptr(x) -> int:
    """Device/host address of a torch tensor, numpy array or raw int."""
    if isinstance(x, int):
        return x
    if hasattr(x, "data_ptr"):
        return x.data_ptr()
    if hasattr(x, "ctypes"):
        return x.ctypes.data
    raise TypeError(type(x))


class FtSgemm:
    """One handle = one device context (cuBLAS handle, checksum workspace, fault counters).

    CUDA graphs: matmul, bmm and linear (bmm and linear forward and backward) can be captured with torch.cuda.graph (its
    default global capture mode) or torch.cuda.make_graphed_callables, first calls of a shape included.  A replay reads the tensors the
    capture used -- copy new inputs into those same static tensors -- and writes C bit for bit as the eager call would; eager
    calls and replays may interleave on one handle in stream order.  stats() synchronises only the stream of the handle's
    last call, so synchronise the replay stream first; inside a capture it raises FtsgemmError(-2), as run_host, verify and
    the baseline with host sync do.  The handle keeps what a graph uses until close(): close it after its graphs
    (include/ftsgemm.h, "CUDA graphs")."""

    def __init__(self):
        self._h = C.c_void_p()
        _check(lib().ftsgemm_create(C.byref(self._h)))

    def close(self):
        if self._h:
            lib().ftsgemm_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _run_checked(self, code):
        if code != 0:
            msg = lib().ftsgemm_error_string(code).decode()
            raise FtsgemmError(code, f"{msg} (cuda/cublas status {lib().ftsgemm_last_cuda_error(self._h)})")

    # the reference kernel contract:  kernel<<<...>>>(M, N, K, dA, dB, dC, alpha, beta)  selected by id
    def run(self, kernel_id: int, M: int, N: int, K: int, dA, dB, dC, alpha: float = 1.0, beta: float = 0.0,
            opts: Opts | None = None) -> None:
        self._run_checked(lib().ftsgemm_run(self._h, kernel_id, M, N, K, _ptr(dA), _ptr(dB), _ptr(dC), alpha, beta,
                                            C.byref(opts) if opts is not None else None))

    def run_ex(self, kernel_id: int, M: int, N: int, K: int, dA, layout_a: int, lda: int, dB, layout_b: int, ldb: int, dC,
               ldc: int, alpha: float = 1.0, beta: float = 0.0, opts: Opts | None = None) -> None:
        """C = alpha * A * B^T + beta * C with a layout (LAYOUT_MN_MAJOR / LAYOUT_K_MAJOR) and a leading dimension per
        operand; C column-major with ldc >= M (include/ftsgemm.h: ftsgemm_run_ex)."""
        self._run_checked(lib().ftsgemm_run_ex(self._h, kernel_id, M, N, K, _ptr(dA), layout_a, lda, _ptr(dB), layout_b, ldb,
                                               _ptr(dC), ldc, alpha, beta, C.byref(opts) if opts is not None else None))

    def run_bias(self, kernel_id: int, M: int, N: int, K: int, dA, layout_a: int, lda: int, dB, layout_b: int, ldb: int, dC,
                 ldc: int, alpha: float = 1.0, beta: float = 0.0, bias=None, bias_mode: int = BIAS_NONE,
                 opts: Opts | None = None) -> None:
        """C = (alpha * A * B^T + beta * C) + bias, the bias added in the store pass under the same ABFT protection:
        bias[m] per row (BIAS_ROW, length M) or bias[n] per column (BIAS_COL, length N) (include/ftsgemm.h:
        ftsgemm_run_bias).  The value in parentheses is bit for bit what run_ex stores."""
        self._run_checked(lib().ftsgemm_run_bias(self._h, kernel_id, M, N, K, _ptr(dA), layout_a, lda, _ptr(dB), layout_b, ldb,
                                                 _ptr(dC), ldc, alpha, beta, _ptr(bias) if bias is not None else None, bias_mode,
                                                 C.byref(opts) if opts is not None else None))

    def run_act(self, kernel_id: int, M: int, N: int, K: int, dA, layout_a: int, lda: int, dB, layout_b: int, ldb: int, dC,
                ldc: int, alpha: float = 1.0, beta: float = 0.0, bias=None, bias_mode: int = BIAS_NONE,
                activation: int = ACT_NONE, dZ=None, opts: Opts | None = None) -> None:
        """C = act(z) with z = (alpha * A * B^T + beta * C) + bias, bit for bit what run_bias stores; z also into dZ (C's
        geometry: M x N column-major, ldc) when given.  ACT_RELU / ACT_GELU are applied in the store pass; ABFT verifies z,
        not the activation's own arithmetic (include/ftsgemm.h: ftsgemm_run_act)."""
        self._run_checked(lib().ftsgemm_run_act(self._h, kernel_id, M, N, K, _ptr(dA), layout_a, lda, _ptr(dB), layout_b, ldb,
                                                _ptr(dC), ldc, alpha, beta, _ptr(bias) if bias is not None else None, bias_mode,
                                                activation, _ptr(dZ) if dZ is not None else None,
                                                C.byref(opts) if opts is not None else None))

    def run_batched(self, kernel_id: int, M: int, N: int, K: int, dA, layout_a: int, lda: int, stride_a: int, dB, layout_b: int,
                    ldb: int, stride_b: int, dC, ldc: int, stride_c: int, batch: int, alpha: float = 1.0, beta: float = 0.0,
                    bias=None, bias_mode: int = BIAS_NONE, opts: Opts | None = None) -> None:
        """`batch` run_bias products in one launch: entry i on dA + i*stride_a, dB + i*stride_b, dC + i*stride_c (element
        strides), one bias shared by all entries (include/ftsgemm.h: ftsgemm_run_batched).  Fault and event rows are stacked
        rows i*M + m."""
        self._run_checked(lib().ftsgemm_run_batched(self._h, kernel_id, M, N, K, _ptr(dA), layout_a, lda, stride_a, _ptr(dB),
                                                    layout_b, ldb, stride_b, _ptr(dC), ldc, stride_c, batch, alpha, beta,
                                                    _ptr(bias) if bias is not None else None, bias_mode,
                                                    C.byref(opts) if opts is not None else None))

    def run_batched_act(self, kernel_id: int, M: int, N: int, K: int, dA, layout_a: int, lda: int, stride_a: int, dB,
                        layout_b: int, ldb: int, stride_b: int, dC, ldc: int, stride_c: int, batch: int, alpha: float = 1.0,
                        beta: float = 0.0, bias=None, bias_mode: int = BIAS_NONE, stride_bias: int = 0,
                        activation: int = ACT_NONE, dZ=None, opts: Opts | None = None) -> None:
        """`batch` run_act products in one launch: entry i is run_act on dA + i*stride_a, dB + i*stride_b, dC + i*stride_c
        with the bias bias + i*stride_bias (0: shared by all entries) and z into dZ + i*stride_c when dZ is given
        (include/ftsgemm.h: ftsgemm_run_batched_act).  Fault and event rows are stacked rows i*M + m."""
        self._run_checked(lib().ftsgemm_run_batched_act(self._h, kernel_id, M, N, K, _ptr(dA), layout_a, lda, stride_a, _ptr(dB),
                                                        layout_b, ldb, stride_b, _ptr(dC), ldc, stride_c, batch, alpha, beta,
                                                        _ptr(bias) if bias is not None else None, bias_mode, stride_bias,
                                                        activation, _ptr(dZ) if dZ is not None else None,
                                                        C.byref(opts) if opts is not None else None))

    def run_out(self, kernel_id: int, M: int, N: int, K: int, dA, layout_a: int, lda: int, dB, layout_b: int, ldb: int, dC,
                ldc: int, dD, alpha: float = 1.0, beta: float = 0.0, bias=None, bias_mode: int = BIAS_NONE,
                activation: int = ACT_NONE, dZ=None, opts: Opts | None = None) -> None:
        """run_act with the result written to dD (C's geometry: ldc) and C read-only: bit for bit run_act on a copy of C in
        dD.  dC may be None with beta = 0 (C is not read); dD == dC is run_act itself (include/ftsgemm.h:
        ftsgemm_run_out)."""
        self._run_checked(lib().ftsgemm_run_out(self._h, kernel_id, M, N, K, _ptr(dA), layout_a, lda, _ptr(dB), layout_b, ldb,
                                                _ptr(dC) if dC is not None else None, ldc, _ptr(dD), alpha, beta,
                                                _ptr(bias) if bias is not None else None, bias_mode, activation,
                                                _ptr(dZ) if dZ is not None else None, C.byref(opts) if opts is not None else None))

    def run_batched_out(self, kernel_id: int, M: int, N: int, K: int, dA, layout_a: int, lda: int, stride_a: int, dB,
                        layout_b: int, ldb: int, stride_b: int, dC, ldc: int, stride_c: int, dD, batch: int, alpha: float = 1.0,
                        beta: float = 0.0, bias=None, bias_mode: int = BIAS_NONE, stride_bias: int = 0,
                        activation: int = ACT_NONE, dZ=None, opts: Opts | None = None) -> None:
        """run_batched_act with the results written to dD (C's geometry: ldc, entry i at dD + i*stride_c) and C read-only:
        bit for bit run_batched_act on a copy of C in dD (include/ftsgemm.h: ftsgemm_run_batched_out)."""
        self._run_checked(lib().ftsgemm_run_batched_out(self._h, kernel_id, M, N, K, _ptr(dA), layout_a, lda, stride_a, _ptr(dB),
                                                        layout_b, ldb, stride_b, _ptr(dC) if dC is not None else None, ldc,
                                                        stride_c, _ptr(dD), batch, alpha, beta,
                                                        _ptr(bias) if bias is not None else None, bias_mode, stride_bias,
                                                        activation, _ptr(dZ) if dZ is not None else None,
                                                        C.byref(opts) if opts is not None else None))

    def run_batched_typed(self, kernel_id: int, M: int, N: int, K: int, dA, layout_a: int, lda: int, stride_a: int, dB,
                          layout_b: int, ldb: int, stride_b: int, ab_type: int, dC, ldc: int, stride_c: int, dD, batch: int,
                          alpha: float = 1.0, beta: float = 0.0, bias=None, bias_mode: int = BIAS_NONE, stride_bias: int = 0,
                          activation: int = ACT_NONE, dZ=None, opts: Opts | None = None) -> None:
        """run_batched_out with A and B of element type ab_type (TYPE_F32: run_batched_out itself; TYPE_BF16: BF16 A and B,
        leading dimensions and entry strides in elements, FP32 accumulate, C / D / Z / bias FP32; include/ftsgemm.h:
        ftsgemm_run_batched_typed)."""
        self._run_checked(lib().ftsgemm_run_batched_typed(self._h, kernel_id, M, N, K, _ptr(dA), layout_a, lda, stride_a,
                                                          _ptr(dB), layout_b, ldb, stride_b, ab_type,
                                                          _ptr(dC) if dC is not None else None, ldc, stride_c, _ptr(dD), batch,
                                                          alpha, beta, _ptr(bias) if bias is not None else None, bias_mode,
                                                          stride_bias, activation, _ptr(dZ) if dZ is not None else None,
                                                          C.byref(opts) if opts is not None else None))

    def run_batched_mixed(self, kernel_id: int, M: int, N: int, K: int, dA, layout_a: int, lda: int, stride_a: int, dB,
                          layout_b: int, ldb: int, stride_b: int, ab_type: int, dC, ldc: int, stride_c: int, dD, cd_type: int,
                          batch: int, alpha: float = 1.0, beta: float = 0.0, bias=None, bias_mode: int = BIAS_NONE,
                          stride_bias: int = 0, activation: int = ACT_NONE, dZ=None, opts: Opts | None = None) -> None:
        """run_batched_typed with C, D and Z of element type cd_type (TYPE_F32: run_batched_typed itself; TYPE_BF16: BF16 C,
        D and Z, BF16 operands only, ldc and stride_c in elements, everything up to the store FP32 and the stored values
        rounded to nearest even; include/ftsgemm.h: ftsgemm_run_batched_mixed)."""
        self._run_checked(lib().ftsgemm_run_batched_mixed(self._h, kernel_id, M, N, K, _ptr(dA), layout_a, lda, stride_a,
                                                          _ptr(dB), layout_b, ldb, stride_b, ab_type,
                                                          _ptr(dC) if dC is not None else None, ldc, stride_c, _ptr(dD), cd_type,
                                                          batch, alpha, beta, _ptr(bias) if bias is not None else None,
                                                          bias_mode, stride_bias, activation,
                                                          _ptr(dZ) if dZ is not None else None,
                                                          C.byref(opts) if opts is not None else None))

    def run_typed(self, kernel_id: int, M: int, N: int, K: int, dA, layout_a: int, lda: int, dB, layout_b: int, ldb: int,
                  ab_type: int, dC, ldc: int, dD, alpha: float = 1.0, beta: float = 0.0, bias=None, bias_mode: int = BIAS_NONE,
                  activation: int = ACT_NONE, dZ=None, opts: Opts | None = None) -> None:
        """run_batched_typed with batch = 1 (include/ftsgemm.h: ftsgemm_run_typed)."""
        self._run_checked(lib().ftsgemm_run_typed(self._h, kernel_id, M, N, K, _ptr(dA), layout_a, lda, _ptr(dB), layout_b, ldb,
                                                  ab_type, _ptr(dC) if dC is not None else None, ldc, _ptr(dD), alpha, beta,
                                                  _ptr(bias) if bias is not None else None, bias_mode, activation,
                                                  _ptr(dZ) if dZ is not None else None, C.byref(opts) if opts is not None else None))

    def bmm(self, a, b, out=None, *, c=None, bias=None, activation=None, preact=None, kernel_id: int = ID_ABFT_AUTO,
            alpha: float = 1.0, beta: float = 0.0, opts: Opts | None = None, out_dtype=None):
        """out = act(alpha * (a @ b) + beta * out + bias) for 3-D float32 CUDA tensors a: (Bt, M, K), b: (Bt, K, N), out:
        (Bt, M, N), an optional bias (N,) shared by all entries or (Bt, N) one per entry, and an optional activation --
        torch.baddbmm plus a bias and an activation -- as ONE run_batched_mixed call; returns out.

        Every matrix may be row- or column-major with any leading stride that keeps 16-byte rows, and is read in place when
        its batch stride is a multiple of 4 floats: contiguous bmm operands and q @ k.transpose(-1, -2) copy nothing.  An
        expanded operand (batch stride 0), a batch stride that is not a multiple of 4, or a matrix matmul could not read in
        place is copied once (bmm_plan); an out that cannot be written in place is computed in a contiguous buffer and copied
        back.  Fault and event coordinates (opts, stats()) are stacked kernel rows entry * kernel_M + row, transposed against
        out when the call is swapped (a row-major out: the kernel's rows are out's columns).  Capturable in a CUDA graph (see
        the class docstring); copies it makes are then graph-pool tensors, refreshed on every replay.

        activation = "relu" | "gelu" stores act(z) with z the value above, in the same store pass, and z into preact when
        given (preact must have out's shape and strides; out and preact must be writable in place, else ValueError), as
        matmul does.

        Autograd: with out=None, grad mode on and any of a, b, bias requiring grad, bmm is differentiable.  The forward is
        the same single call; z is written for GELU only (ReLU's backward reads out > 0).  Backward: grad_z =
        threshold_backward / gelu_backward in torch (grad_out itself without an activation), grad_a = alpha * grad_z @ b^T and
        grad_b = alpha * a^T @ grad_z through bmm with the same kernel id and opts (injected faults stripped, on the stream
        autograd runs the backward on), grad_bias = grad_z summed over the entries' rows (per-entry bias) or over entries
        and rows (shared bias).  An expanded operand is copied as above and autograd sums its gradient.  With out= given
        nothing is recorded (as torch.bmm(out=...)).  Forward and backward can be captured in a CUDA graph, also through
        torch.cuda.make_graphed_callables.

        c: a (Bt, M, N) tensor read in place of out's old values and never written -- out = act(alpha * (a @ b) + beta * c
        + bias), bit for bit what the call gives with out holding a copy of c (the same call with C = c and D = out; without
        c, C = D = out).  beta must not be 0 (c would not be read: ValueError).  With out=None, out is allocated with c's
        strides (c dense) and the call is differentiable in c as well: grad_c = beta * grad_z.  The kernels read c with out's
        geometry: a c with other strides (or a base that is not 16-byte aligned) is copied once into that geometry first.

        a and b may also both be bfloat16 (mixed with float32: TypeError): the same call with TYPE_BF16, on the BF16 kernels,
        FP32 accumulate, with out, c and preact float32 as above and a bfloat16 bias upcast (exactly) into a float32
        temporary; copies pad rows to 8 elements (bmm_plan with bf16).  Autograd as above, with grad_z rounded to bfloat16
        once for the two gradient products (the rounding of torch autocast's BF16 backward), which run on the BF16 kernels
        and write bfloat16 directly; grad_a, grad_b, grad_bias and grad_c come back in the dtypes of a, b, the bias and c.

        The result dtype is out.dtype when out is given, else c.dtype when c is, else out_dtype (None: float32).  A bfloat16
        result needs bfloat16 a and b (else TypeError) and is one run_batched_mixed call with BF16 C / D / Z: the float32
        result of the same call rounded to nearest even, as .to(torch.bfloat16) rounds it, with no separate cast pass.  c
        and preact must have the result dtype, and an out_dtype that contradicts out or c raises ValueError.  A bfloat16 out
        is written in place when its rows and batch stride are multiples of 8 elements; otherwise through a copy with rows
        padded to 8 (bmm_plan with out_bf16).  Autograd: grad_out arrives in the result dtype."""
        import torch
        for name, t in (("a", a), ("b", b)):
            if t.dtype not in (torch.float32, torch.bfloat16) or not t.is_cuda:
                raise TypeError(f"{name} must be a float32 or bfloat16 CUDA tensor")
            if t.dim() != 3:
                raise TypeError(f"{name} must be 3-D")
        if a.dtype != b.dtype:
            raise TypeError(f"a and b must both be float32 or both bfloat16, not {a.dtype} and {b.dtype}")
        bf16 = a.dtype == torch.bfloat16
        rdt = out.dtype if out is not None else c.dtype if c is not None else out_dtype or torch.float32  # result dtype
        if out_dtype is not None and out_dtype != rdt:
            raise ValueError(f"out_dtype {out_dtype} contradicts the {rdt} of {'out' if out is not None else 'c'}")
        if rdt not in (torch.float32, torch.bfloat16):
            raise ValueError(f"the result must be float32 or bfloat16, not {rdt}")
        out16 = rdt == torch.bfloat16
        if out16 and not bf16:
            raise TypeError("a bfloat16 result needs bfloat16 a and b")
        rname = "bfloat16" if out16 else "float32"
        Bt, M, K = a.shape
        N = b.shape[2]
        if b.shape[0] != Bt or b.shape[1] != K or b.device != a.device:
            raise ValueError(f"b must be a ({Bt}, {K}, N) tensor on {a.device}")
        if activation not in ACTIVATIONS:
            raise ValueError(f"activation must be None, 'relu' or 'gelu', not {activation!r}")
        if preact is not None and activation is None:
            raise ValueError("preact needs an activation")
        if c is not None:
            if beta == 0.0:
                raise ValueError("c is not read with beta = 0")
            if c.shape != (Bt, M, N) or c.dtype != rdt or c.device != a.device:
                raise ValueError(f"c must be a {rname} ({Bt}, {M}, {N}) tensor on {a.device}")
        if out is None and c is None and beta != 0.0:
            raise ValueError("beta != 0 needs an out tensor or c")
        if out is None and torch.is_grad_enabled() and any(t is not None and t.requires_grad for t in (a, b, bias, c)):
            # (a bfloat16 bias is upcast inside the forward, which runs without grad: autograd sees the caller's tensor)
            fwd = Opts.from_buffer_copy(opts) if opts is not None else make_opts()
            if not fwd.stream:
                fwd.stream = torch.cuda.current_stream(a.device).cuda_stream
            return _bmm_fn().apply(a, b, bias, preact, c, self, kernel_id, alpha, beta, fwd, activation, rdt)
        if out is None:
            out = (torch.empty_like(c, memory_format=torch.preserve_format) if c is not None else
                   torch.empty(Bt, M, N, device=a.device, dtype=rdt))
        if out.shape != (Bt, M, N) or out.device != a.device:
            raise ValueError(f"out must be a {rname} ({Bt}, {M}, {N}) tensor on {a.device}")
        if bf16 and bias is not None and bias.dtype == torch.bfloat16:
            bias = bias.float()
        if bias is not None and (bias.shape not in ((N,), (Bt, N)) or bias.dtype != torch.float32 or bias.device != a.device):
            raise ValueError(f"bias must be a float32 ({N},) or ({Bt}, {N}) tensor on {a.device}")
        if preact is not None and (preact.shape != out.shape or preact.stride() != out.stride() or
                                   preact.dtype != rdt or preact.device != a.device):
            raise ValueError(f"preact must be a {rname} tensor with out's shape and strides on out's device")
        if Bt == 0:  # an empty batch (torch.bmm accepts it): nothing to compute
            return out
        per_entry = bias is not None and bias.dim() == 2
        bias_stride = bias.stride(-1) if bias is not None else None
        plan = bmm_plan(tuple(a.shape), a.stride(), tuple(b.shape), b.stride(), out.stride(), a.data_ptr(), b.data_ptr(),
                        out.data_ptr(), bias_stride, bias.data_ptr() if bias is not None else 0,
                        bias.stride(0) if per_entry else None, bf16, out16)
        if activation is not None and plan["copy_out"]:
            raise ValueError("out (and so preact) must be writable in place with an activation: 16-byte rows and entries")
        if plan["copy_bias"]:
            bias = (torch.empty(Bt, N, device=a.device, dtype=torch.float32).copy_(bias) if plan["stride_bias"] != 0 else
                    torch.empty(N, device=a.device, dtype=torch.float32).copy_(bias[0] if per_entry else bias))
        pad = _pad8 if bf16 else _pad4
        if plan["copy_a"]:
            a = torch.empty(Bt, M, pad(K), device=a.device, dtype=a.dtype)[:, :, :K].copy_(a)
        if plan["copy_b"]:
            b = torch.empty(Bt, N, pad(K), device=a.device, dtype=b.dtype)[:, :, :K].copy_(b.transpose(1, 2)).transpose(1, 2)
        dst = out
        if plan["copy_out"] and out16:  # (rows padded to 8 elements, plan["ldc"])
            dst = torch.empty(Bt, M, _pad8(N), device=a.device, dtype=rdt)[:, :, :N]
            if beta != 0.0 and c is None:
                dst.copy_(out)
        elif plan["copy_out"]:
            dst = (out.contiguous() if beta != 0.0 and c is None else
                   torch.empty(Bt, M, N, device=a.device, dtype=torch.float32))
            if dst is out:
                dst = out.clone()
        if c is not None and (c.stride() != dst.stride() or c.data_ptr() % 16 != 0):
            c = torch.empty_strided(dst.shape, dst.stride(), device=a.device, dtype=rdt).copy_(c)
        if opts is None:
            opts = make_opts(stream=torch.cuda.current_stream(a.device).cuda_stream)
        kA, kB = (b, a) if plan["swap"] else (a, b)
        self.run_batched_mixed(kernel_id, plan["M"], plan["N"], plan["K"], kA, plan["layout_a"], plan["lda"], plan["stride_a"],
                               kB, plan["layout_b"], plan["ldb"], plan["stride_b"], TYPE_BF16 if bf16 else TYPE_F32,
                               c if c is not None else dst, plan["ldc"], plan["stride_c"], dst, TYPE_BF16 if out16 else TYPE_F32,
                               Bt, alpha, beta, bias, plan["bias_mode"], plan["stride_bias"], ACTIVATIONS[activation], preact,
                               opts)
        if dst is not out:
            out.copy_(dst)
        return out

    def matmul(self, a, b, out=None, *, c=None, bias=None, activation=None, preact=None, kernel_id: int = ID_ABFT_AUTO,
               alpha: float = 1.0, beta: float = 0.0, opts: Opts | None = None, out_dtype=None):
        """out = alpha * (a @ b) + beta * out + bias for 2-D float32 CUDA tensors a: (M, K), b: (K, N) and an optional 1-D
        float32 bias of length N (one value per column of out, added in the fused store pass); returns out.

        a, b and out may each be row-major or column-major (a .t() view is the other layout) with any leading stride that
        keeps 16-byte rows; they are read and written in place -- x @ W.T + b (F.linear) on row-major tensors copies
        nothing.  An operand that cannot be read in place (no unit stride, a base address or, for a and b, a
        leading stride that is not a multiple of 16 bytes) is copied once into an aligned buffer first; an out that cannot
        be written in place is computed in a contiguous buffer and copied back; a bias without unit stride is copied once.
        With out=None a new row-major out is returned and beta must be 0.  The mapping onto the kernel is matmul_plan: a
        row-major out is computed as out^T = b^T a^T, so the kernel's (row, col) is out's (col, row) -- the coordinates of
        injected faults (opts) and of stats() events are the kernel's, transposed against out in that case.  A kernel M or
        N (after the mapping) that is not a multiple of 4 raises FtsgemmError(-2) for the tensor-core ids, as run does.
        Runs on the current torch stream unless opts.stream says otherwise.  No autograd: linear() is the differentiable
        F.linear.  Every call is bmm on a batch of one entry, so one run_batched_mixed call with batch = 1.  Capturable in a
        CUDA graph (see the class docstring).

        activation = "relu" | "gelu" stores act(z) with z the value above, in the same store pass of the same call, and z
        into preact when given.  preact must have out's shape and strides, and out and preact must both be writable in place
        (else ValueError: there is no copy path for them); a, b and the bias are copied as above when needed.

        c: an (M, N) tensor read in place of out's old values and never written -- out = act(alpha * (a @ b) + beta * c +
        bias), bit for bit what the call gives with out holding a copy of c (the same call with C = c and D = out).  beta
        must not be 0 (c would not be read: ValueError).  With out=None, out is allocated with c's strides (c dense).  The
        kernels read c with out's geometry: a c with other strides (or a base that is not 16-byte aligned) is copied once
        into that geometry first.

        a and b may also both be bfloat16 (float32 and bfloat16 mixed raise TypeError): the same call on the BF16 kernels,
        FP32 accumulate, with out, c and preact float32 as above; a bfloat16 bias is upcast (exactly) into a float32
        temporary.  Their copies pad rows to 8 elements (matmul_plan with bf16).

        The result dtype is chosen as in bmm: out.dtype, else c.dtype, else out_dtype (None: float32); a bfloat16 result
        needs bfloat16 a and b and is the float32 result rounded to nearest even in the same store pass."""
        import torch
        # (bmm checks everything else on the batch-of-one views)
        for name, t in (("a", a), ("b", b)):
            if t.dim() != 2:
                raise TypeError(f"{name} must be 2-D")
        M, N = a.shape[0], b.shape[1]
        if out is None:
            if c is not None:
                out = torch.empty_like(c, memory_format=torch.preserve_format)
            elif beta != 0.0:
                raise ValueError("beta != 0 needs an out tensor or c")
            else:
                out = torch.empty(M, N, device=a.device, dtype=out_dtype or torch.float32)
        for name, t in (("c", c), ("out", out), ("preact", preact)):
            if t is not None and t.shape != (M, N):
                raise ValueError(f"{name} must be an ({M}, {N}) tensor")
        if bias is not None and bias.dim() != 1:  # (bmm would take a (1, N) bias as one bias per entry)
            raise ValueError(f"bias must be a ({N},) tensor")
        self.bmm(a[None], b[None], out[None], c=c[None] if c is not None else None, bias=bias, activation=activation,
                 preact=preact[None] if preact is not None else None, kernel_id=kernel_id, alpha=alpha, beta=beta, opts=opts,
                 out_dtype=out_dtype)
        return out

    def linear(self, x, weight, bias=None, *, activation=None, residual=None, kernel_id: int = ID_ABFT_AUTO,
               opts: Opts | None = None, out_dtype=None):
        """F.linear(x, weight, bias) = x @ weight.T + bias under ABFT protection, differentiable: x (..., K), weight (N, K),
        bias (N,) or None, all float32 CUDA tensors; returns (..., N).

        The forward is one matmul, so one run_batched_mixed call, with the bias fused into the store pass, whatever the
        activation and residual (one autograd Function, _linear_fn); x's leading dimensions are flattened as a view
        where the strides allow it (linear_plan) and copied otherwise.  Backward: grad_x = grad_y @ weight and
        grad_weight = grad_y^T @ x through matmul with the same kernel id and opts (both read in place), grad_bias =
        grad_y.sum(0) in torch.  Faults injected through opts land in the forward product only; faults detected in any of
        the three products are counted in stats().  The forward runs on the current torch stream unless opts.stream names
        one; the backward runs on the stream autograd runs it on.  Forward and backward can be captured in a CUDA graph, also
        through torch.cuda.make_graphed_callables (see the class docstring).

        activation = "relu" | "gelu" gives F.relu / F.gelu(F.linear(...)) from the same single matmul, the activation fused
        into its store pass.  The pre-activation value is written only where the backward needs it: for GELU, when grad mode
        is on and an input requires grad (ReLU's backward reads y > 0).  Backward: grad_z = threshold_backward(grad_y, y, 0)
        or gelu_backward(grad_y, z) in torch, then the three gradients as above from grad_z.

        residual = r, a tensor of the output's shape (..., N): y = (x @ weight.T + r) + bias -- the residual connection of a
        transformer block -- from the same single matmul (beta = 1, r read in place of the old output and never written),
        under the same ABFT protection.  The bias is added after the residual, the kernel's order, so y can differ from
        F.linear(x, weight, bias) + r in the last bits.  y has r's strides when r is dense.  Backward: grad_r = grad_y, the
        other gradients as above.  A residual with an activation raises ValueError.

        x and weight may also both be bfloat16 (mixed with float32: TypeError): the product runs on the BF16 kernels (FP32
        accumulate) and y is float32, as are the residual and the pre-activation value; a bfloat16 bias is upcast exactly.
        The backward rounds grad_z to bfloat16 once (the rounding of torch autocast's BF16 backward) and runs grad_x and
        grad_weight on the BF16 kernels, which write them as bfloat16; the gradients come back in the dtypes of x, weight
        and the bias.

        out_dtype=torch.bfloat16 (bfloat16 x and weight only, else TypeError) makes y bfloat16: the float32 y above rounded
        to nearest even in the same store pass, as F.linear on bfloat16 tensors returns it.  The residual must then be
        bfloat16 and the saved pre-activation value is bfloat16; grad_y arrives as bfloat16, grad_z is formed from it in
        torch (rounded to bfloat16 once) and grad_r is grad_y."""
        import torch
        if x.dtype not in (torch.float32, torch.bfloat16) or not x.is_cuda or x.dim() < 1:
            raise TypeError("x must be a float32 or bfloat16 CUDA tensor with at least one dimension")
        if weight.dim() != 2:
            raise TypeError("weight must be 2-D (out_features, in_features)")
        if weight.dtype != x.dtype:
            raise TypeError(f"x and weight must both be float32 or both bfloat16, not {x.dtype} and {weight.dtype}")
        ydt = out_dtype or torch.float32
        if ydt not in (torch.float32, torch.bfloat16):
            raise ValueError(f"out_dtype must be float32 or bfloat16, not {ydt}")
        if ydt == torch.bfloat16 and x.dtype != torch.bfloat16:
            raise TypeError("out_dtype=torch.bfloat16 needs bfloat16 x and weight")
        lp = linear_plan(tuple(x.shape), x.stride(), tuple(weight.shape))
        x2 = (x.as_strided((lp["M"], lp["K"]), lp["view"], x.storage_offset()) if lp["view"] is not None
              else x.reshape(lp["M"], lp["K"]).contiguous())
        r2 = None
        if residual is not None:
            if activation is not None:
                raise ValueError("a residual cannot be combined with an activation")
            if tuple(residual.shape) != lp["out_shape"] or residual.dtype != ydt or residual.device != x.device:
                raise ValueError(f"residual must be a {ydt} {lp['out_shape']} tensor on {x.device}")
            r2 = residual.reshape(lp["M"], lp["N"])
        fwd = Opts.from_buffer_copy(opts) if opts is not None else make_opts()
        if not fwd.stream:
            fwd.stream = torch.cuda.current_stream(x.device).cuda_stream
        grad = torch.is_grad_enabled() and any(t is not None and t.requires_grad for t in (x, weight, bias))
        y = _linear_fn().apply(x2, weight, bias, r2, self, kernel_id, fwd, activation, grad, ydt)
        return y.view(lp["out_shape"])

    def run_host(self, kernel_id: int, M: int, N: int, K: int, hA, hB, hC, alpha: float = 1.0, beta: float = 0.0,
                 opts: Opts | None = None) -> None:
        self._run_checked(lib().ftsgemm_run_host(self._h, kernel_id, M, N, K, _ptr(hA), _ptr(hB), _ptr(hC), alpha,
                                                 beta, C.byref(opts) if opts is not None else None))

    # baseline_ft_sgemm (include/baseline_ft_sgemm.cuh:1)
    def baseline(self, M, N, K, dA, dB, dC, alpha=1.0, beta=0.0, tf32=False, opts: Opts | None = None,
                 residual_out=None) -> None:
        self._run_checked(lib().ftsgemm_baseline(self._h, M, N, K, _ptr(dA), _ptr(dB), _ptr(dC), alpha, beta,
                                                 1 if tf32 else 0, C.byref(opts) if opts is not None else None,
                                                 _ptr(residual_out) if residual_out is not None else None))

    def stats(self) -> dict:
        s = Stats()
        self._run_checked(lib().ftsgemm_get_stats(self._h, C.byref(s)))
        return s.as_dict()

    # fused multi-GPU verdict exchange (include/ftsgemm.h: ftsgemm_peer_*)
    def peer_export(self) -> bytes:
        buf = C.create_string_buffer(64)
        self._run_checked(lib().ftsgemm_peer_export(self._h, buf))
        return buf.raw

    def peer_connect(self, rank: int, world: int, handles) -> None:
        blob = b"".join(handles)
        assert len(blob) == 64 * world
        self._run_checked(lib().ftsgemm_peer_connect(self._h, rank, world, C.create_string_buffer(blob, len(blob))))

    def peer_verdict(self, world: int, timeout_ms: int = 10000):
        out, per = (C.c_double * 8)(), (C.c_double * (8 * world))()
        self._run_checked(lib().ftsgemm_peer_verdict(self._h, out, per, timeout_ms))
        return list(out), [list(per[8 * r:8 * r + 8]) for r in range(world)]

    def launch_count(self) -> int:
        """Kernels of this library launched through the handle so far (include/ftsgemm.h)."""
        return int(lib().ftsgemm_launch_count(self._h))

    def stats_device(self, d_out8, stream=None) -> None:
        """Device-side verdict vector (8 doubles, see include/ftsgemm.h), asynchronous on `stream`, counters not reset."""
        self._run_checked(lib().ftsgemm_stats_device(self._h, _ptr(d_out8), stream))

    def debug_trace(self):
        """Timeline of the last launch made under debug_set("trace", 1): list (per unit) of item dicts, times in ns."""
        cap = 160 * 512
        buf = (C.c_ulonglong * cap)()
        n = lib().ftsgemm_debug_trace(self._h, buf, cap)
        if n < 0:
            self._run_checked(n)
        keys = ("prod_start", "prod_end", "mma_start", "mma_end", "acc_done", "check_done", "epi_end")
        out = []
        for u in range(n):
            items = []
            for i in range(63):
                r = buf[(u * 64 + i) * 8:(u * 64 + i) * 8 + 8]
                if r[4] == 0:  # unused slot, or an encoder item (it has no accumulator / epilogue)
                    continue
                d = dict(zip(keys, r[:7]))
                d["tile"] = r[7] & 0xFFFFFF
                d["kind"] = r[7] >> 24
                items.append(d)
            if items:
                # the unit's front phase: (start after griddepcontrol.wait, last warp added to front_done) per CTA
                f = buf[(u * 64 + 63) * 8:(u * 64 + 63) * 8 + 8]
                items[0]["front"] = [(f[2 * r], f[2 * r + 1]) for r in range(4) if f[2 * r]]
            out.append(items)
        return out

    # verify_matrix (utils/utils.cu:61-77) on device buffers
    def verify(self, d_ref, d_x, M: int, N: int, stream=None):
        bad, rel = C.c_longlong(), C.c_double()
        code = lib().ftsgemm_verify(self._h, _ptr(d_ref), _ptr(d_x), M, N, C.byref(bad), C.byref(rel), stream)
        if code not in (0, -6):
            self._run_checked(code)
        return code == 0, int(bad.value), float(rel.value)


_LINEAR_FN = None


def _linear_fn():
    """The torch.autograd.Function behind FtSgemm.linear (built on first use: torch is imported lazily): one matmul
    forward (so one run_batched_mixed call), the activation's backward in torch, then the products of _linear_grads."""
    global _LINEAR_FN
    if _LINEAR_FN is None:
        import torch

        class LinearFn(torch.autograd.Function):
            @staticmethod
            def forward(ctx, x2, weight, bias, residual, dev, kernel_id, opts, activation, grad, ydt):
                # (grad: grad mode was on and an input requires grad -- forward itself runs with grad mode off.  z is
                # written for GELU's backward only: ReLU's reads y > 0, and without an activation grad_z is grad_y.
                # ydt: the dtype of y, and of z)
                z = None
                if grad and activation == "gelu":
                    z = torch.empty(x2.shape[0], weight.shape[0], device=x2.device, dtype=ydt)
                y = dev.matmul(x2, weight.t(), c=residual, bias=bias, activation=activation, preact=z, kernel_id=kernel_id,
                               beta=0.0 if residual is None else 1.0, opts=opts, out_dtype=ydt)
                ctx.save_for_backward(x2, weight, y if activation == "relu" else z)
                ctx.dev, ctx.kernel_id, ctx.opts, ctx.activation = dev, kernel_id, opts, activation
                ctx.bias_dtype = bias.dtype if bias is not None else None
                return y

            @staticmethod
            def backward(ctx, gy):
                x2, weight, saved = ctx.saved_tensors
                gz = _grad_z(gy, ctx.activation, saved)
                gx, gw, gb = _linear_grads(ctx, gz, x2, weight, _backward_opts(ctx.opts, gy.device))
                return gx, gw, gb, gy if ctx.needs_input_grad[3] else None, None, None, None, None, None, None

        _LINEAR_FN = LinearFn
    return _LINEAR_FN


def _backward_opts(opts, device):
    """The forward's opts for the gradient products: a copy with the injected faults stripped, on the stream autograd runs
    the backward on."""
    import torch
    bwd = Opts.from_buffer_copy(opts)
    bwd.inject_mode, bwd.n_faults = 0, 0
    bwd.stream = torch.cuda.current_stream(device).cuda_stream
    return bwd


def _grad_z(gy, activation, saved):
    """grad_z from grad_y: threshold_backward on the saved output y (ReLU) or gelu_backward on the saved z (GELU) in torch,
    grad_y itself without an activation."""
    import torch
    if activation == "relu":
        return torch.ops.aten.threshold_backward(gy, saved, 0)
    if activation == "gelu":
        return torch.ops.aten.gelu_backward(gy, saved)
    return gy


def _linear_grads(ctx, gz, x2, weight, bwd):
    """grad_x = grad_z @ weight, grad_weight = grad_z^T @ x through matmul, grad_bias = grad_z summed over the rows (the
    needed ones, None otherwise).  BF16 x and weight: grad_z is rounded to bfloat16 once and the products run on the BF16
    kernels, which write bfloat16 gradients directly (the float32 products rounded once, bit for bit); every gradient is
    returned in its input's dtype."""
    import torch
    gx = gw = gb = None
    g = gz.to(torch.bfloat16) if x2.dtype == torch.bfloat16 else gz
    if ctx.needs_input_grad[0]:
        gx = ctx.dev.matmul(g, weight, kernel_id=ctx.kernel_id, opts=bwd, out_dtype=x2.dtype)
    if ctx.needs_input_grad[1]:
        gw = ctx.dev.matmul(g.t(), x2, kernel_id=ctx.kernel_id, opts=bwd, out_dtype=weight.dtype)
    if ctx.needs_input_grad[2]:
        gb = g.float().sum(0).to(ctx.bias_dtype)
    return gx, gw, gb


_BMM_FN = None


def _bmm_fn():
    """The torch.autograd.Function behind a differentiable FtSgemm.bmm: one bmm forward (so one run_batched_mixed call),
    the activation's backward in torch, then the two gradient products through bmm."""
    global _BMM_FN
    if _BMM_FN is None:
        import torch

        class BmmFn(torch.autograd.Function):
            @staticmethod
            def forward(ctx, a, b, bias, preact, c, dev, kernel_id, alpha, beta, opts, activation, rdt):
                # (rdt: the result dtype, which z has too)
                z = preact
                if z is None and activation == "gelu":
                    z = torch.empty(a.shape[0], a.shape[1], b.shape[2], device=a.device, dtype=rdt)
                y = dev.bmm(a, b, c=c, bias=bias, activation=activation, preact=z, kernel_id=kernel_id, alpha=alpha,
                            beta=beta if c is not None else 0.0, opts=opts, out_dtype=rdt)
                ctx.save_for_backward(a, b, y if activation == "relu" else z)
                ctx.dev, ctx.kernel_id, ctx.alpha, ctx.beta, ctx.opts, ctx.activation = dev, kernel_id, alpha, beta, opts, activation
                ctx.per_entry_bias = bias is not None and bias.dim() == 2
                ctx.bias_dtype = bias.dtype if bias is not None else None
                return y

            @staticmethod
            def backward(ctx, gy):
                a, b, saved = ctx.saved_tensors
                gz = _grad_z(gy, ctx.activation, saved)
                bwd = _backward_opts(ctx.opts, gy.device)
                ga = gb = gbias = gc = None
                # (BF16 operands: grad_z rounded to bfloat16 once for the products, which write the gradients in the inputs'
                # dtypes directly)
                g = gz.to(torch.bfloat16) if a.dtype == torch.bfloat16 else gz
                if ctx.needs_input_grad[0]:
                    ga = ctx.dev.bmm(g, b.transpose(1, 2), kernel_id=ctx.kernel_id, alpha=ctx.alpha, opts=bwd, out_dtype=a.dtype)
                if ctx.needs_input_grad[1]:
                    gb = ctx.dev.bmm(a.transpose(1, 2), g, kernel_id=ctx.kernel_id, alpha=ctx.alpha, opts=bwd, out_dtype=b.dtype)
                if ctx.needs_input_grad[2]:
                    gf = g.float() if a.dtype == torch.bfloat16 else gz
                    gbias = (gf.sum(1) if ctx.per_entry_bias else gf.sum((0, 1))).to(ctx.bias_dtype)
                if ctx.needs_input_grad[4]:
                    gc = ctx.beta * gz
                return ga, gb, gbias, None, gc, None, None, None, None, None, None, None

        _BMM_FN = BmmFn
    return _BMM_FN


def run_cli(args, timeout=None) -> subprocess.CompletedProcess:
    """ft_sgemm START END GAP ST_KERNEL END_KERNEL  (sgemm.cu:13-19)."""
    if not CLI_PATH.exists():
        raise FtsgemmError(-4, f"{CLI_PATH} not built")
    return subprocess.run([str(CLI_PATH), *map(str, args)], capture_output=True, text=True, timeout=timeout)
