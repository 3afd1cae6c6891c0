"""BF16 results (ftsgemm_run_batched_mixed with cd_type = FTSGEMM_TYPE_BF16; FtSgemm.matmul / bmm / linear with bfloat16 out,
c, out_dtype or residual).

The definition every GPU test checks against: a call with BF16 C / D / Z is the same call with FP32 C / D / Z on the exact
upcast of C, its D and Z then rounded to bfloat16 to nearest even -- by torch's own .to(torch.bfloat16) on the GPU.  D16
and Z16 must equal that bit for bit, NaN positions included (a NaN's payload may differ)."""
import ctypes as C
import re
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parents[1]
MN, KM = 0, 1
NONE, ROW, COL = 0, 1, 2
RELU, GELU = 1, 2
BF16_IDS = (21, 31, 3, 13, 22, 32, 20, 40)
ABFT = {13, 31, 32, 40}
LAYOUTS = ((MN, MN), (MN, KM), (KM, MN), (KM, KM))
SENTINEL = -12352.0  # exactly a BF16 value (8 significant bits): the padding of D and Z must keep it
INVALID, UNSUPPORTED = -1, -2
F32, BF16 = 0, 1  # FTSGEMM_TYPE_*


def pad8(n):
    return (n + 7) // 8 * 8


# ------------------------------------------------------------------ CPU
def test_plan_bf16_out_in_place_or_copied(ft):
    # a row-major out with a leading stride of 12: written in place as float32, copied (rows padded to 16) as bfloat16
    f32 = ft.matmul_plan((5, 8), (8, 1), (8, 12), (12, 1), (12, 1), bf16=True)
    b16 = ft.matmul_plan((5, 8), (8, 1), (8, 12), (12, 1), (12, 1), bf16=True, out_bf16=True)
    assert not f32["copy_out"] and b16["copy_out"] and b16["ldc"] == 16 and b16["swap"]
    # leading strides that are multiples of 8 are written in place, in either layout
    b16 = ft.matmul_plan((16, 8), (8, 1), (8, 24), (24, 1), (24, 1), bf16=True, out_bf16=True)
    assert not b16["copy_out"] and b16["ldc"] == 24
    b16 = ft.matmul_plan((16, 8), (8, 1), (8, 24), (24, 1), (1, 16), bf16=True, out_bf16=True)
    assert not b16["copy_out"] and b16["ldc"] == 16 and not b16["swap"]
    # an unaligned base is copied
    assert ft.matmul_plan((16, 8), (8, 1), (8, 24), (24, 1), (24, 1), out_ptr=8, bf16=True, out_bf16=True)["copy_out"]


def test_bmm_plan_bf16_out_batch_stride(ft):
    # entries 16 * 20 = 320 elements apart: in place; 16 * 20 + 4: copied into (Bt, M, pad8(N)) = rows of 24
    p = ft.bmm_plan((3, 16, 8), (128, 8, 1), (3, 8, 20), (160, 20, 1), (16 * 24, 24, 1), bf16=True, out_bf16=True)
    assert not p["copy_out"] and p["stride_c"] == 16 * 24
    p = ft.bmm_plan((3, 16, 8), (128, 8, 1), (3, 8, 24), (192, 24, 1), (16 * 24 + 4, 24, 1), bf16=True, out_bf16=True)
    assert p["copy_out"] and p["ldc"] == 24 and p["stride_c"] == 16 * 24
    p = ft.bmm_plan((3, 16, 8), (128, 8, 1), (3, 8, 20), (160, 20, 1), (320, 20, 1), bf16=True, out_bf16=True)
    assert p["copy_out"] and p["ldc"] == 24 and p["stride_c"] == 16 * 24
    # the same float32 out is written in place
    p = ft.bmm_plan((3, 16, 8), (128, 8, 1), (3, 8, 20), (160, 20, 1), (320, 20, 1), bf16=True)
    assert not p["copy_out"]


def test_mixed_signature_matches_header(ft):
    hdr = (ROOT / "include" / "ftsgemm.h").read_text()
    decl = re.search(r"int ftsgemm_run_batched_mixed\(([^;]*)\);", hdr).group(1)
    params = [" ".join(p.split()) for p in decl.split(",")]
    assert "ftsgemm_run_batched_mixed" in ft.EXPORTED_SYMBOLS
    ctype_of = {"ftsgemm_handle_t": C.c_void_p, "int": C.c_int, "long long": C.c_longlong, "float": C.c_float}
    want = []
    for p in params:
        typ = p.rsplit(" ", 1)[0]
        if "*" in p:
            want.append(C.POINTER(ft.Opts) if "ftsgemm_opts" in p else C.c_void_p)
        else:
            want.append(ctype_of[typ])
    assert len(want) == 28
    names = [p.rsplit(" ", 1)[1].lstrip("*") for p in params]
    assert names[13:20] == ["ab_type", "C", "ldc", "stride_c", "D", "cd_type", "batch"]
    got = ft.lib().ftsgemm_run_batched_mixed.argtypes
    assert [a.__name__ if hasattr(a, "__name__") else a for a in got] == [w.__name__ for w in want]


# ------------------------------------------------------------------ GPU harness
@pytest.fixture(scope="module")
def dev(cuda, ft):
    cuda.cuda.set_device(0)
    h = ft.FtSgemm()
    yield h
    h.close()


def same16(t, x, y):
    """bfloat16 tensors equal bit for bit, except that NaN only has to meet NaN"""
    nx, ny = t.isnan(x), t.isnan(y)
    return bool(t.equal(nx, ny)) and bool(((x.view(t.int16) == y.view(t.int16)) | nx).all())


def bf(t, g, shape, scale=1.0):
    return (t.randn(shape, generator=g, device="cuda") * scale).to(t.bfloat16)


def pack(t, X, layout, ld, batch_dims=()):
    """(..., rows, K) -> a flat buffer in the layout (MN: X[r, k] at r + k*ld; KM: at k + r*ld) per entry, padding NaN"""
    rows, K = X.shape[-2:]
    if layout == MN:
        buf = t.full((*batch_dims, K, ld), float("nan"), device="cuda", dtype=X.dtype)
        buf[..., :rows] = X.transpose(-1, -2)
    else:
        buf = t.full((*batch_dims, rows, ld), float("nan"), device="cuda", dtype=X.dtype)
        buf[..., :K] = X
    return buf.reshape(-1)


def mixed_pair(t, dev, kid, A, B, la=KM, lb=KM, alpha=1.0, beta=0.0, C16=None, bias=None, mode=NONE, act=0, z=False,
               sep=False, opts=None, ldc=None, bias_per_entry=False):
    """One run_batched_mixed call with BF16 C / D / Z and its definition: the same call with FP32 C / D / Z on C16.float().
    A (Bt, M, K), B (Bt, N, K) bfloat16; C column-major per entry (N, ldc), padding SENTINEL.  Checks that C keeps its bytes
    when D != C and that no padding of D or Z was written.  Returns (D16, Z16, D32, Z32) as (Bt, M, N) views."""
    Bt, M, K = A.shape
    N = B.shape[1]
    ldc = ldc or pad8(M)
    lda = (pad8(M) if la == MN else pad8(K)) + 8
    ldb = (pad8(N) if lb == MN else pad8(K)) + 8
    sa, sb, sc = lda * (K if la == MN else M), ldb * (K if lb == MN else N), N * ldc
    dA, dB = pack(t, A, la, lda, (Bt,)), pack(t, B, lb, ldb, (Bt,))
    c16 = t.full((Bt, N, ldc), SENTINEL, device="cuda", dtype=t.bfloat16)
    if C16 is not None:
        c16[:, :, :M] = C16.transpose(1, 2)
    else:
        c16[:, :, :M] = 0
    c32 = c16.float()
    before = c16.clone()
    out = {}
    for tag, cbuf, cd in (("f32", c32, F32), ("bf16", c16, BF16)):
        dbuf = t.full_like(cbuf, SENTINEL) if sep else cbuf
        zbuf = t.full_like(cbuf, SENTINEL) if z else None
        stride_bias = (bias.shape[-1] if bias_per_entry else 0) if bias is not None else 0
        dev.run_batched_mixed(kid, M, N, K, dA, la, lda, sa, dB, lb, ldb, sb, 1, cbuf, ldc, sc, dbuf, cd, Bt, alpha, beta,
                              bias, mode, stride_bias, act, zbuf, opts)
        t.cuda.synchronize()
        if ldc > M:
            assert bool((dbuf[:, :, M:].float() == SENTINEL).all()), "D's padding was written"
            if z:
                assert bool((zbuf[:, :, M:].float() == SENTINEL).all()), "Z's padding was written"
        out[tag] = (dbuf[:, :, :M].transpose(1, 2), zbuf[:, :, :M].transpose(1, 2) if z else None)
    if sep:
        assert t.equal(c16.view(t.int16), before.view(t.int16)), "C was written"
    (d32, z32), (d16, z16) = out["f32"], out["bf16"]
    return d16, z16, d32, z32


def check_definition(t, d16, z16, d32, z32, tag):
    assert d16.dtype == t.bfloat16
    assert same16(t, d16, d32.to(t.bfloat16)), tag
    if z16 is not None:
        assert same16(t, z16, z32.to(t.bfloat16)), tag


def quiet(st, tag):
    assert st["detected"] == 0 and st["epilogue_faults"] == 0 and st["uncorrectable"] == 0, (tag, st)


# ------------------------------------------------------------------ GPU: the definition
@pytest.mark.gpu
@pytest.mark.parametrize("kid", BF16_IDS)
def test_definition_every_id_layout_and_option(cuda, ft, dev, kid):
    """Every BF16 id and layout pair over beta 0 / != 0, D == C / D != C, bias none / row / col (and per entry), activation
    none / ReLU / GELU with and without Z, protect_epilogue 0 / 1 / 2, batch 1 and a ragged batch: D16 and Z16 equal the
    FP32-output call rounded by .to(torch.bfloat16)."""
    t = cuda
    g = t.Generator(device="cuda").manual_seed(kid)
    rng = np.random.default_rng(kid)
    M, N, K = 200, 332, 136
    levels = (0, 1, 2) if kid in ABFT else (0,)
    case = 0
    for la, lb in LAYOUTS:
        for beta, sep in ((0.0, False), (-1.5, False), (0.0, True), (0.75, True)):
            Bt = (1, 3)[case % 2]
            mode = (NONE, ROW, COL)[case % 3]
            act = (0, RELU, GELU)[(case // 3) % 3]
            z = act != 0 and case % 2 == 0
            level = levels[case % len(levels)]
            case += 1
            A, B = bf(t, g, (Bt, M, K)), bf(t, g, (Bt, N, K))
            C16 = bf(t, g, (Bt, M, N), 4.0)
            per_entry = Bt > 1 and mode != NONE and case % 2 == 0
            blen = M if mode == ROW else N
            bias = (t.randn((Bt, blen) if per_entry else (blen,), generator=g, device="cuda") if mode != NONE else None)
            alpha = float(rng.choice([1.0, 0.5, -2.0]))
            opts = ft.make_opts(protect_epilogue=level)
            d16, z16, d32, z32 = mixed_pair(t, dev, kid, A, B, la, lb, alpha, beta, C16, bias, mode, act, z, sep, opts,
                                            ldc=pad8(M) + 8, bias_per_entry=per_entry)
            tag = (kid, la, lb, beta, sep, Bt, mode, act, z, level)
            check_definition(t, d16, z16, d32, z32, tag)
            quiet(dev.stats(), tag)


@pytest.mark.gpu
def test_comparator_catches_one_ulp(cuda, ft, dev):
    """The comparator of these tests fails on a one-ulp change of one BF16 element of D, and so does the float64 one of
    tests/test_bf16_exact.py (round_bf16 / mismatch16), which names that element; on integer data whose results need
    rounding D meets both.  (Its sensitivity to the rounding mode is test_bf16_out_exact.test_rounding_edge_data.)"""
    from test_bf16_exact import mismatch16, round_bf16
    t = cuda
    g = t.Generator(device="cuda").manual_seed(1)
    A, B = bf(t, g, (1, 128, 64)), bf(t, g, (1, 256, 64))
    d16, _, d32, _ = mixed_pair(t, dev, 31, A, B)
    want = d32.to(t.bfloat16)
    assert same16(t, d16, want)
    bad = d16.clone()
    bad.view(t.int16)[0, 17, 33] ^= 1
    assert not same16(t, bad, want)
    Ai, Bi = _ints(t, g, (1, 128, 64), 15).to(t.bfloat16), _ints(t, g, (1, 256, 64), 15).to(t.bfloat16)
    d16, _, _, _ = mixed_pair(t, dev, 31, Ai, Bi)
    bits = round_bf16(Ai[0].double() @ Bi[0].double().T)
    assert mismatch16(d16[0], bits) == ""
    bad = d16.clone()
    bad.view(t.int16)[0, 17, 33] ^= 1
    assert mismatch16(bad[0], bits).startswith("1 elements differ, e.g. (17, 33)")


# ------------------------------------------------------------------ GPU: exactness
def _ints(t, g, shape, amax):
    return t.randint(-amax, amax + 1, shape, generator=g, device="cuda", dtype=t.int32).float()


@pytest.mark.gpu
@pytest.mark.parametrize("shape", [(256, 256, 64), (260, 132, 80), (384, 520, 200), (8192, 8192, 8192)])
def test_exact_rounded_once(cuda, ft, dev, shape):
    """Integer data whose products need more than 8 significant bits: D16 is the float64 product rounded once to BF16, at
    tile edges and at 8192^3; cuBLAS with BF16 C (id 7) is within one BF16 ulp (it sums in another order)."""
    t = cuda
    M, N, K = shape
    g = t.Generator(device="cuda").manual_seed(M + N + K)
    amax = 15 if K <= 256 else 3
    A, B = _ints(t, g, (1, M, K), amax).to(t.bfloat16), _ints(t, g, (1, N, K), amax).to(t.bfloat16)
    want = (A[0].double() @ B[0].double().T).to(t.bfloat16)  # exact in float64, rounded once
    for kid in (31, 32, 21):
        d16, _, _, _ = mixed_pair(t, dev, kid, A, B, KM, KM)
        assert same16(t, d16[0], want), (kid, shape)
        quiet(dev.stats(), (kid, shape))
    # cuBLAS: in place with BF16 C (ldc a multiple of 8 elements)
    ldc = pad8(M)
    c = t.zeros(N * ldc, device="cuda", dtype=t.bfloat16)
    dev.run_batched_mixed(7, M, N, K, A.reshape(-1), KM, K, 0, B.reshape(-1), KM, K, 0, 1, c, ldc, 0, c, 1, 1)
    t.cuda.synchronize()
    cub = c.view(N, ldc)[:, :M].t()
    ulp = (want.float().abs() * 2.0 ** -7).clamp_min(2.0 ** -126)
    assert bool(((cub.float() - want.float()).abs() <= ulp).all())


# ------------------------------------------------------------------ GPU: faults
@pytest.mark.gpu
@pytest.mark.slow
def test_fault_campaign_bf16_out(cuda, ft, dev):
    """Accumulator upsets at 8192^3 with BF16 output (id 31): bits >= 22 detected and repaired 100 %, the repaired D16 bit
    for bit the fault-free one; epilogue upsets (modes 2 and 3) under level 1 (beta = 0, and beta != 0 with D != C) and
    level 2 store the fault-free bits."""
    t = cuda
    n, kid = 8192, 31
    g = t.Generator(device="cuda").manual_seed(7)
    # entries -1, 0, 1: every accumulator, checksum and correction is exact, so a repair restores the fault-free bits
    A = _ints(t, g, (n * n,), 1).to(t.bfloat16)
    B = _ints(t, g, (n * n,), 1).to(t.bfloat16)
    C16 = (t.randn(n * n, generator=g, device="cuda")).to(t.bfloat16)

    def call(beta=0.0, sep=False, opts=None, cd=BF16):
        typ = t.bfloat16 if cd == BF16 else t.float32
        c = C16.to(typ, copy=True)
        d = t.empty(n * n, device="cuda", dtype=typ) if sep else c
        dev.run_batched_mixed(kid, n, n, n, A, MN, n, 0, B, MN, n, 0, 1, c, n, 0, d, cd, 1, 1.0, beta, opts=opts)
        t.cuda.synchronize()
        return d

    dev.stats()
    cases = ((0.0, False), (-1.5, True))
    clean = {cs: call(*cs) for cs in cases}
    # upsets only where every clean FP32 value is at least 1 (a flip of a zero's exponent can stay below the threshold)
    big = (call(*cases[0], cd=F32).abs() >= 1) & (call(*cases[1], cd=F32).abs() >= 1)
    quiet(dev.stats(), "clean")
    rng = np.random.default_rng(0)
    for bit in (31, 30, 29, 27, 25, 23, 22):
        faults, seen = [], set()
        while len(faults) < ft.MAX_FAULTS:
            r, c = int(rng.integers(n)), int(rng.integers(n))
            if (r, c // 256) in seen or not bool(big[r + c * n]):
                continue
            seen.add((r, c // 256))
            faults.append({"row": r, "col": c, "xor": 1 << bit})
        d = call(opts=ft.make_opts(faults=faults))
        st = dev.stats()
        assert st["detected"] == len(faults) and st["uncorrectable"] == 0, (bit, st)
        assert st["corrected"] + st["recomputed"] == st["detected"], (bit, st)
        assert t.equal(d.view(t.int16), clean[(0.0, False)].view(t.int16)), bit
    r, c = next((r, c) for r in range(3000, n) for c in (4000,) if bool(big[r + c * n]))
    for level, where in ((1, "epilogue_tmem"), (1, "epilogue_value"), (2, "epilogue_tmem"), (2, "epilogue_value")):
        for beta, sep in cases:
            f = [{"row": r, "col": c, "xor": 1 << 27, "where": where}]
            d = call(beta, sep, ft.make_opts(protect_epilogue=level, faults=f))
            st = dev.stats()
            assert st["epilogue_faults"] >= 1 and st["uncorrectable"] == 0, (level, where, beta, st)
            assert t.equal(d.view(t.int16), clean[(beta, sep)].view(t.int16)), (level, where, beta)


@pytest.mark.gpu
@pytest.mark.parametrize("la,lb", LAYOUTS)
def test_repairs_store_fault_free_bits(cuda, ft, dev, la, lb):
    """The row recompute (two upsets in one row of a tile), level 1's segment recompute into D (D != C, beta != 0) and level
    2's chunk recompute store the bits of a fault-free BF16 call, in every layout pair and in entry 2 of a batch."""
    t = cuda
    g = t.Generator(device="cuda").manual_seed(la * 2 + lb)
    Bt, M, N, K = 3, 512, 768, 256
    # integer operands: the recomputes on CUDA cores sum exactly what the tensor cores sum
    A, B = _ints(t, g, (Bt, M, K), 4).to(t.bfloat16), _ints(t, g, (Bt, N, K), 4).to(t.bfloat16)
    C16 = bf(t, g, (Bt, M, N))
    bias = t.randn(N, generator=g, device="cuda")
    clean, _, _, _ = mixed_pair(t, dev, 31, A, B, la, lb, 1.0, -1.5, C16, bias, COL, GELU, False, True)
    quiet(dev.stats(), "clean")
    row = 2 * M + 300  # entry 2, stacked rows
    cases = (
        ("row recompute", ft.make_opts(faults=[{"row": row, "col": 40, "xor": 1 << 30}, {"row": row, "col": 41, "xor": 1 << 29}])),
        ("level 1", ft.make_opts(protect_epilogue=1, faults=[{"row": row, "col": 40, "xor": 1 << 27, "where": "epilogue_value"}])),
        ("level 2", ft.make_opts(protect_epilogue=2, faults=[{"row": row, "col": 40, "xor": 1 << 27, "where": "epilogue_value"}])),
    )
    for tag, opts in cases:
        d16, _, _, _ = mixed_pair(t, dev, 31, A, B, la, lb, 1.0, -1.5, C16, bias, COL, GELU, False, True, opts)
        st = dev.stats()
        assert st["uncorrectable"] == 0 and st["recomputed"] >= 1, (tag, st)
        assert same16(t, d16, clean), tag


# ------------------------------------------------------------------ GPU: values
@pytest.mark.gpu
def test_nonfinite_overflow_and_subnormal(cuda, ft, dev):
    """Inf and NaN in the operands and in the old C, FP32 results past the BF16 range (+-Inf, no alarm) and results in the
    BF16 subnormal range: all as the definition rounds them, under every protection level."""
    t = cuda
    g = t.Generator(device="cuda").manual_seed(3)
    M, N, K = 256, 256, 64
    A, B, C16 = bf(t, g, (1, M, K)), bf(t, g, (1, N, K)), bf(t, g, (1, M, N))
    A[0, 5, 3], A[0, 9, 1], B[0, 7, 2] = float("inf"), float("nan"), float("-inf")
    C16[0, 100, 10], C16[0, 101, 11] = float("nan"), float("inf")
    for level in (0, 1, 2):
        d16, _, d32, _ = mixed_pair(t, dev, 31, A, B, KM, MN, 1.0, 2.0, C16, opts=ft.make_opts(protect_epilogue=level))
        check_definition(t, d16, None, d32, None, ("nonfinite", level))
        assert bool(t.isnan(d16[0, 9]).all()) and bool(t.isnan(d16[0, 100, 10]))
        dev.stats()
    # FP32 results just below FLT_MAX but above the BF16 range round to +-Inf and raise no alarm
    ones_a = t.zeros(1, M, K, device="cuda", dtype=t.bfloat16)
    ones_b = t.zeros(1, N, K, device="cuda", dtype=t.bfloat16)
    # (one +1 and one -1 per 32 columns: the check sums of every chunk stay finite)
    ones_a[0, :, 0] = 1.0
    ones_b[0, 0::32, 0], ones_b[0, 16::32, 0] = 1.0, -1.0
    for level in (0, 1, 2):
        d16, _, d32, _ = mixed_pair(t, dev, 31, ones_a, ones_b, KM, KM, 3.4e38, opts=ft.make_opts(protect_epilogue=level))
        assert bool(t.isfinite(d32).all()) and float(d32.abs().max()) > 3.39e38
        assert bool((d16[0, :, 0::32] == float("inf")).all()) and bool((d16[0, :, 16::32] == float("-inf")).all())
        check_definition(t, d16, None, d32, None, ("overflow", level))
        quiet(dev.stats(), ("overflow", level))
    # the BF16 subnormal range
    ia, ib = _ints(t, g, (1, M, K), 7).to(t.bfloat16), _ints(t, g, (1, N, K), 7).to(t.bfloat16)
    for alpha in (2.0 ** -133, 2.0 ** -140, 3.0 * 2.0 ** -138):
        d16, _, d32, _ = mixed_pair(t, dev, 31, ia, ib, KM, KM, alpha)
        check_definition(t, d16, None, d32, None, ("subnormal", alpha))
        sub = (d16 != 0) & (d16.float().abs() < 2.0 ** -126)
        assert bool(sub.any())
        dev.stats()


# ------------------------------------------------------------------ GPU: arguments
@pytest.mark.gpu
def test_argument_rules(cuda, ft, dev):
    t = cuda
    M = N = K = 128
    a = t.zeros(2 * M * K, device="cuda", dtype=t.bfloat16)  # (room for the batch of two below)
    b = t.zeros(2 * N * K, device="cuda", dtype=t.bfloat16)
    a32, b32 = t.zeros(M * K, device="cuda"), t.zeros(N * K, device="cuda")
    big = t.zeros(4 * M * N + 64, device="cuda", dtype=t.bfloat16)
    c, d, z = big[:M * N], big[M * N:2 * M * N], big[2 * M * N:3 * M * N]

    def code(kid=31, A=a, B=b, ab=1, Cb=c, ldc=M, sc=0, Db=c, cd=1, batch=1, beta=0.0, act=0, Z=None, opts=None, bias=None,
             mode=NONE):
        try:
            dev.run_batched_mixed(kid, M, N, K, A, KM, K, M * K, B, KM, K, N * K, ab, Cb, ldc, sc, Db, cd, batch, 1.0, beta,
                                  bias, mode, 0, act, Z, opts)
            t.cuda.synchronize()
            return 0
        except ft.FtsgemmError as e:
            return e.code

    assert code() == 0
    assert code(cd=2) == INVALID and code(cd=-1) == INVALID
    assert code(A=a32, B=b32, ab=0) == UNSUPPORTED
    for kid in (1, 2, 4, 5, 6, 10, 11, 12, 14, 15, 16, 30):
        assert code(kid=kid) == UNSUPPORTED, kid
    assert code(kid=7) == 0 and code(kid=0) == 0
    assert code(kid=7, Db=d) == UNSUPPORTED  # cuBLAS: in place only
    assert code(ldc=M + 4) == INVALID
    assert code(batch=2, sc=M * N + 4, Cb=big, Db=big) == INVALID
    assert code(batch=2, sc=M * N, Cb=big, Db=big) == 0
    off = big[3 * M * N + 4:4 * M * N + 4]  # 8-byte aligned only (and clear of c and d)
    assert code(Cb=off, Db=off) == INVALID
    assert code(Cb=c, Db=off) == INVALID
    assert code(Cb=off, Db=d, beta=1.0) == INVALID       # C is read: it must be aligned
    assert code(Cb=off, Db=d, beta=0.0) == 0             # C is not read
    assert code(act=GELU, Z=big[2 * M * N + 4:]) == INVALID
    # byte footprints: D starts 1.5 C-footprints in floats after C but past its BF16 footprint -> accepted
    assert code(Cb=c, Db=big[M * N:], beta=1.0) == 0
    assert code(Cb=c, Db=big[M * N - 8:], beta=1.0) == INVALID
    assert code(Cb=c, Db=d, act=GELU, Z=big[2 * M * N - 8:], beta=1.0) == INVALID
    assert code(opts=ft.make_opts(check_segments=2)) == UNSUPPORTED
    assert code(opts=ft.make_opts(precision=1)) == INVALID
    dev.stats()


# ------------------------------------------------------------------ GPU: graphs and launches
@pytest.mark.gpu
@pytest.mark.parametrize("n", [1024, 2048])
def test_graph_replay_and_launch_count(cuda, ft, dev, n):
    """A captured BF16-output call replays bit-identically to the eager one, and launches as often as the FP32-output BF16
    call: 2 below 8 MB of B (n = 1024), 1 from there (n = 2048)."""
    t = cuda
    g = t.Generator(device="cuda").manual_seed(n)
    A, B = bf(t, g, (n * n,)), bf(t, g, (n * n,))
    C16 = bf(t, g, (n * n,))
    bias = t.randn(n, generator=g, device="cuda")
    counts = {}
    for cd in (0, 1):
        Cb = C16.float() if cd == 0 else C16
        D = t.empty_like(Cb)
        c0 = dev.launch_count()
        dev.run_batched_mixed(31, n, n, n, A, MN, n, 0, B, KM, n, 0, 1, Cb, n, 0, D, cd, 1, 1.0, -1.5, bias, COL)
        t.cuda.synchronize()
        counts[cd] = dev.launch_count() - c0
    assert counts[0] == counts[1] == (1 if n >= 2048 else 2), counts
    eager = t.empty_like(C16)
    dev.run_batched_mixed(31, n, n, n, A, MN, n, 0, B, KM, n, 0, 1, C16, n, 0, eager, 1, 1, 1.0, -1.5, bias, COL)
    t.cuda.synchronize()
    D = t.full_like(C16, SENTINEL)
    s = t.cuda.Stream()
    s.wait_stream(t.cuda.current_stream())
    graph = t.cuda.CUDAGraph()
    with t.cuda.stream(s):
        opts = ft.make_opts(stream=s.cuda_stream)
        with t.cuda.graph(graph, stream=s):
            dev.run_batched_mixed(31, n, n, n, A, MN, n, 0, B, KM, n, 0, 1, C16, n, 0, D, 1, 1, 1.0, -1.5, bias, COL,
                                  opts=opts)
    t.cuda.current_stream().wait_stream(s)
    for _ in range(2):
        D.fill_(SENTINEL)
        graph.replay()
        t.cuda.synchronize()
        assert t.equal(D.view(t.int16), eager.view(t.int16))
    quiet(dev.stats(), n)


# ------------------------------------------------------------------ GPU: torch layer
@pytest.mark.gpu
def test_matmul_bmm_linear_bf16_results(cuda, ft, dev):
    """matmul, bmm and linear with bfloat16 results (out=, c=, out_dtype=, residual=, preact) equal their float32 results
    rounded by .to(torch.bfloat16)."""
    t = cuda
    g = t.Generator(device="cuda").manual_seed(11)
    M, N, K = 192, 264, 96
    a, b = bf(t, g, (M, K)), bf(t, g, (K, N))
    bias = bf(t, g, (N,))
    y = dev.matmul(a, b, bias=bias, out_dtype=t.bfloat16)
    assert y.dtype == t.bfloat16 and same16(t, y, dev.matmul(a, b, bias=bias).to(t.bfloat16))
    # a BF16 out that cannot be written in place (rows of 264 + 4) is computed in a padded copy
    wide = t.full((M, N + 4), 7.0, device="cuda", dtype=t.bfloat16)
    out = wide[:, 2:N + 2]
    dev.matmul(a, b, out, bias=bias)
    assert same16(t, out, y) and bool((wide[:, :2] == 7).all()) and bool((wide[:, N + 2:] == 7).all())
    # c (bfloat16): out = a b - 1.5 c
    c16 = bf(t, g, (M, N), 3.0)
    y = dev.matmul(a, b, c=c16, beta=-1.5)
    assert y.dtype == t.bfloat16 and same16(t, y, dev.matmul(a, b, c=c16.float(), beta=-1.5).to(t.bfloat16))
    # activation with preact
    for act in ("relu", "gelu"):
        out16, z16 = t.empty(M, N, device="cuda", dtype=t.bfloat16), t.empty(M, N, device="cuda", dtype=t.bfloat16)
        out32, z32 = t.empty(M, N, device="cuda"), t.empty(M, N, device="cuda")
        dev.matmul(a, b, out16, bias=bias, activation=act, preact=z16)
        dev.matmul(a, b, out32, bias=bias, activation=act, preact=z32)
        assert same16(t, out16, out32.to(t.bfloat16)) and same16(t, z16, z32.to(t.bfloat16)), act
    # bmm: a batch with a per-entry bias, and c
    Bt = 3
    ab, bb = bf(t, g, (Bt, M, K)), bf(t, g, (Bt, K, N))
    pb = t.randn(Bt, N, generator=g, device="cuda")
    y = dev.bmm(ab, bb, bias=pb, out_dtype=t.bfloat16, activation="gelu")
    assert same16(t, y, dev.bmm(ab, bb, bias=pb, activation="gelu").to(t.bfloat16))
    cb = bf(t, g, (Bt, M, N))
    y = dev.bmm(ab, bb, c=cb, beta=0.5)
    assert same16(t, y, dev.bmm(ab, bb, c=cb.float(), beta=0.5).to(t.bfloat16))
    # linear: out_dtype, residual, GELU
    x, W = bf(t, g, (2, 96, K)), bf(t, g, (N, K))
    y = dev.linear(x, W, bias, out_dtype=t.bfloat16)
    assert y.shape == (2, 96, N) and same16(t, y, dev.linear(x, W, bias).to(t.bfloat16))
    r = bf(t, g, (2, 96, N))
    y = dev.linear(x, W, bias, residual=r, out_dtype=t.bfloat16)
    assert same16(t, y, dev.linear(x, W, bias, residual=r.float()).to(t.bfloat16))
    y = dev.linear(x, W, bias, activation="gelu", out_dtype=t.bfloat16)
    assert same16(t, y, dev.linear(x, W, bias, activation="gelu").to(t.bfloat16))
    quiet(dev.stats(), "torch layer")


@pytest.mark.gpu
def test_dtype_errors(cuda, ft, dev):
    t = cuda
    a32, b32 = t.zeros(64, 32, device="cuda"), t.zeros(32, 64, device="cuda")
    a, b = a32.bfloat16(), b32.bfloat16()
    with pytest.raises(TypeError):
        dev.matmul(a32, b32, out_dtype=t.bfloat16)
    with pytest.raises(TypeError):
        dev.matmul(a32, b32, t.empty(64, 64, device="cuda", dtype=t.bfloat16))
    with pytest.raises(TypeError):
        dev.linear(a32, b32.t(), out_dtype=t.bfloat16)
    with pytest.raises(ValueError):  # out_dtype contradicts out / c
        dev.matmul(a, b, t.empty(64, 64, device="cuda"), out_dtype=t.bfloat16)
    with pytest.raises(ValueError):
        dev.matmul(a, b, c=t.zeros(64, 64, device="cuda", dtype=t.bfloat16), beta=1.0, out_dtype=t.float32)
    with pytest.raises(ValueError):  # c and preact must have the result dtype
        dev.matmul(a, b, t.empty(64, 64, device="cuda", dtype=t.bfloat16), c=t.zeros(64, 64, device="cuda"), beta=1.0)
    with pytest.raises(ValueError):
        dev.matmul(a, b, t.empty(64, 64, device="cuda", dtype=t.bfloat16), activation="gelu",
                   preact=t.empty(64, 64, device="cuda"))
    with pytest.raises(ValueError):  # the residual must have y's dtype
        dev.linear(a, b.t(), residual=t.zeros(64, 64, device="cuda"), out_dtype=t.bfloat16)
    with pytest.raises(ValueError):
        dev.linear(a, b.t(), residual=t.zeros(64, 64, device="cuda", dtype=t.bfloat16))
    with pytest.raises(ValueError):
        dev.matmul(a, b, out_dtype=t.float16)
    with pytest.raises(ValueError):  # an activation still needs an out written in place
        dev.matmul(a, b, t.empty(64, 68, device="cuda", dtype=t.bfloat16)[:, :64], activation="relu")


@pytest.mark.gpu
def test_autograd_bf16_output(cuda, ft, dev):
    """linear and bmm with bfloat16 results: grad_y arrives as bfloat16, and the gradients are within one bfloat16 rounding of
    float64 products of the bfloat16 grad_z (FP32 accumulation adds its own bound)."""
    t = cuda
    g = t.Generator(device="cuda").manual_seed(5)
    T, N, K = 256, 192, 128
    x = bf(t, g, (T, K)).requires_grad_()
    W = bf(t, g, (N, K)).requires_grad_()
    bias = bf(t, g, (N,)).requires_grad_()
    r = bf(t, g, (T, N)).requires_grad_()
    gy = bf(t, g, (T, N))

    def close(got, ref, bound):
        assert got.dtype == t.bfloat16
        err = (got.double() - ref).abs()
        assert bool((err <= ref.abs() * 2.0 ** -8 + bound).all()), float((err - ref.abs() * 2.0 ** -8 - bound).max())

    for act, res in (("gelu", None), (None, r)):
        y = dev.linear(x, W, bias, activation=act, residual=res, out_dtype=t.bfloat16)
        assert y.dtype == t.bfloat16
        y.backward(gy)
        if act == "gelu":
            z = dev.linear(x.detach(), W.detach(), bias.detach(), out_dtype=t.bfloat16)
            gz = t.ops.aten.gelu_backward(gy, z)
        else:
            gz = gy
            assert r.grad.dtype == t.bfloat16 and t.equal(r.grad, gy)
        assert gz.dtype == t.bfloat16
        gzd = gz.double()
        close(x.grad, gzd @ W.detach().double(), K * 2.0 ** -23 * (gzd.abs() @ W.detach().double().abs()))
        close(W.grad, gzd.t() @ x.detach().double(), T * 2.0 ** -23 * (gzd.abs().t() @ x.detach().double().abs()))
        assert bias.grad.dtype == t.bfloat16
        close(bias.grad, gzd.sum(0), T * 2.0 ** -23 * gzd.abs().sum(0))
        for p in (x, W, bias, r):
            p.grad = None
    Bt = 2
    a, bm = bf(t, g, (Bt, 64, K)).requires_grad_(), bf(t, g, (Bt, K, 96)).requires_grad_()
    c = bf(t, g, (Bt, 64, 96)).requires_grad_()
    y = dev.bmm(a, bm, c=c, beta=0.5)
    assert y.dtype == t.bfloat16
    gyb = bf(t, g, (Bt, 64, 96))
    y.backward(gyb)
    gd = gyb.double()
    close(a.grad, gd @ bm.detach().double().transpose(1, 2), 96 * 2.0 ** -23 * (gd.abs() @ bm.detach().double().abs().transpose(1, 2)))
    close(bm.grad, a.detach().double().transpose(1, 2) @ gd, 64 * 2.0 ** -23 * (a.detach().double().abs().transpose(1, 2) @ gd.abs()))
    assert c.grad.dtype == t.bfloat16 and same16(t, c.grad, (0.5 * gyb.float()).to(t.bfloat16))
    dev.stats()


@pytest.mark.gpu
def test_float32_output_gradients_unchanged(cuda, ft, dev):
    """The gradients of a float32-output BF16 linear / bmm, now written as bfloat16 by the products themselves, are bit for
    bit the float32 products rounded by .to(torch.bfloat16) -- what the backward computed before."""
    t = cuda
    g = t.Generator(device="cuda").manual_seed(6)
    T, N, K = 320, 200, 136
    x, W = bf(t, g, (T, K)).requires_grad_(), bf(t, g, (N, K)).requires_grad_()
    gy = t.randn(T, N, generator=g, device="cuda")
    for act in (None, "relu", "gelu"):
        y = dev.linear(x, W, activation=act)
        assert y.dtype == t.float32
        y.backward(gy)
        if act is None:
            gz = gy
        elif act == "relu":
            gz = t.ops.aten.threshold_backward(gy, y.detach(), 0)
        else:
            gz = t.ops.aten.gelu_backward(gy, dev.linear(x.detach(), W.detach()))
        g16 = gz.to(t.bfloat16)
        assert same16(t, x.grad, dev.matmul(g16, W.detach()).to(t.bfloat16)), act
        assert same16(t, W.grad, dev.matmul(g16.t(), x.detach()).to(t.bfloat16)), act
        x.grad = W.grad = None
    a, bm = bf(t, g, (3, 64, K)).requires_grad_(), bf(t, g, (3, K, 72)).requires_grad_()
    y = dev.bmm(a, bm, alpha=0.5)
    gyb = t.randn(3, 64, 72, generator=g, device="cuda")
    y.backward(gyb)
    g16 = gyb.to(t.bfloat16)
    assert same16(t, a.grad, dev.bmm(g16, bm.detach().transpose(1, 2), alpha=0.5).to(t.bfloat16))
    assert same16(t, bm.grad, dev.bmm(a.detach().transpose(1, 2), g16, alpha=0.5).to(t.bfloat16))
    dev.stats()
