"""BF16 operands (ftsgemm_run_typed / ftsgemm_run_batched_typed, FtSgemm.matmul with bfloat16 tensors): BF16 A and B read in
place in either layout, FP32 accumulate, FP32 C / D / Z / bias, and the ABFT check on a three-term BF16 checksum operand.

Exact tier: small integers are BF16 values, every product of two of them is exact in FP32, and as long as every partial
sum, row sum, expected checksum and stored value stays at or below 2^24 (test_exact.budget) every correct path returns the
float64 product bit for bit and every row check closes with a residual of exactly zero.  cuBLAS (BF16 A / B, FP32 compute)
is the witness on the same data.  Rounding tier: standard-normal BF16 operands against the float64 product of the same
BF16 values."""
import numpy as np
import pytest

from test_exact import LIMIT, budget, knobs, mismatch

MN, KM = 0, 1
NONE, ROW, COL = 0, 1, 2
RELU, GELU = 1, 2
BF16_IDS = (21, 31, 3, 13, 22, 32, 20, 40)      # the two-CTA tiles and AUTO
ABFT = {13, 31, 32, 40}
SENTINEL = -12345.5


def pad8(n):
    return (n + 7) // 8 * 8


def ld_bf16(layout, rows, K, pad):
    """a leading dimension the BF16 path accepts (a multiple of 8), 8 more when padded"""
    base = pad8(rows) if layout == MN else pad8(K)
    return base + 8 if pad else base


def exact_budget_ok(K, amax, bmax, alpha=1.0, beta=0.0, cmax=0.0, bias_max=0.0, BN=256):
    """test_exact.budget's limits, with the BF16 encode: the weighted column-block sum sum_j (j + 1) b_j <= 2^24 (three
    BF16 terms hold 24 significant bits), in place of the TF32 encode limit"""
    b = budget(K, BN, amax, bmax, alpha, beta, cmax, bias_max)
    weighted = BN * (BN + 1) // 2 * bmax
    return b["out"] is not None and max(b["acc"], b["rowsum"], b["checksum"], b["out"], weighted) <= LIMIT


# ------------------------------------------------------------------ CPU
def test_plan_pads_bf16_rows_to_8(ft):
    assert ft._pad8(1) == 8 and ft._pad8(8) == 8 and ft._pad8(13) == 16
    # a row-major a with a leading stride of 12: 16-byte rows in FP32, not in BF16 (copied, padded to 16)
    f32 = ft.matmul_plan((5, 12), (12, 1), (12, 8), (8, 1), (8, 1))
    bf = ft.matmul_plan((5, 12), (12, 1), (12, 8), (8, 1), (8, 1), bf16=True)
    assert not f32["copy_a"] and bf["copy_a"] and bf["ldb"] == 16
    # strides that are multiples of 8 are read in place in both layouts
    bf = ft.matmul_plan((16, 24), (24, 1), (24, 32), (1, 24), (32, 1), bf16=True)
    assert not (bf["copy_a"] or bf["copy_b"] or bf["copy_out"]) and bf["lda"] == 24 and bf["ldb"] == 24


def test_typed_symbols_and_types(ft):
    assert {"ftsgemm_run_typed", "ftsgemm_run_batched_typed"} <= set(ft.EXPORTED_SYMBOLS)
    assert (ft.TYPE_F32, ft.TYPE_BF16) == (0, 1)


def test_exact_budget_of_bf16_encode():
    assert exact_budget_ok(256, 8, 8) and exact_budget_ok(4096, 2, 2)
    assert not exact_budget_ok(16384 + 64, 2, 2)     # the expected checksum would pass 2^24
    assert not exact_budget_ok(8, 1024, 1024)        # the weighted column-block sum would pass 2^24


# ------------------------------------------------------------------ GPU harness
@pytest.fixture(scope="module")
def dev(cuda, ft):
    cuda.cuda.set_device(0)
    h = ft.FtSgemm()
    yield h
    h.close()


def ints(t, g, shape, amax):
    return t.randint(-amax, amax + 1, shape, generator=g, device="cuda", dtype=t.int32).float()


def pack16(t, X, layout, ld):
    """rows x K float32 matrix -> flat BF16 buffer in the layout (MN: X[r, k] at r + k*ld; KM: at k + r*ld), padding NaN"""
    rows, K = X.shape
    if layout == MN:
        buf = t.full((K, ld), float("nan"), device="cuda")
        buf[:, :rows] = X.T
    else:
        buf = t.full((rows, ld), float("nan"), device="cuda")
        buf[:, :K] = X
    return buf.reshape(-1).to(t.bfloat16)


def reference(A, B, alpha=1.0, beta=0.0, C0=None, bias=None, mode=NONE):
    """float64 alpha * A B^T + beta * C0 (+ bias) of the BF16 values (A: M x K, B: N x K)"""
    out = alpha * (A.to(_t().bfloat16).double() @ B.to(_t().bfloat16).double().T)
    if beta != 0.0:
        out = out + beta * C0.double()
    if mode == ROW:
        out = out + bias.double()[:, None]
    elif mode == COL:
        out = out + bias.double()[None, :]
    return out


def _t():
    import torch
    return torch


def run16(t, dev, kid, A, B, la=KM, lb=KM, pad=False, alpha=1.0, beta=0.0, C0=None, bias=None, mode=NONE, act=0, z=False,
          out_of_place=False, opts=None, ldc=None):
    """one run_typed call on BF16 copies of A (M x K) and B (N x K); C column-major (ldc, padding SENTINEL).  Returns (D, Z)
    as M x N views, and checks that C kept its bytes when D != C and that no padding was written."""
    M, K = A.shape
    N = B.shape[0]
    lda, ldb, ldc = ld_bf16(la, M, K, pad), ld_bf16(lb, N, K, pad), ldc or M
    dA, dB = pack16(t, A, la, lda), pack16(t, B, lb, ldb)
    cbuf = t.full((N, ldc), SENTINEL, device="cuda")
    cbuf[:, :M] = 0.0 if C0 is None else C0.T
    c_before = cbuf.clone()
    dbuf = t.full((N, ldc), SENTINEL, device="cuda") if out_of_place else cbuf
    zbuf = t.full((N, ldc), SENTINEL, device="cuda") if z else None
    dev.run_typed(kid, M, N, K, dA, la, lda, dB, lb, ldb, 1, cbuf, ldc, dbuf, alpha, beta, bias, mode, act, zbuf, opts)
    t.cuda.synchronize()
    if out_of_place:
        assert t.equal(cbuf.view(t.int32), c_before.view(t.int32)), "C was written"
    if ldc > M:
        assert bool((dbuf[:, M:] == SENTINEL).all()), "D's padding was written"
    return dbuf[:, :M].t(), (zbuf[:, :M].t() if z else None)


def zero_residual(st, kid, tag):
    assert st["detected"] == 0 and st["recomputed"] == 0 and st["epilogue_faults"] == 0 and not st["events"], (tag, st)
    if kid in ABFT:
        assert st["rows_checked"] > 0 and st["max_abs_residual"] == 0.0, (tag, st)


def exact(got, want, tag):
    msg = mismatch(got, want)
    assert not msg, f"{tag}: {msg}"


# ------------------------------------------------------------------ GPU: exact data
@pytest.mark.gpu
@pytest.mark.parametrize("kid", BF16_IDS + (7, 0))
def test_exact_every_id_and_layout(cuda, ft, dev, kid):
    """Every supported id, all four layout pairs, padded or tight leading dimensions, ragged M / N / K: D equals the float64
    product of the BF16 integers at every element, bit for bit, and every row check closes exactly (cuBLAS, ids 7 / 0,
    witnesses the same data)."""
    t = cuda
    g = t.Generator(device="cuda").manual_seed(1000 + kid)
    shapes = [(260, 292, 200), (4, 8, 1), (512, 384, 1031), (132, 516, 64)]
    for i, (M, N, K) in enumerate(shapes):
        amax = 8 if exact_budget_ok(K, 8, 8) else 2
        A, B = ints(t, g, (M, K), amax), ints(t, g, (N, K), amax)
        want = reference(A, B)
        for la in (MN, KM):
            for lb in (MN, KM):
                got, _ = run16(t, dev, kid, A, B, la, lb, pad=(i + la + lb) % 2 == 1, ldc=M + 4 * (i % 2))
                exact(got, want, (kid, M, N, K, la, lb))
                zero_residual(dev.stats(), kid, (kid, M, N, K, la, lb))


@pytest.mark.gpu
@pytest.mark.parametrize("kid", (31, 13))
def test_exact_options(cuda, ft, dev, kid):
    """beta 0 / 1 / -1.5 with an integer C, D != C (C's bytes unchanged), ROW / COL bias, ReLU (bit-identical to torch.relu)
    and GELU (within 2 ulp of torch's on the exact pre-activation, which Z holds bit for bit), check_segments, both
    protect_epilogue levels and split-K plans: all exact."""
    t = cuda
    g = t.Generator(device="cuda").manual_seed(77 + kid)
    M, N, K = 516, 388, 1100
    amax = 4
    A, B = ints(t, g, (M, K), amax), ints(t, g, (N, K), amax)
    C0 = ints(t, g, (M, N), 64)
    brow, bcol = ints(t, g, (M,), 64), ints(t, g, (N,), 64)
    cases = [dict(beta=0.0), dict(beta=1.0), dict(beta=-1.5), dict(beta=-1.5, out_of_place=True),
             dict(beta=1.0, mode=ROW), dict(beta=0.0, mode=COL, out_of_place=True)]
    for c in cases:
        mode = c.get("mode", NONE)
        bias = brow if mode == ROW else (bcol if mode == COL else None)
        want = reference(A, B, 1.0, c["beta"], C0, bias, mode)
        for opts_kw in ({}, {"check_segments": 3}, {"protect_epilogue": 1}, {"protect_epilogue": 2}):
            opts = ft.make_opts(**opts_kw)
            got, _ = run16(t, dev, kid, A, B, MN, KM, alpha=1.0, beta=c["beta"], C0=C0, bias=bias, mode=mode,
                           out_of_place=c.get("out_of_place", False), opts=opts)
            exact(got, want, (kid, c, opts_kw))
            zero_residual(dev.stats(), kid, (kid, c, opts_kw))
    for sk in (0, 2, 3):
        with knobs(ft, splitk=sk):
            got, _ = run16(t, dev, kid, A, B, KM, MN)
        exact(got, reference(A, B), (kid, "splitk", sk))
        zero_residual(dev.stats(), kid, (kid, "splitk", sk))
    zexp = reference(A, B, 1.0, 1.0, C0, bcol, COL)
    got, z = run16(t, dev, kid, A, B, KM, KM, beta=1.0, C0=C0, bias=bcol, mode=COL, act=RELU, z=True)
    exact(z, zexp, (kid, "relu z"))
    assert t.equal(got, t.relu(zexp.float())), (kid, "relu")
    got, z = run16(t, dev, kid, A, B, MN, MN, beta=1.0, C0=C0, bias=bcol, mode=COL, act=GELU, z=True, out_of_place=True)
    exact(z, zexp, (kid, "gelu z"))
    ref = t.nn.functional.gelu(zexp.float())
    ulp = (got.view(t.int32).long() - ref.view(t.int32).long()).abs()
    assert int(ulp.max()) <= 2, (kid, "gelu", int(ulp.max()))
    zero_residual(dev.stats(), kid, (kid, "act"))


@pytest.mark.gpu
@pytest.mark.parametrize("kid", (31, 21))
def test_exact_batches(cuda, ft, dev, kid):
    """Strided batches of 1-7 entries (both layouts, per-entry COL bias, beta -1.5) through run_batched_typed: every entry
    exact."""
    t = cuda
    g = t.Generator(device="cuda").manual_seed(5 + kid)
    for Bt, (M, N, K), la, lb in ((1, (260, 132, 96), KM, KM), (3, (132, 260, 200), MN, KM), (7, (68, 72, 33), MN, MN)):
        A, B = ints(t, g, (Bt, M, K), 4), ints(t, g, (Bt, N, K), 4)
        C0 = ints(t, g, (Bt, M, N), 64)
        bias = ints(t, g, (Bt, N), 64)
        lda, ldb = ld_bf16(la, M, K, True), ld_bf16(lb, N, K, False)
        dA = t.stack([pack16(t, A[i], la, lda) for i in range(Bt)])
        dB = t.stack([pack16(t, B[i], lb, ldb) for i in range(Bt)])
        dC = C0.transpose(1, 2).contiguous()
        dev.run_batched_typed(kid, M, N, K, dA, la, lda, dA[0].numel(), dB, lb, ldb, dB[0].numel(), ft.TYPE_BF16, dC, M, M * N,
                              dC, Bt, 1.0, -1.5, bias, COL, N)
        t.cuda.synchronize()
        for i in range(Bt):
            exact(dC[i].t(), reference(A[i], B[i], 1.0, -1.5, C0[i], bias[i], COL), (kid, Bt, i))
        zero_residual(dev.stats(), kid, (kid, Bt))


@pytest.mark.gpu
def test_layouts_bit_identical_and_launch_count(cuda, ft, dev):
    """The four layout pairs give bit-identical D on rounding data; a fault-tolerant BF16 call is two launches (encode
    pre-pass + GEMM), a plain one one; reuse_b_checksums reuses a BF16 encode but never an FP32 one of the same bytes."""
    t = cuda
    g = t.Generator(device="cuda").manual_seed(3)
    M, N, K = 1024, 768, 2000
    A = t.randn(M, K, generator=g, device="cuda")
    B = t.randn(N, K, generator=g, device="cuda")
    outs = [run16(t, dev, 31, A, B, la, lb)[0].clone() for la in (MN, KM) for lb in (MN, KM)]
    for o in outs[1:]:
        assert t.equal(o.view(t.int32), outs[0].view(t.int32))
    assert dev.stats()["detected"] == 0
    dA, dB = pack16(t, A, KM, K), pack16(t, B, KM, K)
    C = t.empty(N, M, device="cuda")
    n0 = dev.launch_count()
    dev.run_typed(31, M, N, K, dA, KM, K, dB, KM, K, ft.TYPE_BF16, C, M, C)
    assert dev.launch_count() - n0 == 2
    n0 = dev.launch_count()
    dev.run_typed(21, M, N, K, dA, KM, K, dB, KM, K, ft.TYPE_BF16, C, M, C)
    assert dev.launch_count() - n0 == 1
    reuse = ft.make_opts(reuse_b_checksums=True)
    dev.run_typed(31, M, N, K, dA, KM, K, dB, KM, K, ft.TYPE_BF16, C, M, C, opts=reuse)
    n0 = dev.launch_count()
    dev.run_typed(31, M, N, K, dA, KM, K, dB, KM, K, ft.TYPE_BF16, C, M, C, opts=reuse)
    assert dev.launch_count() - n0 == 1          # the BF16 encode of the same B is reused
    # the same pointer, shape and leading dimension read as FP32 is another B: encoded afresh (B below 8 MB: the pre-pass),
    # and so is the BF16 B after it
    dBx = t.zeros(2 * N * K, device="cuda", dtype=t.bfloat16)
    dBx[:N * K] = dB
    dAx = t.zeros(2 * M * K, device="cuda", dtype=t.bfloat16)
    dev.run_typed(31, M, N, K, dA, KM, K, dBx, KM, K, ft.TYPE_BF16, C, M, C, opts=reuse)
    n0 = dev.launch_count()
    dev.run_typed(31, M, N, K, dAx, KM, K, dBx, KM, K, ft.TYPE_F32, C, M, C, opts=reuse)
    assert dev.launch_count() - n0 == 2
    n0 = dev.launch_count()
    dev.run_typed(31, M, N, K, dA, KM, K, dBx, KM, K, ft.TYPE_BF16, C, M, C, opts=reuse)
    t.cuda.synchronize()
    assert dev.launch_count() - n0 == 2
    dev.stats()


@pytest.mark.gpu
@pytest.mark.parametrize("kid", (31, 13))
def test_front_phase_encode_exact_and_one_launch(cuda, ft, dev, kid):
    """The encode of B runs in the GEMM kernel's front phase from 8 MB of B (2 bytes per BF16 element), by the FP32 rule: such
    a fault-tolerant BF16 call is one launch, a smaller one two (the pre-pass).  Forced either way (the enc_front knob), every
    layout pair and a batch give the float64 product bit for bit with zero checksum residuals."""
    t = cuda
    g = t.Generator(device="cuda").manual_seed(500 + kid)
    M, N, K = 516, 2048, 2048                      # B: 2048 x 2048 BF16 = 8 MB
    A, B = ints(t, g, (M, K), 2), ints(t, g, (N, K), 2)
    want = reference(A, B)
    for la in (MN, KM):
        for lb in (MN, KM):
            n0 = dev.launch_count()
            got, _ = run16(t, dev, kid, A, B, la, lb)
            assert dev.launch_count() - n0 == 1, (kid, la, lb)
            exact(got, want, (kid, "8 MB", la, lb))
            zero_residual(dev.stats(), kid, (kid, "8 MB", la, lb))
    n0 = dev.launch_count()
    got, _ = run16(t, dev, kid, A, B[: N // 2 - 4], MN, MN)   # B below 8 MB: the pre-pass
    assert dev.launch_count() - n0 == 2
    exact(got, reference(A, B[: N // 2 - 4]), (kid, "pre-pass"))
    zero_residual(dev.stats(), kid, (kid, "pre-pass"))
    Bt, (m, n, k) = 3, (132, 260, 200)
    Ab, Bb = ints(t, g, (Bt, m, k), 4), ints(t, g, (Bt, n, k), 4)
    for front in (0, 1):
        for la, lb in ((MN, MN), (KM, KM), (MN, KM)):
            with knobs(ft, enc_front=front):
                lda, ldb = ld_bf16(la, m, k, False), ld_bf16(lb, n, k, True)
                dA = t.stack([pack16(t, Ab[i], la, lda) for i in range(Bt)])
                dB = t.stack([pack16(t, Bb[i], lb, ldb) for i in range(Bt)])
                dC = t.zeros(Bt, n, m, device="cuda")
                n0 = dev.launch_count()
                dev.run_batched_typed(kid, m, n, k, dA, la, lda, dA[0].numel(), dB, lb, ldb, dB[0].numel(), ft.TYPE_BF16, dC, m,
                                      m * n, dC, Bt)
                t.cuda.synchronize()
                assert dev.launch_count() - n0 == (1 if front else 2)
            for i in range(Bt):
                exact(dC[i].t(), reference(Ab[i], Bb[i]), (kid, "batch", front, la, lb, i))
            zero_residual(dev.stats(), kid, (kid, "batch", front, la, lb))


@pytest.mark.gpu
def test_no_operand_copies(cuda, ft, dev):
    """A BF16 call with both operands MN-major makes no K-major copies of them.  On a fresh handle (after a warm-up call on
    another one) it allocates less than one K-major copy of A would take (64 MB at 4096^2), and more than one copy less than
    the FP32 call with the same layouts, whose front phase writes two (A^T and B^T, 128 MB; the workspaces both calls allocate
    took about 34 MB on an H100)."""
    t = cuda
    n = 4096
    a16 = t.zeros(n * n, device="cuda", dtype=t.bfloat16)
    b16 = t.zeros(n * n, device="cuda", dtype=t.bfloat16)
    a32 = t.zeros(n * n, device="cuda")
    b32 = t.zeros(n * n, device="cuda")
    c = t.zeros(n * n, device="cuda")
    t.cuda.synchronize()

    def call16(h):
        h.run_typed(31, n, n, n, a16, MN, n, b16, MN, n, ft.TYPE_BF16, c, n, c)

    def call32(h):
        h.run_ex(31, n, n, n, a32, MN, n, b32, MN, n, c, n)

    def footprint(call):
        h = ft.FtSgemm()
        try:
            t.cuda.synchronize()
            free0 = t.cuda.mem_get_info()[0]
            call(h)
            t.cuda.synchronize()
            return free0 - t.cuda.mem_get_info()[0]
        finally:
            h.stats()
            h.close()
    footprint(call16)
    footprint(call32)
    used16, used32 = footprint(call16), footprint(call32)
    assert used16 < n * n * 4, (used16, used32)                    # less than one copy
    assert used32 - used16 > n * n * 4, (used16, used32)           # the FP32 front phase's A^T and B^T


@pytest.mark.gpu
def test_argument_checks(cuda, ft, dev):
    t = cuda
    M = N = K = 64
    a = t.zeros(M * K, device="cuda", dtype=t.bfloat16)
    b = t.zeros(N * K, device="cuda", dtype=t.bfloat16)
    c = t.zeros(M * N, device="cuda")
    for kid in (1, 2, 4, 5, 6, 11, 12, 14, 15, 16, 10, 30):
        with pytest.raises(ft.FtsgemmError) as e:
            dev.run_typed(kid, M, N, K, a, KM, K, b, KM, K, ft.TYPE_BF16, c, M, c)
        assert e.value.code == -2, kid
    for bad in (dict(lda=K + 4), dict(ab_type=2), dict(ab_type=-1), dict(precision=1)):
        with pytest.raises(ft.FtsgemmError) as e:
            dev.run_typed(31, M, N, K, a, KM, bad.get("lda", K), b, KM, K, bad.get("ab_type", ft.TYPE_BF16), c, M, c,
                          opts=ft.make_opts(precision=bad.get("precision", 0)))
        assert e.value.code == -1, bad
    x32 = t.zeros(M, K, device="cuda")
    with pytest.raises(TypeError):
        dev.matmul(x32, t.zeros(K, N, device="cuda", dtype=t.bfloat16))


# ------------------------------------------------------------------ GPU: rounding tier
@pytest.mark.gpu
@pytest.mark.parametrize("kid", (31, 13, 21))
def test_rounding_tier(cuda, ft, dev, kid):
    """Standard-normal BF16 operands: every element within (K + 8) 2^-23 (|A| |B|^T)(m, n) + 2^-23 |beta C0| of the float64
    product of the BF16 values, with no alarm."""
    t = cuda
    g = t.Generator(device="cuda").manual_seed(40 + kid)
    worst = 0.0
    for M, N, K, beta in ((1024, 1024, 4096, 0.0), (512, 768, 1000, -1.5), (2048, 2048, 8192, 1.0)):
        A = t.randn(M, K, generator=g, device="cuda").to(t.bfloat16).float()
        B = t.randn(N, K, generator=g, device="cuda").to(t.bfloat16).float()
        C0 = t.randn(M, N, generator=g, device="cuda")
        got, _ = run16(t, dev, kid, A, B, KM, MN, beta=beta, C0=C0)
        want = reference(A, B, 1.0, beta, C0)
        bound = (K + 8) * 2.0 ** -23 * (A.abs().double() @ B.abs().double().T) + 2.0 ** -23 * abs(beta) * C0.abs().double()
        frac = float(((got.double() - want).abs() / bound).max())
        worst = max(worst, frac)
        assert frac <= 1.0, (kid, M, N, K, frac)
        st = dev.stats()
        assert st["detected"] == 0, (kid, M, N, K, st)
    print(f"bf16 rounding tier, id {kid}: largest fraction of the bound {worst:.4f}")


# ------------------------------------------------------------------ GPU: faults, non-finite values, graphs
@pytest.mark.gpu
def test_fault_repair(cuda, ft, dev):
    """Single-bit flips of accumulators (bits 22..30), the self-test injector and post-check upsets (modes 2 / 3 under
    protect_epilogue 1 / 2) on id 31 BF16: detected and repaired, D exact."""
    t = cuda
    g = t.Generator(device="cuda").manual_seed(9)
    M, N, K = 1024, 1024, 1024
    A, B = ints(t, g, (M, K), 4), ints(t, g, (N, K), 4)
    want = reference(A, B)
    rng = np.random.default_rng(0)
    for bit in range(22, 31):
        r, c = int(rng.integers(0, M)), int(rng.integers(0, N))
        got, _ = run16(t, dev, 31, A, B, MN, KM, opts=ft.make_opts(faults=[{"row": r, "col": c, "xor": 1 << bit}]))
        st = dev.stats()
        exact(got, want, ("bit", bit))
        assert st["detected"] >= 1 and st["corrected"] + st["recomputed"] >= 1, (bit, st)
    got, _ = run16(t, dev, 31, A, B, KM, KM, opts=ft.make_opts(selftest=(1000.0, 5, 7)))
    st = dev.stats()
    exact(got, want, "selftest")
    assert st["detected"] >= 1, st
    for level, where in ((1, "epilogue_tmem"), (2, "epilogue_value")):
        got, _ = run16(t, dev, 31, A, B, MN, MN, opts=ft.make_opts(
            protect_epilogue=level, faults=[{"row": 300, "col": 40, "xor": 1 << 27, "where": where}]))
        st = dev.stats()
        exact(got, want, (level, where))
        assert st["epilogue_faults"] >= 1, (level, where, st)


@pytest.mark.gpu
def test_nonfinite_values(cuda, ft, dev):
    """Inf / NaN in BF16 operands land where float64 puts them, and such rows are not flagged."""
    t = cuda
    g = t.Generator(device="cuda").manual_seed(21)
    M, N, K = 512, 256, 300
    A, B = ints(t, g, (M, K), 4), ints(t, g, (N, K), 4)
    A[3, 10] = float("inf")
    A[100, 7] = float("nan")
    B[9, 250] = float("-inf")
    want = reference(A, B)
    for kid in (31, 13, 7):
        got, _ = run16(t, dev, kid, A, B, MN, KM)
        exact(got, want, kid)
        assert dev.stats()["detected"] == 0


@pytest.mark.gpu
def test_graph_replay(cuda, ft, dev):
    """A captured BF16 call replays bit-identically (beta != 0 with D != C: every replay writes the same D)."""
    t = cuda
    g = t.Generator(device="cuda").manual_seed(2)
    M, N, K = 512, 512, 777
    A = t.randn(M, K, generator=g, device="cuda")
    B = t.randn(N, K, generator=g, device="cuda")
    dA, dB = pack16(t, A, MN, pad8(M)), pack16(t, B, KM, pad8(K))
    C = t.randn(N, M, generator=g, device="cuda")
    D0, D = t.empty_like(C), t.empty_like(C)
    s = t.cuda.Stream()
    opts = ft.make_opts(stream=s.cuda_stream)
    with t.cuda.stream(s):
        dev.run_typed(31, M, N, K, dA, MN, pad8(M), dB, KM, pad8(K), ft.TYPE_BF16, C, M, D0, 1.0, 0.5, opts=opts)
    s.synchronize()
    graph = t.cuda.CUDAGraph()
    with t.cuda.graph(graph, stream=s):
        dev.run_typed(31, M, N, K, dA, MN, pad8(M), dB, KM, pad8(K), ft.TYPE_BF16, C, M, D, 1.0, 0.5, opts=opts)
    for _ in range(3):
        D.fill_(0.0)
        graph.replay()
        t.cuda.synchronize()
        assert t.equal(D.view(t.int32), D0.view(t.int32))
    dev.stats()


# ------------------------------------------------------------------ GPU: torch layer
@pytest.mark.gpu
def test_matmul_bf16(cuda, ft, dev):
    """FtSgemm.matmul with bfloat16 a and b: float32 out equal to the float64 product of the BF16 values on exact data (row-
    and column-major operands, a padded copy for an unaligned stride, a bfloat16 bias upcast exactly, c), and within the
    rounding bound on normal data."""
    t = cuda
    g = t.Generator(device="cuda").manual_seed(4)
    M, K, N = 300, 204, 260
    a = ints(t, g, (M, K), 4).to(t.bfloat16)
    b = ints(t, g, (K, N), 4).to(t.bfloat16)
    want = a.double() @ b.double()
    exact(dev.matmul(a, b, kernel_id=31), want, "row-major")
    exact(dev.matmul(a.t().contiguous().t(), b.t().contiguous().t(), kernel_id=13), want, "column-major")
    wide = t.zeros(M, K + 4, device="cuda", dtype=t.bfloat16)
    wide[:, :K] = a
    exact(dev.matmul(wide[:, :K], b, kernel_id=40), want, "copied a")
    bias = ints(t, g, (N,), 16).to(t.bfloat16)
    c = ints(t, g, (M, N), 16)
    exact(dev.matmul(a, b, c=c, beta=1.0, bias=bias), want + c.double() + bias.double(), "c + bias")
    out = dev.matmul(a, b, activation="relu")
    assert t.equal(out, t.relu(want.float()))
    an = t.randn(M, K, generator=g, device="cuda").to(t.bfloat16)
    bn = t.randn(K, N, generator=g, device="cuda").to(t.bfloat16)
    got = dev.matmul(an, bn)
    ref = an.double() @ bn.double()
    bound = (K + 8) * 2.0 ** -23 * (an.double().abs() @ bn.double().abs())
    assert bool(((got.double() - ref).abs() <= bound).all())
    assert dev.stats()["detected"] == 0


def close_to(got, want, bound, tag):
    err = (got.double() - want).abs()
    assert bool((err <= bound).all()), (tag, float((err / bound.clamp_min(1e-300)).max()))


@pytest.mark.gpu
def test_linear_bf16_autograd(cuda, ft, dev):
    """FtSgemm.linear with bfloat16 x, weight and bias: float32 y within the rounding bound of the float64 product; the
    backward rounds grad_y to bfloat16 once, and grad_x, grad_weight and grad_bias (in bfloat16) lie within one bfloat16
    rounding of the float64 products of that rounded grad_y; the residual and the GELU forms too; mixed dtypes refused."""
    t = cuda
    g = t.Generator(device="cuda").manual_seed(31)
    Bt, T, K, N = 2, 96, 200, 136
    x = t.randn(Bt, T, K, generator=g, device="cuda").to(t.bfloat16).requires_grad_()
    W = t.randn(N, K, generator=g, device="cuda").to(t.bfloat16).requires_grad_()
    b = t.randn(N, generator=g, device="cuda").to(t.bfloat16).requires_grad_()
    r = t.randn(Bt, T, N, generator=g, device="cuda")
    gy = t.randn(Bt, T, N, generator=g, device="cuda")
    xd, Wd, bd = x.detach().double().reshape(-1, K), W.detach().double(), b.detach().double()
    for form in ("plain", "residual", "gelu"):
        x.grad = W.grad = b.grad = None
        if form == "plain":
            y = dev.linear(x, W, b)
            z = xd @ Wd.T + bd
            want = z
        elif form == "residual":
            y = dev.linear(x, W, b, residual=r)
            z = xd @ Wd.T + r.double().reshape(-1, N) + bd
            want = z
        else:
            y = dev.linear(x, W, b, activation="gelu")
            z = xd @ Wd.T + bd
            want = t.nn.functional.gelu(z)
        assert y.dtype == t.float32 and y.shape == (Bt, T, N)
        bound = (K + 8) * 2.0 ** -23 * (xd.abs() @ Wd.abs().T) + 2.0 ** -22 * (z.abs() + bd.abs()) + 1e-6
        close_to(y.reshape(-1, N), want, bound, form)
        y.backward(gy)
        assert x.grad.dtype == W.grad.dtype == b.grad.dtype == t.bfloat16
        gz = gy.reshape(-1, N)
        # (GELU: the reference's z is the float64 one rounded to FP32, which may differ from the kernel's in the last bit, and
        # so grad_z in one bfloat16 rounding: a term of 2^-8 of the magnitudes covers it)
        tol_mag = 2.0 ** -15  # (the FP32 accumulation over at most 256 terms)
        if form == "gelu":
            gz = t.ops.aten.gelu_backward(gz, z.float())
            tol_mag = 2.0 ** -8
        g16 = gz.to(t.bfloat16).double()
        for got, want_g, mag in ((x.grad.reshape(-1, K), g16 @ Wd, g16.abs() @ Wd.abs()),
                                 (W.grad, g16.T @ xd, g16.abs().T @ xd.abs()),
                                 (b.grad, g16.sum(0), g16.abs().sum(0))):
            close_to(got, want_g, 2.0 ** -8 * want_g.abs() + tol_mag * mag + 1e-6, (form, "grad"))
    with pytest.raises(TypeError):
        dev.linear(x.detach().float(), W.detach())
    assert dev.stats()["detected"] == 0


@pytest.mark.gpu
def test_bmm_bf16_autograd(cuda, ft, dev):
    """FtSgemm.bmm with bfloat16 a, b and a per-entry bfloat16 bias, ReLU fused: forward within the rounding bound, and the
    gradients (grad_z rounded to bfloat16 once) within one bfloat16 rounding of the float64 products; exact data exact."""
    t = cuda
    g = t.Generator(device="cuda").manual_seed(32)
    Bt, M, K, N = 3, 72, 100, 48
    a = t.randn(Bt, M, K, generator=g, device="cuda").to(t.bfloat16).requires_grad_()
    b = t.randn(Bt, K, N, generator=g, device="cuda").to(t.bfloat16).requires_grad_()
    bias = t.randn(Bt, N, generator=g, device="cuda").to(t.bfloat16).requires_grad_()
    y = dev.bmm(a, b, bias=bias, activation="relu")
    ad, bdd, biasd = a.detach().double(), b.detach().double(), bias.detach().double()
    z = ad @ bdd + biasd[:, None, :]
    bound = (K + 8) * 2.0 ** -23 * (ad.abs() @ bdd.abs()) + 2.0 ** -22 * z.abs() + 1e-6
    close_to(y, t.relu(z), bound, "forward")
    gy = t.randn(Bt, M, N, generator=g, device="cuda")
    y.backward(gy)
    gz = t.ops.aten.threshold_backward(gy, y.detach(), 0).to(t.bfloat16).double()
    for got, want_g, mag in ((a.grad, gz @ bdd.transpose(1, 2), gz.abs() @ bdd.abs().transpose(1, 2)),
                             (b.grad, ad.transpose(1, 2) @ gz, ad.abs().transpose(1, 2) @ gz.abs()),
                             (bias.grad, gz.sum(1), gz.abs().sum(1))):
        assert got.dtype == t.bfloat16
        close_to(got, want_g, 2.0 ** -8 * want_g.abs() + 2.0 ** -15 * mag + 1e-6, "grad")
    assert dev.stats()["detected"] == 0  # (and resets the counters: the rounding data above leave nonzero residuals)
    ai, bi = ints(t, g, (Bt, M, K), 4).to(t.bfloat16), ints(t, g, (Bt, K, N), 4).to(t.bfloat16)
    exact(dev.bmm(ai, bi, kernel_id=31), ai.double() @ bi.double(), "exact bmm")
    zero_residual(dev.stats(), 31, "bmm")


@pytest.mark.gpu
def test_graphed_linear_bf16(cuda, ft, dev):
    """A BF16 FtSgemm.linear captured in a CUDA graph replays bit-identically to the eager call."""
    t = cuda
    g = t.Generator(device="cuda").manual_seed(33)
    x = t.randn(256, 512, generator=g, device="cuda").to(t.bfloat16)
    W = t.randn(384, 512, generator=g, device="cuda").to(t.bfloat16)
    b = t.randn(384, generator=g, device="cuda")
    want = dev.linear(x, W, b)
    s = t.cuda.Stream()
    s.wait_stream(t.cuda.current_stream())
    with t.cuda.stream(s):
        dev.linear(x, W, b)
    t.cuda.current_stream().wait_stream(s)
    graph = t.cuda.CUDAGraph()
    with t.cuda.graph(graph):
        y = dev.linear(x, W, b)
    for _ in range(2):
        graph.replay()
        t.cuda.synchronize()
        assert t.equal(y.view(t.int32), want.view(t.int32))
    dev.stats()


@pytest.mark.gpu
@pytest.mark.slow
def test_fault_campaign_floors_bf16(cuda, ft, dev):
    """test_gpu_parity's fault campaign on BF16 operands at the real size (M = N = K = 8192, id 31): single-bit flips of
    accumulators.  Bits >= 22 detected and repaired 100 % with the error left <= 1e-4 max|C|; lower bits: whatever is
    detected is repaired, and what stays undetected is below the detection threshold (< 5e-4 max|C|)."""
    t = cuda
    n, kid = 8192, 31
    g = t.Generator(device="cuda").manual_seed(7)
    dA = ((t.randint(0, 10, (n * n,), generator=g, device="cuda").float() * 0.1) *
          (t.randint(0, 2, (n * n,), generator=g, device="cuda").float() * 2 - 1)).to(t.bfloat16)
    dB = ((t.randint(0, 10, (n * n,), generator=g, device="cuda").float() * 0.1) *
          (t.randint(0, 2, (n * n,), generator=g, device="cuda").float() * 2 - 1)).to(t.bfloat16)
    clean = t.zeros(n * n, device="cuda")
    dev.stats()
    dev.run_typed(kid, n, n, n, dA, MN, n, dB, MN, n, ft.TYPE_BF16, clean, n, clean)
    t.cuda.synchronize()
    assert dev.stats()["detected"] == 0
    scale = float(clean.abs().max())
    rng = np.random.default_rng(0)
    dC = t.zeros(n * n, device="cuda")
    for bit in (31, 30, 29, 27, 25, 23, 22, 21, 19, 16, 10):
        faults, seen = [], set()
        while len(faults) < ft.MAX_FAULTS:
            r, c = int(rng.integers(n)), int(rng.integers(n))
            if (r, c // 256) in seen:
                continue
            seen.add((r, c // 256))
            faults.append({"row": r, "col": c, "xor": 1 << bit})
        dC.zero_()
        dev.run_typed(kid, n, n, n, dA, MN, n, dB, MN, n, ft.TYPE_BF16, dC, n, dC, opts=ft.make_opts(faults=faults))
        t.cuda.synchronize()
        st = dev.stats()
        assert st["uncorrectable"] == 0 and st["checksum_faults"] == 0, (bit, st)
        assert st["corrected"] + st["recomputed"] == st["detected"], (bit, st)
        worst = float((dC - clean).abs().max())
        assert worst <= 5e-4 * scale, (bit, worst, scale)
        if bit >= 22:
            assert st["detected"] == len(faults) and worst <= 1e-4 * scale, (bit, st, worst, scale)


@pytest.mark.gpu
def test_deep_k_alarms_reported(cuda, ft, dev):
    """Fault-free standard-normal BF16 operands at K = 16384 (512 x 512, six calls, id 31): the alarms the default threshold
    raises there are counted and printed (the FP32 path raises some at this depth too, DESIGN.md section 4); a call without
    alarms is within the rounding bound."""
    t = cuda
    g = t.Generator(device="cuda").manual_seed(16384)
    M = N = 512
    K = 16384
    flagged = 0
    for _ in range(6):
        A = t.randn(M, K, generator=g, device="cuda").to(t.bfloat16).float()
        B = t.randn(N, K, generator=g, device="cuda").to(t.bfloat16).float()
        got, _ = run16(t, dev, 31, A, B, KM, KM)
        want = reference(A, B)
        bound = (K + 8) * 2.0 ** -23 * (A.abs().double() @ B.abs().double().T)
        detected = dev.stats()["detected"]
        if detected == 0:
            assert bool(((got.double() - want).abs() <= bound).all())
        flagged += detected
    print(f"bf16 K = 16384: {flagged} rows flagged over six fault-free calls")
