"""Operand layouts and leading dimensions (ftsgemm_run_ex, FtSgemm.run_ex / matmul).

The product C = alpha * A * B^T + beta * C does not depend on how the operands are stored: with each of A and B MN-major
(the reference's layout) or K-major, and with padded leading dimensions, every tensor-core kernel gives C bit for bit as
ftsgemm_run does on the same data, and writes nothing outside C's M x N block.  The CPU tests check the ABI's NULL-handle
answer and the torch stride mapping of matmul; the rest run on the GPU.

Tolerances as in tests/test_gpu_parity.py: TOL_NORM = 1e-3 norm-wise against the FP32 CPU product, TOL_MODEL = 5e-5
norm-wise against a float64 product of TF32-truncated operands (or between two fault-tolerant runs).
"""
import numpy as np
import pytest

TOL_NORM = 1e-3
TOL_MODEL = 5e-5
MN, KM = 0, 1
NAMES = ["small", "medium", "large", "tall", "wide", "huge", "giant", "pair128"]


# ------------------------------------------------------------------ CPU
def test_run_ex_null_handle(ft):
    assert ft.lib().ftsgemm_run_ex(None, 16, 128, 128, 128, None, 0, 128, None, 0, 128, None, 128, 1.0, 0.0, None) == -4


def _plan(ft, a_rm, b_rm, o_rm, M=64, N=96, K=40, pad=0):
    """strides of a (M, K), b (K, N), out (M, N): row-major (rm) or column-major, leading stride padded by `pad`"""
    def st(rows, cols, rm):
        return (cols + pad, 1) if rm else (1, rows + pad)
    return ft.matmul_plan((M, K), st(M, K, a_rm), (K, N), st(K, N, b_rm), st(M, N, o_rm), 256, 512, 1024)


@pytest.mark.parametrize("a_rm", [True, False])
@pytest.mark.parametrize("b_rm", [True, False])
@pytest.mark.parametrize("o_rm", [True, False])
def test_matmul_plan_strides(ft, a_rm, b_rm, o_rm):
    M, N, K = 64, 96, 40
    for pad in (0, 4):
        p = _plan(ft, a_rm, b_rm, o_rm, M, N, K, pad)
        assert not (p["copy_a"] or p["copy_b"] or p["copy_out"]), p
        lay_a = KM if a_rm else MN            # a(m, k) contiguous along k
        lay_b = MN if b_rm else KM            # b(k, n) as a (n, k) operand: row-major b is contiguous along n
        ld_a = (K if a_rm else M) + pad
        ld_b = (N if b_rm else K) + pad
        ld_o = (N if o_rm else M) + pad
        if o_rm:  # out^T = b^T a^T: kernel A is b^T, kernel B is a
            want = dict(M=N, N=M, K=K, layout_a=lay_b, lda=ld_b, layout_b=lay_a, ldb=ld_a, ldc=ld_o, swap=True)
        else:
            want = dict(M=M, N=N, K=K, layout_a=lay_a, lda=ld_a, layout_b=lay_b, ldb=ld_b, ldc=ld_o, swap=False)
        assert {k: p[k] for k in want} == want, (pad, p)
    # x @ W.T with row-major x, W and out: both kernel operands K-major, nothing copied
    p = ft.matmul_plan((M, K), (K, 1), (K, N), (1, K), (N, 1))
    assert p["swap"] and p["layout_a"] == KM and p["layout_b"] == KM and p["lda"] == K and p["ldb"] == K


def test_matmul_plan_marks_copies(ft):
    M, N, K = 64, 96, 40
    # no unit stride
    p = ft.matmul_plan((M, K), (2 * K, 2), (K, N), (N, 1), (N, 1))
    assert p["copy_a"] and not p["copy_b"] and not p["copy_out"]
    assert p["layout_b"] == KM and p["ldb"] == K  # the copy of a: row-major, rows padded to 16 bytes
    # leading stride not a multiple of 16 bytes (K = 42 floats)
    p = ft.matmul_plan((M, 42), (42, 1), (42, N), (N, 1), (N, 1))
    assert p["copy_a"] and not p["copy_b"] and p["ldb"] == 44
    # misaligned base address
    p = ft.matmul_plan((M, K), (K, 1), (K, N), (N, 1), (N, 1), a_ptr=256, b_ptr=260)
    assert p["copy_b"] and not p["copy_a"] and p["layout_a"] == KM and p["lda"] == K  # the copy of b: column-major
    # out: no unit stride -> computed in a contiguous row-major buffer
    p = ft.matmul_plan((M, K), (K, 1), (K, N), (N, 1), (2 * N, 2))
    assert p["copy_out"] and p["swap"] and p["ldc"] == N
    # out's leading stride needs no 16-byte multiple, only its base does
    p = ft.matmul_plan((M, K), (K, 1), (K, N), (N, 1), (N + 1, 1))
    assert not p["copy_out"] and p["ldc"] == N + 1
    p = ft.matmul_plan((M, K), (K, 1), (K, N), (N, 1), (N, 1), out_ptr=1028)
    assert p["copy_out"]
    with pytest.raises(ValueError):
        ft.matmul_plan((M, K), (K, 1), (K + 1, N), (N, 1), (N, 1))


# ------------------------------------------------------------------ GPU helpers
def _rand(rng, shape):
    return (rng.integers(0, 10, shape) * 0.1 * rng.choice([-1.0, 1.0], shape)).astype(np.float32)


def _pack(X, layout, ld):
    """rows x K matrix X -> flat buffer in the layout (MN: X[r, k] at r + k*ld; KM: at k + r*ld), padding = NaN"""
    rows, K = X.shape
    if layout == MN:
        buf = np.full((K, ld), np.nan, np.float32)
        buf[:, :rows] = X.T
    else:
        buf = np.full((rows, ld), np.nan, np.float32)
        buf[:, :K] = X
    return buf.reshape(-1)


def _ld(layout, rows, K, pad=True):
    if not pad:
        return rows if layout == MN else K
    return rows + 4 if layout == MN else (K + 3) // 4 * 4 + 4


SENTINEL = np.float32(-12345.5)


class _Case:
    """One product on the GPU: A (M x K), B (N x K), C0 (M x N) as 2-D numpy arrays."""

    def __init__(self, cuda, dev, A, B, C0):
        self.cuda, self.dev, self.A, self.B, self.C0 = cuda, dev, A, B, C0
        self.M, self.K = A.shape
        self.N = B.shape[0]

    def run(self, kid, alpha=1.0, beta=0.0, opts=None):
        """ftsgemm_run on the reference layout: C as an M x N array"""
        t = self.cuda
        dA = t.from_numpy(_pack(self.A, MN, self.M)).cuda()
        dB = t.from_numpy(_pack(self.B, MN, self.N)).cuda()
        dC = t.from_numpy(np.ascontiguousarray(self.C0.T).reshape(-1)).cuda()
        self.dev.run(kid, self.M, self.N, self.K, dA, dB, dC, alpha, beta, opts)
        t.cuda.synchronize()
        return dC.cpu().numpy().reshape(self.N, self.M).T

    def run_ex(self, kid, la, lda, lb, ldb, ldc, alpha=1.0, beta=0.0, opts=None):
        t = self.cuda
        dA = t.from_numpy(_pack(self.A, la, lda)).cuda()
        dB = t.from_numpy(_pack(self.B, lb, ldb)).cuda()
        cbuf = np.full((self.N, ldc), SENTINEL, np.float32)
        cbuf[:, :self.M] = self.C0.T
        dC = t.from_numpy(cbuf.reshape(-1)).cuda()
        self.dev.run_ex(kid, self.M, self.N, self.K, dA, la, lda, dB, lb, ldb, dC, ldc, alpha, beta, opts)
        t.cuda.synchronize()
        out = dC.cpu().numpy().reshape(self.N, ldc)
        assert np.all(out[:, self.M:] == SENTINEL), "C's padding was written"
        return out[:, :self.M].T

    def layouts(self, pad=True):
        for la in (MN, KM):
            for lb in (MN, KM):
                yield la, _ld(la, self.M, self.K, pad), lb, _ld(lb, self.N, self.K, pad)


def _rel(ref, x):
    ref, x = ref.astype(np.float64), x.astype(np.float64)
    return float(np.linalg.norm(ref - x) / np.linalg.norm(ref))


@pytest.fixture(scope="module")
def dev(cuda, ft):
    cuda.cuda.set_device(0)
    h = ft.FtSgemm()
    yield h
    h.close()


# ------------------------------------------------------------------ GPU: bit-identity
@pytest.mark.gpu
@pytest.mark.parametrize("splitk", [0, 2])
def test_layouts_bit_identical_to_run(cuda, ft, dev, splitk):
    """Every named variant, plain and fault-tolerant, with cut tiles off and forced: all four layout pairs with padded leading
    dimensions (lda = rows + 4 or K + 4, ldc = M + 8) and the reference layout with dense ones give C bit for bit as run."""
    rng = np.random.default_rng(21)
    M, N, K = 260, 388, 201  # ragged in M, N and K (K % 4 != 0)
    case = _Case(cuda, dev, _rand(rng, (M, K)), _rand(rng, (N, K)), rng.standard_normal((M, N)).astype(np.float32))
    try:
        ft.debug_set("splitk", splitk)
        for name in NAMES:
            for kid in (ft.SGEMM_IDS[name], ft.ABFT_IDS[name]):
                dev.stats()
                ref = case.run(kid, 0.75, -1.5)
                got = case.run_ex(kid, MN, M, MN, N, M, 0.75, -1.5)
                assert np.array_equal(ref, got), (kid, "dense")
                for la, lda, lb, ldb in case.layouts():
                    got = case.run_ex(kid, la, lda, lb, ldb, M + 8, 0.75, -1.5)
                    assert np.array_equal(ref, got), (kid, la, lb)
                if kid >= 10:
                    assert dev.stats()["detected"] == 0, kid
    finally:
        ft.debug_set("splitk", -1)


# ------------------------------------------------------------------ GPU: cuBLAS rows
@pytest.mark.gpu
def test_cublas_ids_through_run_ex(cuda, ft, dev, oracle):
    rng = np.random.default_rng(22)
    M, N, K = 256, 384, 300
    A, B, C0 = _rand(rng, (M, K)), _rand(rng, (N, K)), rng.standard_normal((M, N)).astype(np.float32)
    case = _Case(cuda, dev, A, B, C0)
    want = oracle.sgemm_nt(M, N, K, 0.75, _pack(A, MN, M), _pack(B, MN, N), -1.5,
                           np.ascontiguousarray(C0.T).reshape(-1)).reshape(N, M).T
    for kid in (0, 7):
        ref = case.run(kid, 0.75, -1.5)
        for la, lda, lb, ldb in case.layouts():
            got = case.run_ex(kid, la, lda, lb, ldb, M + 8, 0.75, -1.5)
            assert _rel(ref, got) < (1e-5 if kid == 0 else TOL_MODEL), (kid, la, lb, _rel(ref, got))
            assert _rel(want, got) < TOL_NORM, (kid, la, lb)


# ------------------------------------------------------------------ GPU: ABFT with a K-major B
def _faults_per_tile(clean, rng, bits, tile_n):
    M = clean.shape[0]
    cand = np.argwhere(np.abs(clean) >= 2.0)
    faults, seen = [], set()
    for r, c in rng.permutation(cand):
        if (r, c // tile_n) in seen:
            continue
        seen.add((r, c // tile_n))
        faults.append({"row": int(r), "col": int(c), "xor": 1 << bits[len(faults)]})
        if len(faults) == len(bits):
            break
    assert len(faults) == len(bits) and M > 0
    return faults


@pytest.mark.gpu
@pytest.mark.parametrize("NK", [1024, 2048])  # B = 4 MB: encode pre-pass; 16 MB: encode in the kernel's front phase
def test_abft_with_k_major_b(cuda, ft, dev, NK):
    rng = np.random.default_rng(NK)
    M, N, K = 512, NK, NK
    kid = 31
    case = _Case(cuda, dev, _rand(rng, (M, K)), _rand(rng, (N, K)), rng.standard_normal((M, N)).astype(np.float32))
    launches = dev.launch_count()
    dev.stats()
    clean = case.run(kid)
    ref_rel = dev.stats()["max_rel_residual"]
    assert dev.launch_count() - launches == (2 if NK == 1024 else 1)
    for la, lda in ((KM, K), (MN, M + 4), (KM, K + 4)):
        for ldb in (K, K + 4):
            launches = dev.launch_count()
            got = case.run_ex(kid, la, lda, KM, ldb, M)
            st = dev.stats()
            assert dev.launch_count() - launches == (2 if NK == 1024 else 1)
            assert np.array_equal(got, clean) and st["detected"] == 0, (la, ldb, st)
            assert st["max_rel_residual"] <= 4 * ref_rel, (st["max_rel_residual"], ref_rel)
    # single-bit flips in the exponent, sign and top mantissa bit: detected and corrected
    faults = _faults_per_tile(clean, rng, [22, 25, 30, 31], 256)
    got = case.run_ex(kid, KM, K, KM, K + 4, M, opts=ft.make_opts(faults=faults))
    st = dev.stats()
    assert st["detected"] == 4 == st["corrected"], st
    assert {(e["row"], e["col"]) for e in st["events"]} == {(f["row"], f["col"]) for f in faults}
    assert np.abs(got - clean).max() < 2e-2
    # two upsets in one row: the row segment is recomputed from the operands in their own layouts
    two = [{"row": 40, "col": 10, "add": 100.0}, {"row": 40, "col": 25, "add": -37.0}]
    ref_beta = case.run(kid, 0.75, -1.5)
    for la, lda in ((KM, K + 4), (MN, M + 4)):
        got = case.run_ex(kid, la, lda, KM, K + 4, M + 8, 0.75, -1.5, opts=ft.make_opts(faults=two))
        st = dev.stats()
        assert st["detected"] == 1 and st["recomputed"] == 1 and st["uncorrectable"] == 0, (la, st)
        assert _rel(ref_beta, got) < TOL_MODEL
        assert set(np.argwhere(got != ref_beta)[:, 0].tolist()) <= {40}
    # protected epilogue, beta = 0: an upset after the check is recomputed, with a K-major A as well
    for la, lda in ((KM, K + 4), (MN, M)):
        f = [{"row": 37, "col": 5, "xor": 1 << 27, "where": "epilogue_tmem"}]
        got = case.run_ex(kid, la, lda, KM, K, M, 0.75, 0.0, opts=ft.make_opts(faults=f, protect_epilogue=True))
        st = dev.stats()
        assert st["epilogue_faults"] == 1 and st["recomputed"] == 1 and st["uncorrectable"] == 0, (la, st)
        clean_a = case.run(kid, 0.75, 0.0)
        assert np.abs(got - clean_a).max() <= 1e-4 * float(np.abs(clean_a).max())
        assert set(np.argwhere(got != clean_a)[:, 0].tolist()) <= {37}


# ------------------------------------------------------------------ GPU: option interactions
@pytest.mark.gpu
def test_check_segments_and_3xtf32_layouts(cuda, ft, dev, oracle):
    rng = np.random.default_rng(23)
    M, N, K = 384, 640, 1000
    A = rng.standard_normal((M, K)).astype(np.float32)
    B = rng.standard_normal((N, K)).astype(np.float32)
    C0 = rng.standard_normal((M, N)).astype(np.float32)
    case = _Case(cuda, dev, A, B, C0)
    want = oracle.sgemm_nt(M, N, K, 0.75, _pack(A, MN, M), _pack(B, MN, N), -1.5,
                           np.ascontiguousarray(C0.T).reshape(-1)).reshape(N, M).T
    rms = float(np.sqrt(np.mean(want.astype(np.float64) ** 2)))
    for kid in (31, 16):
        for opts in (dict(check_segments=4), dict(precision=1), dict(check_segments=3, precision=1)):
            dev.stats()
            ref = case.run(kid, 0.75, -1.5, opts=ft.make_opts(**opts))
            for la, lda, lb, ldb in case.layouts():
                got = case.run_ex(kid, la, lda, lb, ldb, M + 8, 0.75, -1.5, opts=ft.make_opts(**opts))
                assert np.array_equal(ref, got), (kid, opts, la, lb)
            assert dev.stats()["detected"] == 0
            if opts.get("precision"):  # element-wise parity with the FP32 product
                d = np.abs(got.astype(np.float64) - want.astype(np.float64))
                assert np.all(d <= 1e-3 * np.abs(want) + 1e-5 * rms), (kid, float(d.max()))


# ------------------------------------------------------------------ GPU: checksum reuse
@pytest.mark.gpu
def test_reuse_b_checksums_keyed_on_layout(cuda, ft, dev):
    """The same B pointer read in the other layout (N = K: B or B^T) is another operand: its checksums are not reused."""
    t = cuda
    rng = np.random.default_rng(24)
    M, N = 512, 1024
    A, Bbuf = _rand(rng, M * N), _rand(rng, N * N)
    dA, dB = t.from_numpy(A).cuda(), t.from_numpy(Bbuf).cuda()

    def once(n, k, lb, ldb, reuse):
        dC = t.zeros(M * n, device="cuda")
        dev.run_ex(31, M, n, k, dA, MN, M, dB, lb, ldb, dC, M, 1.0, 0.0, ft.make_opts(reuse_b_checksums=reuse))
        return dC
    for first, second in (((N, N, MN, N), (N, N, KM, N)),                # B, then the same pointer read as B^T
                          ((N, N, KM, N), (N, N, MN, N)),
                          ((512, 1020, KM, 1024), (512, 1020, KM, 1020))):  # same layout, another row stride
        dev.stats()
        once(*first, False)
        got = once(*second, True)
        st = dev.stats()
        assert st["detected"] == 0, (first, second, st)
        assert t.equal(got, once(*second, False))
        assert dev.stats()["detected"] == 0
    # the checksums of the same operand are reused, with the same result
    once(N, N, KM, N, False)
    assert t.equal(once(N, N, KM, N, True), once(N, N, KM, N, False)) and dev.stats()["detected"] == 0


# ------------------------------------------------------------------ GPU: argument checks
@pytest.mark.gpu
def test_run_ex_argument_checks(cuda, ft, dev):
    t = cuda
    M, N, K = 256, 256, 128
    dA = t.zeros(4096 * 64, device="cuda")
    dB = t.zeros(4096 * 64, device="cuda")
    dC = t.zeros(4096 * 64, device="cuda")

    def code(kid=31, la=MN, lda=M, lb=MN, ldb=N, ldc=M, a=dA, b=dB):
        try:
            dev.run_ex(kid, M, N, K, a, la, lda, b, lb, ldb, dC, ldc)
            t.cuda.synchronize()
            return 0
        except ft.FtsgemmError as e:
            return e.code
    assert code() == 0 and code(la=KM, lda=K, lb=KM, ldb=K) == 0
    for la in (2, -1):
        assert code(la=la) == -1 and code(lb=la) == -1
    assert code(lda=M - 4) == -1 and code(ldb=N - 4) == -1 and code(ldc=M - 1) == -1
    assert code(la=KM, lda=K - 4) == -1 and code(lb=KM, ldb=K - 4) == -1
    assert code(lda=M + 2) == -1 and code(lb=KM, ldb=K + 2) == -1      # rows not 16-byte multiples
    assert code(a=dA.data_ptr() + 4) == -1 and code(b=dB.data_ptr() + 8) == -1
    for kid in (10, 30):
        assert code(kid) == 0
        assert code(kid, la=KM, lda=K) == -2 and code(kid, lb=KM, ldb=K) == -2 and code(kid, lda=M + 4) == -2
        assert code(kid, ldc=M + 4) == -2
    for kid in (0, 7):  # cuBLAS takes any leading dimension
        assert code(kid, la=KM, lda=K + 2, ldc=M + 1) == 0


# ------------------------------------------------------------------ GPU: torch matmul
@pytest.mark.gpu
def test_matmul_strides(cuda, ft, dev):
    t = cuda
    g = t.Generator(device="cuda").manual_seed(25)
    M, N, K = 192, 320, 264

    def mat(rows, cols, row_major):
        x = t.randn(rows, cols, device="cuda", generator=g)
        return x if row_major else x.t().contiguous().t()
    for a_rm in (True, False):
        for b_rm in (True, False):
            for o_rm in (True, False):
                a, b, o0 = mat(M, K, a_rm), mat(K, N, b_rm), mat(M, N, o_rm)
                want = 0.5 * (a.double() @ b.double()) - 1.5 * o0.double()
                out = o0.clone(memory_format=t.preserve_format)
                assert out.stride() == o0.stride()
                r = dev.matmul(a, b, out, alpha=0.5, beta=-1.5)
                assert r is out
                err = float((out.double() - want).norm() / want.norm())
                assert err < TOL_NORM, (a_rm, b_rm, o_rm, err)
    # views with padded leading strides, an unaligned view (copied once) and out=None
    big = t.randn(M, K + 8, device="cuda", generator=g)
    a = big[:, :K]
    bT = t.randn(N, K + 4, device="cuda", generator=g)[:, :K]
    want = a.double() @ bT.double().t()
    for aa in (a, big[:, 1:K + 1]):
        out = dev.matmul(aa, bT.t())
        w = aa.double() @ bT.double().t()
        assert float((out.double() - w).norm() / w.norm()) < TOL_NORM
    assert float((dev.matmul(a, bT.t(), kernel_id=7).double() - want).norm() / want.norm()) < TOL_NORM
    with pytest.raises(ft.FtsgemmError) as ei:
        dev.matmul(t.randn(6, K, device="cuda"), t.randn(K, 6, device="cuda"))
    assert ei.value.code == -2


@pytest.mark.gpu
def test_matmul_linear_copies_nothing(cuda, ft, dev):
    """x @ W.T on row-major tensors: no operand copy (the memory torch allocates grows by out only), and with the kernel's
    B operand (x) >= 8 MB exactly one launch of this library per call (encode in the kernel's front phase)."""
    t = cuda
    M, N, K = 2048, 1024, 2048
    x = t.randn(M, K, device="cuda")
    W = t.randn(N, K, device="cuda")
    dev.matmul(x, W.t())  # warm-up: workspace, plans, cuBLAS-free path
    t.cuda.synchronize()
    t.cuda.reset_peak_memory_stats()
    base = t.cuda.memory_allocated()
    launches = dev.launch_count()
    out = dev.matmul(x, W.t())
    t.cuda.synchronize()
    assert t.cuda.max_memory_allocated() - base <= out.numel() * 4
    assert dev.launch_count() - launches == 1
    for _ in range(3):
        dev.matmul(x, W.t(), out)
    assert dev.launch_count() - launches == 4
    want = x.double() @ W.double().t()
    assert float((out.double() - want).norm() / want.norm()) < TOL_NORM
    assert dev.stats()["detected"] == 0
