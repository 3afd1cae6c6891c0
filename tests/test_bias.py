"""Bias fused into the store pass (ftsgemm_run_bias, FtSgemm.run_bias / matmul(bias=) / linear).

C = (alpha * A * B^T + beta * C) + bias, with bias[m] per row (BIAS_ROW) or bias[n] per column (BIAS_COL).  The value in
parentheses is bit for bit what run_ex stores, and the add is one FP32 rounding, so every biased C here must equal the
unbiased C followed by a float32 numpy add of the broadcast bias, bit for bit.  The ABFT check runs on the accumulator before
the bias; the recompute fallback and the protected store pass include it.  The CPU tests check the ABI's NULL-handle answer
and the torch mappings of matmul and linear; the rest run on the GPU.

Tolerances as in tests/test_gpu_parity.py: TOL_MODEL = 5e-5 norm-wise against a float64 product of TF32-truncated operands.
"""
import numpy as np
import pytest

TOL_MODEL = 5e-5
MN, KM = 0, 1
NONE, ROW, COL = 0, 1, 2
NAMES = ["small", "medium", "large", "tall", "wide", "huge", "giant", "pair128"]


# ------------------------------------------------------------------ CPU
def test_run_bias_null_handle(ft):
    assert ft.lib().ftsgemm_run_bias(None, 16, 128, 128, 128, None, 0, 128, None, 0, 128, None, 128, 1.0, 0.0, None, 0,
                                     None) == -4
    assert (ft.BIAS_NONE, ft.BIAS_ROW, ft.BIAS_COL) == (NONE, ROW, COL)


@pytest.mark.parametrize("a_rm", [True, False])
@pytest.mark.parametrize("b_rm", [True, False])
@pytest.mark.parametrize("o_rm", [True, False])
def test_matmul_plan_bias_mode(ft, a_rm, b_rm, o_rm):
    """A bias over out's columns is per kernel row when out is row-major (computed swapped), per kernel column otherwise."""
    M, N, K = 64, 96, 40

    def st(rows, cols, rm):
        return (cols, 1) if rm else (1, rows)
    args = ((M, K), st(M, K, a_rm), (K, N), st(K, N, b_rm), st(M, N, o_rm), 256, 512, 1024)
    p = ft.matmul_plan(*args, bias_stride=1, bias_ptr=2048)
    assert p["swap"] == o_rm and p["bias_mode"] == (ROW if o_rm else COL) and not p["copy_bias"], p
    assert not (p["copy_a"] or p["copy_b"] or p["copy_out"])
    q = ft.matmul_plan(*args)
    assert q["bias_mode"] == NONE and not q["copy_bias"]
    assert {k: v for k, v in p.items() if "bias" not in k} == {k: v for k, v in q.items() if "bias" not in k}
    assert ft.matmul_plan(*args, bias_stride=2, bias_ptr=2048)["copy_bias"]
    assert ft.matmul_plan(*args, bias_stride=1, bias_ptr=2050)["copy_bias"]


def test_linear_plan(ft):
    K, N = 40, 24
    p = ft.linear_plan((6, K), (K, 1), (N, K))
    assert (p["M"], p["K"], p["N"], p["out_shape"], p["view"]) == (6, K, N, (6, N), (K, 1))
    # (B, T, K) contiguous, and a slice of wider rows: the leading dimensions collapse into one stride
    assert ft.linear_plan((3, 5, K), (5 * K, K, 1), (N, K))["view"] == (K, 1)
    p = ft.linear_plan((3, 5, K), (5 * (K + 8), K + 8, 1), (N, K))
    assert (p["M"], p["out_shape"], p["view"]) == (15, (3, 5, N), (K + 8, 1))
    # size-1 dimensions do not matter; a 1-D x is one row
    assert ft.linear_plan((1, 5, 1, K), (7, K, 3, 1), (N, K))["view"] == (K, 1)
    p = ft.linear_plan((K,), (1,), (N, K))
    assert p["M"] == 1 and p["out_shape"] == (N,) and p["view"] == (K, 1)
    # a transposed batch (T, B, K).transpose(0, 1) does not nest: copied
    assert ft.linear_plan((3, 5, K), (K, 3 * K, 1), (N, K))["view"] is None
    with pytest.raises(ValueError):
        ft.linear_plan((3, K), (K, 1), (N, K + 1))


# ------------------------------------------------------------------ GPU helpers
def _rand(rng, shape):
    return (rng.integers(0, 10, shape) * 0.1 * rng.choice([-1.0, 1.0], shape)).astype(np.float32)


def _ints(rng, shape):
    """small integers: every TF32 product and FP32 sum of these shapes is exact, so a corrected or recomputed element is
    bit-identical to the fault-free one"""
    return rng.integers(-3, 4, shape).astype(np.float32)


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


def _add_bias(C, bias, mode):
    """the reference: float32 add of the broadcast bias"""
    if mode == NONE:
        return C
    return (C + (bias[:, None] if mode == ROW else bias[None, :])).astype(np.float32)


SENTINEL = np.float32(-12345.5)


class _Case:
    """One product on the GPU: A (M x K), B (N x K), C0 (M x N) as 2-D numpy arrays."""

    def __init__(self, cuda, dev, A, B, C0):
        self.cuda, self.dev, self.A, self.B, self.C0 = cuda, dev, A, B, C0
        self.M, self.K = A.shape
        self.N = B.shape[0]

    def run(self, kid, la=MN, lda=None, lb=MN, ldb=None, ldc=None, alpha=1.0, beta=0.0, bias=None, mode=NONE, opts=None):
        """run_bias (mode NONE: the pointer is NULL and the call is run_ex); C as an M x N array, its padding checked"""
        t = self.cuda
        lda = lda or _ld(la, self.M, self.K, False)
        ldb = ldb or _ld(lb, self.N, self.K, False)
        ldc = ldc or self.M
        dA = t.from_numpy(_pack(self.A, la, lda)).cuda()
        dB = t.from_numpy(_pack(self.B, lb, ldb)).cuda()
        cbuf = np.full((self.N, ldc), SENTINEL, np.float32)
        cbuf[:, :self.M] = self.C0.T
        dC = t.from_numpy(cbuf.reshape(-1)).cuda()
        db = t.from_numpy(bias).cuda() if mode != NONE else None
        if mode == NONE:
            self.dev.run_ex(kid, self.M, self.N, self.K, dA, la, lda, dB, lb, ldb, dC, ldc, alpha, beta, opts)
        else:
            self.dev.run_bias(kid, self.M, self.N, self.K, dA, la, lda, dB, lb, ldb, dC, ldc, alpha, beta, db, mode, opts)
        t.cuda.synchronize()
        out = dC.cpu().numpy().reshape(self.N, ldc)
        assert np.all(out[:, self.M:] == SENTINEL), "C's padding was written"
        return out[:, :self.M].T

    def bias(self, rng, mode, scale=1.0):
        return (scale * rng.standard_normal(self.M if mode == ROW else self.N)).astype(np.float32)

    def layouts(self):
        for la in (MN, KM):
            for lb in (MN, KM):
                yield la, _ld(la, self.M, self.K), lb, _ld(lb, self.N, self.K)


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
def test_bias_bit_identical_to_run_ex_plus_add(cuda, ft, dev, splitk):
    """Every named variant, plain and fault-tolerant, with cut tiles off and forced, both bias modes, all four layout pairs
    with padded leading dimensions and ldc = M + 8, beta = 0 and -1.5: C = run_ex + float32 add, bit for bit."""
    rng = np.random.default_rng(31)
    M, N, K = 260, 388, 201  # ragged in M, N and K (K % 4 != 0)
    case = _Case(cuda, dev, _rand(rng, (M, K)), _rand(rng, (N, K)), rng.standard_normal((M, N)).astype(np.float32))
    biases = {mode: case.bias(rng, mode) for mode in (ROW, COL)}
    try:
        ft.debug_set("splitk", splitk)
        for name in NAMES:
            for kid in (ft.SGEMM_IDS[name], ft.ABFT_IDS[name]):
                dev.stats()
                for la, lda, lb, ldb in case.layouts():
                    for beta in (0.0, -1.5):
                        ref = case.run(kid, la, lda, lb, ldb, M + 8, 0.75, beta)
                        for mode, b in biases.items():
                            got = case.run(kid, la, lda, lb, ldb, M + 8, 0.75, beta, b, mode)
                            assert np.array_equal(_add_bias(ref, b, mode), got), (kid, la, lb, beta, mode)
                if kid >= 10:
                    assert dev.stats()["detected"] == 0, kid
    finally:
        ft.debug_set("splitk", -1)


@pytest.mark.gpu
def test_bias_added_once_with_3xtf32_and_segments(cuda, ft, dev):
    rng = np.random.default_rng(32)
    M, N, K = 384, 640, 1000
    case = _Case(cuda, dev, rng.standard_normal((M, K)).astype(np.float32), rng.standard_normal((N, K)).astype(np.float32),
                 rng.standard_normal((M, N)).astype(np.float32))
    for kid in (31, 16):
        for opts in (dict(check_segments=4), dict(precision=1), dict(check_segments=3, precision=1)):
            dev.stats()
            for la, lb in ((MN, MN), (KM, KM)):
                ref = case.run(kid, la, None, lb, None, M + 8, 0.75, -1.5, opts=ft.make_opts(**opts))
                for mode in (ROW, COL):
                    b = case.bias(rng, mode, 10.0)
                    got = case.run(kid, la, None, lb, None, M + 8, 0.75, -1.5, b, mode, ft.make_opts(**opts))
                    assert np.array_equal(_add_bias(ref, b, mode), got), (kid, opts, la, mode)
            assert dev.stats()["detected"] == 0


# ------------------------------------------------------------------ GPU: ABFT with a bias
def _faults_per_tile(clean, rng, bits, tile_n, floor):
    cand = np.argwhere(np.abs(clean) >= floor)
    faults, seen = [], set()
    for r, c in rng.permutation(cand):
        if (r, c // tile_n) in seen:
            continue
        seen.add((r, c // tile_n))
        faults.append({"row": int(r), "col": int(c), "xor": 1 << bits[len(faults)]})
        if len(faults) == len(bits):
            break
    assert len(faults) == len(bits)
    return faults


def _cancel_case(cuda, dev, rng, mode, M=512, N=1024, K=1024):
    """a product whose rows (COL) or columns (ROW) are all equal, so that one bias vector equals -C exactly (integer data: with
    equal columns the rounding errors of a row's checksums add up coherently, beyond the threshold's model of independent
    errors, and the accumulator check would flag rows without any bias)"""
    A, B = _ints(rng, (M, K)), _ints(rng, (N, K))
    if mode == COL:
        A[:] = A[0]
    else:
        B[:] = B[0]
    case = _Case(cuda, dev, A, B, np.zeros((M, N), np.float32))
    clean = case.run(31)
    bias = -(clean[0, :] if mode == COL else clean[:, 0]).copy()
    return case, bias


@pytest.mark.gpu
def test_abft_with_bias(cuda, ft, dev):
    rng = np.random.default_rng(33)
    M, N, K = 512, 1024, 1024
    kid = 31
    case = _Case(cuda, dev, _ints(rng, (M, K)), _ints(rng, (N, K)), _ints(rng, (M, N)))
    dev.stats()
    clean = case.run(kid)
    scale = float(np.abs(clean).max())
    for mode in (ROW, COL):
        # no false alarm with a bias 1e3 x the product's magnitude
        big = case.bias(rng, mode, 1e3 * scale)
        got = case.run(kid, KM, None, KM, None, None, 1.0, 0.0, big, mode)
        st = dev.stats()
        assert st["detected"] == 0 and np.array_equal(got, _add_bias(clean, big, mode)), st
        # single-bit flips in the exponent, sign and top mantissa bit: corrected, C bit-identical to the fault-free biased C
        b = np.round(case.bias(rng, mode, 50.0))
        want = _add_bias(clean, b, mode)
        faults = _faults_per_tile(clean, rng, [22, 25, 30, 31], 256, 64.0)
        got = case.run(kid, KM, None, KM, None, None, 1.0, 0.0, b, mode, ft.make_opts(faults=faults))
        st = dev.stats()
        assert st["detected"] == 4 == st["corrected"], st
        assert np.array_equal(got, want)
    # two upsets in one row: the row is recomputed, with the bias counted once (data of the magnitude of
    # tests/test_layouts.py: with the integer products above the locator's tolerance accepts this pair as one upset)
    small = _Case(cuda, dev, _rand(rng, (M, K)), _rand(rng, (N, K)), rng.standard_normal((M, N)).astype(np.float32))
    two = [{"row": 40, "col": 10, "add": 100.0}, {"row": 40, "col": 25, "add": -37.0}]
    for mode in (ROW, COL):
        b = small.bias(rng, mode, 10.0)
        ref_beta = _add_bias(small.run(kid, alpha=0.75, beta=-1.5), b, mode)
        dev.stats()
        for la in (KM, MN):
            got = small.run(kid, la, None, KM, None, M + 8, 0.75, -1.5, b, mode, ft.make_opts(faults=two))
            st = dev.stats()
            assert st["detected"] == 1 and st["recomputed"] == 1 and st["uncorrectable"] == 0, (la, st)
            assert _rel(ref_beta, got) < TOL_MODEL
            assert _rel(ref_beta[40], got[40]) < TOL_MODEL
            assert set(np.argwhere(got != ref_beta)[:, 0].tolist()) <= {40}
    # no false alarm with a bias that cancels the product: C = 0
    for mode in (ROW, COL):
        cc, cancel = _cancel_case(cuda, dev, rng, mode)
        dev.stats()
        got = cc.run(kid, KM, None, KM, None, None, 1.0, 0.0, cancel, mode)
        assert dev.stats()["detected"] == 0 and np.all(got == 0.0)


@pytest.mark.gpu
def test_protect_epilogue_with_bias(cuda, ft, dev):
    rng = np.random.default_rng(34)
    M, N, K = 512, 1024, 1024
    kid = 31
    case = _Case(cuda, dev, _ints(rng, (M, K)), _ints(rng, (N, K)), _ints(rng, (M, N)))
    clean = case.run(kid)
    scale = float(np.abs(clean).max())
    prot = dict(protect_epilogue=True)
    for mode in (ROW, COL):
        dev.stats()
        # fault-free: large and cancelling bias
        big = case.bias(rng, mode, 1e3 * scale)
        got = case.run(kid, KM, None, KM, None, None, 1.0, 0.0, big, mode, ft.make_opts(**prot))
        st = dev.stats()
        assert st["epilogue_faults"] == 0 and st["detected"] == 0 and np.array_equal(got, _add_bias(clean, big, mode)), st
        cc, cancel = _cancel_case(cuda, dev, rng, mode)
        dev.stats()
        got = cc.run(kid, KM, None, KM, None, None, 1.0, 0.0, cancel, mode, ft.make_opts(**prot))
        st = dev.stats()
        assert st["epilogue_faults"] == 0 and st["detected"] == 0 and np.all(got == 0.0), st
        # upsets after the check with beta = 0: detected, recomputed, C equal to the clean biased C
        b = np.round(case.bias(rng, mode, 50.0))
        want = _add_bias(clean, b, mode)
        col = next(c for c in range(5, N) if clean[37, c] != 0 and want[37, c] != 0)  # (a flipped exponent bit of 0 is 2^-111)
        for where in ("epilogue_value", "epilogue_tmem"):
            f = [{"row": 37, "col": col, "xor": 1 << 27, "where": where}]
            got = case.run(kid, KM, None, MN, None, None, 1.0, 0.0, b, mode, ft.make_opts(faults=f, **prot))
            st = dev.stats()
            assert st["epilogue_faults"] == 1 and st["recomputed"] == 1 and st["uncorrectable"] == 0, (where, st)
            assert np.array_equal(got, want), where
        # beta != 0: the old values are gone, the row segment is reported (status 7)
        f = [{"row": 37, "col": col, "xor": 1 << 27, "where": "epilogue_value"}]
        case.run(kid, KM, None, KM, None, None, 1.0, -1.5, b, mode, ft.make_opts(faults=f, **prot))
        st = dev.stats()
        assert st["epilogue_faults"] == 1 and st["uncorrectable"] == 1 and st["recomputed"] == 0, st
        assert [e["status"] for e in st["events"]] == [7]


@pytest.mark.gpu
def test_reuse_b_checksums_with_bias(cuda, ft, dev):
    """The bias never enters the checksums: reused checksums give the same C as fresh ones, biased or not."""
    rng = np.random.default_rng(35)
    M, N, K = 512, 1024, 1024
    case = _Case(cuda, dev, _rand(rng, (M, K)), _rand(rng, (N, K)), rng.standard_normal((M, N)).astype(np.float32))
    b = case.bias(rng, COL, 5.0)
    t = cuda
    dA = t.from_numpy(_pack(case.A, KM, K)).cuda()
    dB = t.from_numpy(_pack(case.B, KM, K)).cuda()
    db = t.from_numpy(b).cuda()

    def once(mode, reuse):
        dC = t.zeros(M * N, device="cuda")
        dev.run_bias(31, M, N, K, dA, KM, K, dB, KM, K, dC, M, 1.0, 0.0, db, mode, ft.make_opts(reuse_b_checksums=reuse))
        return dC
    dev.stats()
    fresh = {mode: once(mode, False) for mode in (NONE, COL)}
    for first, second in ((COL, NONE), (NONE, COL), (COL, COL)):
        once(first, False)
        assert t.equal(once(second, True), fresh[second]), (first, second)
    assert dev.stats()["detected"] == 0


# ------------------------------------------------------------------ GPU: launches and copies
@pytest.mark.gpu
def test_bias_adds_no_launch_and_no_copy(cuda, ft, dev):
    t = cuda
    g = t.Generator(device="cuda").manual_seed(36)
    for M, K, N, launches in ((2048, 2048, 1024, 1), (512, 1024, 1024, 2)):  # kernel B = x: 16 MB / 2 MB
        x = t.randn(M, K, device="cuda", generator=g)
        W = t.randn(N, K, device="cuda", generator=g)
        b = t.randn(N, device="cuda", generator=g)
        dev.linear(x, W, b)  # warm-up: workspace, plans
        dev.matmul(x, W.t(), bias=b)
        t.cuda.synchronize()
        t.cuda.reset_peak_memory_stats()
        base = t.cuda.memory_allocated()
        n0 = dev.launch_count()
        y = dev.linear(x, W, b)
        assert dev.launch_count() - n0 == launches
        out = dev.matmul(x, W.t(), bias=b)
        assert dev.launch_count() - n0 == 2 * launches
        dev.matmul(x, W.t(), out)
        assert dev.launch_count() - n0 == 3 * launches
        t.cuda.synchronize()
        assert t.cuda.max_memory_allocated() - base <= 2 * out.numel() * 4
        assert t.equal(y, dev.matmul(x, W.t(), bias=b))
        assert dev.stats()["detected"] == 0


# ------------------------------------------------------------------ GPU: argument checks
@pytest.mark.gpu
def test_run_bias_argument_checks(cuda, ft, dev):
    t = cuda
    M, N, K = 256, 256, 128
    dA, dB, dC = (t.zeros(M * N, device="cuda") for _ in range(3))
    bias = t.zeros(M + 4, device="cuda")

    def code(kid=31, b=bias.data_ptr(), mode=ROW):
        try:
            dev.run_bias(kid, M, N, K, dA, MN, M, dB, MN, N, dC, M, 1.0, 0.0, b, mode)
            t.cuda.synchronize()
            return 0
        except ft.FtsgemmError as e:
            return e.code
    assert code() == 0 and code(mode=COL) == 0 and code(b=bias.data_ptr() + 4) == 0
    for mode in (3, -1):
        assert code(mode=mode) == -1
    assert code(b=None) == -1 and code(b=None, mode=COL) == -1
    assert code(b=bias.data_ptr() + 2) == -1 and code(b=bias.data_ptr() + 1, mode=COL) == -1
    assert code(b=None, mode=NONE) == 0 and code(b=bias.data_ptr() + 2, mode=NONE) == 0  # ignored
    for kid in (0, 7, 10, 30):
        assert code(kid) == -2 and code(kid, mode=COL) == -2
        assert code(kid, b=None, mode=NONE) == 0


# ------------------------------------------------------------------ GPU: linear
def _tf32(x):
    return (x.contiguous().view(__import__("torch").int32) & -8192).view(__import__("torch").float32).double()


@pytest.mark.gpu
def test_linear_forward_and_backward(cuda, ft, dev):
    t = cuda
    g = t.Generator(device="cuda").manual_seed(37)
    K, N = 520, 392
    for shape in ((300, K), (3, 100, K)):
        x = t.randn(*shape, device="cuda", generator=g, requires_grad=True)
        W = t.randn(N, K, device="cuda", generator=g, requires_grad=True)
        b = t.randn(N, device="cuda", generator=g, requires_grad=True)
        dev.stats()
        y = dev.linear(x, W, b)
        assert y.shape == (*shape[:-1], N)
        x2 = x.detach().reshape(-1, K)
        want = _tf32(x2) @ _tf32(W.detach()).t() + b.detach().double()
        assert float((y.detach().reshape(-1, N).double() - want).norm() / want.norm()) < TOL_MODEL
        gy = t.randn(*y.shape, device="cuda", generator=g)
        y.backward(gy)
        gy2 = gy.reshape(-1, N)
        gx = _tf32(gy2) @ _tf32(W.detach())
        gw = _tf32(gy2).t() @ _tf32(x2)
        assert float((x.grad.reshape(-1, K).double() - gx).norm() / gx.norm()) < TOL_MODEL
        assert float((W.grad.double() - gw).norm() / gw.norm()) < TOL_MODEL
        assert t.equal(b.grad, gy2.sum(0))
        assert dev.stats()["detected"] == 0
    # without a bias, and with a fault injected through opts: corrected in the forward, gradients unchanged
    x = t.randn(256, K, device="cuda", generator=g, requires_grad=True)
    W = t.randn(N, K, device="cuda", generator=g, requires_grad=True)
    gy = t.randn(256, N, device="cuda", generator=g)
    grads = []
    for opts in (None, ft.make_opts(faults=[{"row": 5, "col": 7, "add": 1000.0}])):  # kernel (row, col) = y's (col, row)
        x.grad = W.grad = None
        dev.stats()
        y = dev.linear(x, W, opts=opts)
        y.backward(gy)
        st = dev.stats()
        assert st["detected"] == st["corrected"] == (0 if opts is None else 1), st
        want = _tf32(x.detach()) @ _tf32(W.detach()).t()
        assert float((y.detach().double() - want).norm() / want.norm()) < TOL_MODEL
        grads.append((x.grad.clone(), W.grad.clone()))
    assert t.equal(grads[0][0], grads[1][0]) and t.equal(grads[0][1], grads[1][1])
