"""Strided batches with an activation and a per-entry bias (ftsgemm_run_batched_act, FtSgemm.run_batched_act, bmm(bias=,
activation=, preact=) and bmm's autograd).

Entry i of run_batched_act is run_act on entry i alone, with the bias bias + i*stride_bias and Z at dZ + i*stride_c: the same
device code, so C and Z must match bit for bit, GELU included, and the padding and the gaps between entries stay untouched.
Integer operands make every product and sum exact, so a repaired run equals the fault-free one bit for bit, and bmm can be
held to torch's FP32 baddbmm bit for bit (GELU within a few ulp).  The CPU tests check the ABI's NULL-handle answer and
bmm_plan's handling of a (Bt, N) bias; the rest run on the GPU.
"""
import numpy as np
import pytest

MN, KM = 0, 1
NONE, ROW, COL = 0, 1, 2
ACT_NONE, RELU, GELU = 0, 1, 2
NAMES = ["small", "medium", "large", "tall", "wide", "huge", "giant", "pair128"]
GELU_ULP = 2
SENTINEL = -12345.5
Z_SENTINEL = 7777.25
GAP = 8  # floats between the entries of every buffer


# ------------------------------------------------------------------ CPU
def test_run_batched_act_null_handle(ft):
    assert ft.lib().ftsgemm_run_batched_act(None, 16, 128, 128, 128, None, 0, 128, 0, None, 0, 128, 0, None, 128, 0, 2, 1.0,
                                            0.0, None, 0, 0, 1, None, None) == -4
    assert "ftsgemm_run_batched_act" in ft.EXPORTED_SYMBOLS


def _strides(rows, cols, row_major):
    return (rows * cols, cols, 1) if row_major else (rows * cols, 1, rows)


@pytest.mark.parametrize("a_rm", [True, False])
@pytest.mark.parametrize("b_rm", [True, False])
@pytest.mark.parametrize("out_rm", [True, False])
def test_bmm_plan_per_entry_bias(ft, a_rm, b_rm, out_rm):
    Bt, M, K, N = 3, 8, 12, 16
    args = ((Bt, M, K), _strides(M, K, a_rm), (Bt, K, N), _strides(K, N, b_rm), _strides(M, N, out_rm), 256, 512, 1024)

    def plan(bias_stride=1, bias_ptr=4096, entry=None, shape=args):
        return ft.bmm_plan(*shape, bias_stride, bias_ptr, entry)
    p = plan(entry=N)  # a contiguous (Bt, N) bias
    assert p["swap"] == out_rm and p["bias_mode"] == (ROW if out_rm else COL)
    assert p["stride_bias"] == N and not p["copy_bias"]
    assert not (p["copy_a"] or p["copy_b"] or p["copy_out"])
    assert plan(entry=N + 3)["stride_bias"] == N + 3 and not plan(entry=N + 3)["copy_bias"]  # (any entry stride >= 0)
    # an expanded (Bt, N) bias and a shared (N,) one: stride_bias 0, read in place
    for entry in (0, None):
        p = plan(entry=entry)
        assert p["stride_bias"] == 0 and not p["copy_bias"] and p["bias_mode"] == (ROW if out_rm else COL)
    # copied: no unit element stride, a negative entry stride, a base that is not 4-byte aligned -> dense (Bt, N)
    for kw in (dict(bias_stride=2, entry=2 * N), dict(entry=-N), dict(bias_ptr=4098, entry=N)):
        p = plan(**kw)
        assert p["copy_bias"] and p["stride_bias"] == N, kw
    # an expanded bias without unit stride is copied as one shared (N,) vector
    p = plan(bias_stride=2, entry=0)
    assert p["copy_bias"] and p["stride_bias"] == 0
    # one entry: the entry stride is ignored
    one = ((1, M, K), args[1], (1, K, N), args[3], args[4], 256, 512, 1024)
    assert plan(entry=N, shape=one)["stride_bias"] == 0 and plan(entry=-N, shape=one)["stride_bias"] == 0
    # no bias
    p = ft.bmm_plan(*args)
    assert p["stride_bias"] == 0 and p["bias_mode"] == NONE and not p["copy_bias"]


# ------------------------------------------------------------------ GPU helpers
def _ints(rng, shape, lo=-3, hi=4):
    return rng.integers(lo, hi, shape).astype(np.float32)


def _ld(layout, rows, K, pad=True):
    if not pad:
        return rows if layout == MN else K
    return rows + 4 if layout == MN else (K + 3) // 4 * 4 + 4


def _bits(t, x):
    return x.contiguous().view(t.int32)


def _same(t, x, y):
    return t.equal(_bits(t, x), _bits(t, y))


def _ulp(t, a, b):
    def key(x):
        i = x.contiguous().view(t.int32).long()
        return t.where(i < 0, -(i & 0x7FFFFFFF), i)
    return (key(a) - key(b)).abs()


def _check_act(t, C, Z, act):
    """C = act(Z): bit for bit for ReLU, within GELU_ULP for GELU (same NaN positions, same Inf signs)"""
    ref = t.relu(Z) if act == RELU else t.nn.functional.gelu(Z)
    assert t.equal(t.isnan(C), t.isnan(ref))
    fin = t.isfinite(ref)
    assert t.equal(fin, t.isfinite(C))
    inf = t.isinf(ref)
    assert t.equal(C[inf], ref[inf])
    if act == RELU:
        assert _same(t, C[fin], ref[fin])
        return 0
    d = int(_ulp(t, C[fin], ref[fin]).max()) if bool(fin.any()) else 0
    assert d <= GELU_ULP, d
    return d


class _Batch:
    """Bt products on the GPU: A (Bt, M, K), B (Bt, N, K), C0 (Bt, M, N) as numpy arrays.  Every device buffer holds the
    entries GAP floats apart, with padded leading dimensions; operand padding is NaN, C's and Z's padding a sentinel."""

    def __init__(self, t, dev, A, B, C0):
        self.t, self.dev, self.A, self.B, self.C0 = t, dev, A, B, C0
        self.Bt, self.M, self.K = A.shape
        self.N = B.shape[1]
        self._ops = {}

    def op(self, which, layout, ld):
        """(buffer, entry stride) of A or B in the layout"""
        key = (which, layout, ld)
        if key not in self._ops:
            X = self.A if which == "a" else self.B
            rows = X.shape[1]
            span = (self.K if layout == MN else rows) * ld
            stride = span + GAP
            buf = np.full(self.Bt * stride, np.nan, np.float32)
            for i in range(self.Bt):
                e = buf[i * stride:i * stride + span]
                if layout == MN:
                    e.reshape(self.K, ld)[:, :rows] = X[i].T
                else:
                    e.reshape(rows, ld)[:, :self.K] = X[i]
            self._ops[key] = (self.t.from_numpy(buf).cuda(), stride)
        return self._ops[key]

    def c_stride(self, ldc):
        return self.N * ldc + GAP

    def cbuf(self, ldc, fill=None):
        sc = self.c_stride(ldc)
        buf = np.full(self.Bt * sc, SENTINEL if fill is None else fill, np.float32)
        if fill is None:
            for i in range(self.Bt):
                buf[i * sc:i * sc + self.N * ldc].reshape(self.N, ldc)[:, :self.M] = self.C0[i].T
        return self.t.from_numpy(buf).cuda()

    def entry(self, buf, i, ldc):
        """entry i of a C or Z buffer as an M x N view"""
        sc = self.c_stride(ldc)
        return buf[i * sc:i * sc + self.N * ldc].view(self.N, ldc)[:, :self.M].t()

    def untouched(self, buf, ldc, value):
        """everything outside the entries' M x N values still holds value"""
        mask = self.t.ones_like(buf, dtype=self.t.bool)
        for i in range(self.Bt):
            self.entry(mask, i, ldc).fill_(False)
        return bool((buf[mask] == value).all())

    def bias(self, rng, mode, per_entry, scale=20.0, integer=True):
        """(tensor, stride_bias): a shared vector, or one per entry 3 floats apart"""
        L = self.M if mode == ROW else self.N
        if not per_entry:
            b = scale * rng.standard_normal(L)
            return self.t.from_numpy((np.round(b) if integer else b).astype(np.float32)).cuda(), 0
        b = scale * rng.standard_normal((self.Bt, L + 3))
        return self.t.from_numpy((np.round(b) if integer else b).astype(np.float32).reshape(-1)).cuda(), L + 3

    def run(self, kid, la=KM, lda=None, lb=KM, ldb=None, ldc=None, alpha=1.0, beta=0.0, bias=None, mode=NONE, sbias=0,
            act=None, z=False, opts=None, single=False):
        """the batch as one run_batched_act call, or (single) entry by entry through run_act / run_bias: (C, Z) buffers, Z
        None unless z; padding and gaps checked"""
        t, M, N, K = self.t, self.M, self.N, self.K
        lda = lda or _ld(la, M, K, False)
        ldb = ldb or _ld(lb, N, K, False)
        ldc = ldc or M
        (dA, sa), (dB, sb) = self.op("a", la, lda), self.op("b", lb, ldb)
        sc = self.c_stride(ldc)
        cbuf = self.cbuf(ldc)
        zbuf = self.cbuf(ldc, Z_SENTINEL) if z else None
        if not single:
            self.dev.run_batched_act(kid, M, N, K, dA, la, lda, sa, dB, lb, ldb, sb, cbuf, ldc, sc, self.Bt, alpha, beta, bias,
                                     mode, sbias, act or ACT_NONE, zbuf, opts)
        else:
            for i in range(self.Bt):
                pa, pb, pc = dA.data_ptr() + 4 * i * sa, dB.data_ptr() + 4 * i * sb, cbuf.data_ptr() + 4 * i * sc
                pbias = bias.data_ptr() + 4 * i * sbias if bias is not None else None
                if act is None:
                    self.dev.run_bias(kid, M, N, K, pa, la, lda, pb, lb, ldb, pc, ldc, alpha, beta, pbias, mode, opts)
                else:
                    pz = zbuf.data_ptr() + 4 * i * sc if z else None
                    self.dev.run_act(kid, M, N, K, pa, la, lda, pb, lb, ldb, pc, ldc, alpha, beta, pbias, mode, act, pz, opts)
        t.cuda.synchronize()
        assert self.untouched(cbuf, ldc, SENTINEL), "C's padding or gaps were written"
        if z:
            assert self.untouched(zbuf, ldc, Z_SENTINEL), "Z's padding or gaps were written"
        return cbuf, zbuf

    def layouts(self):
        for la in (MN, KM):
            for lb in (MN, KM):
                yield la, _ld(la, self.M, self.K), lb, _ld(lb, self.N, self.K)


@pytest.fixture(scope="module")
def dev(cuda, ft):
    cuda.cuda.set_device(0)
    h = ft.FtSgemm()
    yield h
    h.close()


@pytest.fixture
def fp32(cuda):
    """torch's matmuls in FP32 for the reference (other tests may have allowed TF32)"""
    prev = cuda.backends.cuda.matmul.allow_tf32
    cuda.backends.cuda.matmul.allow_tf32 = False
    yield
    cuda.backends.cuda.matmul.allow_tf32 = prev


def _batch(t, dev, rng, Bt, M, N, K, c_grid=True):
    C0 = (np.round(64 * rng.standard_normal((Bt, M, N))) / 64).astype(np.float32) if c_grid else _ints(rng, (Bt, M, N))
    return _Batch(t, dev, _ints(rng, (Bt, M, K)), _ints(rng, (Bt, N, K)), C0)


# ------------------------------------------------------------------ GPU: bit identity per entry
@pytest.mark.gpu
def test_batched_act_equals_run_act_per_entry(cuda, ft, dev):
    """Every named variant, plain and fault-tolerant, cut tiles off and forced, all four layout pairs with padded leading
    dimensions, ldc = M + 8 and gaps between the entries, a ragged shape, beta 0 and -1.5, ReLU and GELU; the bias (none,
    row, column; shared or per entry) and whether Z is written rotate through the sweep.  Entry i equals run_act on entry i
    alone, bit for bit, in C and Z."""
    t = cuda
    rng = np.random.default_rng(61)
    case = _batch(t, dev, rng, 3, 132, 196, 201)
    biases = [(NONE, None, 0), (ROW, *case.bias(rng, ROW, True)), (COL, *case.bias(rng, COL, True)),
              (ROW, *case.bias(rng, ROW, False)), (COL, *case.bias(rng, COL, False))]
    ldc = case.M + 8
    n = 0
    try:
        for splitk in (0, 2):
            ft.debug_set("splitk", splitk)
            for name in NAMES:
                for kid in (ft.SGEMM_IDS[name], ft.ABFT_IDS[name]):
                    dev.stats()
                    for la, lda, lb, ldb in case.layouts():
                        for beta in (0.0, -1.5):
                            for act in (RELU, GELU):
                                mode, b, sb = biases[n % len(biases)]
                                z = n % 3 != 2
                                n += 1
                                args = (kid, la, lda, lb, ldb, ldc, 0.75, beta, b, mode, sb, act, z)
                                c, zb = case.run(*args)
                                c1, z1 = case.run(*args, single=True)
                                assert _same(t, c, c1), (name, kid, splitk, la, lb, beta, act, mode, sb)
                                assert not z or _same(t, zb, z1), (name, kid, splitk, la, lb, beta, act, mode, sb)
                    if kid >= 10:
                        assert dev.stats()["detected"] == 0, kid
    finally:
        ft.debug_set("splitk", -1)


@pytest.mark.gpu
def test_per_entry_bias_without_activation(cuda, ft, dev):
    """entry i of a per-entry bias call equals run_bias with entry i's bias, bit for bit (the BIAS x BATCH kernels)"""
    t = cuda
    rng = np.random.default_rng(62)
    case = _batch(t, dev, rng, 4, 256, 384, 160)
    for kid in (21, 31, 12, 16):
        for mode in (ROW, COL):
            b, sb = case.bias(rng, mode, True, integer=False)
            for beta in (0.0, -1.5):
                c, _ = case.run(kid, MN, None, KM, None, None, 1.0, beta, b, mode, sb)
                c1, _ = case.run(kid, MN, None, KM, None, None, 1.0, beta, b, mode, sb, single=True)
                assert _same(t, c, c1), (kid, mode, beta)
        assert kid < 10 or dev.stats()["detected"] == 0


@pytest.mark.gpu
def test_wrappers_are_the_same_call(cuda, ft, dev):
    """run_batched_act(ACT_NONE, stride_bias = 0, dZ = NULL) gives run_batched's bits and launches as many kernels"""
    t = cuda
    rng = np.random.default_rng(63)
    case = _batch(t, dev, rng, 3, 256, 512, 512)
    M, N, K, Bt = case.M, case.N, case.K, case.Bt
    (dA, sa), (dB, sb) = case.op("a", KM, K), case.op("b", MN, N)
    sc = case.c_stride(M)
    for kid in (40, 31, 16):
        for bias, mode in ((None, NONE), (case.bias(rng, COL, False)[0], COL)):
            for opt in (dict(), dict(precision=1), dict(check_segments=4)):
                outs, launches = [], []
                for fn in ("run_batched", "run_batched_act"):
                    c = case.cbuf(M)
                    n0 = dev.launch_count()
                    if fn == "run_batched":
                        dev.run_batched(kid, M, N, K, dA, KM, K, sa, dB, MN, N, sb, c, M, sc, Bt, 1.0, -1.5, bias, mode,
                                        ft.make_opts(**opt))
                    else:
                        dev.run_batched_act(kid, M, N, K, dA, KM, K, sa, dB, MN, N, sb, c, M, sc, Bt, 1.0, -1.5, bias, mode, 0,
                                            ACT_NONE, None, ft.make_opts(**opt))
                    t.cuda.synchronize()
                    launches.append(dev.launch_count() - n0)
                    outs.append(c)
                assert _same(t, outs[0], outs[1]) and launches[0] == launches[1], (kid, mode, opt, launches)
    assert dev.stats()["detected"] == 0


@pytest.mark.gpu
def test_3xtf32_and_segments_apply_once(cuda, ft, dev):
    """3xTF32 and check_segments = 4: the bias and the activation go to the last pass / segment; entries equal run_act"""
    t = cuda
    rng = np.random.default_rng(64)
    Bt, M, N, K = 3, 256, 384, 256
    C0 = rng.standard_normal((Bt, M, N)).astype(np.float32)
    case = _Batch(t, dev, rng.standard_normal((Bt, M, K)).astype(np.float32),
                  rng.standard_normal((Bt, N, K)).astype(np.float32), C0)
    for kid in (31, 16):
        for opt in (dict(precision=1), dict(check_segments=4), dict(check_segments=4, precision=1)):
            dev.stats()
            for mode in (ROW, COL):
                b, sb = case.bias(rng, mode, True, 5.0, integer=False)
                for act in (RELU, GELU):
                    args = (kid, MN, None, KM, None, None, 0.75, -1.5, b, mode, sb, act, True, ft.make_opts(**opt))
                    c, z = case.run(*args)
                    c1, z1 = case.run(*args, single=True)
                    assert _same(t, c, c1) and _same(t, z, z1), (kid, opt, mode, act)
                    for i in range(Bt):
                        _check_act(t, case.entry(c, i, M), case.entry(z, i, M), act)
            assert dev.stats()["detected"] == 0, (kid, opt)


# ------------------------------------------------------------------ GPU: fault tolerance
@pytest.mark.gpu
def test_abft_in_one_entry(cuda, ft, dev):
    """single-bit flips in several entries and two upsets in one row of entry 2 (stacked fault rows i*M + m): corrected or
    recomputed, C and Z both right, events on stacked rows"""
    t = cuda
    rng = np.random.default_rng(65)
    Bt, M, N, K = 3, 512, 1024, 512
    kid = 31
    case = _batch(t, dev, rng, Bt, M, N, K, c_grid=False)
    acc = [case.A[i] @ case.B[i].T for i in range(Bt)]
    # bit 30 of an accumulator value of magnitude >= 64 (its exponent: a large, locatable upset), one per entry
    faults = []
    for i, (r, col0) in enumerate(((17, 100), (57, 400), (97, 700))):
        col = next(cc for cc in range(col0, N) if abs(acc[i][r, cc]) >= 64)
        faults.append({"row": i * M + r, "col": col, "xor": 1 << 30})
    for mode in (ROW, COL):
        b, sb = case.bias(rng, mode, True, 50.0)
        for act in (RELU, GELU):
            dev.stats()
            want_c, want_z = case.run(kid, bias=b, mode=mode, sbias=sb, act=act, z=True)
            assert dev.stats()["detected"] == 0
            c, z = case.run(kid, bias=b, mode=mode, sbias=sb, act=act, z=True, opts=ft.make_opts(faults=faults))
            st = dev.stats()
            assert st["detected"] == st["corrected"] == Bt and st["uncorrectable"] == 0, st
            assert _same(t, c, want_c) and _same(t, z, want_z), (mode, act)
            assert sorted(e["row"] for e in st["events"]) == [f["row"] for f in faults], st
            # two upsets in one row of entry 2 that the checksums cannot place: recomputed
            two = [{"row": 2 * M + 40, "col": 10, "add": 100.0}, {"row": 2 * M + 40, "col": 25, "add": -50.0}]
            for la in (KM, MN):
                c, z = case.run(kid, la, bias=b, mode=mode, sbias=sb, act=act, z=True, opts=ft.make_opts(faults=two))
                st = dev.stats()
                assert st["detected"] == 1 and st["recomputed"] == 1 and st["uncorrectable"] == 0, (la, st)
                assert [e["row"] for e in st["events"]] == [2 * M + 40], st
                assert _same(t, c, want_c) and _same(t, z, want_z), (mode, act, la)


@pytest.mark.gpu
def test_protected_store_pass_in_later_entries(cuda, ft, dev):
    """mode-3 upsets (the value about to be stored, i.e. z) in entries 1 and 2: level 1 with beta = 0 recomputes the row,
    level 2 recomputes the failed chunks with beta != 0 too; C and Z restored, events on stacked rows with status 6"""
    t = cuda
    rng = np.random.default_rng(66)
    Bt, M, N, K = 3, 256, 512, 512
    kid = 31
    case = _batch(t, dev, rng, Bt, M, N, K, c_grid=False)
    for mode in (ROW, COL):
        b, sb = case.bias(rng, mode, True, 50.0)
        for act in (RELU, GELU):
            for level, beta in ((1, 0.0), (2, 0.0), (2, -1.5)):
                want_c, want_z = case.run(kid, beta=beta, bias=b, mode=mode, sbias=sb, act=act, z=True)
                dev.stats()
                # fault-free under protection: no alarm, the unprotected bits
                c, z = case.run(kid, beta=beta, bias=b, mode=mode, sbias=sb, act=act, z=True,
                                opts=ft.make_opts(protect_epilogue=level))
                st = dev.stats()
                assert st["epilogue_faults"] == 0 and st["detected"] == 0, st
                assert _same(t, c, want_c) and _same(t, z, want_z)
                wz = [case.entry(want_z, i, M).cpu().numpy() for i in range(Bt)]
                rows = []
                for i, (r, col0) in ((1, (37, 5)), (2, (150, 260))):
                    col = next(cc for cc in range(col0, N) if wz[i][r, cc] != 0)
                    rows.append((i * M + r, col))
                f = [{"row": r, "col": col, "xor": 1 << 27, "where": "epilogue_value"} for r, col in rows]
                c, z = case.run(kid, beta=beta, bias=b, mode=mode, sbias=sb, act=act, z=True,
                                opts=ft.make_opts(faults=f, protect_epilogue=level))
                st = dev.stats()
                assert st["epilogue_faults"] == 2 and st["recomputed"] == 2 and st["uncorrectable"] == 0, (level, beta, st)
                assert sorted(e["row"] for e in st["events"]) == [r for r, _ in rows], st
                assert all(e["status"] == 6 for e in st["events"]), st
                assert _same(t, c, want_c) and _same(t, z, want_z), (mode, act, level, beta)


@pytest.mark.gpu
def test_nonfinite_stays_in_its_entry(cuda, ft, dev):
    """Inf and NaN in entry 1's A: the other entries are finite, and every entry is run_act's bits on it"""
    t = cuda
    rng = np.random.default_rng(67)
    case = _batch(t, dev, rng, 3, 256, 384, 96)
    case.A[1, 3, 5], case.A[1, 70, 9], case.A[1, 100, 50] = np.inf, -np.inf, np.nan
    case._ops.clear()
    for kid in (21, 31, 11):
        dev.stats()
        for mode in (ROW, COL):
            b, sb = case.bias(rng, mode, True, 5.0)
            for act in (RELU, GELU):
                args = (kid, MN, None, KM, None, None, 1.0, -1.5, b, mode, sb, act, True)
                c, z = case.run(*args)
                c1, z1 = case.run(*args, single=True)
                assert _same(t, c, c1) and _same(t, z, z1), (kid, mode, act)
                zs = [case.entry(z, i, case.M) for i in range(3)]
                assert bool(t.isfinite(zs[0]).all()) and bool(t.isfinite(zs[2]).all())
                assert bool(t.isnan(zs[1]).any()) and bool(t.isinf(zs[1]).any())
        assert dev.stats()["detected"] == 0, kid


# ------------------------------------------------------------------ GPU: argument checks
@pytest.mark.gpu
def test_run_batched_act_argument_checks(cuda, ft, dev):
    t = cuda
    Bt, M, N, K = 2, 256, 256, 128
    dA, dB, dC, dZ = (t.zeros(Bt * M * N + 16, device="cuda") for _ in range(4))
    bias = t.zeros(2 * N, device="cuda")

    def code(kid=31, act=RELU, z=dZ.data_ptr(), c=dC.data_ptr(), b=None, mode=NONE, sbias=0):
        try:
            dev.run_batched_act(kid, M, N, K, dA, MN, M, M * K, dB, MN, N, N * K, c, M, M * N, Bt, 1.0, 0.0, b, mode, sbias,
                                act, z)
            t.cuda.synchronize()
            return 0
        except ft.FtsgemmError as e:
            return e.code
    assert code() == 0 and code(act=GELU) == 0 and code(z=None) == 0 and code(act=ACT_NONE, z=None) == 0
    assert code(b=bias, mode=COL, sbias=N) == 0 and code(b=bias, mode=COL, sbias=0) == 0
    assert code(b=bias, mode=COL, sbias=-N) == -1                 # negative entry stride of the bias
    assert code(b=None, mode=NONE, sbias=-N) == 0                 # (ignored without a bias)
    for act in (3, -1):
        assert code(act=act) == -1 and code(act=act, z=None) == -1
    assert code(act=ACT_NONE) == -1                               # Z without an activation
    assert code(z=dC.data_ptr()) == -1                            # Z == C
    assert code(z=dZ.data_ptr() + 2) == -1                        # Z not 4-byte aligned
    for kid in (0, 7, 10, 30):
        assert code(kid, act=GELU, z=None) == -2                  # an activation
        assert code(kid, act=ACT_NONE, z=None, b=bias, mode=COL, sbias=N) == -2  # a per-entry bias
    assert code(0, act=ACT_NONE, z=None) == 0                     # (cuBLAS: the plain strided batch)


# ------------------------------------------------------------------ GPU: the torch layer
def _t_ints(t, g, shape, lo=-3, hi=4):
    return t.randint(lo, hi, shape, device="cuda", generator=g).float()


def _torch_ref(t, a, b, bias, act, alpha):
    """act(baddbmm) in FP32 on the same tensors: differentiable through torch's autograd"""
    if bias is None:
        z = alpha * t.bmm(a, b)
    else:
        z = t.baddbmm(bias.unsqueeze(1) if bias.dim() == 2 else bias, a, b, alpha=alpha)
    y = z if act is None else (t.relu(z) if act == "relu" else t.nn.functional.gelu(z))
    return y, z


@pytest.mark.gpu
def test_bmm_forward_matches_torch(cuda, ft, dev, fp32):
    t = cuda
    g = t.Generator(device="cuda").manual_seed(68)
    Bt, M, K, N = 4, 132, 72, 200
    a = _t_ints(t, g, (Bt, M, K))
    bmat = _t_ints(t, g, (Bt, K, N))
    with t.no_grad():
        for per_entry in (False, True):
            bias = _t_ints(t, g, (Bt, N) if per_entry else (N,), -20, 21)
            for act in (None, "relu", "gelu"):
                for out_rm in (True, False):
                    for b_op in (bmat, bmat.transpose(1, 2).contiguous().transpose(1, 2)):
                        out = t.empty(Bt, M, N, device="cuda") if out_rm else t.empty(Bt, N, M, device="cuda").transpose(1, 2)
                        pre = t.empty_like(out) if act is not None else None
                        y = dev.bmm(a, b_op, out, bias=bias, activation=act, preact=pre, alpha=0.5)
                        want, z = _torch_ref(t, a, b_op, bias, act, 0.5)
                        if act is None:
                            assert _same(t, y, want), (per_entry, out_rm)
                        else:
                            assert _same(t, pre, z), (per_entry, act, out_rm)
                            if act == "relu":
                                assert _same(t, y, want)
                            else:
                                _check_act(t, y, z, GELU)
        # an expanded bias is the shared one; a (Bt, N) bias of one entry too
        bias = _t_ints(t, g, (N,), -20, 21)
        y1 = dev.bmm(a, bmat, bias=bias.expand(Bt, N), activation="relu")
        assert _same(t, y1, dev.bmm(a, bmat, bias=bias, activation="relu"))
        # invalid: preact strides, an out that cannot be written in place, preact without activation, unknown activation
        out = t.empty(Bt, M, N, device="cuda")
        with pytest.raises(ValueError):
            dev.bmm(a, bmat, out, activation="relu", preact=t.empty(Bt, N, M, device="cuda").transpose(1, 2))
        with pytest.raises(ValueError):
            dev.bmm(a, bmat, t.empty(Bt, M, 2 * N, device="cuda")[:, :, ::2], activation="relu")
        with pytest.raises(ValueError):
            dev.bmm(a, bmat, out, preact=t.empty_like(out))
        with pytest.raises(ValueError):
            dev.bmm(a, bmat, out, activation="tanh")
        with pytest.raises(ValueError):
            dev.bmm(a, bmat, out, bias=t.zeros(Bt + 1, N, device="cuda"))
    assert dev.stats()["detected"] == 0


@pytest.mark.gpu
def test_bmm_attention_scores_copy_nothing(cuda, ft, dev):
    """q @ k^T of contiguous q, k: read in place, one launch (B of all entries >= 8 MiB: the encode is fused), and with GELU
    and no input requiring grad no Z either"""
    t = cuda
    g = t.Generator(device="cuda").manual_seed(69)
    Bt, S, d = 8, 1024, 256
    q = t.randn(Bt, S, d, device="cuda", generator=g)
    k = t.randn(Bt, S, d, device="cuda", generator=g)
    for act in (None, "gelu"):
        dev.bmm(q, k.transpose(-1, -2), activation=act)  # warm-up: workspaces, plans
        t.cuda.synchronize()
        t.cuda.reset_peak_memory_stats()
        base = t.cuda.memory_allocated()
        n0 = dev.launch_count()
        y = dev.bmm(q, k.transpose(-1, -2), activation=act)
        assert dev.launch_count() - n0 == 1, act
        t.cuda.synchronize()
        assert t.cuda.max_memory_allocated() - base <= y.numel() * 4, act
        assert y.grad_fn is None
        del y
    assert dev.stats()["detected"] == 0


@pytest.mark.gpu
@pytest.mark.parametrize("act", [None, "relu", "gelu"])
def test_bmm_autograd_matches_torch(cuda, ft, dev, fp32, act):
    """gradients of a, b and the bias (per entry and shared) against torch's autograd of act(baddbmm) on the same integer
    inputs: bit for bit without an activation and with ReLU (every sum exact), close for GELU (grad_z is not an integer,
    and the products read it as TF32); an expanded operand; the forward bits as in the no-grad call"""
    t = cuda
    g = t.Generator(device="cuda").manual_seed(70)
    Bt, M, K, N = 3, 136, 96, 204
    for per_entry, expand_a in ((True, False), (False, False), (True, True)):
        if expand_a:
            a0 = _t_ints(t, g, (1, M, K)).requires_grad_()
            a = a0.expand(Bt, M, K)
        else:
            a0 = a = _t_ints(t, g, (Bt, M, K)).requires_grad_()
        bmat = _t_ints(t, g, (Bt, K, N)).requires_grad_()
        bias = _t_ints(t, g, (Bt, N) if per_entry else (N,), -20, 21).requires_grad_()
        gy = _t_ints(t, g, (Bt, M, N))
        leaves = (a0, bmat, bias)

        def grads(y):
            for v in leaves:
                v.grad = None
            y.backward(gy)
            return [v.grad.clone() for v in leaves]
        y = dev.bmm(a, bmat, bias=bias, activation=act, alpha=0.5)
        assert y.grad_fn is not None
        got = grads(y)
        with t.no_grad():
            assert _same(t, y, dev.bmm(a, bmat, bias=bias, activation=act, alpha=0.5))
        want_y, _ = _torch_ref(t, a, bmat, bias, act, 0.5)
        want = grads(want_y)
        for name, x, w in zip(("a", "b", "bias"), got, want):
            assert x.shape == w.shape, name
            if act != "gelu":
                assert _same(t, x, w), (name, per_entry, expand_a)
            else:
                err = float((x - w).norm() / w.norm())
                assert err < 3e-3, (name, per_entry, expand_a, err)
    assert dev.stats()["detected"] == 0


@pytest.mark.gpu
def test_bmm_graphed_attention_and_expert_ffn(cuda, ft):
    """make_graphed_callables of softmax(q k^T) v and of gelu(bmm(x, W1^T, bias=b1)), forward and backward: the replays
    equal eager calls bit for bit"""
    t = cuda
    t.cuda.set_device(0)
    g = t.Generator(device="cuda").manual_seed(71)
    dev, ref = ft.FtSgemm(), ft.FtSgemm()

    def attention(d):
        def fn(q, k, v):
            return d.bmm(t.softmax(d.bmm(q, k.transpose(1, 2), alpha=0.125), dim=-1), v)
        return fn

    def expert(d):
        def fn(x, w1, b1):
            return d.bmm(x, w1.transpose(1, 2), bias=b1, activation="gelu")
        return fn
    try:
        cases = [(attention, [(4, 256, 64), (4, 256, 64), (4, 256, 64)], (4, 256, 64)),
                 (expert, [(4, 128, 256), (4, 512, 256), (4, 512)], (4, 128, 512))]
        for make, shapes, out_shape in cases:
            sample = tuple(t.randn(*s, device="cuda", generator=g).requires_grad_() for s in shapes)
            graphed = t.cuda.make_graphed_callables(make(dev), sample)
            eager = make(ref)
            for r in range(2):
                xs = [t.randn(*s, device="cuda", generator=g) for s in shapes]
                gy = t.randn(*out_shape, device="cuda", generator=g)
                xg = [x.clone().requires_grad_() for x in xs]
                xe = [x.clone().requires_grad_() for x in xs]
                y = graphed(*xg)
                y.backward(gy)
                ye = eager(*xe)
                ye.backward(gy)
                t.cuda.synchronize()
                assert _same(t, y, ye), (make.__name__, r)
                for i, (u, v) in enumerate(zip(xg, xe)):
                    assert _same(t, u.grad, v.grad), (make.__name__, r, i)
        assert dev.stats()["detected"] == 0
    finally:
        dev.close()
        ref.close()
