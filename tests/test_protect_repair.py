"""The repairing protected store pass (opts.protect_epilogue = 2).

Level 2 verifies every 32-column chunk of C before it writes it, so a chunk that fails is recomputed from A, B and the old C,
whatever beta is, and it covers tiles that are ragged in N.  Fault-free, it stores exactly what the unprotected kernel
stores.  Integer operands and an integer (or 1/64-grid) old C make every product and sum exact, so a recomputed row equals
the fault-free one bit for bit.  The CPU tests check the option mapping and the NULL-handle answer; the rest run on the GPU.
"""
import ctypes

import numpy as np
import pytest

MN, KM = 0, 1
NONE, ROW, COL = 0, 1, 2
RELU, GELU = 1, 2
SENTINEL = -12345.5
FT_IDS = (11, 12, 13, 14, 15, 16, 31, 32, 40)


# ------------------------------------------------------------------ CPU
def test_make_opts_maps_every_level(ft):
    for value, want in ((False, 0), (True, 1), (0, 0), (1, 1), (2, 2)):
        assert ft.make_opts(protect_epilogue=value).protect_epilogue == want, value


def test_level2_null_handle(ft):
    o = ft.make_opts(protect_epilogue=2)
    rc = ft.lib().ftsgemm_run(None, 31, 128, 128, 128, None, None, None, ctypes.c_float(1.0), ctypes.c_float(0.0),
                              ctypes.byref(o))
    assert rc in (-1, -4), rc


# ------------------------------------------------------------------ GPU helpers
def _ints(rng, shape, lo=-3, hi=4):
    return rng.integers(lo, hi, shape).astype(np.float32)


def _bits_equal(t, a, b):
    """same NaN positions, and the same bits everywhere else"""
    na, nb = t.isnan(a), t.isnan(b)
    if not t.equal(na, nb):
        return False
    return t.equal(a.contiguous().view(t.int32)[~na], b.contiguous().view(t.int32)[~nb])


class _Prod:
    """One product on the GPU: A (M x K), B (N x K), C0 (M x N) as numpy arrays; C and Z come back as M x N tensors."""

    def __init__(self, t, ft, dev, A, B, C0):
        self.t, self.ft, self.dev = t, ft, dev
        self.M, self.K = A.shape
        self.N = B.shape[0]
        self.A, self.B = A, B
        self.C0T = t.from_numpy(np.ascontiguousarray(C0.T)).cuda()
        self._ops = {}

    def op(self, which, layout):
        key = (which, layout)
        if key not in self._ops:
            X = self.A if which == "a" else self.B
            arr = np.ascontiguousarray(X.T if layout == MN else X)  # MN: (r, k) at r + k*rows; KM: at k + r*K
            self._ops[key] = (self.t.from_numpy(arr.reshape(-1)).cuda(), X.shape[0] if layout == MN else self.K)
        return self._ops[key]

    def run(self, kid, level, layout=KM, alpha=1.0, beta=0.0, bias=None, mode=NONE, act=None, z=False, **opt):
        t, M, N = self.t, self.M, self.N
        (dA, lda), (dB, ldb) = self.op("a", layout), self.op("b", layout)
        cbuf = self.C0T.clone()
        zbuf = t.full((N, M), SENTINEL, device="cuda") if z else None
        opts = self.ft.make_opts(protect_epilogue=level, **opt)
        if act is None:
            self.dev.run_bias(kid, M, N, self.K, dA, layout, lda, dB, layout, ldb, cbuf, M, alpha, beta, bias, mode, opts)
        else:
            self.dev.run_act(kid, M, N, self.K, dA, layout, lda, dB, layout, ldb, cbuf, M, alpha, beta, bias, mode, act, zbuf,
                             opts)
        t.cuda.synchronize()
        return cbuf.t(), (zbuf.t() if z else None)

    def bias(self, rng, mode, scale=20.0, integer=False):
        b = scale * rng.standard_normal(self.M if mode == ROW else self.N)
        return self.t.from_numpy((np.round(b) if integer else b).astype(np.float32)).cuda()


@pytest.fixture(scope="module")
def dev(cuda, ft):
    cuda.cuda.set_device(0)
    h = ft.FtSgemm()
    yield h
    h.close()


def _expect_repaired(st, n=1):
    assert st["epilogue_faults"] == n and st["recomputed"] == n and st["uncorrectable"] == 0, st
    assert [e["status"] for e in st["events"]] == [6] * n, st


def _row_where(clean, col, rows, also=None):
    """the first row of `rows` whose clean value at col (and at also[row, col]) is non-zero: an upset there changes the sums"""
    return next(r for r in rows if clean[r, col] != 0 and (also is None or also[r, col] != 0))


# ------------------------------------------------------------------ GPU: arguments
@pytest.mark.gpu
def test_level_arguments(cuda, ft, dev):
    """3 and -1 are INVALID_ARG; 2 is accepted by every entry point"""
    t = cuda
    rng = np.random.default_rng(50)
    M = N = K = 256
    A, B = _ints(rng, (M, K)), _ints(rng, (N, K))
    dA, dB = t.from_numpy(np.ascontiguousarray(A.T)).cuda(), t.from_numpy(np.ascontiguousarray(B.T)).cuda()
    want = t.from_numpy(A @ B.T).cuda()
    for bad in (3, -1):
        o = ft.make_opts(protect_epilogue=bad)
        dC = t.zeros(N, M, device="cuda")
        with pytest.raises(ft.FtsgemmError) as e:
            dev.run_ex(31, M, N, K, dA, MN, M, dB, MN, N, dC, M, 1.0, 0.0, o)
        assert e.value.code == -1
    o = ft.make_opts(protect_epilogue=2)
    dev.stats()
    outs = []
    dC = t.zeros(N, M, device="cuda")
    dev.run(31, M, N, K, dA, dB, dC, 1.0, 0.0, o)
    outs.append(dC)
    dC = t.zeros(N, M, device="cuda")
    dev.run_ex(16, M, N, K, dA, MN, M, dB, MN, N, dC, M, 1.0, 0.0, o)
    outs.append(dC)
    dC = t.zeros(N, M, device="cuda")
    dev.run_bias(31, M, N, K, dA, MN, M, dB, MN, N, dC, M, 1.0, 0.0, t.zeros(M, device="cuda"), ft.BIAS_ROW, o)
    outs.append(dC)
    dC, dZ = t.zeros(N, M, device="cuda"), t.zeros(N, M, device="cuda")
    dev.run_act(31, M, N, K, dA, MN, M, dB, MN, N, dC, M, 1.0, 0.0, None, ft.BIAS_NONE, ft.ACT_RELU, dZ, o)
    outs.append(dZ)
    dC = t.zeros(2, N, M, device="cuda")
    dev.run_batched(31, M, N, K, t.cat([dA, dA]), MN, M, M * K, t.cat([dB, dB]), MN, N, N * K, dC, M, M * N, 2, 1.0, 0.0,
                    None, ft.BIAS_NONE, o)
    outs += [dC[0], dC[1]]
    hC = np.zeros(M * N, np.float32)
    dev.run_host(31, M, N, K, np.ascontiguousarray(A.T).reshape(-1), np.ascontiguousarray(B.T).reshape(-1), hC, 1.0, 0.0,
                 o)
    t.cuda.synchronize()
    outs.append(t.from_numpy(hC.reshape(N, M)).cuda())
    for c in outs:
        assert t.equal(c.t(), want)
    st = dev.stats()
    assert st["detected"] == 0 and st["epilogue_faults"] == 0, st


# ------------------------------------------------------------------ GPU: fault-free
@pytest.mark.gpu
@pytest.mark.parametrize("shape", [(260, 260, 96), (200, 132, 64)])
def test_level2_fault_free_is_level0(cuda, ft, dev, shape):
    """Every fault-tolerant id, both layouts, beta 0 / 1 / -1.5, no / row / column bias, ReLU and GELU with and without Z,
    shapes ragged in M and in N (N = 256 + 4, 128 + 4): level 2 stores C and Z bit for bit as level 0, with no flag."""
    t = cuda
    rng = np.random.default_rng(51)
    M, N, K = shape
    C0 = (np.round(64 * rng.standard_normal((M, N))) / 64).astype(np.float32)
    case = _Prod(t, ft, dev, _ints(rng, (M, K)), _ints(rng, (N, K)), C0)
    biases = {NONE: None, ROW: case.bias(rng, ROW), COL: case.bias(rng, COL)}
    dev.stats()
    for kid in FT_IDS:
        for layout in (MN, KM):
            for beta in (0.0, 1.0, -1.5):
                for mode, b in biases.items():
                    for act, z in ((None, False), (RELU, False), (RELU, True), (GELU, False), (GELU, True)):
                        c0, z0 = case.run(kid, 0, layout, 0.75, beta, b, mode, act, z)
                        c2, z2 = case.run(kid, 2, layout, 0.75, beta, b, mode, act, z)
                        key = (kid, layout, beta, mode, act, z)
                        assert _bits_equal(t, c0, c2), key
                        assert not z or _bits_equal(t, z0, z2), key
        st = dev.stats()
        assert st["detected"] == 0 and st["epilogue_faults"] == 0, (kid, st)


@pytest.mark.gpu
def test_level2_nonfinite_old_c(cuda, ft, dev):
    """Inf / NaN in the old C cannot be verified and are not flagged: level 2 stores what level 0 stores"""
    t = cuda
    rng = np.random.default_rng(52)
    M, N, K = 256, 516, 96
    C0 = _ints(rng, (M, N))
    C0[5, 7], C0[100, 300], C0[9, 9], C0[200, 514] = np.inf, -np.inf, np.nan, np.nan
    case = _Prod(t, ft, dev, _ints(rng, (M, K)), _ints(rng, (N, K)), C0)
    dev.stats()
    for kid in (31, 16, 11):
        for beta in (1.0, -1.5):
            for mode in (NONE, COL):
                b = case.bias(rng, mode) if mode != NONE else None
                for act in (None, GELU):
                    c0, z0 = case.run(kid, 0, KM, 1.0, beta, b, mode, act, act is not None)
                    c2, z2 = case.run(kid, 2, KM, 1.0, beta, b, mode, act, act is not None)
                    assert bool(t.isnan(c2).any()) and _bits_equal(t, c0, c2), (kid, beta, mode, act)
                    assert act is None or _bits_equal(t, z0, z2)
        st = dev.stats()
        assert st["detected"] == 0 and st["epilogue_faults"] == 0, (kid, st)


@pytest.mark.gpu
def test_level2_realistic_deep_k(cuda, ft, dev):
    """normal operands, K = 8192, beta = -1.5: no false alarm from the per-chunk tolerance, C bit for bit level 0's"""
    t = cuda
    g = t.Generator(device="cuda").manual_seed(53)
    M, N, K = 1024, 1024, 8192
    dA = t.randn(K * M, device="cuda", generator=g)
    dB = t.randn(K * N, device="cuda", generator=g)
    C0 = t.randn(N, M, device="cuda", generator=g) * 50
    outs = []
    dev.stats()
    for level in (0, 2):
        dC = C0.clone()
        dev.run(31, M, N, K, dA, dB, dC, 1.0, -1.5, ft.make_opts(protect_epilogue=level))
        outs.append(dC)
    t.cuda.synchronize()
    st = dev.stats()
    assert st["detected"] == 0 and st["epilogue_faults"] == 0, st
    assert _bits_equal(t, outs[0], outs[1])


# ------------------------------------------------------------------ GPU: repair with beta != 0
def _repair_case(t, ft, dev, rng, M=512, N=1000, K=256):
    """id 31 tiles are 256 wide: chunks [0, 4) go to the epilogue warp, [4, 8) to its helper; N = 1000 leaves a last tile
    column [768, 1000) with full chunks and one chunk [992, 1024) that straddles N"""
    return _Prod(t, ft, dev, _ints(rng, (M, K)), _ints(rng, (N, K)), _ints(rng, (M, N), -20, 21))


# (tile column of the fault: first / last column of a chunk, the helper's half, a ragged-N tile's full and straddling chunk)
REPAIR_COLS = (0, 31, 96, 128, 191, 255, 800, 831, 992, 995, 999)


@pytest.mark.gpu
@pytest.mark.parametrize("where", ["epilogue_value", "epilogue_tmem"])
def test_level2_repairs_with_beta(cuda, ft, dev, where):
    t = cuda
    rng = np.random.default_rng(54)
    case = _repair_case(t, ft, dev, rng)
    acc = case.A @ case.B.T
    for beta in (1.0, -1.5):
        want, _ = case.run(31, 0, KM, 1.0, beta)
        wz = want.cpu().numpy()
        for col in REPAIR_COLS:
            r = _row_where(acc, col, range(37, case.M), wz)
            f = [{"row": r, "col": col, "xor": 1 << 27, "where": where}]
            dev.stats()
            c, _ = case.run(31, 2, KM, 1.0, beta, faults=f)
            st = dev.stats()
            _expect_repaired(st)
            assert st["events"][0]["row"] == r
            assert t.equal(c, want), (beta, col)
            # level 1 cannot repair this with beta != 0 (and does not see a ragged-N tile at all)
            c1, _ = case.run(31, 1, KM, 1.0, beta, faults=f)
            st = dev.stats()
            if col < 768:
                assert [e["status"] for e in st["events"]] == [7], (col, st)
            else:
                assert st["epilogue_faults"] == 0, (col, st)


@pytest.mark.gpu
def test_level2_repairs_bias_activation_and_z(cuda, ft, dev):
    t = cuda
    rng = np.random.default_rng(55)
    case = _repair_case(t, ft, dev, rng)
    acc = case.A @ case.B.T
    for mode, act in ((ROW, GELU), (COL, RELU), (NONE, GELU)):
        b = case.bias(rng, mode, 30.0, integer=True) if mode != NONE else None
        for beta in (1.0, -1.5):
            want_c, want_z = case.run(31, 0, KM, 1.0, beta, b, mode, act, True)
            wz = want_z.cpu().numpy()
            for col, where in ((5, "epilogue_value"), (200, "epilogue_tmem"), (995, "epilogue_value"), (800, "epilogue_tmem")):
                r = _row_where(acc, col, range(60, case.M), wz)
                f = [{"row": r, "col": col, "xor": 1 << 27, "where": where}]
                dev.stats()
                c, z = case.run(31, 2, KM, 1.0, beta, b, mode, act, True, faults=f)
                _expect_repaired(dev.stats())
                assert t.equal(c, want_c) and t.equal(z, want_z), (mode, act, beta, col, where)


# ------------------------------------------------------------------ GPU: other paths
@pytest.mark.gpu
def test_level2_batched(cuda, ft, dev):
    """an upset in entry 2 of a strided batch: repaired, and the event carries the stacked row 2*M + r"""
    t = cuda
    rng = np.random.default_rng(56)
    Bt, M, N, K = 3, 256, 516, 128
    A, B = _ints(rng, (Bt, M, K)), _ints(rng, (Bt, N, K))
    C0 = _ints(rng, (Bt, N, M), -20, 21)  # entry i: C[m + n*M]
    dA, dB = t.from_numpy(A).cuda(), t.from_numpy(B).cuda()

    def run(level, faults=None):
        dC = t.from_numpy(C0).cuda()
        dev.run_batched(31, M, N, K, dA, KM, K, M * K, dB, KM, K, N * K, dC, M, M * N, Bt, 1.0, -1.5, None, ft.BIAS_NONE,
                        ft.make_opts(protect_epilogue=level, faults=faults))
        t.cuda.synchronize()
        return dC

    want = run(0)
    acc2 = A[2] @ B[2].T
    for col, where in ((40, "epilogue_value"), (300, "epilogue_tmem"), (514, "epilogue_value")):
        r = _row_where(acc2, col, range(9, M), (C0[2].T * -1.5 + acc2))
        dev.stats()
        got = run(2, [{"row": 2 * M + r, "col": col, "xor": 1 << 27, "where": where}])
        st = dev.stats()
        _expect_repaired(st)
        assert st["events"][0]["row"] == 2 * M + r
        assert t.equal(got, want), (col, where)


@pytest.mark.gpu
def test_level2_3xtf32_repairs_main_product(cuda, ft, dev):
    """3xTF32 runs its main product with beta = 1 even when the caller passes 0: level 1 reports the upset (7), level 2
    repairs it"""
    t = cuda
    rng = np.random.default_rng(57)
    case = _repair_case(t, ft, dev, rng, N=1024)
    acc = case.A @ case.B.T
    want, _ = case.run(31, 0, KM, 1.0, 0.0, precision=1)
    r = _row_where(acc, 70, range(30, case.M))
    f = [{"row": r, "col": 70, "xor": 1 << 27, "where": "epilogue_value"}]
    dev.stats()
    case.run(31, 1, KM, 1.0, 0.0, precision=1, faults=f)
    assert [e["status"] for e in dev.stats()["events"]] == [7]
    c, _ = case.run(31, 2, KM, 1.0, 0.0, precision=1, faults=f)
    _expect_repaired(dev.stats())
    assert t.equal(c, want)


@pytest.mark.gpu
def test_level2_check_segments(cuda, ft, dev):
    t = cuda
    rng = np.random.default_rng(58)
    case = _repair_case(t, ft, dev, rng, N=1000, K=256)
    acc = case.A @ case.B.T
    acc = case.A[:, :64] @ case.B[:, :64].T  # faults go to the first of the four segments, k in [0, 64)
    want, _ = case.run(31, 0, KM, 1.0, 1.0, check_segments=4)
    for col in (70, 993):
        r = _row_where(acc, col, range(30, case.M))
        dev.stats()
        c, _ = case.run(31, 2, KM, 1.0, 1.0, check_segments=4,
                        faults=[{"row": r, "col": col, "xor": 1 << 27, "where": "epilogue_tmem"}])
        _expect_repaired(dev.stats())
        assert t.equal(c, want), col


@pytest.mark.gpu
def test_level2_graph_replay_repairs(cuda, ft, dev):
    t = cuda
    rng = np.random.default_rng(59)
    M, N, K = 512, 1000, 256
    A, B, C0 = _ints(rng, (M, K)), _ints(rng, (N, K)), _ints(rng, (N, M), -20, 21)
    dA, dB = t.from_numpy(A).cuda(), t.from_numpy(B).cuda()
    dC = t.from_numpy(C0).cuda()
    ref = dC.clone()
    dev.run_ex(31, M, N, K, dA, KM, K, dB, KM, K, ref, M, 1.0, -1.5, ft.make_opts())
    acc = A @ B.T
    r = _row_where(acc, 997, range(3, M), acc - 1.5 * C0.T)
    f = [{"row": r, "col": 997, "xor": 1 << 27, "where": "epilogue_value"}]
    t.cuda.synchronize()
    dev.stats()
    g = t.cuda.CUDAGraph()
    with t.cuda.graph(g):
        dev.run_ex(31, M, N, K, dA, KM, K, dB, KM, K, dC, M, 1.0, -1.5,
                   ft.make_opts(stream=t.cuda.current_stream().cuda_stream, faults=f, protect_epilogue=2))
    for _ in range(2):
        dC.copy_(t.from_numpy(C0).cuda())
        t.cuda.synchronize()
        dev.stats()
        g.replay()
        t.cuda.synchronize()
        _expect_repaired(dev.stats())
        assert t.equal(dC, ref)


@pytest.mark.gpu
def test_level2_linear_ragged_tokens(cuda, ft, dev):
    """FtSgemm.linear runs y^T = W x^T: the kernel's N is the token count, and 1000 tokens leave a ragged last tile column"""
    t = cuda
    rng = np.random.default_rng(60)
    T, K, O = 1000, 256, 512
    x = t.from_numpy(_ints(rng, (T, K))).cuda()
    W = t.from_numpy(_ints(rng, (O, K))).cuda()
    b = t.from_numpy(_ints(rng, (O,), -50, 51)).cuda()
    with t.no_grad():
        want = dev.linear(x, W, b)
        acc = (x @ W.t()).cpu().numpy()  # integers: exact in any order
        tok = 996
        feat = next(o for o in range(100, O) if acc[tok, o] != 0 and acc[tok, o] + b[o].item() != 0)
        for where in ("epilogue_value", "epilogue_tmem"):
            t.cuda.synchronize()
            dev.stats()
            f = [{"row": feat, "col": tok, "xor": 1 << 27, "where": where}]
            y = dev.linear(x, W, b, opts=ft.make_opts(faults=f, protect_epilogue=2))
            t.cuda.synchronize()
            _expect_repaired(dev.stats())
            assert t.equal(y, want), where


# ------------------------------------------------------------------ GPU: several upsets, no_recompute
@pytest.mark.gpu
def test_level2_several_upsets_and_no_recompute(cuda, ft, dev):
    t = cuda
    rng = np.random.default_rng(61)
    case = _repair_case(t, ft, dev, rng)
    acc = case.A @ case.B.T
    want, _ = case.run(31, 0, KM, 1.0, -1.5)
    wz = want.cpu().numpy()
    # two upsets in different chunks of one row (one row segment: one count), and two more rows of the same warp, one of
    # them in the helper's half and the ragged tile
    r0 = next(r for r in range(64, 96) if all(acc[r, c] != 0 and wz[r, c] != 0 for c in (5, 70)))
    r1 = next(r for r in range(64, 96) if r != r0 and acc[r, 200] != 0 and wz[r, 200] != 0)
    r2 = next(r for r in range(64, 96) if r not in (r0, r1) and acc[r, 996] != 0 and wz[r, 996] != 0)
    for where in ("epilogue_value", "epilogue_tmem"):
        f = [{"row": r0, "col": 5, "xor": 1 << 27, "where": where}, {"row": r0, "col": 70, "xor": 1 << 30, "where": where},
             {"row": r1, "col": 200, "xor": 1 << 26, "where": where}, {"row": r2, "col": 996, "xor": 1 << 31, "where": where}]
        dev.stats()
        c, _ = case.run(31, 2, KM, 1.0, -1.5, faults=f)
        st = dev.stats()
        _expect_repaired(st, 3)
        assert sorted(e["row"] for e in st["events"]) == sorted([r0, r1, r2])
        assert t.equal(c, want), where
    # two chunks of one row segment in the ragged tile as well
    r3 = next(r for r in range(64, 96) if all(acc[r, c] != 0 and wz[r, c] != 0 for c in (780, 830)))
    f = [{"row": r3, "col": 780, "xor": 1 << 27, "where": "epilogue_value"},
         {"row": r3, "col": 830, "xor": 1 << 22, "where": "epilogue_value"}]
    dev.stats()
    c, _ = case.run(31, 2, KM, 1.0, -1.5, faults=f)
    _expect_repaired(dev.stats())
    assert t.equal(c, want)
    # no_recompute / detect_only: the chunk is stored as computed and reported
    mask = 1 << 27
    for opt in (dict(no_recompute=True), dict(detect_only=True)):
        for col in (70, 996):
            r = _row_where(acc, col, range(40, case.M), wz)
            dev.stats()
            c, _ = case.run(31, 2, KM, 1.0, -1.5, faults=[{"row": r, "col": col, "xor": mask, "where": "epilogue_value"}],
                            **opt)
            st = dev.stats()
            assert st["epilogue_faults"] == 1 and st["uncorrectable"] == 1 and st["recomputed"] == 0, st
            assert [e["status"] for e in st["events"]] == [7]
            diff = (c != want).nonzero().tolist()
            assert diff == [[r, col]], diff
            got_bits = int(c[r, col:col + 1].view(t.int32).item()) & 0xFFFFFFFF
            want_bits = int(want[r, col:col + 1].view(t.int32).item()) & 0xFFFFFFFF
            assert got_bits == want_bits ^ mask


# ------------------------------------------------------------------ GPU: mini campaign
@pytest.mark.gpu
def test_level2_campaign(cuda, ft, dev):
    """id 31 at 4096^3 with beta = -1.5: random single-bit flips of the value about to be stored, at most one per row and
    tile.  Every detected flip is repaired; a flip of bit >= 22 at an element whose |z| is at least 5 % of its chunk's mean
    |z| is always detected (below that the chunk's tolerance can hide it, as at level 1); the error left is <= 1e-4 max|C|."""
    t = cuda
    n, kid = 4096, 31
    g = t.Generator(device="cuda").manual_seed(62)

    def operand():
        return (t.randint(0, 10, (n * n,), generator=g, device="cuda").float() * 0.1) * \
            (t.randint(0, 2, (n * n,), generator=g, device="cuda").float() * 2 - 1)
    dA, dB = operand(), operand()
    C0 = t.randn(n * n, device="cuda", generator=g)
    clean = C0.clone()
    dev.stats()
    dev.run(kid, n, n, n, dA, dB, clean, 1.0, -1.5, None)
    t.cuda.synchronize()
    assert dev.stats()["detected"] == 0
    z = clean.view(n, n).t().contiguous()  # z[m, nn]
    zabs = z.abs().view(n, n // 32, 32)
    chunk_mean = zabs.mean(dim=2).cpu().numpy()
    zc = z.cpu().numpy()
    scale = float(clean.abs().max())
    rng = np.random.default_rng(0)
    dC = t.empty_like(clean)
    worst = 0.0
    for bit in (31, 30, 27, 25, 23, 22, 21, 19, 17, 14):
        for _ in range(2):
            faults, rows = [], set()
            while len(faults) < ft.MAX_FAULTS:
                r, c = int(rng.integers(n)), int(rng.integers(n))
                if r in rows:  # (one per row: each event names its fault)
                    continue
                rows.add(r)
                faults.append({"row": r, "col": c, "xor": 1 << bit, "where": "epilogue_value"})
            dC.copy_(C0)
            dev.run(kid, n, n, n, dA, dB, dC, 1.0, -1.5, ft.make_opts(faults=faults, protect_epilogue=2))
            t.cuda.synchronize()
            st = dev.stats()
            assert st["uncorrectable"] == 0 and st["recomputed"] == st["epilogue_faults"], (bit, st)
            assert all(e["status"] == 6 for e in st["events"]), st
            seen = {e["row"] for e in st["events"]}
            assert len(seen) == st["epilogue_faults"] <= len(faults)
            for f in faults:
                r, c = f["row"], f["col"]
                if bit >= 22 and abs(zc[r, c]) >= 0.05 * chunk_mean[r, c // 32]:
                    assert r in seen, (bit, f, float(zc[r, c]), float(chunk_mean[r, c // 32]))
            worst = max(worst, float((dC - clean).abs().max()))
    assert worst <= 1e-4 * scale, (worst, scale)
