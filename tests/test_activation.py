"""Activation fused into the store pass (ftsgemm_run_act, FtSgemm.run_act / matmul(activation=) / linear(activation=)).

z = (alpha * A * B^T + beta * C) + bias is bit for bit what run_bias stores; the call stores C = act(z) and, when asked, z
into Z.  ReLU is torch.relu's clamp_min, so C must equal torch.relu(Z) bit for bit.  GELU is torch's exact erf form; it goes
through the device's erff, so C is held to within GELU_ULP ulp of F.gelu(Z) (the maximum measured is printed).  The ABFT
check runs on the accumulator, and the protected store pass verifies z before the activation: every repair restores C and Z.
Integer operands make every product and sum exact, so C and Z of a repaired run equal the fault-free ones bit for bit.
The CPU tests check the ABI's NULL-handle answer and the constants; the rest run on the GPU.
"""
import numpy as np
import pytest

MN, KM = 0, 1
NONE, ROW, COL = 0, 1, 2
RELU, GELU = 1, 2
NAMES = ["small", "medium", "large", "tall", "wide", "huge", "giant", "pair128"]
GELU_ULP = 2
SENTINEL = -12345.5
Z_SENTINEL = 7777.25


# ------------------------------------------------------------------ CPU
def test_run_act_null_handle(ft):
    assert ft.lib().ftsgemm_run_act(None, 16, 128, 128, 128, None, 0, 128, None, 0, 128, None, 128, 1.0, 0.0, None, 0, 1,
                                    None, None) == -4


def test_activation_constants_mirror_the_header(ft):
    assert (ft.ACT_NONE, ft.ACT_RELU, ft.ACT_GELU) == (0, 1, 2)
    assert ft.ACTIVATIONS == {None: 0, "relu": 1, "gelu": 2}
    header = (ft.HERE.parent / "include" / "ftsgemm.h").read_text()
    for name, value in (("NONE", 0), ("RELU", 1), ("GELU", 2)):
        assert f"FTSGEMM_ACT_{name} = {value}" in header
    assert "int ftsgemm_run_act(" in header and "ftsgemm_run_act" in ft.EXPORTED_SYMBOLS


# ------------------------------------------------------------------ GPU helpers
def _ints(rng, shape, lo=-3, hi=4):
    return rng.integers(lo, hi, shape).astype(np.float32)


def _pack(t, X, layout, ld):
    """rows x K matrix X -> flat device buffer in the layout (MN: X[r, k] at r + k*ld; KM: at k + r*ld), padding = NaN"""
    rows, K = X.shape
    if layout == MN:
        buf = np.full((K, ld), np.nan, np.float32)
        buf[:, :rows] = X.T
    else:
        buf = np.full((rows, ld), np.nan, np.float32)
        buf[:, :K] = X
    return t.from_numpy(buf.reshape(-1)).cuda()


def _ld(layout, rows, K, pad=True):
    if not pad:
        return rows if layout == MN else K
    return rows + 4 if layout == MN else (K + 3) // 4 * 4 + 4


def _ulp(a, b):
    """elementwise ulp distance of two float32 tensors (finite or equal non-finite elements)"""
    import torch

    def key(x):
        i = x.contiguous().view(torch.int32).long()
        return torch.where(i < 0, -(i & 0x7FFFFFFF), i)
    return (key(a) - key(b)).abs()


def _act_ref(t, Z, act):
    return t.relu(Z) if act == RELU else t.nn.functional.gelu(Z)


def _check_act(t, C, Z, act):
    """C = act(Z): bit for bit for ReLU, within GELU_ULP for GELU (same NaN positions, same Inf signs); returns the max ulp"""
    ref = _act_ref(t, Z, act)
    assert t.equal(t.isnan(C), t.isnan(ref))
    fin = t.isfinite(ref)
    assert t.equal(fin, t.isfinite(C))
    inf = t.isinf(ref)
    assert t.equal(C[inf], ref[inf])
    if act == RELU:
        assert t.equal(C.view(t.int32)[fin], ref.view(t.int32)[fin])
        return 0
    d = int(_ulp(C[fin], ref[fin]).max()) if bool(fin.any()) else 0
    assert d <= GELU_ULP, d
    return d


class _Case:
    """One product on the GPU: A (M x K), B (N x K), C0 (M x N) as numpy arrays, operands uploaded once per layout."""

    def __init__(self, t, dev, A, B, C0):
        self.t, self.dev, self.A, self.B = t, dev, A, B
        self.M, self.K = A.shape
        self.N = B.shape[0]
        self.C0T = t.from_numpy(np.ascontiguousarray(C0.T)).cuda()
        self._ops = {}

    def op(self, which, layout, ld):
        key = (which, layout, ld)
        if key not in self._ops:
            self._ops[key] = _pack(self.t, self.A if which == "a" else self.B, layout, ld)
        return self._ops[key]

    def run(self, kid, la=KM, lda=None, lb=KM, ldb=None, ldc=None, alpha=1.0, beta=0.0, bias=None, mode=NONE, act=None,
            z=False, opts=None):
        """run_bias (act None) or run_act: (C, Z) as M x N device tensors (Z None unless z), the padding of both checked"""
        t, M, N = self.t, self.M, self.N
        lda = lda or _ld(la, M, self.K, False)
        ldb = ldb or _ld(lb, N, self.K, False)
        ldc = ldc or M
        dA, dB = self.op("a", la, lda), self.op("b", lb, ldb)
        cbuf = t.full((N, ldc), SENTINEL, device="cuda")
        cbuf[:, :M] = self.C0T
        zbuf = t.full((N, ldc), Z_SENTINEL, device="cuda") if z else None
        if act is None:
            self.dev.run_bias(kid, M, N, self.K, dA, la, lda, dB, lb, ldb, cbuf, ldc, alpha, beta, bias, mode, opts)
        else:
            self.dev.run_act(kid, M, N, self.K, dA, la, lda, dB, lb, ldb, cbuf, ldc, alpha, beta, bias, mode, act, zbuf, opts)
        t.cuda.synchronize()
        assert bool((cbuf[:, M:] == SENTINEL).all()), "C's padding was written"
        if z:
            assert bool((zbuf[:, M:] == Z_SENTINEL).all()), "Z's padding was written"
        return cbuf[:, :M].t(), (zbuf[:, :M].t() if z else None)

    def bias(self, rng, mode, scale=1.0, integer=False):
        b = scale * rng.standard_normal(self.M if mode == ROW else self.N)
        return self.t.from_numpy((np.round(b) if integer else b).astype(np.float32)).cuda()

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


# ------------------------------------------------------------------ GPU: correctness
@pytest.mark.gpu
@pytest.mark.parametrize("shape", [(260, 388, 201), (256, 512, 128)])
def test_act_matches_run_bias_then_torch(cuda, ft, dev, shape):
    """Every named variant, plain and fault-tolerant, cut tiles off and forced, all four layout pairs with padded leading
    dimensions and ldc = M + 8, beta 0 and -1.5, no / row / column bias, ReLU and GELU, with and without Z: Z = run_bias's C
    and C = act(Z) (see _check_act), C the same across variants, layouts and splitk, padding untouched."""
    t = cuda
    rng = np.random.default_rng(41)
    M, N, K = shape
    # integer operands and an old C on a 1/64 grid: alpha * acc + beta * C_old is exact, whatever the variant, tile edge or
    # contraction, so C may be compared across variants (the bias add is the one rounding)
    C0 = (np.round(64 * rng.standard_normal((M, N))) / 64).astype(np.float32)
    case = _Case(t, dev, _ints(rng, (M, K)), _ints(rng, (N, K)), C0)
    biases = {NONE: None, ROW: case.bias(rng, ROW, 20.0), COL: case.bias(rng, COL, 20.0)}
    first = {}
    worst = 0
    try:
        for splitk in (0, 2):
            ft.debug_set("splitk", splitk)
            for name in NAMES:
                for kid in (ft.SGEMM_IDS[name], ft.ABFT_IDS[name]):
                    dev.stats()
                    for la, lda, lb, ldb in case.layouts():
                        for beta in (0.0, -1.5):
                            for mode, b in biases.items():
                                ref, _ = case.run(kid, la, lda, lb, ldb, M + 8, 0.75, beta, b, mode)
                                for act in (RELU, GELU):
                                    c, z = case.run(kid, la, lda, lb, ldb, M + 8, 0.75, beta, b, mode, act, True)
                                    assert t.equal(z, ref), (kid, la, lb, beta, mode, act)
                                    worst = max(worst, _check_act(t, c, z, act))
                                    c2, _ = case.run(kid, la, lda, lb, ldb, M + 8, 0.75, beta, b, mode, act, False)
                                    assert t.equal(c, c2), (kid, la, lb, beta, mode, act)
                                    key = (beta, mode, act)
                                    first.setdefault(key, c.clone())
                                    assert t.equal(first[key], c), (kid, splitk, la, lb, key)
                    if kid >= 10:
                        assert dev.stats()["detected"] == 0, kid
    finally:
        ft.debug_set("splitk", -1)
    print(f"max GELU ulp against F.gelu(Z), shape {shape}: {worst}")


def _segment_case(t, dev, rng):
    """a ReLU case where z > 0 at the end but the partial sum after the first and second of three K-segments is < 0: an
    activation applied per segment or per 3xTF32 pass would store something else"""
    M, N, K = 256, 384, 192  # 6 k-blocks: segments [0, 64), [64, 128), [128, 192)
    A = _ints(rng, (M, K), 1, 4)
    A[:, :64], A[:, 128:] = 1.0, 3.0
    B = _ints(rng, (N, K))
    B[::2, :64], B[::2, 128:] = -3.0, 3.0
    p1 = A[:, :64] @ B[:, :64].T
    p2 = p1 + A[:, 64:128] @ B[:, 64:128].T
    full = A @ B.T
    assert int(((p1 < 0) & (p2 < 0) & (full > 0)).sum()) >= M * N // 4
    return _Case(t, dev, A, B, rng.standard_normal((M, N)).astype(np.float32))


@pytest.mark.gpu
def test_act_applied_once_with_3xtf32_and_segments(cuda, ft, dev):
    t = cuda
    rng = np.random.default_rng(42)
    case = _segment_case(t, dev, rng)
    for kid in (31, 16):
        for opts in (dict(check_segments=3), dict(precision=1), dict(check_segments=3, precision=1)):
            dev.stats()
            for la, lb in ((MN, MN), (KM, KM)):
                for beta in (0.0, -1.5):
                    for mode in (NONE, ROW, COL):
                        b = case.bias(rng, mode, 10.0) if mode != NONE else None
                        ref, _ = case.run(kid, la, None, lb, None, case.M + 8, 0.75, beta, b, mode, opts=ft.make_opts(**opts))
                        for act in (RELU, GELU):
                            c, z = case.run(kid, la, None, lb, None, case.M + 8, 0.75, beta, b, mode, act, True,
                                            ft.make_opts(**opts))
                            assert t.equal(z, ref), (kid, opts, la, beta, mode, act)
                            _check_act(t, c, z, act)
            assert dev.stats()["detected"] == 0


@pytest.mark.gpu
def test_act_nonfinite(cuda, ft, dev):
    """Inf / NaN in A, B, the bias and the old C: C has the NaN positions and Inf signs of torch's relu / gelu of Z, and Z is
    run_bias's C (same NaN positions, equal elsewhere)."""
    t = cuda
    rng = np.random.default_rng(43)
    M, N, K = 256, 384, 96
    A, B = _ints(rng, (M, K)), _ints(rng, (N, K))
    A[3, 5], A[70, 9], B[11, 2], B[200, 40] = np.inf, -np.inf, np.nan, np.inf
    C0 = rng.standard_normal((M, N)).astype(np.float32)
    C0[5, 7], C0[100, 300], C0[9, 9] = np.inf, -np.inf, np.nan
    case = _Case(t, dev, A, B, C0)
    for mode in (ROW, COL):
        b = case.bias(rng, mode, 5.0)
        b[1], b[17] = float("inf"), float("nan")
        for kid in (21, 31, 11):
            for beta in (0.0, -1.5):
                dev.stats()
                ref, _ = case.run(kid, MN, None, KM, None, None, 1.0, beta, b, mode)
                for act in (RELU, GELU):
                    c, z = case.run(kid, MN, None, KM, None, None, 1.0, beta, b, mode, act, True)
                    assert t.equal(t.isnan(z), t.isnan(ref)) and t.equal(z[~t.isnan(ref)], ref[~t.isnan(ref)])
                    assert bool(t.isinf(z).any()) and bool(t.isnan(z).any())
                    _check_act(t, c, z, act)
                assert dev.stats()["detected"] == 0, (kid, beta, mode)


# ------------------------------------------------------------------ GPU: fault tolerance
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


@pytest.mark.gpu
def test_abft_with_activation(cuda, ft, dev):
    t = cuda
    rng = np.random.default_rng(44)
    M, N, K = 512, 1024, 1024
    kid = 31
    case = _Case(t, dev, _ints(rng, (M, K)), _ints(rng, (N, K)), _ints(rng, (M, N)))
    clean = case.run(kid)[0].cpu().numpy()
    for mode in (ROW, COL):
        b = case.bias(rng, mode, 50.0, integer=True)
        for act in (RELU, GELU):
            dev.stats()
            want_c, want_z = case.run(kid, bias=b, mode=mode, act=act, z=True)
            assert dev.stats()["detected"] == 0
            # accumulator upsets (mode 1: exponent, sign and top mantissa bits; mode 0: added values): corrected
            faults = _faults_per_tile(clean, rng, [22, 25, 30, 31], 256, 64.0)
            r0 = next(r for r in range(300, M) if all(f["row"] not in (r, r + 1) for f in faults))
            faults += [{"row": r0, "col": 900, "add": 1e4}, {"row": r0 + 1, "col": 100, "add": -512.0}]
            c, z = case.run(kid, bias=b, mode=mode, act=act, z=True, opts=ft.make_opts(faults=faults))
            st = dev.stats()
            assert st["detected"] == 6 == st["corrected"], st
            assert t.equal(c, want_c) and t.equal(z, want_z), (mode, act)
            # two upsets in one row that the two checksums cannot place (d2 / d1 = -4): the row is recomputed
            two = [{"row": 40, "col": 10, "add": 100.0}, {"row": 40, "col": 25, "add": -50.0}]
            for la in (KM, MN):
                c, z = case.run(kid, la, bias=b, mode=mode, act=act, z=True, opts=ft.make_opts(faults=two))
                st = dev.stats()
                assert st["detected"] == 1 and st["recomputed"] == 1 and st["uncorrectable"] == 0, (la, st)
                assert t.equal(c, want_c) and t.equal(z, want_z), (mode, act, la)


@pytest.mark.gpu
def test_protect_epilogue_with_activation(cuda, ft, dev):
    t = cuda
    rng = np.random.default_rng(45)
    M, N, K = 512, 1024, 1024
    kid = 31
    case = _Case(t, dev, _ints(rng, (M, K)), _ints(rng, (N, K)), _ints(rng, (M, N)))
    clean = case.run(kid)[0].cpu().numpy()
    scale = float(np.abs(clean).max())
    prot = dict(protect_epilogue=True)
    for mode in (ROW, COL):
        for act in (RELU, GELU):
            # fault-free, with a bias 1e3 x the product's magnitude: no alarm, C and Z those of the unprotected kernel
            big = case.bias(rng, mode, 1e3 * scale)
            want_c, want_z = case.run(kid, bias=big, mode=mode, act=act, z=True)
            dev.stats()
            c, z = case.run(kid, bias=big, mode=mode, act=act, z=True, opts=ft.make_opts(**prot))
            st = dev.stats()
            assert st["epilogue_faults"] == 0 and st["detected"] == 0, st
            assert t.equal(c, want_c) and t.equal(z, want_z)
            # upsets after the check with beta = 0 (mode 3 hits z): detected, recomputed, C and Z restored
            b = case.bias(rng, mode, 50.0, integer=True)
            want_c, want_z = case.run(kid, bias=b, mode=mode, act=act, z=True)
            wz = want_z.cpu().numpy()
            col = next(c for c in range(5, N) if clean[37, c] != 0 and wz[37, c] != 0)
            for where in ("epilogue_value", "epilogue_tmem"):
                f = [{"row": 37, "col": col, "xor": 1 << 27, "where": where}]
                for z_out in (True, False):
                    c, z = case.run(kid, KM, None, MN, None, None, 1.0, 0.0, b, mode, act, z_out,
                                    ft.make_opts(faults=f, **prot))
                    st = dev.stats()
                    assert st["epilogue_faults"] == 1 and st["recomputed"] == 1 and st["uncorrectable"] == 0, (where, st)
                    assert t.equal(c, want_c), (where, mode, act)
                    assert not z_out or t.equal(z, want_z), (where, mode, act)
            # beta != 0: the old values are gone, the row segment is reported (status 7)
            f = [{"row": 37, "col": col, "xor": 1 << 27, "where": "epilogue_value"}]
            case.run(kid, KM, None, KM, None, None, 1.0, -1.5, b, mode, act, True, ft.make_opts(faults=f, **prot))
            st = dev.stats()
            assert st["epilogue_faults"] == 1 and st["uncorrectable"] == 1 and st["recomputed"] == 0, st
            assert [e["status"] for e in st["events"]] == [7]


# ------------------------------------------------------------------ GPU: the torch layer
@pytest.mark.gpu
@pytest.mark.parametrize("act", ["relu", "gelu"])
def test_linear_activation_equals_unfused_chain(cuda, ft, dev, act):
    """forward = F.act(ft.linear(...)) (ReLU bit for bit, GELU within GELU_ULP) and grad_x, grad_W, grad_b bit-identical to
    the unfused chain through the same library"""
    t = cuda
    F = t.nn.functional
    fn = F.relu if act == "relu" else F.gelu
    g = t.Generator(device="cuda").manual_seed(46)
    K, N = 520, 392
    for shape, with_bias in (((300, K), True), ((3, 100, K), True), ((256, K), False)):
        x = t.randn(*shape, device="cuda", generator=g, requires_grad=True)
        W = t.randn(N, K, device="cuda", generator=g, requires_grad=True)
        b = t.randn(N, device="cuda", generator=g, requires_grad=True) if with_bias else None
        gy = t.randn(*shape[:-1], N, device="cuda", generator=g)
        leaves = [v for v in (x, W, b) if v is not None]

        def grads(y):
            for v in leaves:
                v.grad = None
            y.backward(gy)
            return [v.grad.clone() for v in leaves]
        y_unf = fn(dev.linear(x, W, b))
        g_unf = grads(y_unf)
        y = dev.linear(x, W, b, activation=act)
        g_fused = grads(y)
        assert y.shape == y_unf.shape
        if act == "relu":
            assert t.equal(y, y_unf)
        else:
            _check_act(t, y.detach(), dev.linear(x, W, b).detach(), GELU)
        for a, c in zip(g_fused, g_unf):
            assert t.equal(a, c), (shape, with_bias)
        assert dev.stats()["detected"] == 0


@pytest.mark.gpu
def test_linear_activation_no_grad_is_one_launch_and_y_only(cuda, ft, dev):
    t = cuda
    g = t.Generator(device="cuda").manual_seed(47)
    M, K, N = 2048, 2048, 1024  # kernel B = x: 16 MB, so the encode runs in the kernel's front phase
    x = t.randn(M, K, device="cuda", generator=g)
    W = t.randn(N, K, device="cuda", generator=g)
    b = t.randn(N, device="cuda", generator=g)
    with t.no_grad():
        for act in ("relu", "gelu"):
            dev.linear(x, W, b, activation=act)  # warm-up: workspace, plans
            t.cuda.synchronize()
            t.cuda.reset_peak_memory_stats()
            base = t.cuda.memory_allocated()
            n0 = dev.launch_count()
            y = dev.linear(x, W, b, activation=act)
            assert dev.launch_count() - n0 == 1
            t.cuda.synchronize()
            assert t.cuda.max_memory_allocated() - base <= y.numel() * 4, act
            del y
    # with grad: GELU keeps z for its backward, ReLU does not
    xr = x.clone().requires_grad_()
    for act, extra in (("relu", 0), ("gelu", 1)):
        dev.linear(xr, W, b, activation=act)
        t.cuda.synchronize()
        t.cuda.reset_peak_memory_stats()
        base = t.cuda.memory_allocated()
        y = dev.linear(xr, W, b, activation=act)
        t.cuda.synchronize()
        assert t.cuda.max_memory_allocated() - base <= (1 + extra) * y.numel() * 4, act
        del y
    assert dev.stats()["detected"] == 0


@pytest.mark.gpu
@pytest.mark.parametrize("act", ["relu", "gelu"])
def test_linear_activation_mlp_graph_replay(cuda, ft, act):
    t = cuda
    t.cuda.set_device(0)
    dev = ft.FtSgemm()
    try:
        g = t.Generator(device="cuda").manual_seed(48)
        dims = [256, 1024, 512, 768, 384]
        ws = [t.randn(dims[i + 1], dims[i], device="cuda", generator=g) * dims[i] ** -0.5 for i in range(4)]
        bs = [t.randn(dims[i + 1], device="cuda", generator=g) for i in range(4)]
        x = t.zeros(128, dims[0], device="cuda")
        outs = []

        def stack(h, out):
            out.clear()
            for w, b in zip(ws, bs):
                h = dev.linear(h, w, b, activation=act)
                out.append(h)

        stack(x, outs)  # eager warm-up of every shape
        graph = t.cuda.CUDAGraph()
        with t.cuda.graph(graph):
            stack(x, outs)
        for r in range(2):
            x.copy_(t.randn(*x.shape, device="cuda", generator=g))
            want = []
            stack(x.clone(), want)
            graph.replay()
            t.cuda.synchronize()
            for i, (a, b) in enumerate(zip(outs, want)):
                assert t.equal(a, b), (r, i)
        assert dev.stats()["detected"] == 0
    finally:
        dev.close()


@pytest.mark.gpu
def test_matmul_activation_mapping_and_preact(cuda, ft, dev):
    """matmul(activation=, preact=) on column- and row-major out (swapped): out = act(preact), preact = matmul(bias=)"""
    t = cuda
    g = t.Generator(device="cuda").manual_seed(49)
    M, K, N = 192, 136, 320
    a = t.randn(M, K, device="cuda", generator=g)
    bmat = t.randn(K, N, device="cuda", generator=g)
    bias = t.randn(N, device="cuda", generator=g)
    for out_rm in (True, False):
        def fresh():
            return t.empty(M, N, device="cuda") if out_rm else t.empty(N, M, device="cuda").t()
        ref = dev.matmul(a, bmat, fresh(), bias=bias)
        for act in ("relu", "gelu"):
            out, z = fresh(), fresh()
            dev.matmul(a, bmat, out, bias=bias, activation=act, preact=z)
            assert t.equal(z, ref)
            _check_act(t, out, z, RELU if act == "relu" else GELU)
            out2 = dev.matmul(a, bmat, fresh(), bias=bias, activation=act)
            assert t.equal(out2, out)
    # preact with other strides than out, out that cannot be written in place, preact without an activation: ValueError
    out = t.empty(M, N, device="cuda")
    with pytest.raises(ValueError):
        dev.matmul(a, bmat, out, activation="relu", preact=t.empty(N, M, device="cuda").t())
    with pytest.raises(ValueError):
        dev.matmul(a, bmat, t.empty(M, 2 * N, device="cuda")[:, ::2], activation="relu")
    with pytest.raises(ValueError):
        dev.matmul(a, bmat, out, preact=t.empty(M, N, device="cuda"))
    with pytest.raises(ValueError):
        dev.matmul(a, bmat, out, activation="tanh")
    with pytest.raises(ValueError):
        dev.linear(a, bmat.t(), activation="silu")


# ------------------------------------------------------------------ GPU: argument checks
@pytest.mark.gpu
def test_run_act_argument_checks(cuda, ft, dev):
    t = cuda
    M, N, K = 256, 256, 128
    dA, dB, dC, dZ = (t.zeros(M * N + 16, device="cuda") for _ in range(4))  # (room for a Z offset by one float)

    def code(kid=31, act=RELU, z=dZ.data_ptr(), c=dC.data_ptr()):
        try:
            dev.run_act(kid, M, N, K, dA, MN, M, dB, MN, N, c, M, 1.0, 0.0, None, NONE, act, z)
            t.cuda.synchronize()
            return 0
        except ft.FtsgemmError as e:
            return e.code
    assert code() == 0 and code(act=GELU) == 0 and code(z=None) == 0 and code(act=NONE, z=None) == 0
    assert code(z=dZ.data_ptr() + 4) == 0
    for act in (3, -1):
        assert code(act=act) == -1 and code(act=act, z=None) == -1
    assert code(act=NONE) == -1                                  # Z without an activation
    assert code(z=dC.data_ptr()) == -1                           # Z == C
    assert code(z=dZ.data_ptr() + 2) == -1 and code(z=dZ.data_ptr() + 1) == -1  # Z not 4-byte aligned
    for kid in (0, 7, 10, 30):
        assert code(kid) == -2 and code(kid, act=GELU, z=None) == -2
        assert code(kid, act=NONE, z=None) == 0
