"""A separate output D with C read-only (ftsgemm_run_out, ftsgemm_run_batched_out, matmul / bmm(c=), linear(residual=)).

An out-of-place call is defined as the in-place call on a copy of C: D0 = C.clone(), then run_batched_act on D0.  Every
test here holds D to D0 bit for bit and C to its bytes before the call, and the gaps and padding of D to what they held.
The exceptions are the ones the separate output exists for: at protect_epilogue = 1 a failed row segment is repaired with
beta != 0 (the in-place call leaves it in C), and a captured call with beta != 0 replays to the same D every time.
Integer operands make every product and sum exact, so a repaired D equals the fault-free one bit for bit.  The CPU tests
check the ABI's NULL-handle answer; the rest run on the GPU.
"""
import numpy as np
import pytest

MN, KM = 0, 1
NONE, ROW, COL = 0, 1, 2
ACT_NONE, RELU, GELU = 0, 1, 2
IDS = [1, 2, 3, 4, 5, 6, 11, 12, 13, 14, 15, 16, 20, 21, 22, 31, 32, 40]
GAP = 8  # floats between the entries of C, D and Z
SENTINEL = -12345.5


# ------------------------------------------------------------------ CPU
def test_run_out_null_handle(ft):
    assert ft.lib().ftsgemm_run_batched_out(None, 16, 128, 128, 128, None, 0, 128, 0, None, 0, 128, 0, None, 128, 0, None, 1,
                                            1.0, 0.0, None, 0, 0, 0, None, None) == -4
    assert ft.lib().ftsgemm_run_out(None, 16, 128, 128, 128, None, 0, 128, None, 0, 128, None, 128, None, 1.0, 0.0, None, 0, 0,
                                    None, None) == -4
    assert {"ftsgemm_run_out", "ftsgemm_run_batched_out"} <= set(ft.EXPORTED_SYMBOLS)


# ------------------------------------------------------------------ GPU helpers
def _ints(rng, shape, lo=-3, hi=4):
    return rng.integers(lo, hi, shape).astype(np.float32)


def _bits(t, x):
    return x.contiguous().view(t.int32)


def _same(t, x, y):
    return t.equal(_bits(t, x), _bits(t, y))


@pytest.fixture(scope="module")
def dev(cuda, ft):
    cuda.cuda.set_device(0)
    h = ft.FtSgemm()
    yield h
    h.close()


class _Case:
    """Bt products: A (Bt, M, K), B (Bt, N, K), C0 (Bt, M, N) as numpy arrays, on device buffers with padded leading
    dimensions (operand padding NaN) and entries GAP floats apart.  out() runs one out-of-place call and its in-place
    definition, checks C's bytes, D's gaps and Z, and returns (D, D0) as (Bt, M, N) tensors."""

    def __init__(self, t, ft, dev, A, B, C0, ldc=None):
        self.t, self.ft, self.dev = t, ft, dev
        self.Bt, self.M, self.K = A.shape
        self.N = B.shape[1]
        self.A, self.B = A, B
        self.ldc = ldc or self.M + 4
        self.sc = self.N * self.ldc + GAP
        buf = np.full(self.Bt * self.sc, SENTINEL, np.float32)
        for i in range(self.Bt):
            buf[i * self.sc:i * self.sc + self.N * self.ldc].reshape(self.N, self.ldc)[:, :self.M] = C0[i].T
        self.C = t.from_numpy(buf).cuda()
        self._ops = {}

    def op(self, which, layout, pad=4):
        key = (which, layout, pad)
        if key not in self._ops:
            X = self.A if which == "a" else self.B
            rows = X.shape[1]
            ld = (rows if layout == MN else (self.K + 3) // 4 * 4) + pad
            span = (self.K if layout == MN else rows) * ld
            stride = span + GAP
            buf = np.full(self.Bt * stride, np.nan, np.float32)
            for i in range(self.Bt):
                e = buf[i * stride:i * stride + span]
                if layout == MN:
                    e.reshape(self.K, ld)[:, :rows] = X[i].T
                else:
                    e.reshape(rows, ld)[:, :self.K] = X[i]
            self._ops[key] = (self.t.from_numpy(buf).cuda(), ld, stride)
        return self._ops[key]

    def view(self, buf):
        return buf.as_strided((self.Bt, self.N, self.M), (self.sc, self.ldc, 1)).transpose(1, 2)

    def bias(self, rng, mode, per_entry=False):
        n = self.M if mode == ROW else self.N
        b = np.round(20 * rng.standard_normal((self.Bt if per_entry else 1) * n)).astype(np.float32)
        return self.t.from_numpy(b).cuda(), (n if per_entry else 0)

    def call(self, kid, C, D, la=KM, lb=KM, alpha=1.0, beta=1.0, bias=None, mode=NONE, sbias=0, act=ACT_NONE, Z=None,
             opts=None, **opt):
        (dA, lda, sa), (dB, ldb, sb) = self.op("a", la), self.op("b", lb)
        opts = opts if opts is not None else self.ft.make_opts(**opt)
        if D is None:  # the in-place call
            self.dev.run_batched_act(kid, self.M, self.N, self.K, dA, la, lda, sa, dB, lb, ldb, sb, C, self.ldc, self.sc, self.Bt,
                                     alpha, beta, bias, mode, sbias, act, Z, opts)
        else:
            self.dev.run_batched_out(kid, self.M, self.N, self.K, dA, la, lda, sa, dB, lb, ldb, sb, C, self.ldc, self.sc, D,
                                     self.Bt, alpha, beta, bias, mode, sbias, act, Z, opts)

    def out(self, kid, z=False, **kw):
        t = self.t
        D0 = self.C.clone()
        Z0 = t.full_like(self.C, SENTINEL) if z else None
        self.call(kid, D0, None, Z=Z0, **kw)
        D = t.full_like(self.C, SENTINEL)
        Z = t.full_like(self.C, SENTINEL) if z else None
        before = self.C.clone()
        C = None if kw.get("beta", 1.0) == 0.0 else self.C
        self.call(kid, C, D, Z=Z, **kw)
        t.cuda.synchronize()
        assert _same(t, self.C, before), "C was written"
        keep = t.ones_like(D, dtype=t.bool)
        self.view(keep).fill_(False)
        assert bool((D[keep] == SENTINEL).all()), "D's padding or gaps were written"
        if z:
            assert _same(t, self.view(Z), self.view(Z0)), "Z differs"
        return self.view(D), self.view(D0)


def _case(t, ft, dev, rng, Bt=1, M=200, N=136, K=96, ldc=None, c0=None):
    C0 = c0 if c0 is not None else (np.round(64 * rng.standard_normal((Bt, M, N))) / 64).astype(np.float32)
    return _Case(t, ft, dev, _ints(rng, (Bt, M, K)), _ints(rng, (Bt, N, K)), C0, ldc)


def _check(t, D, D0, what):
    assert _same(t, D, D0), what


# ------------------------------------------------------------------ GPU: the definition
@pytest.mark.gpu
@pytest.mark.parametrize("kid", IDS)
def test_every_id_and_beta(cuda, ft, dev, kid):
    """every wgmma id, beta 0 (C = NULL) / 1 / -1.5, batch 1 and 3, at a ragged shape: D = the in-place result on a copy"""
    t = cuda
    rng = np.random.default_rng(kid)
    for Bt in (1, 3):
        case = _case(t, ft, dev, rng, Bt)
        for beta in (0.0, 1.0, -1.5):
            D, D0 = case.out(kid, alpha=0.75, beta=beta)
            _check(t, D, D0, (kid, Bt, beta))


@pytest.mark.gpu
@pytest.mark.parametrize("shape", [(256, 256, 128), (200, 136, 100)])
def test_layouts_and_padding(cuda, ft, dev, shape):
    """all four layout pairs with padded leading dimensions and ldc, at a full and a ragged shape"""
    t = cuda
    rng = np.random.default_rng(3)
    M, N, K = shape
    case = _case(t, ft, dev, rng, 2, M, N, K, ldc=M + 12)
    for la in (MN, KM):
        for lb in (MN, KM):
            for kid in (6, 16, 31, 40):
                D, D0 = case.out(kid, la=la, lb=lb, beta=-1.5)
                _check(t, D, D0, (kid, la, lb))


@pytest.mark.gpu
@pytest.mark.parametrize("Bt", [1, 3])
def test_bias_and_activation(cuda, ft, dev, Bt):
    """every bias mode (per-entry included with a batch), no activation / ReLU / GELU, with and without Z"""
    t = cuda
    rng = np.random.default_rng(10 + Bt)
    case = _case(t, ft, dev, rng, Bt)
    biases = [(NONE, None, 0)]
    for mode in (ROW, COL):
        biases.append((mode, *case.bias(rng, mode)))
        if Bt > 1:
            biases.append((mode, *case.bias(rng, mode, per_entry=True)))
    for kid in (11, 31, 40):
        for mode, b, sbias in biases:
            for act in (ACT_NONE, RELU, GELU):
                for z in ((False, True) if act != ACT_NONE else (False,)):
                    for beta in (0.0, -1.5):
                        D, D0 = case.out(kid, z, beta=beta, bias=b, mode=mode, sbias=sbias, act=act)
                        _check(t, D, D0, (kid, mode, sbias, act, z, beta))


@pytest.mark.gpu
def test_options(cuda, ft, dev):
    """3xTF32, check_segments, protect_epilogue 0 / 1 / 2 and the splitk knob, each with a bias and beta != 0"""
    t = cuda
    rng = np.random.default_rng(20)
    case = _case(t, ft, dev, rng, 2, 256, 256, 320)
    b, sbias = case.bias(rng, ROW, per_entry=True)
    variants = [dict(precision=1), dict(check_segments=3), dict(check_segments=2, precision=1)]
    variants += [dict(protect_epilogue=lvl) for lvl in (0, 1, 2)]
    try:
        for splitk in (0, 2):
            ft.debug_set("splitk", splitk)
            for kid in (31, 40, 15):
                for opt in variants:
                    for act in (ACT_NONE, GELU):
                        D, D0 = case.out(kid, act == GELU, beta=-1.5, bias=b, mode=ROW, sbias=sbias, act=act, **opt)
                        _check(t, D, D0, (splitk, kid, opt, act))
                        assert dev.stats()["detected"] == 0
    finally:
        ft.debug_set("splitk", -1)


@pytest.mark.gpu
def test_nonfinite(cuda, ft, dev):
    """Inf / NaN in C with beta = 0 leave D unaffected; Inf / NaN in A or B give the in-place result"""
    t = cuda
    rng = np.random.default_rng(30)
    M, N, K = 128, 128, 64
    C0 = _ints(rng, (1, M, N))
    C0[0, 5, 7], C0[0, 9, 3], C0[0, 100, 100] = np.inf, np.nan, -np.inf
    case = _case(t, ft, dev, rng, 1, M, N, K, c0=C0)
    clean = _Case(t, ft, dev, case.A, case.B, np.zeros_like(C0))
    for kid in (16, 31):
        D, D0 = case.out(kid, beta=0.0)
        assert bool(t.isfinite(D).all())
        _check(t, D, D0, kid)
        Dc, _ = clean.out(kid, beta=0.0)
        _check(t, D, Dc, kid)
    A = _ints(rng, (1, M, K))
    B = _ints(rng, (1, N, K))
    A[0, 3, 5], B[0, 8, 2], A[0, 40, 1], B[0, 60, 1] = np.inf, np.nan, -np.inf, np.inf
    bad = _Case(t, ft, dev, A, B, _ints(rng, (1, M, N)))
    for kid in (16, 31):
        for beta in (0.0, 1.0):
            for opt in ({}, dict(precision=1), dict(protect_epilogue=2)):
                D, D0 = bad.out(kid, beta=beta, **opt)
                assert t.equal(t.isnan(D), t.isnan(D0)) and bool(t.isnan(D).any())
                _check(t, D, D0, (kid, beta, opt))


# ------------------------------------------------------------------ GPU: faults
def _col_where(D, row, lo, hi):
    return next(c for c in range(lo, hi) if D[row, c] != 0)


@pytest.mark.gpu
@pytest.mark.parametrize("level", [0, 1, 2])
def test_accumulator_upsets_corrected(cuda, ft, dev, level):
    """upsets of the accumulator (modes 0 / 1): corrected, D = the fault-free D, C untouched"""
    t = cuda
    rng = np.random.default_rng(40)
    case = _case(t, ft, dev, rng, 1, 256, 256, 256)
    want, _ = case.out(31, beta=1.0)
    want = want.clone()
    for f in ({"row": 37, "col": 70, "add": 4096.0}, {"row": 130, "col": 201, "xor": 1 << 30}):
        dev.stats()
        D, _ = case.out(31, beta=1.0, faults=[f], protect_epilogue=level)
        st = dev.stats()
        assert st["corrected"] >= 1 and st["uncorrectable"] == 0, st
        _check(t, D, want, f)


@pytest.mark.gpu
@pytest.mark.parametrize("act", [ACT_NONE, GELU])
def test_level1_repairs_any_beta(cuda, ft, dev, act):
    """an upset of the stored value (mode 3) at protect_epilogue = 1 with beta != 0: in place it stays in C (status 7); with
    D != C the segment is recomputed into D from the intact C (status 6) and D = the fault-free D.  Level 2 the same."""
    t = cuda
    rng = np.random.default_rng(41)
    for Bt in (1, 2):
        case = _case(t, ft, dev, rng, Bt, 256, 256, 256)
        b, sbias = case.bias(rng, COL, per_entry=Bt > 1)
        kw = dict(beta=-1.5, bias=b, mode=COL, sbias=sbias, act=act)
        want, _ = case.out(31, act == GELU, **kw)
        want = want.clone()
        entry = Bt - 1
        col = _col_where(want[entry], 37, 40, 256)
        f = [{"row": entry * 256 + 37, "col": col, "xor": 1 << 27, "where": "epilogue_value"}]
        for level in (1, 2):
            # the in-place definition: reported, left in C
            D0 = case.C.clone()
            dev.stats()
            case.call(31, D0, None, faults=f, protect_epilogue=level, **kw)
            st = dev.stats()
            assert st["epilogue_faults"] == 1, st
            assert [e["status"] for e in st["events"]] == ([7] if level == 1 else [6]), (level, st)
            # out of place: repaired
            D = t.full_like(case.C, SENTINEL)
            before = case.C.clone()
            case.call(31, case.C, D, faults=f, protect_epilogue=level, **kw)
            st = dev.stats()
            assert st["epilogue_faults"] == 1 and st["recomputed"] == 1 and st["uncorrectable"] == 0, (level, st)
            assert [e["status"] for e in st["events"]] == [6], (level, st)
            assert _same(t, case.C, before)
            _check(t, case.view(D), want, (Bt, level))
        # no_recompute: left as computed, status 7
        D = t.full_like(case.C, SENTINEL)
        case.call(31, case.C, D, faults=f, protect_epilogue=1, no_recompute=True, **kw)
        st = dev.stats()
        assert st["uncorrectable"] == 1 and st["recomputed"] == 0 and [e["status"] for e in st["events"]] == [7], st


# ------------------------------------------------------------------ GPU: arguments
@pytest.mark.gpu
def test_argument_checks(cuda, ft, dev):
    t = cuda
    rng = np.random.default_rng(50)
    case = _case(t, ft, dev, rng, 2, 128, 128, 64)
    n = case.C.numel()

    def code(C, D, kid=31, Z=None, act=ACT_NONE, beta=1.0):
        with pytest.raises(ft.FtsgemmError) as e:
            case.call(kid, C, D, beta=beta, Z=Z, act=act)
        return e.value.code

    big = t.zeros(3 * n + 64, device="cuda")
    C = big[:n]
    assert code(C, 0) == -1                                         # D NULL
    assert code(C, big[n + 1:2 * n + 1]) == -1                      # misaligned D
    assert code(C, big[case.ldc:case.ldc + n]) == -1                # D overlaps C by one column
    assert code(C, big[case.sc:case.sc + n]) == -1                  # ... and by one entry
    D = big[2 * n + 16:3 * n + 16]
    assert code(C, D, Z=D, act=RELU) == -1                          # dZ == D
    assert code(C, D, Z=big[2 * n + 16 + 4:], act=RELU) == -1        # Z overlapping D
    assert code(C, D, Z=C, act=RELU) == -1                          # Z overlapping (here: equal to) C
    assert code(None, D, beta=1.0) == -1                            # C NULL with beta != 0
    single = _case(t, ft, dev, rng, 1, 128, 128, 64)
    (dA, lda, _), (dB, ldb, _) = single.op("a", MN), single.op("b", MN)
    for kid in (0, 7, 10, 30):
        D1 = t.zeros_like(single.C)
        with pytest.raises(ft.FtsgemmError) as e:
            dev.run_out(kid, 128, 128, 64, dA, MN, lda, dB, MN, ldb, single.C, single.ldc, D1, 1.0, 1.0)
        assert e.value.code == -2, kid
    # D == C is the in-place call, on every id
    want = single.C.clone()
    single.call(31, want, None, la=MN, lb=MN)
    got = single.C.clone()
    single.call(31, got, got, la=MN, lb=MN)
    t.cuda.synchronize()
    assert _same(t, got, want)


# ------------------------------------------------------------------ GPU: graphs
@pytest.mark.gpu
def test_graph_replay_is_idempotent(cuda, ft, dev):
    """a captured out-of-place call with beta = 1 replays to the same D every time, C untouched, D = the eager call"""
    t = cuda
    rng = np.random.default_rng(60)
    case = _case(t, ft, dev, rng, 2, 512, 384, 256)
    b = case.bias(rng, ROW)[0]
    want, _ = case.out(40, beta=1.0, bias=b, mode=ROW)
    want = want.clone()
    before = case.C.clone()
    D = t.full_like(case.C, SENTINEL)
    g = t.cuda.CUDAGraph()
    with t.cuda.graph(g):
        case.call(40, case.C, D, beta=1.0, bias=b, mode=ROW,
                  opts=ft.make_opts(stream=t.cuda.current_stream().cuda_stream))
    for r in range(3):
        g.replay()
        t.cuda.synchronize()
        _check(t, case.view(D), want, r)
        assert _same(t, case.C, before), r
    assert dev.stats()["detected"] == 0


# ------------------------------------------------------------------ GPU: the torch layer
def _lin(t, g, *shape, scale=1.0):
    return (scale * t.randn(*shape, device="cuda", generator=g)).requires_grad_()


@pytest.mark.gpu
@pytest.mark.parametrize("tokens", [512, 300])
def test_linear_residual_forward(cuda, ft, dev, tokens):
    """y = linear(x, W, b, residual=r) is bit for bit r.clone() + matmul(out=, beta=1), within TF32 of float64, from one
    launch like linear(x, W, b), and r is not written"""
    t = cuda
    g = t.Generator(device="cuda").manual_seed(70)
    K, N = 512, 384
    with t.no_grad():
        x, W, b, r = (_lin(t, g, 2, tokens // 2, K), _lin(t, g, N, K, scale=K ** -0.5), _lin(t, g, N), _lin(t, g, 2, tokens // 2, N))
        r0 = r.clone()
        n0 = dev.launch_count()
        dev.linear(x, W, b)
        n_plain = dev.launch_count() - n0
        n0 = dev.launch_count()
        y = dev.linear(x, W, b, residual=r)
        assert dev.launch_count() - n0 == n_plain
        ref = r.clone()
        dev.matmul(x.reshape(-1, K), W.t(), out=ref.view(-1, N), bias=b, beta=1.0)
        t.cuda.synchronize()
        assert _same(t, r, r0)
        assert _same(t, y, ref)
        want = (x.double().reshape(-1, K) @ W.double().t() + b.double()).view(2, tokens // 2, N) + r.double()
        err = (y.double() - want).abs().max().item()
        assert err <= 1e-2 * want.abs().max().item(), err
        with pytest.raises(ValueError):
            dev.linear(x, W, b, residual=r, activation="relu")
        with pytest.raises(ValueError):
            dev.linear(x, W, b, residual=r[:, :, :-4])


@pytest.mark.gpu
def test_linear_residual_gradients(cuda, ft, dev):
    """grad_x, grad_W, grad_b match the unfused chain linear(x, W, b) + r bit for bit; grad_r = grad_y; r unmodified"""
    t = cuda
    g = t.Generator(device="cuda").manual_seed(71)
    K, N, T = 384, 256, 264
    x, W, b, r = _lin(t, g, T, K), _lin(t, g, N, K, scale=K ** -0.5), _lin(t, g, N), _lin(t, g, T, N)
    r0 = r.detach().clone()
    gy = t.randn(T, N, device="cuda", generator=g)
    y = dev.linear(x, W, b, residual=r)
    y.backward(gy)
    grads = [p.grad.clone() for p in (x, W, b, r)]
    for p in (x, W, b, r):
        p.grad = None
    (dev.linear(x, W, b) + r).backward(gy)
    for got, p in zip(grads, (x, W, b, r)):
        assert _same(t, got, p.grad)
    assert _same(t, grads[3], gy)
    assert _same(t, r.detach(), r0)


@pytest.mark.gpu
def test_matmul_and_bmm_c(cuda, ft, dev):
    """matmul(c=) / bmm(c=) forward = the in-place call on a copy of c (c with other strides copied once), c never written,
    out allocated with c's strides; bmm's grad_c = beta * grad_z"""
    t = cuda
    g = t.Generator(device="cuda").manual_seed(72)
    M, K, N = 200, 96, 136
    a, b = t.randn(M, K, device="cuda", generator=g), t.randn(K, N, device="cuda", generator=g)
    bias = t.randn(N, device="cuda", generator=g)
    for c in (t.randn(M, N, device="cuda", generator=g), t.randn(N, M, device="cuda", generator=g).t()):
        c0 = c.clone()
        for act in (None, "relu", "gelu"):
            ref = c.clone()
            dev.matmul(a, b, out=ref, bias=bias, activation=act, beta=-1.5)
            out = dev.matmul(a, b, c=c, bias=bias, activation=act, beta=-1.5)
            assert out.stride() == c.stride()
            assert _same(t, out, ref), act
            o2 = t.empty(M, N, device="cuda")  # row-major out, c possibly column-major: copied into out's geometry
            dev.matmul(a, b, o2, c=c, bias=bias, activation=act, beta=-1.5)
            assert (o2 - ref).abs().max().item() <= 1e-3 * ref.abs().max().item()
        assert _same(t, c, c0)
    with pytest.raises(ValueError):
        dev.matmul(a, b, c=c, beta=0.0)
    Bt = 3
    A = t.randn(Bt, M, K, device="cuda", generator=g, requires_grad=True)
    B = t.randn(Bt, K, N, device="cuda", generator=g, requires_grad=True)
    Cc = t.randn(Bt, M, N, device="cuda", generator=g, requires_grad=True)
    pb = t.randn(Bt, N, device="cuda", generator=g, requires_grad=True)
    C0 = Cc.detach().clone()
    for act in (None, "gelu"):
        with t.no_grad():
            ref = Cc.detach().clone()
            dev.bmm(A.detach(), B.detach(), ref, bias=pb.detach(), activation=act, alpha=0.5, beta=-1.5)
        y = dev.bmm(A, B, c=Cc, bias=pb, activation=act, alpha=0.5, beta=-1.5)
        assert _same(t, y.detach(), ref)
        gy = t.randn(Bt, M, N, device="cuda", generator=g)
        y.backward(gy)
        if act is None:
            assert _same(t, Cc.grad, -1.5 * gy)
        # grad_c = beta * grad_z and grad_bias = grad_z summed over each entry's rows
        assert t.allclose(Cc.grad.sum(1), -1.5 * pb.grad, rtol=1e-5, atol=1e-4)
        for p in (A, B, Cc, pb):
            p.grad = None
    assert _same(t, Cc.detach(), C0)


@pytest.mark.gpu
def test_graphed_transformer_block(cuda, ft, dev):
    """attention output projection + residual and FFN + residual, captured and replayed: the same y as eager, every replay,
    and the residual stream input untouched"""
    t = cuda
    g = t.Generator(device="cuda").manual_seed(73)
    T, E, H = 512, 256, 1024
    x = t.randn(T, E, device="cuda", generator=g)
    attn = t.randn(T, E, device="cuda", generator=g)
    Wo, bo = t.randn(E, E, device="cuda", generator=g) * E ** -0.5, t.randn(E, device="cuda", generator=g)
    W1, b1 = t.randn(H, E, device="cuda", generator=g) * E ** -0.5, t.randn(H, device="cuda", generator=g)
    W2, b2 = t.randn(E, H, device="cuda", generator=g) * H ** -0.5, t.randn(E, device="cuda", generator=g)

    def block():
        h = dev.linear(attn, Wo, bo, residual=x)
        f = dev.linear(h, W1, b1, activation="gelu")
        return dev.linear(f, W2, b2, residual=h)

    with t.no_grad():
        want = block().clone()
        x0 = x.clone()
        s = t.cuda.Stream()
        s.wait_stream(t.cuda.current_stream())
        with t.cuda.stream(s):
            block()
        t.cuda.current_stream().wait_stream(s)
        gr = t.cuda.CUDAGraph()
        with t.cuda.graph(gr):
            y = block()
        for r in range(3):
            gr.replay()
            t.cuda.synchronize()
            assert _same(t, y, want), r
            assert _same(t, x, x0), r
    assert dev.stats()["detected"] == 0
