"""Inf, NaN and overflow through every GEMM path (include/ftsgemm.h: ftsgemm_run, ftsgemm_stats.detected; DESIGN.md §3.3-3.5, §4).

The contract:
  * every tensor-core id stores what IEEE FP32 arithmetic gives on TF32-truncated operands: the NaN positions and the +-Inf
    positions and signs of a float64 reference (precision = 1: FP32 on the untruncated operands);
  * beta == 0: C is not read, on every id and entry point;
  * a row whose expected checksum is non-finite cannot be verified: it is not flagged, not counted, and stored bit for bit as
    the plain twin stores it;
  * with a finite expected checksum, an upset to +-Inf or NaN is detected, located and repaired.

The reference below is float64 on TF32-truncated operands, formed without BLAS (einsum with optimize=False): reference BLAS
skips zero terms, which would hide 0 * Inf.  Inputs are small integers wherever rounding is not what a test checks, so every
finite element is exact and compares equal, and any re-rounding (a recomputed row) shows.
"""
import numpy as np
import pytest

MN, KM = 0, 1
NONE, ROW, COL = 0, 1, 2
NAMES = ["small", "medium", "large", "tall", "wide", "huge", "giant", "pair128"]
INF, NAN = np.float32(np.inf), np.float32(np.nan)
SENTINEL = np.float32(-12345.5)


# ------------------------------------------------------------------ helpers (no GPU)
def tf32(x):
    """the tensor core's operand truncation: keep the top 19 bits (keeps +-Inf and the canonical NaN)"""
    x = np.ascontiguousarray(x, np.float32)
    return (x.view(np.uint32) & np.uint32(0xFFFFE000)).view(np.float32)


def reference(A, B, C0=None, alpha=1.0, beta=0.0, truncate=True):
    """alpha * A * B^T + beta * C0 in float64, rounded once to float32; A: M x K, B: N x K.  No BLAS, and C0 is not read when
    beta == 0."""
    a = (tf32(A) if truncate else np.asarray(A, np.float32)).astype(np.float64)
    b = (tf32(B) if truncate else np.asarray(B, np.float32)).astype(np.float64)
    with np.errstate(all="ignore"):
        out = alpha * np.einsum("mk,nk->mn", a, b, optimize=False)
        if beta != 0.0:
            out = out + beta * np.asarray(C0, np.float64)
        return out.astype(np.float32)


def add_bias(C, bias, mode):
    """the store pass's bias add: one float32 rounding of the broadcast bias"""
    if mode == NONE:
        return C
    with np.errstate(all="ignore"):
        return (C + (bias[:, None] if mode == ROW else bias[None, :])).astype(np.float32)


def mismatch(got, want):
    """'' when got and want have the same NaN mask, the same +-Inf mask and signs and equal finite values (+0 == -0);
    otherwise a description of the first differences"""
    got, want = np.asarray(got, np.float32), np.asarray(want, np.float32)
    if got.shape != want.shape:
        return f"shape {got.shape} != {want.shape}"
    bad = ((np.isnan(got) != np.isnan(want)) | (np.isposinf(got) != np.isposinf(want)) | (np.isneginf(got) != np.isneginf(want))
           | (np.isfinite(want) & np.isfinite(got) & (got != want)))
    if not bad.any():
        return ""
    idx = np.argwhere(bad)[:6]
    return f"{int(bad.sum())} elements differ, e.g. " + ", ".join(f"{tuple(i)}: got {got[tuple(i)]} want {want[tuple(i)]}" for i in idx)


def bits(x):
    return np.ascontiguousarray(x, np.float32).view(np.uint32)


def same_bits(x, y):
    return x.shape == y.shape and np.array_equal(bits(x), bits(y))


def xor_mask(value, target):
    """the xor mask that turns the float32 `value` into exactly `target` (+Inf, -Inf, NaN): an injected upset"""
    return int(np.float32(value).view(np.uint32)) ^ int(np.float32(target).view(np.uint32))


def clean_stats(st):
    """nothing detected or counted, and the residual statistics untouched by non-finite rows"""
    return (all(st[k] == 0 for k in ("detected", "corrected", "uncorrectable", "recomputed", "checksum_faults", "epilogue_faults"))
            and np.isfinite(st["max_abs_residual"]) and np.isfinite(st["max_rel_residual"]) and not st["events"])


def ints(rng, shape):
    return rng.integers(-4, 5, shape).astype(np.float32)


def pad4(n):
    return (n + 3) // 4 * 4


def ld_of(layout, rows, K, pad):
    base = rows if layout == MN else pad4(K)
    return base + 4 if pad else base


def pack(X, layout, ld):
    """rows x K matrix -> flat buffer in the layout (MN: X[r, k] at r + k*ld; KM: at k + r*ld), padding = NaN"""
    rows, K = X.shape
    if layout == MN:
        buf = np.full((K, ld), np.nan, np.float32)
        buf[:, :rows] = X.T
    else:
        buf = np.full((rows, ld), np.nan, np.float32)
        buf[:, :K] = X
    return buf.reshape(-1)


def poison(rng, shape):
    """an old C made of NaN, +Inf and -Inf only"""
    return rng.choice(np.array([np.nan, np.inf, -np.inf], np.float32), shape)


# ------------------------------------------------------------------ CPU
def test_reference_hand_cases():
    A = np.array([[0.0, 1.0], [1.0, 1.0], [2.0 ** 64, 2.0 ** 64], [1.0, 0.0]], np.float32)
    B = np.array([[np.inf, 0.0], [np.inf, -np.inf], [2.0 ** 64, 2.0 ** 64], [-(2.0 ** 64), -(2.0 ** 64)]], np.float32)
    C = reference(A, B)
    assert np.isnan(C[0, 0])                         # 0 * Inf
    assert np.isnan(C[1, 1])                         # Inf + (-Inf)
    assert C[3, 0] == np.inf                         # 1 * Inf + 0 * 0
    assert np.isnan(C[3, 1])                         # 1 * Inf + 0 * (-Inf): the zero term is not skipped
    assert C[2, 2] == np.inf and C[2, 3] == -np.inf  # 2^64 * 2^64 * 2: same-sign overflow, both signs
    assert C[0, 2] == np.float32(2.0 ** 64)
    # beta = 0 never reads C; beta != 0 does
    C0 = np.full((4, 4), np.nan, np.float32)
    assert np.array_equal(reference(A, B, C0, 1.0, 0.0), C, equal_nan=True)
    assert np.all(np.isnan(reference(A, B, C0, 1.0, 0.5)))
    # TF32 truncation keeps Inf, -Inf and NaN, and a finite value's top bits
    t = tf32(np.array([np.inf, -np.inf, np.nan, 1.0 + 2.0 ** -12, 3.0], np.float32))
    assert t[0] == np.inf and t[1] == -np.inf and np.isnan(t[2]) and t[3] == 1.0 and t[4] == 3.0


def test_mismatch_and_bits():
    x = np.array([1.0, np.nan, np.inf, -np.inf, 0.0], np.float32)
    assert mismatch(x, x.copy()) == ""
    assert mismatch(x, np.array([1.0, np.nan, np.inf, -np.inf, -0.0], np.float32)) == ""
    for i, v in ((0, 2.0), (1, 1.0), (2, -np.inf), (3, np.nan), (4, np.inf)):
        y = x.copy()
        y[i] = v
        assert mismatch(x, y), (i, v)
    assert same_bits(x, x.copy()) and not same_bits(x, np.array([1.0, np.nan, np.inf, -np.inf, -0.0], np.float32))


def test_xor_mask():
    assert xor_mask(1.0, np.inf) == 1 << 30        # bit 30 of an exact 1.0 is the whole exponent
    assert xor_mask(-1.0, -np.inf) == 1 << 30
    for v in (1.0, -3.0, 0.0, 2.5e-3, 7.0e30):
        for target in (np.inf, -np.inf, np.nan):
            got = np.uint32(int(np.float32(v).view(np.uint32)) ^ xor_mask(v, target)).view(np.float32)
            assert (np.isnan(got) if np.isnan(target) else got == target), (v, target)


def test_poison_has_only_nonfinite():
    p = poison(np.random.default_rng(0), (64, 64))
    assert not np.isfinite(p).any() and np.isnan(p).any() and np.isposinf(p).any() and np.isneginf(p).any()


# ------------------------------------------------------------------ GPU helpers
@pytest.fixture(scope="module")
def dev(cuda, ft):
    cuda.cuda.set_device(0)
    h = ft.FtSgemm()
    yield h
    h.close()


class Case:
    """One product on the GPU: A (M x K), B (N x K) as 2-D numpy arrays."""

    def __init__(self, cuda, dev, A, B):
        self.cuda, self.dev, self.A, self.B = cuda, dev, A, B
        self.M, self.K = A.shape
        self.N = B.shape[0]

    def run(self, kid, la=MN, lb=MN, pad=False, ldc=None, alpha=1.0, beta=0.0, C0=None, bias=None, mode=NONE, opts=None):
        """run_bias (mode NONE: run_ex); returns C as an M x N array and checks that C's padding was not written"""
        t, M, N, K = self.cuda, self.M, self.N, self.K
        lda, ldb, ldc = ld_of(la, M, K, pad), ld_of(lb, N, K, pad), ldc or M
        dA = t.from_numpy(pack(self.A, la, lda)).cuda()
        dB = t.from_numpy(pack(self.B, lb, ldb)).cuda()
        cbuf = np.full((N, ldc), SENTINEL, np.float32)
        cbuf[:, :M] = (np.zeros((M, N), np.float32) if C0 is None else C0).T
        dC = t.from_numpy(cbuf.reshape(-1)).cuda()
        if mode == NONE:
            self.dev.run_ex(kid, M, N, K, dA, la, lda, dB, lb, ldb, dC, ldc, alpha, beta, opts)
        else:
            self.dev.run_bias(kid, M, N, K, dA, la, lda, dB, lb, ldb, dC, ldc, alpha, beta, t.from_numpy(bias).cuda(), mode, opts)
        t.cuda.synchronize()
        out = dC.cpu().numpy().reshape(N, ldc)
        assert np.all(out[:, M:] == SENTINEL), "C's padding was written"
        return np.ascontiguousarray(out[:, :M].T)


def run_batched(cuda, dev, kid, A, B, C0=None, beta=0.0, opts=None):
    """A (Bt, M, K), B (Bt, N, K), both K-major with rows padded to 4, C (Bt, M, N) column-major, in one run_batched call"""
    t = cuda
    Bt, M, K = A.shape
    N = B.shape[1]
    ld = pad4(K)
    dA = t.from_numpy(np.concatenate([pack(a, KM, ld) for a in A])).cuda()
    dB = t.from_numpy(np.concatenate([pack(b, KM, ld) for b in B])).cuda()
    c = np.zeros((Bt, M, N), np.float32) if C0 is None else C0
    dC = t.from_numpy(np.ascontiguousarray(c.transpose(0, 2, 1)).reshape(-1)).cuda()
    dev.run_batched(kid, M, N, K, dA, KM, ld, M * ld, dB, KM, ld, N * ld, dC, M, M * N, Bt, 1.0, beta, None, NONE, opts)
    t.cuda.synchronize()
    return np.ascontiguousarray(dC.cpu().numpy().reshape(Bt, N, M).transpose(0, 2, 1))


def tile_n(ft):
    return {k["id"]: k["tile"][1] for k in ft.kernel_table()}


def twins(ft):
    """(plain id, ABFT id) of every named wgmma variant"""
    return [(ft.SGEMM_IDS[n], ft.ABFT_IDS[n]) for n in NAMES]


# ------------------------------------------------------------------ GPU 1: beta = 0 never reads C
@pytest.mark.gpu
def test_beta_zero_ignores_c(cuda, ft, dev):
    """C0 made of NaN and +-Inf, beta = 0: the result equals the same call with C0 = 0, bit for bit, on every id, with full-N
    tiles and with a ragged N tail, under every ABFT option, in a batch and through run_host."""
    rng = np.random.default_rng(101)
    ids = [i for pair in twins(ft) for i in pair] + [ft.ID_SGEMM_AUTO, ft.ID_ABFT_AUTO, ft.ID_CUBLAS, ft.ID_CUBLAS_TF32,
                                                     ft.ID_ABFT_BASELINE, ft.ID_ABFT_BASELINE_TF32]
    for M, N, K in ((256, 512, 128), (260, 388, 201)):
        case = Case(cuda, dev, ints(rng, (M, K)), ints(rng, (N, K)))
        bad = poison(rng, (M, N))
        for kid in ids:
            want = case.run(kid, alpha=0.75)
            got = case.run(kid, alpha=0.75, C0=bad)
            assert same_bits(got, want), (kid, M, N, mismatch(got, want))
    # the ABFT options, on the ragged shape, data of 0.1 steps (so that two upsets in one row are not taken for one)
    M, N, K = 260, 388, 201
    A = (rng.integers(-9, 10, (M, K)) * 0.1).astype(np.float32)
    B = (rng.integers(-9, 10, (N, K)) * 0.1).astype(np.float32)
    case = Case(cuda, dev, A, B)
    bad = poison(rng, (M, N))
    two = [{"row": 40, "col": 10, "add": 100.0}, {"row": 40, "col": 25, "add": -37.0}]
    bias = {ROW: rng.standard_normal(M).astype(np.float32), COL: rng.standard_normal(N).astype(np.float32)}
    for kid in (31, 16):
        for opts, mode in ((dict(protect_epilogue=True), NONE), (dict(precision=1), NONE), (dict(check_segments=4), NONE),
                           ({}, ROW), ({}, COL), (dict(faults=two), NONE), (dict(faults=two, protect_epilogue=True), COL)):
            b = bias.get(mode)
            dev.stats()
            want = case.run(kid, KM, MN, True, M + 8, 0.75, 0.0, None, b, mode, ft.make_opts(**opts))
            st_want = dev.stats()
            got = case.run(kid, KM, MN, True, M + 8, 0.75, 0.0, bad, b, mode, ft.make_opts(**opts))
            st_got = dev.stats()
            assert same_bits(got, want), (kid, opts, mode, mismatch(got, want))
            if "faults" in opts:  # the row went through recompute_row (id 31, as in tests/test_bias.py)
                assert st_want["detected"] == st_got["detected"] == 1, (st_want, st_got)
                assert st_want["recomputed"] == st_got["recomputed"] == (1 if kid == 31 else st_got["recomputed"]), (st_want, st_got)
            else:
                assert st_got["detected"] == st_want["detected"] == 0
    # a 3-entry batch
    Ab, Bb = ints(rng, (3, 260, 201)), ints(rng, (3, 388, 201))
    for kid in (31, 21, 14):
        want = run_batched(cuda, dev, kid, Ab, Bb)
        got = run_batched(cuda, dev, kid, Ab, Bb, poison(rng, (3, 260, 388)))
        assert same_bits(got, want), kid
    # run_host with a host C full of NaN (no upload of C when beta == 0)
    hA = np.ascontiguousarray(case.A.T).reshape(-1)  # column-major M x K
    hB = np.ascontiguousarray(case.B.T).reshape(-1)  # column-major N x K
    for kid in (31, 6, ft.ID_CUBLAS):
        outs = []
        for fill in (0.0, np.nan):
            hC = np.full(M * N, fill, np.float32)
            dev.run_host(kid, M, N, K, hA, hB, hC, 0.75, 0.0)
            outs.append(hC)
        assert same_bits(outs[1], outs[0]), kid
    assert dev.stats()["detected"] == 0


# ------------------------------------------------------------------ GPU 2: non-finite operands follow IEEE
def plant(A, B, bn):
    """Inf / NaN in A rows and B columns at the tile edges of tile width bn (n = bn - 1, bn, the ragged last column and row
    tiles) and at k = 0 and K - 1 (the ragged last k-block); 0 * Inf and Inf + (-Inf) both occur"""
    A, B = A.copy(), B.copy()
    M, K = A.shape
    N = B.shape[0]
    B[bn - 1, 0], B[bn - 1, K - 1] = INF, -INF  # +Inf at k = 0 and -Inf at k = K-1 in one column: NaN where a0 * aK1 > 0
    B[bn, K - 1] = -INF
    B[N - 1, K // 2] = NAN
    A[3, 0] = NAN
    A[7, 0] = 0.0                               # 0 * Inf
    A[9, 0], A[9, K - 1] = 2.0, 3.0             # Inf + (-Inf)
    A[M - 1, K - 1] = INF
    return A, B


@pytest.mark.gpu
@pytest.mark.parametrize("splitk", [0, 2])
def test_nonfinite_operands_follow_ieee(cuda, ft, dev, splitk):
    """Every named id, all four layout pairs with padded leading dimensions (NaN in the padding), cut tiles off and forced:
    C is the IEEE result, and each ABFT id is bit-identical to its plain twin with nothing detected or counted -- also with
    no_recompute and detect_only."""
    rng = np.random.default_rng(102 + splitk)
    M, N, K = 260, 388, 201
    A0, B0 = ints(rng, (M, K)), ints(rng, (N, K))
    bn_of = tile_n(ft)
    try:
        ft.debug_set("splitk", splitk)
        for bn in sorted({bn_of[p] for p, _ in twins(ft)}):
            A, B = plant(A0, B0, bn)
            want = reference(A, B)
            assert np.isnan(want[7, bn - 1]) and np.isnan(want[9, bn - 1]) and np.isnan(want[3]).all()
            assert np.isinf(want[:, bn]).any() and not np.isfinite(want[M - 1]).any()
            case = Case(cuda, dev, A, B)
            for plain, abft in twins(ft):
                if bn_of[plain] != bn:
                    continue
                for la in (MN, KM):
                    for lb in (MN, KM):
                        x = case.run(plain, la, lb, True, M + 8)
                        assert not mismatch(x, want), (plain, la, lb, mismatch(x, want))
                        dev.stats()
                        y = case.run(abft, la, lb, True, M + 8)
                        st = dev.stats()
                        assert same_bits(y, x), (abft, la, lb, mismatch(y, x))
                        assert clean_stats(st), (abft, la, lb, st)
                for opts in (dict(no_recompute=True), dict(detect_only=True)):
                    y = case.run(abft, opts=ft.make_opts(**opts))
                    st = dev.stats()
                    assert same_bits(y, case.run(plain)) and clean_stats(st), (abft, opts, st)
            if bn == 256:  # cuBLAS (FP32, no truncation: the data is TF32-exact) as an independent IEEE witness
                z = case.run(ft.ID_CUBLAS)
                assert not mismatch(z, want), mismatch(z, want)
    finally:
        ft.debug_set("splitk", -1)


@pytest.mark.gpu
def test_one_inf_in_random_normal_b(cuda, ft, dev):
    """Random-normal data, where a recomputed row would be re-rounded: one Inf in B leaves every ABFT id bit-identical to its
    plain twin, with nothing detected."""
    rng = np.random.default_rng(104)
    M, N, K = 512, 768, 1000
    A = rng.standard_normal((M, K)).astype(np.float32)
    B = rng.standard_normal((N, K)).astype(np.float32)
    B[300, 17] = INF
    case = Case(cuda, dev, A, B)
    want = reference(A, B)
    for plain, abft in twins(ft):
        x = case.run(plain)
        dev.stats()
        y = case.run(abft)
        st = dev.stats()
        assert same_bits(y, x), (abft, mismatch(y, x))
        assert clean_stats(st), (abft, st)
        assert np.array_equal(np.isposinf(x), np.isposinf(want)) and np.array_equal(np.isneginf(x), np.isneginf(want))
        assert not np.isnan(x).any()


# ------------------------------------------------------------------ GPU 3: overflow
@pytest.mark.gpu
def test_overflow(cuda, ft, dev):
    """Finite operands (1) whose same-sign products exceed FLT_MAX in chosen elements and (2) whose B column-block sums
    overflow in the encode while C stays finite: C is the IEEE result (cuBLAS agrees), each ABFT id equals its plain twin and
    nothing is counted."""
    rng = np.random.default_rng(105)
    M, N, K = 260, 388, 201
    big = np.float32(2.0 ** 64)
    A, B = ints(rng, (M, K)), ints(rng, (N, K))
    # one huge term per element (k = 10, 30, 31 are zero elsewhere): two of them could cancel, and the sum of the small
    # terms left over would then depend on rounding, in float64 as well as in FP32
    A[:, [10, 30, 31]] = 0.0
    B[:, [10, 30, 31]] = 0.0
    A[5, 10], B[20, 10] = big, big      # 2^128 + small: +Inf
    A[70, 30], B[300, 30] = -big, big   # -Inf
    A[70, 31], B[300, 31] = -big, big   # (same sign as the term before)
    want = reference(A, B)
    assert want[5, 20] == np.inf and want[70, 300] == -np.inf and np.isfinite(np.delete(want.reshape(-1), [5 * N + 20, 70 * N + 300])).all()
    # encode overflow: two columns of 2^127 in one column block at k = 40 (e = 2^128 > FLT_MAX) with |a| <= 1 there
    A2, B2 = ints(rng, (M, K)), ints(rng, (N, K))
    A2[:, 40] = rng.integers(-1, 2, M)
    B2[0, 40] = B2[1, 40] = np.float32(2.0 ** 127)
    want2 = reference(A2, B2)
    assert np.isfinite(want2).all()
    for a, b, w in ((A, B, want), (A2, B2, want2)):
        case = Case(cuda, dev, a, b)
        z = case.run(ft.ID_CUBLAS)
        assert not mismatch(z, w), mismatch(z, w)
        for plain, abft in twins(ft):
            x = case.run(plain, KM, KM)
            assert not mismatch(x, w), (plain, mismatch(x, w))
            dev.stats()
            y = case.run(abft, KM, KM)
            st = dev.stats()
            assert same_bits(y, x), (abft, mismatch(y, x))
            assert clean_stats(st), (abft, st)


# ------------------------------------------------------------------ GPU 4: upsets to +-Inf and NaN are repaired
def upsets(clean, bn, rows):
    """five upsets in five rows: +Inf at column 0, -Inf at bn - 1, NaN in the ragged last tile-column, bit 30 of an exact 1.0
    (+Inf) and add: +Inf at column bn"""
    N = clean.shape[1]
    r1, c1 = next((int(r), int(c)) for r, c in np.argwhere(clean == 1.0) if r not in rows)
    f = [{"row": rows[0], "col": 0, "xor": xor_mask(clean[rows[0], 0], INF)},
         {"row": rows[1], "col": bn - 1, "xor": xor_mask(clean[rows[1], bn - 1], -INF)},
         {"row": rows[2], "col": N - 1, "xor": xor_mask(clean[rows[2], N - 1], NAN)},
         {"row": r1, "col": c1, "xor": 1 << 30},
         {"row": rows[3], "col": bn, "add": float("inf")}]
    return f


@pytest.mark.gpu
def test_upsets_to_inf_and_nan_are_repaired(cuda, ft, dev):
    """alpha = 1, beta = 0 (the accumulator is the clean C): every ABFT id, with the helper warp's column half, forced cut
    tiles, ROW / COL bias and protect_epilogue: detected == corrected == 5 and C bit-identical to the clean run."""
    rng = np.random.default_rng(106)
    M, N, K = 260, 388, 201
    case = Case(cuda, dev, ints(rng, (M, K)), ints(rng, (N, K)))
    bias = {ROW: np.round(10 * rng.standard_normal(M)).astype(np.float32), COL: np.round(10 * rng.standard_normal(N)).astype(np.float32)}
    bn_of = tile_n(ft)
    rows = [0, 100, 200, M - 1]  # M - 1: the ragged last row tile
    for _, kid in twins(ft):
        bn = bn_of[kid]
        dev.stats()
        clean = case.run(kid, KM, MN)
        faults = upsets(clean, bn, rows)
        assert N % bn != 0  # column N - 1 is in a ragged tile-column
        for variant in ("plain", "splitk", ROW, COL, "protect"):
            opts, mode, b = {}, NONE, None
            if variant in (ROW, COL):
                mode, b = variant, bias[variant]
            if variant == "protect":
                opts = dict(protect_epilogue=True)
            try:
                if variant == "splitk":
                    ft.debug_set("splitk", 2)
                want = case.run(kid, KM, MN, bias=b, mode=mode, opts=ft.make_opts(**opts))
                dev.stats()
                got = case.run(kid, KM, MN, bias=b, mode=mode, opts=ft.make_opts(faults=faults, **opts))
                st = dev.stats()
            finally:
                ft.debug_set("splitk", -1)
            assert st["detected"] == st["corrected"] == 5 and st["recomputed"] == st["uncorrectable"] == 0, (kid, variant, st)
            assert st["epilogue_faults"] == 0, (kid, variant, st)
            assert same_bits(got, want), (kid, variant, mismatch(got, want))
            assert np.array_equal(want, add_bias(clean, b, mode))


@pytest.mark.gpu
def test_inf_upsets_with_3xtf32_and_segments(cuda, ft, dev):
    """precision = 1 and check_segments = 4: the injected pass's accumulator is not C, so the upsets add +-Inf"""
    rng = np.random.default_rng(107)
    M, N, K = 260, 388, 201
    case = Case(cuda, dev, ints(rng, (M, K)), ints(rng, (N, K)))
    bn_of = tile_n(ft)
    for kid in (31, 16, 14):
        bn = bn_of[kid]
        faults = [{"row": 11, "col": 0, "add": float("inf")}, {"row": 150, "col": bn - 1, "add": float("-inf")},
                  {"row": M - 2, "col": N - 2, "add": float("inf")}]
        for opts in (dict(precision=1), dict(check_segments=4), dict(precision=1, check_segments=3)):
            dev.stats()
            want = case.run(kid, opts=ft.make_opts(**opts))
            assert dev.stats()["detected"] == 0
            got = case.run(kid, opts=ft.make_opts(faults=faults, **opts))
            st = dev.stats()
            assert st["detected"] == st["corrected"] == 3 and st["recomputed"] == 0, (kid, opts, st)
            assert same_bits(got, want), (kid, opts, mismatch(got, want))


# ------------------------------------------------------------------ GPU 5: isolation in a batch
@pytest.mark.gpu
def test_nonfinite_entry_is_isolated_in_a_batch(cuda, ft, dev):
    """NaN in entry 1's A and Inf in entry 1's B: entries 0 and 2 are bit-identical to single products, entry 1 is the IEEE
    result; upsets in entries 0 and 2, and in a tile-column of entry 1 without non-finite data, are corrected."""
    rng = np.random.default_rng(108)
    Bt, M, N, K = 3, 256, 512, 200
    A, B = ints(rng, (Bt, M, K)), ints(rng, (Bt, N, K))
    A[1, 5, 3] = NAN
    B[1, 7, 10] = INF
    for kid in (31, 16):
        dev.stats()
        got = run_batched(cuda, dev, kid, A, B)
        assert clean_stats(dev.stats()), kid
        for i in (0, 2):
            single = Case(cuda, dev, A[i], B[i]).run(kid, KM, KM)
            assert same_bits(got[i], single), (kid, i)
        assert not mismatch(got[1], reference(A[1], B[1])), (kid, mismatch(got[1], reference(A[1], B[1])))
        # column 300 of entry 1 is in the second tile-column (BN = 256 and 128), which holds no Inf or NaN in row 20
        faults = [{"row": 0 * M + 9, "col": 4, "xor": xor_mask(got[0, 9, 4], INF)},
                  {"row": 2 * M + 99, "col": 500, "xor": xor_mask(got[2, 99, 500], NAN)},
                  {"row": 1 * M + 20, "col": 300, "add": float("-inf")}]
        assert np.isfinite(got[1, 20, 256:]).all() and np.isfinite(got[1, 20, 300])
        dev.stats()
        fixed = run_batched(cuda, dev, kid, A, B, opts=ft.make_opts(faults=faults))
        st = dev.stats()
        assert st["detected"] == st["corrected"] == 3 and st["recomputed"] == 0, (kid, st)
        assert same_bits(fixed, got), kid


# ------------------------------------------------------------------ GPU 6: 3xTF32
@pytest.mark.gpu
def test_3xtf32_nonfinite(cuda, ft, dev):
    """opts.precision = 1 with Inf, -Inf and NaN in A and in B, next to TF32-exact and to random-normal values: the non-finite
    elements are those of FP32 on the untruncated operands, the finite ones within the element-wise bound of
    tests/test_gpu_parity.py::test_3xtf32_elementwise_fp32_parity, and nothing is detected.  Dense operands and padded
    rows take the two split kernels; a batch of two entries the batched split."""
    rng = np.random.default_rng(109)
    M, N, K = 260, 388, 201
    A = rng.standard_normal((M, K)).astype(np.float32)
    B = rng.standard_normal((N, K)).astype(np.float32)
    A[:, 12] = rng.integers(-2, 3, M)   # TF32-exact (lo = 0), zeros included, against Inf in B at k = 12
    B[40, 12], B[41, 12] = INF, -INF
    B[300, 77] = INF                    # next to random-normal A values
    B[N - 1, K - 1] = NAN
    A[8, 150] = -INF
    B[:, 150] = rng.integers(-2, 3, N)  # TF32-exact in B against Inf in A
    A[100, 0] = INF
    A[200, 199] = NAN
    want = reference(A, B, truncate=False)
    fin = np.isfinite(want)
    assert (~fin).sum() > M + N and fin.sum() > M * N // 2 and np.isnan(want).any() and np.isneginf(want).any()
    rms = float(np.sqrt(np.mean(want[fin].astype(np.float64) ** 2)))

    def check(got, tag):
        assert np.array_equal(np.isnan(got), np.isnan(want)), (tag, mismatch(got, want))
        assert np.array_equal(np.isposinf(got), np.isposinf(want)) and np.array_equal(np.isneginf(got), np.isneginf(want)), tag
        d = np.abs(got[fin].astype(np.float64) - want[fin].astype(np.float64))
        assert np.all(d <= 1e-3 * np.abs(want[fin]) + 1e-5 * rms), (tag, float(d.max()))
    case = Case(cuda, dev, A, B)
    for kid in (31, 16, ft.ID_ABFT_AUTO):
        for la, lb, pad in ((MN, MN, False), (KM, KM, False), (KM, MN, True), (MN, KM, True)):
            dev.stats()
            got = case.run(kid, la, lb, pad, opts=ft.make_opts(precision=1))
            assert clean_stats(dev.stats()), (kid, la, lb, pad)
            check(got, (kid, la, lb, pad))
    dev.stats()
    got = run_batched(cuda, dev, 31, np.stack([A, A[::-1]]), np.stack([B, B]), opts=ft.make_opts(precision=1))
    assert clean_stats(dev.stats())
    check(got[0], "batch entry 0")
    want1 = reference(A[::-1], B, truncate=False)
    assert np.array_equal(np.isnan(got[1]), np.isnan(want1)) and np.array_equal(np.isinf(got[1]), np.isinf(want1))


# ------------------------------------------------------------------ GPU 7: bias and the torch surface
@pytest.mark.gpu
def test_nonfinite_bias(cuda, ft, dev):
    """A bias holding +-Inf and NaN touches only its row or column: C is the float32 add onto the clean C, with no detection
    and no epilogue fault."""
    rng = np.random.default_rng(110)
    M, N, K = 260, 388, 201
    case = Case(cuda, dev, ints(rng, (M, K)), ints(rng, (N, K)))
    for kid in (31, 16, 12):
        clean = case.run(kid, KM, KM)
        for mode, L in ((ROW, M), (COL, N)):
            b = np.round(5 * rng.standard_normal(L)).astype(np.float32)
            b[3], b[10], b[L - 1] = INF, -INF, NAN
            for opts in ({}, dict(protect_epilogue=True)):
                dev.stats()
                got = case.run(kid, KM, KM, bias=b, mode=mode, opts=ft.make_opts(**opts))
                st = dev.stats()
                assert not mismatch(got, add_bias(clean, b, mode)), (kid, mode, opts, mismatch(got, add_bias(clean, b, mode)))
                assert clean_stats(st), (kid, mode, opts, st)
                lines = np.delete(got, [3, 10, L - 1], axis=0 if mode == ROW else 1)
                assert np.isfinite(lines).all()


@pytest.mark.gpu
def test_linear_and_bmm_with_inf_in_x(cuda, ft, dev):
    t = cuda
    rng = np.random.default_rng(111)
    M, K, N = 96, 40, 64
    x, W, b = ints(rng, (M, K)), ints(rng, (N, K)), ints(rng, N)
    x[5, 7], x[60, 0], x[61, 39] = INF, -INF, NAN
    want = add_bias(reference(x, W), b, COL)
    dev.stats()
    y = dev.linear(t.from_numpy(x).cuda(), t.from_numpy(W).cuda(), t.from_numpy(b).cuda())
    t.cuda.synchronize()
    assert not mismatch(y.cpu().numpy(), want), mismatch(y.cpu().numpy(), want)
    assert clean_stats(dev.stats())
    a = np.stack([ints(rng, (M, K)), x, ints(rng, (M, K))])
    bb = np.stack([ints(rng, (K, N)) for _ in range(3)])
    out = dev.bmm(t.from_numpy(a).cuda(), t.from_numpy(bb).cuda())
    t.cuda.synchronize()
    got = out.cpu().numpy()
    for i in range(3):
        w = reference(a[i], bb[i].T)
        assert not mismatch(got[i], w), (i, mismatch(got[i], w))
    assert clean_stats(dev.stats())
