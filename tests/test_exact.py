"""Exact, element-wise checks of every GEMM path against a float64 reference (DESIGN.md §3.1, §3.3, §4).

Operands are small integers (optionally with random bits below the TF32 mantissa, optionally scaled by powers of two per
row) chosen so that every product, every partial sum over k, every row sum over a tile width, every expected row checksum
and every stored value alpha*acc + beta*c (+ b) is an integer (or a dyadic fraction) below 2^24.  FP32 then represents
every intermediate exactly, so any correct path -- whatever its summation order, work plan, layout or tile -- returns the
float64 result bit for bit at every element, and every ABFT row check closes with a residual d1 = r1 - s1 of exactly zero.
A dropped, duplicated or misplaced k-block, tile, row or column, a leak between batch entries, or a rounding that should not
happen is a nonzero difference.  `budget` states the worst-case magnitudes; the generators refuse what exceeds 2^24.

Where the data cannot be exact (standard-normal operands), the rounding tier checks every element against a worst-case
bound of truncating FP32 accumulation instead.
"""
import contextlib

import numpy as np
import pytest

MN, KM = 0, 1
NONE, ROW, COL = 0, 1, 2
RELU, GELU = 1, 2
NAMES = ["small", "medium", "large", "tall", "wide", "huge", "giant", "pair128"]
LIMIT = 1 << 24          # every integer of magnitude <= 2^24 is an FP32 value, and so is every partial sum below it
ENC_LIMIT = 1 << 11      # a column-block sum E = sum_n b of at most 2^11 is TF32-exact: the encode's lo plane is zero
DYADIC = (0.0, 0.5, -0.5, 1.0, -1.0, 2.0, -2.0, 0.75, -0.75)
SENTINEL = -12345.5
Z_SENTINEL = 7777.25
GELU_ULP = 2
TOL_MODEL = 5e-5         # the suite's norm-wise bound against the TF32 model (tests/test_gpu_parity.py)


# ------------------------------------------------------------------ exact-data helpers (no GPU)
def frac_bits(x, most=8):
    """number of fractional bits of the dyadic value x (0.75 -> 2), None if x needs more than `most`"""
    for f in range(most + 1):
        v = float(x) * (1 << f)
        if v == int(v):
            return f
    return None


def budget(K, BN, amax, bmax, alpha=1.0, beta=0.0, cmax=0.0, bias_max=0.0):
    """Worst-case magnitudes of one product with |a| <= amax, |b| <= bmax, |C0| <= cmax, |bias| <= bias_max:
      acc       every accumulator element, K * amax * bmax;
      rowsum    every row sum over a tile width BN (the check's s1);
      checksum  every expected row checksum sum_k a * E_k with E_k = sum_{n in tile} b (the check's r1);
      encode    every column-block sum E_k (must stay TF32-exact: <= 2^11);
      out       every stored alpha * acc + beta * c (+ b), in units of the finest fraction of alpha and beta.
    All must be <= 2^24 for the data to be exact; alpha and beta must be dyadic (None in 'out' otherwise)."""
    acc = K * amax * bmax
    f = [frac_bits(alpha), frac_bits(beta)]
    out = None if None in f else (abs(alpha) * acc + abs(beta) * cmax + bias_max) * (1 << max(f))
    return {"acc": acc, "rowsum": BN * acc, "checksum": K * amax * BN * bmax, "encode": BN * bmax, "out": out}


def refusal(K, BN, amax, bmax, alpha=1.0, beta=0.0, cmax=0.0, bias_max=0.0):
    """'' when the parameter set is exact, else why not"""
    b = budget(K, BN, amax, bmax, alpha, beta, cmax, bias_max)
    if b["out"] is None:
        return f"alpha {alpha} / beta {beta} not dyadic"
    if b["encode"] > ENC_LIMIT:
        return f"column-block sum {b['encode']} > 2^11 (not TF32-exact)"
    over = [k for k in ("acc", "rowsum", "checksum", "out") if b[k] > LIMIT]
    return f"{', '.join(over)} above 2^24: {b}" if over else ""


def pick_amax(K, BN, alpha=1.0, beta=0.0, cmax=0.0, bias_max=0.0, choices=(8, 4, 2, 1)):
    """the widest integer range [-a, a] (for A and B alike) that keeps the set exact"""
    for a in choices:
        if not refusal(K, BN, a, a, alpha, beta, cmax, bias_max):
            return a
    raise ValueError(refusal(K, BN, 1, 1, alpha, beta, cmax, bias_max))


def tf32(x):
    """the tensor core's operand truncation: clear the 13 low mantissa bits (the int32 & -8192 view)"""
    return (x.contiguous().view(dtype=_torch().int32) & -8192).view(dtype=_torch().float32)


def _torch():
    import torch
    return torch


def ints(g, shape, amax, device, garbage=False):
    """integers in [-amax, amax] as float32; garbage: random bits in the 13 low mantissa bits of every nonzero value, so
    tf32(x) is still the integer"""
    t = _torch()
    x = t.randint(-amax, amax + 1, shape, generator=g, device=device, dtype=t.int32).float()
    return with_garbage(g, x) if garbage else x


def with_garbage(g, x):
    t = _torch()
    bits = t.randint(0, 1 << 13, x.shape, generator=g, device=x.device, dtype=t.int32)
    return t.where(x != 0, (x.view(dtype=t.int32) | bits).view(dtype=t.float32), x)


def scale_rows(g, x, spread):
    """x with row i multiplied by 2^e_i, e_i uniform in [-spread, spread] (exact: a power of two)"""
    t = _torch()
    e = t.randint(-spread, spread + 1, (x.shape[0], 1), generator=g, device=x.device, dtype=t.int32)
    return t.ldexp(x, e.float()).float()


def reference(A, B, alpha=1.0, beta=0.0, C0=None, bias=None, mode=NONE, truncate=True):
    """float64 alpha * A~ * B~^T + beta * C0 (+ bias) with A~, B~ the TF32-truncated operands (A: M x K, B: N x K); C0 is not
    read when beta == 0"""
    a = (tf32(A) if truncate else A).double()
    b = (tf32(B) if truncate else B).double()
    out = alpha * (a @ b.T)
    if beta != 0.0:
        out = out + beta * C0.double()
    if mode == ROW:
        out = out + bias.double()[:, None]
    elif mode == COL:
        out = out + bias.double()[None, :]
    return out


def mismatch(got, want, show=4):
    """'' when got (float32) equals want (float64) at every element (NaN == NaN, +0 == -0); otherwise the count and the
    first few (m, n, got, want)"""
    t = _torch()
    if tuple(got.shape) != tuple(want.shape):
        return f"shape {tuple(got.shape)} != {tuple(want.shape)}"
    g = got.double()
    bad = (g != want) & ~(t.isnan(g) & t.isnan(want))
    n = int(bad.sum())
    if n == 0:
        return ""
    idx = bad.nonzero()[:show].tolist()
    return f"{n} elements differ, e.g. " + ", ".join(
        f"{tuple(i)}: got {float(got[tuple(i)])!r} want {float(want[tuple(i)])!r}" for i in idx)


def pad4(n):
    return (n + 3) // 4 * 4


def ld_of(layout, rows, K, pad):
    base = rows if layout == MN else pad4(K)
    return base + 4 if pad else base


def pack(X, layout, ld):
    """rows x K matrix -> flat buffer in the layout (MN: X[r, k] at r + k*ld; KM: at k + r*ld), padding = NaN"""
    t = _torch()
    rows, K = X.shape
    if layout == MN:
        buf = t.full((K, ld), float("nan"), device=X.device)
        buf[:, :rows] = X.T
    else:
        buf = t.full((rows, ld), float("nan"), device=X.device)
        buf[:, :K] = X
    return buf.reshape(-1)


def fuzz_case(seed):
    """the parameters of one seeded exact fuzz case (no GPU): shape, variant, layouts, alpha/beta, entry point, knobs"""
    rng = np.random.default_rng(7000 + seed)
    p = {"seed": seed, "M": int(rng.integers(1, 200)) * 4, "N": int(rng.integers(1, 200)) * 4,
         "K": int(rng.choice([int(rng.integers(1, 64)), int(rng.integers(1, 1500))])),
         "name": NAMES[seed % len(NAMES)], "la": int(rng.integers(0, 2)), "lb": int(rng.integers(0, 2)),
         "pad": bool(rng.integers(0, 2)), "alpha": float(rng.choice(DYADIC)), "beta": float(rng.choice([0.0, 1.0, -0.5, 2.0])),
         "entry": ["run_ex", "run_bias_row", "run_bias_col", "run_act_relu", "batched"][seed % 5],
         "garbage": bool(rng.integers(0, 2)),
         "knobs": {"splitk": int(rng.choice([-1, 0, 2, 3])), "wave_sync": int(rng.choice([0, 1])), "pdl": int(rng.choice([0, 1])),
                   "epi_assist": int(rng.choice([0, 1])), "chk_slices": int(rng.choice([1, 2, 3])),
                   "enc_front": int(rng.choice([0, 1]))}}
    p["cmax"] = 0 if p["beta"] == 0.0 else 64
    p["bias_max"] = 64 if p["entry"] != "run_ex" else 0
    p["amax"] = pick_amax(p["K"], 256, p["alpha"], p["beta"], p["cmax"], p["bias_max"])
    return p


# ------------------------------------------------------------------ CPU tests of the helpers
def test_budget_refuses_sets_that_would_round():
    assert not refusal(16384, 256, 2, 2)                       # ints in [-2, 2] up to K = 16384 at BN = 256
    assert not refusal(65536, 256, 1, 1)                       # {-1, 0, 1} up to K = 65536
    assert budget(16384, 256, 2, 2)["checksum"] == LIMIT       # ... with no room left
    assert "checksum" in refusal(16384 + 4, 256, 2, 2)
    assert "checksum" in refusal(65536 + 4, 256, 1, 1)
    # what is refused would round: an odd integer of that size is not an FP32 value
    worst = budget(16384 + 4, 256, 2, 2)["checksum"] - 1
    assert float(np.float32(worst)) != worst
    assert float(np.float32(LIMIT - 1)) == LIMIT - 1 and float(np.float32(LIMIT)) == LIMIT
    # the encode's lo plane: E = sum_n b over 256 columns of |b| <= 8 is exact, of |b| <= 16 is not TF32-exact
    assert not refusal(8, 256, 8, 8) and "2^11" in refusal(8, 256, 16, 16)
    # alpha and beta: dyadic only, and a fraction costs bits of the budget
    assert "dyadic" in refusal(16, 64, 2, 2, alpha=0.1) and "dyadic" in refusal(16, 64, 2, 2, beta=1.0 / 3.0)
    for a in DYADIC:
        assert not refusal(1000, 256, 2, 2, alpha=a, beta=-0.75, cmax=1000, bias_max=100), a
    assert not refusal(8192, 256, 2, 2, alpha=1.0) and "out" in refusal(8192, 256, 2, 2, alpha=0.75, beta=0.75, cmax=LIMIT // 2)
    assert pick_amax(2088, 256) == 4 and pick_amax(16384, 256) == 2 and pick_amax(65536, 256) == 1
    with pytest.raises(ValueError):
        pick_amax(65540, 256)


def test_garbage_operands_truncate_to_the_integers():
    t = _torch()
    g = t.Generator().manual_seed(1)
    x = ints(g, (64, 64), 8, "cpu")
    y = with_garbage(g, x)
    assert t.equal(tf32(y).view(dtype=t.int32), x.view(dtype=t.int32))         # bit for bit, signs of zero included
    nz = x != 0
    assert bool((y[nz] != x[nz]).float().mean() > 0.99) and t.equal(y[~nz], x[~nz])
    assert float((y - x).abs().max()) < 8 * 2.0 ** -10                          # below the TF32 mantissa
    # scaled rows stay exact, and so does their truncation
    s = scale_rows(g, y, 40)
    ratio = tf32(s).double() / x.double()
    r = ratio[nz.all(1)]
    assert bool((r == r[:, :1]).all()) and bool((t.log2(r[:, 0]) == t.log2(r[:, 0]).round()).all())


def test_reference_equals_numpy_einsum():
    t = _torch()
    rng = np.random.default_rng(3)
    for M, N, K in ((4, 8, 1), (12, 20, 33), (36, 4, 70)):
        A = rng.standard_normal((M, K)).astype(np.float32)
        B = rng.standard_normal((N, K)).astype(np.float32)
        C0 = rng.standard_normal((M, N)).astype(np.float32)
        bias = rng.standard_normal(M).astype(np.float32)
        at = (A.view(np.uint32) & np.uint32(0xFFFFE000)).view(np.float32).astype(np.float64)
        bt = (B.view(np.uint32) & np.uint32(0xFFFFE000)).view(np.float32).astype(np.float64)
        want = -0.75 * np.einsum("mk,nk->mn", at, bt, optimize=False) + 2.0 * C0 + bias[:, None]
        got = reference(t.from_numpy(A), t.from_numpy(B), -0.75, 2.0, t.from_numpy(C0), t.from_numpy(bias), ROW).numpy()
        assert np.allclose(got, want, rtol=1e-13, atol=1e-13)
        want_u = np.einsum("mk,nk->mn", A.astype(np.float64), B.astype(np.float64), optimize=False)
        got_u = reference(t.from_numpy(A), t.from_numpy(B), truncate=False).numpy()
        assert np.allclose(got_u, want_u, rtol=1e-13, atol=1e-13)
        # C0 is not read when beta == 0
        nan = t.full((M, N), float("nan"))
        assert not t.isnan(reference(t.from_numpy(A), t.from_numpy(B), 1.0, 0.0, nan)).any()


def test_mismatch_reports_elements():
    t = _torch()
    want = t.arange(12, dtype=t.float64).reshape(3, 4)
    got = want.float().clone()
    assert mismatch(got, want) == ""
    got[2, 1] += 1
    got[0, 3] = -0.0 if want[0, 3] == 0 else got[0, 3]
    msg = mismatch(got, want)
    assert msg.startswith("1 elements differ") and "(2, 1)" in msg
    assert mismatch(t.tensor([0.0, float("nan")]), t.tensor([-0.0, float("nan")], dtype=t.float64)) == ""


def test_fuzz_cases_are_within_budget():
    for seed in range(40):
        p = fuzz_case(seed)
        assert not refusal(p["K"], 256, p["amax"], p["amax"], p["alpha"], p["beta"], p["cmax"], p["bias_max"]), p
        assert p["M"] % 4 == 0 and p["N"] % 4 == 0 and p["K"] >= 1
    assert {fuzz_case(s)["entry"] for s in range(40)} == {"run_ex", "run_bias_row", "run_bias_col", "run_act_relu", "batched"}
    assert 0.0 in {fuzz_case(s)["alpha"] for s in range(40)}


# ------------------------------------------------------------------ GPU harness
@pytest.fixture(scope="module")
def dev(cuda, ft):
    cuda.cuda.set_device(0)
    h = ft.FtSgemm()
    yield h
    h.close()


@contextlib.contextmanager
def knobs(ft, **kv):
    try:
        for k, v in kv.items():
            ft.debug_set(k, v)
        yield
    finally:
        for k in kv:
            ft.debug_set(k, -1)


def tiles(ft):
    """id -> (rows, columns) of its work unit"""
    return {k["id"]: k["tile"][:2] for k in ft.kernel_table()}


def abft_ids(ft):
    return set(ft.ABFT_IDS.values()) | {ft.ID_ABFT_AUTO}


class Prod:
    """One product on the GPU: A (M x K), B (N x K) float32 device tensors, packed per layout on demand."""

    def __init__(self, t, A, B):
        self.t, self.A, self.B = t, A, B
        self.M, self.K = A.shape
        self.N = B.shape[0]
        self._ops = {}

    def op(self, which, layout, ld):
        key = (which, layout, ld)
        if key not in self._ops:
            self._ops[key] = pack(self.A if which == "a" else self.B, layout, ld)
        return self._ops[key]

    def run(self, dev, kid, la=KM, lb=KM, pad=False, ldc=None, alpha=1.0, beta=0.0, C0=None, bias=None, mode=NONE,
            act=None, z=False, opts=None):
        """run_bias (act None) or run_act; returns (C, Z) as M x N views (Z None unless z) and checks C's and Z's padding"""
        t, M, N, K = self.t, self.M, self.N, self.K
        lda, ldb, ldc = ld_of(la, M, K, pad), ld_of(lb, N, K, pad), ldc or M
        cbuf = t.full((N, ldc), SENTINEL, device="cuda")
        cbuf[:, :M] = 0.0 if C0 is None else C0.T
        zbuf = t.full((N, ldc), Z_SENTINEL, device="cuda") if z else None
        dA, dB = self.op("a", la, lda), self.op("b", lb, ldb)
        if act is None:
            dev.run_bias(kid, M, N, K, dA, la, lda, dB, lb, ldb, cbuf, ldc, alpha, beta, bias, mode, opts)
        else:
            dev.run_act(kid, M, N, K, dA, la, lda, dB, lb, ldb, cbuf, ldc, alpha, beta, bias, mode, act, zbuf, opts)
        t.cuda.synchronize()
        if ldc > M:
            assert bool((cbuf[:, M:] == SENTINEL).all()), "C's padding was written"
            if z:
                assert bool((zbuf[:, M:] == Z_SENTINEL).all()), "Z's padding was written"
        return cbuf[:, :M].t(), (zbuf[:, :M].t() if z else None)


def pack_batch(X, layout, ld):
    """(Bt, rows, K) -> (flat buffer, entry stride): each entry packed as `pack` packs it, padding = NaN"""
    t = _torch()
    Bt, rows, K = X.shape
    if layout == MN:
        buf = t.full((Bt, K, ld), float("nan"), device=X.device)
        buf[:, :, :rows] = X.transpose(1, 2)
    else:
        buf = t.full((Bt, rows, ld), float("nan"), device=X.device)
        buf[:, :, :K] = X
    return buf.reshape(-1), buf[0].numel()


def run_batched(t, dev, kid, A, B, alpha=1.0, beta=0.0, C0=None, bias=None, mode=NONE, act=None, z=False, opts=None,
                la=KM, lb=KM, pad=False):
    """A (Bt, M, K), B (Bt, N, K) in the layouts la / lb (leading dimensions of ld_of, padding NaN), C (Bt, M, N) column-major
    per entry, one bias per entry (Bt, len) or None; one run_batched_act call.  Returns (C, Z) as (Bt, M, N) views."""
    Bt, M, K = A.shape
    N = B.shape[1]
    lda, ldb = ld_of(la, M, K, pad), ld_of(lb, N, K, pad)
    dA, sa = pack_batch(A, la, lda)
    dB, sb = pack_batch(B, lb, ldb)
    dC = (t.zeros(Bt, N, M, device="cuda") if C0 is None else C0.transpose(1, 2).contiguous())
    dZ = t.full((Bt, N, M), Z_SENTINEL, device="cuda") if z else None
    sbias = 0 if bias is None else bias.shape[1]
    dev.run_batched_act(kid, M, N, K, dA, la, lda, sa, dB, lb, ldb, sb, dC, M, M * N, Bt, alpha, beta, bias, mode, sbias,
                        act or 0, dZ, opts)
    t.cuda.synchronize()
    return dC.transpose(1, 2), (dZ.transpose(1, 2) if z else None)


def batched_reference(A, B, alpha=1.0, beta=0.0, C0=None, bias=None, mode=NONE):
    t = _torch()
    out = alpha * t.bmm(tf32(A).double(), tf32(B).double().transpose(1, 2))
    if beta != 0.0:
        out = out + beta * C0.double()
    if mode == ROW:
        out = out + bias.double()[:, :, None]
    elif mode == COL:
        out = out + bias.double()[:, None, :]
    return out


def zero_residual(st, kid, ft, tag):
    """the zero-residual rule of exact data: nothing detected, counted or repaired, every row check closes exactly"""
    assert st["detected"] == 0 and st["recomputed"] == 0 and st["epilogue_faults"] == 0 and not st["events"], (tag, st)
    if kid in abft_ids(ft):
        assert st["rows_checked"] > 0 and st["max_abs_residual"] == 0.0, (tag, st)


def exact(got, want, tag):
    msg = mismatch(got, want)
    assert not msg, f"{tag}: {msg}"


# ------------------------------------------------------------------ GPU 1: tile edges
def sweep(ft, kid, seed):
    """a seeded pairwise subset of the tile-edge grid of one id: every M, every N and every K value at least once, each
    with a layout pair, padded or not, an ldc > M or not, a splitk setting and alpha / beta"""
    tm, tn = tiles(ft)[kid]
    Ms = [4, tm - 4, tm, tm + 4, 2 * tm + 4]
    Ns = sorted({4, max(4, tn - 36), max(4, tn - 28), tn - 4, tn, tn + 4, tn + 28})
    Ks = [1, 3, 4, 31, 32, 33, 127, 129, 1000, 2088]
    rng = np.random.default_rng(seed)
    n = max(len(Ms), len(Ns), len(Ks))
    off = int(rng.integers(0, 30))   # the layout / alpha / splitk pairing differs between variants as well
    cols = [rng.permutation(np.resize(v, n)) for v in (Ms, Ns, Ks)]
    ab = [(1.0, 0.0), (0.5, 0.0), (-2.0, 1.0), (0.0, -0.5), (0.75, 2.0)]
    for j in range(n):
        i = j + off
        yield {"M": int(cols[0][j]), "N": int(cols[1][j]), "K": int(cols[2][j]), "la": i % 2, "lb": (i // 2) % 2,
               "pad": i % 3 != 0, "ldc": i % 2 == 1, "splitk": (-1, 0, 2)[i % 3], "ab": ab[i % len(ab)],
               "garbage": i % 2 == 0}


@pytest.mark.gpu
@pytest.mark.parametrize("name", NAMES + ["auto"])
def test_tile_edges_exact(cuda, ft, dev, name):
    """Every named variant, plain and ABFT (ids 20 / 40 for 'auto'), at M, N and K around the tile edges, all four layout
    pairs, padded leading dimensions (NaN padding), ldc > M (sentinel untouched), splitk -1 / 0 / 2, dyadic alpha / beta
    (alpha = 0 included) with an integer C0: C equals the float64 reference at every element, and every ABFT row check
    closes with a residual of exactly zero."""
    t = cuda
    pair = (ft.ID_SGEMM_AUTO, ft.ID_ABFT_AUTO) if name == "auto" else (ft.SGEMM_IDS[name], ft.ABFT_IDS[name])
    tile_of = tiles(ft)
    g = t.Generator(device="cuda").manual_seed(11 + NAMES.index(name) if name in NAMES else 19)
    for c in sweep(ft, pair[1] if name != "auto" else 31, 100 + (NAMES + ["auto"]).index(name)):
        M, N, K = c["M"], c["N"], c["K"]
        alpha, beta = c["ab"]
        amax = pick_amax(K, 256, alpha, beta, 64)
        A, B = ints(g, (M, K), amax, "cuda", c["garbage"]), ints(g, (N, K), amax, "cuda", c["garbage"])
        C0 = ints(g, (M, N), 64, "cuda")
        want = reference(A, B, alpha, beta, C0)
        p = Prod(t, A, B)
        for kid in pair:
            tag = (kid, tile_of.get(kid), c)
            with knobs(ft, splitk=c["splitk"]):
                dev.stats()
                got, _ = p.run(dev, kid, c["la"], c["lb"], c["pad"], M + 8 if c["ldc"] else None, alpha, beta, C0)
                st = dev.stats()
            exact(got, want, tag)
            zero_residual(st, kid, ft, tag)


@pytest.mark.gpu
def test_power_of_two_scaling_exact(cuda, ft, dev):
    """Rows of A scaled by 2^r (r in [-40, 40]), with garbage low bits: every term of C(m, n) has the same scale, so C is exact
    and every row check still closes with zero residual.

    Rows of A and of B scaled together (2^(r_m + s_n)): C is still exact, but a tile row now mixes scales, so its row sum and
    its expected checksum round.  With mixed-sign operands a row whose largest-scale element happens to be small or zero
    has a threshold (relative to sum_n |acc|) below that rounding, and the check can flag it (DESIGN.md §4): the plain ids
    and detect_only are exact, and with repairs on nothing but flagged rows may change (at most one element each).  With
    operands of one sign no row sum cancels, and nothing is flagged."""
    t = cuda
    g = t.Generator(device="cuda").manual_seed(51)
    M, N, K = 516, 388, 301
    A = scale_rows(g, ints(g, (M, K), 4, "cuda", True), 40)
    B = ints(g, (N, K), 4, "cuda", True)
    p = Prod(t, A, B)
    want = reference(A, B, -0.5)
    for kid in (31, 16, 12, 21, 6):
        for la, lb in ((MN, KM), (KM, MN)):
            dev.stats()
            got, _ = p.run(dev, kid, la, lb, alpha=-0.5)
            exact(got, want, (kid, la, lb, "2^r"))
            zero_residual(dev.stats(), kid, ft, (kid, la, lb, "2^r"))
    A2 = scale_rows(g, ints(g, (M, K), 2, "cuda", True), 40)
    B2 = scale_rows(g, ints(g, (N, K), 2, "cuda", True), 40)
    p2 = Prod(t, A2, B2)
    want = reference(A2, B2)
    flagged, changed = {}, {}
    for plain, kid in ((21, 31), (6, 16), (2, 12)):
        for la, lb in ((MN, MN), (KM, KM)):
            got, _ = p2.run(dev, plain, la, lb)
            exact(got, want, (plain, la, lb, "2^r 2^s"))
            dev.stats()
            got, _ = p2.run(dev, kid, la, lb, opts=ft.make_opts(detect_only=True))
            st = dev.stats()
            exact(got, want, (kid, la, lb, "2^r 2^s, detect_only"))
            flagged[kid] = flagged.get(kid, 0) + st["detected"]
            got, _ = p2.run(dev, kid, la, lb)
            st2 = dev.stats()
            bad = int((got.double() != want).sum())
            assert st2["detected"] == st["detected"] and bad <= st2["detected"], (kid, la, lb, bad, st2)
            changed[kid] = changed.get(kid, 0) + bad
    print("2^r 2^s scaling, mixed signs: rows flagged", flagged, "elements changed by a repair", changed)
    A3 = scale_rows(g, ints(g, (M, K), 2, "cuda").abs() + 1.0, 40)
    B3 = scale_rows(g, ints(g, (N, K), 2, "cuda").abs() + 1.0, 40)
    p2 = Prod(t, A3, B3)
    want = reference(A3, B3)
    for kid in (31, 16, 12):
        for la, lb in ((MN, MN), (KM, KM)):
            dev.stats()
            got, _ = p2.run(dev, kid, la, lb)
            st = dev.stats()
            exact(got, want, (kid, la, lb, "2^r 2^s, one sign"))
            assert st["detected"] == 0 and st["rows_checked"] > 0, (kid, la, lb, st)


# ------------------------------------------------------------------ GPU 2: production sizes, whole output
def _free(t):
    t.cuda.synchronize()
    t.cuda.empty_cache()


def _whole(t, dev, ft, M, N, K, ids, amax, seed, garbage=False, beta=0.0, saturate=False):
    g = t.Generator(device="cuda").manual_seed(seed)
    dA = ints(g, (K, M), amax, "cuda", garbage)          # MN-major A: A(m, k) at m + k*M
    dB = ints(g, (K, N), amax, "cuda", garbage)
    if saturate:  # row 0 of A and the first 256 columns of B all amax: acc(0, n < 256) = K * amax^2, r1 = s1 = 2^24 there
        dA[:, 0] = amax
        dB[:, :256] = amax
    C0 = ints(g, (N, M), 64, "cuda") if beta != 0.0 else None   # column-major C
    want = (tf32(dA).double().T @ tf32(dB).double()).T           # (N, M): column-major C
    if beta != 0.0:
        want += beta * C0.double()
    for kid in ids:
        dC = C0.clone() if C0 is not None else t.zeros(N, M, device="cuda")
        dev.stats()
        dev.run(kid, M, N, K, dA, dB, dC, 1.0, beta, None)
        t.cuda.synchronize()
        st = dev.stats()
        tag = (kid, M, N, K, garbage, beta)
        bad = int((dC.double() != want).sum())
        assert bad == 0, (tag, mismatch(dC.T, want.T))
        zero_residual(st, kid, ft, tag)
        del dC
    del dA, dB, C0, want
    _free(t)


@pytest.mark.gpu
@pytest.mark.slow
def test_production_sizes_whole_output(cuda, ft, dev):
    """The sizes the project is measured at, every output element against float64: 4096^3 (ids 6, 16, 15, 21, 31, 40 and
    cuBLAS-TF32 7 as an independent witness of exact FP32 accumulation), 8192^3 (21, 31, 16), 16384^3 (id 31: the wave
    re-synchronisation path), and deep K at the planner's own choices (split-K head, checksum K-slices) with a row whose
    checksum reaches 2^24; garbage low bits and beta != 0 with an integer C0.  Peak device memory ~10 GB."""
    t = cuda
    _whole(t, dev, ft, 4096, 4096, 4096, (6, 16, 15, 21, 31, 40, ft.ID_CUBLAS_TF32), 2, 1)
    _whole(t, dev, ft, 4096, 4096, 4096, (31, 16), 2, 2, garbage=True)
    _whole(t, dev, ft, 8192, 8192, 8192, (21, 31, 16), 2, 3)
    _whole(t, dev, ft, 8192, 8192, 8192, (31,), 2, 4, beta=-1.0)
    _whole(t, dev, ft, 16384, 16384, 16384, (31,), 2, 5)
    _whole(t, dev, ft, 256, 256, 65536, (31, 40, 16, ft.ID_CUBLAS_TF32), 1, 6, saturate=True)
    _whole(t, dev, ft, 512, 1024, 32768, (31, 40, 16), 1, 7, garbage=True)
    _whole(t, dev, ft, 512, 1024, 32768, (31,), 1, 8, beta=2.0)


@pytest.mark.gpu
def test_cublas_tf32_does_not_truncate(cuda, ft, dev):
    """cuBLAS-TF32 (id 7) does not drop the low mantissa bits as this library's tensor-core path does: on integers with
    garbage low bits it is not the product of the truncated operands (the fused ids are, test_production_sizes_whole_output),
    but it stays within TF32's rounding of the untruncated product, (K + 8) 2^-22 + 2^-10 of |A| |B|^T.  So it witnesses
    exact accumulation on TF32-exact operands only."""
    t = cuda
    g = t.Generator(device="cuda").manual_seed(9)
    M = N = K = 2048
    dA, dB = ints(g, (K, M), 2, "cuda", True), ints(g, (K, N), 2, "cuda", True)
    dC = t.zeros(N, M, device="cuda")
    dev.run(ft.ID_CUBLAS_TF32, M, N, K, dA, dB, dC, 1.0, 0.0, None)
    t.cuda.synchronize()
    want = (tf32(dA).double().T @ tf32(dB).double()).T
    assert float((dC.double() != want).float().mean()) > 0.5
    bound = ((K + 8) * 2.0 ** -22 + 2.0 ** -10) * (dA.double().abs().T @ dB.double().abs()).T
    assert bool(((dC.double() - (dA.double().T @ dB.double()).T).abs() <= bound).all())


# ------------------------------------------------------------------ GPU 3: every entry point
SHAPES = ((260, 388, 201), (512, 512, 256))   # ragged multi-tile, full tiles


@pytest.mark.gpu
@pytest.mark.parametrize("shape", SHAPES)
def test_entry_points_exact(cuda, ft, dev, shape):
    """run_bias ROW / COL, run_act (ReLU exact, Z exact, GELU within the ulp rule of gelu(Z)), precision = 1,
    check_segments 2 / 3 / 20, protect_epilogue 1 / 2, reuse_b_checksums, run_host, cuBLAS 0 / 7 and the baseline 10 / 30:
    exact on integer data, every ABFT check closing with zero residual."""
    t = cuda
    M, N, K = shape
    g = t.Generator(device="cuda").manual_seed(M + K)
    A, B = ints(g, (M, K), 4, "cuda"), ints(g, (N, K), 4, "cuda")
    C0 = ints(g, (M, N), 64, "cuda")
    bias = {ROW: ints(g, (M,), 64, "cuda"), COL: ints(g, (N,), 64, "cuda")}
    p = Prod(t, A, B)
    for kid in (31, 16, 12, 14, 40):
        for mode in (ROW, COL):
            for alpha, beta in ((1.0, 0.0), (-0.5, 2.0)):
                want = reference(A, B, alpha, beta, C0, bias[mode], mode)
                dev.stats()
                got, _ = p.run(dev, kid, MN, KM, True, M + 4, alpha, beta, C0, bias[mode], mode)
                exact(got, want, (kid, mode, alpha, beta))
                zero_residual(dev.stats(), kid, ft, (kid, mode))
                for act in (RELU, GELU):
                    dev.stats()
                    c, z = p.run(dev, kid, KM, MN, False, None, alpha, beta, C0, bias[mode], mode, act, True)
                    zero_residual(dev.stats(), kid, ft, (kid, mode, act))
                    exact(z, want, (kid, mode, act, "Z"))
                    if act == RELU:
                        exact(c, t.relu(want), (kid, mode, "relu"))
                    else:
                        ref = t.nn.functional.gelu(z)
                        assert t.equal(t.isfinite(c), t.isfinite(ref))
                        key = lambda x: t.where(x.view(dtype=t.int32) < 0, -(x.view(dtype=t.int32) & 0x7FFFFFFF),
                                                x.view(dtype=t.int32)).long()
                        assert int((key(c.contiguous()) - key(ref.contiguous())).abs().max()) <= GELU_ULP, (kid, mode)
        want = reference(A, B, 0.75, -1.0, C0)
        for opts in (dict(precision=1), dict(check_segments=2), dict(check_segments=3), dict(check_segments=20),
                     dict(precision=1, check_segments=3), dict(protect_epilogue=1), dict(protect_epilogue=2),
                     dict(protect_epilogue=2, precision=1)):
            dev.stats()
            got, _ = p.run(dev, kid, KM, KM, False, None, 0.75, -1.0, C0, opts=ft.make_opts(**opts))
            exact(got, want, (kid, opts))
            zero_residual(dev.stats(), kid, ft, (kid, opts))
        # reuse_b_checksums: the second call encodes nothing and still closes every check exactly
        for reuse in (False, True):
            dev.stats()
            got, _ = p.run(dev, kid, KM, KM, opts=ft.make_opts(reuse_b_checksums=reuse))
            exact(got, reference(A, B), (kid, "reuse", reuse))
            zero_residual(dev.stats(), kid, ft, (kid, "reuse", reuse))
    # the cuBLAS ids (FP32 and TF32) and the non-fused baseline (FP32 and TF32): reference layout only
    want = reference(A, B, 0.5, 1.0, C0)
    for kid in (ft.ID_CUBLAS, ft.ID_CUBLAS_TF32, ft.ID_ABFT_BASELINE, ft.ID_ABFT_BASELINE_TF32):
        got, _ = p.run(dev, kid, MN, MN, False, None, 0.5, 1.0, C0)
        exact(got, want, kid)
    dev.stats()
    # run_host: column-major host buffers
    hA = A.T.contiguous().cpu().numpy().reshape(-1)
    hB = B.T.contiguous().cpu().numpy().reshape(-1)
    for kid in (31, 16, ft.ID_CUBLAS):
        hC = C0.T.contiguous().cpu().numpy().reshape(-1).copy()
        dev.stats()
        dev.run_host(kid, M, N, K, hA, hB, hC, -2.0, 0.5)
        zero_residual(dev.stats(), kid, ft, (kid, "run_host"))
        exact(t.from_numpy(hC.reshape(N, M).T.copy()).cuda(), reference(A, B, -2.0, 0.5, C0), (kid, "run_host"))


@pytest.mark.gpu
def test_batched_exact(cuda, ft, dev):
    """run_batched_act with a per-entry bias: M not a multiple of the tile (rows past M must not leak into the next entry),
    batch 1 / 2 / 7, ReLU with Z; and 65537 tiny entries (4 x 4 x 6, rows padded to 8 or 12), past the 65535 grid rows of
    the encode pre-pass (B below the front-phase encode's 8 MiB, and forced with enc_front = 0) and of the strided 3xTF32
    split kernel (padded rows): every entry exact, in both layouts of B."""
    t = cuda
    g = t.Generator(device="cuda").manual_seed(21)
    for kid in (31, 16, 13):
        for Bt, (M, N, K) in ((1, (260, 388, 201)), (2, (132, 260, 96)), (7, (260, 132, 129))):
            A, B = ints(g, (Bt, M, K), 4, "cuda"), ints(g, (Bt, N, K), 4, "cuda")
            C0 = ints(g, (Bt, M, N), 64, "cuda")
            for mode, L in ((ROW, M), (COL, N)):
                bias = ints(g, (Bt, L), 64, "cuda")
                want = batched_reference(A, B, -1.0, 0.5, C0, bias, mode)
                dev.stats()
                c, z = run_batched(t, dev, kid, A, B, -1.0, 0.5, C0, bias, mode, RELU, True)
                zero_residual(dev.stats(), kid, ft, (kid, Bt, mode))
                exact(z, want, (kid, Bt, mode, "Z"))
                exact(c, t.relu(want), (kid, Bt, mode, "C"))
    Bt, M, N, K = 65537, 4, 4, 6
    assert 4 * N * K * Bt < 8 << 20   # below the size from which B is encoded in the GEMM kernel's front phase
    A, B = ints(g, (Bt, M, K), 8, "cuda"), ints(g, (Bt, N, K), 8, "cuda")
    Bg = with_garbage(g, B)   # 3xTF32 would see these bits (its lo parts): it runs on B itself
    bias = ints(g, (Bt, N), 64, "cuda")
    want = batched_reference(A, B, 1.0, 0.0, None, bias, COL)
    for kid, opts, b, lb, pad in ((31, {}, Bg, KM, False), (16, {}, Bg, MN, True), (31, dict(precision=1), B, KM, False),
                                  (16, dict(precision=1), B, MN, True), (ft.ID_ABFT_AUTO, dict(protect_epilogue=2), Bg, KM, True)):
        for front in (-1, 0):
            with knobs(ft, enc_front=front):
                dev.stats()
                c, _ = run_batched(t, dev, kid, A, b, bias=bias, mode=COL, opts=ft.make_opts(**opts), lb=lb, pad=pad)
                st = dev.stats()
            zero_residual(st, kid, ft, (kid, Bt, opts, lb, pad, front))
            assert st["rows_checked"] >= Bt * M, st
            exact(c, want, (kid, Bt, opts, lb, pad, front))
    del A, B, Bg, bias, want
    _free(t)


@pytest.mark.gpu
def test_torch_surface_exact(cuda, ft, dev):
    """matmul, linear (with ReLU) and bmm (per-entry bias), forward and backward: with integer data and an integer grad_y
    every output and gradient equals float64 torch autograd bit for bit."""
    t = cuda
    g = t.Generator(device="cuda").manual_seed(31)
    dev.stats()
    # matmul into a column-major out with beta
    a, b = ints(g, (260, 201), 4, "cuda"), ints(g, (201, 388), 4, "cuda")
    out = ints(g, (388, 260), 64, "cuda").t()
    want = 0.5 * (a.double() @ b.double()) + 2.0 * out.double()
    dev.matmul(a, b, out, alpha=0.5, beta=2.0)
    t.cuda.synchronize()
    exact(out, want, "matmul")
    for act in (None, "relu"):
        x = ints(g, (3, 100, 200), 4, "cuda").requires_grad_()
        W = ints(g, (388, 200), 4, "cuda").requires_grad_()
        bias = ints(g, (388,), 64, "cuda").requires_grad_()
        y = dev.linear(x, W, bias, activation=act)
        gy = ints(g, y.shape, 4, "cuda")
        y.backward(gy)
        x64, W64, b64 = (v.detach().double().requires_grad_() for v in (x, W, bias))
        y64 = t.nn.functional.linear(x64, W64, b64)
        if act == "relu":
            y64 = t.relu(y64)
        y64.backward(gy.double())
        for name, got, w in (("y", y, y64), ("dx", x.grad, x64.grad), ("dW", W.grad, W64.grad), ("db", bias.grad, b64.grad)):
            exact(got.detach(), w.detach(), ("linear", act, name))
    a = ints(g, (3, 132, 200), 4, "cuda").requires_grad_()
    b = ints(g, (3, 200, 260), 4, "cuda").requires_grad_()
    bias = ints(g, (3, 260), 64, "cuda").requires_grad_()
    y = dev.bmm(a, b, bias=bias, alpha=2.0)
    gy = ints(g, y.shape, 4, "cuda")
    y.backward(gy)
    a64, b64, c64 = (v.detach().double().requires_grad_() for v in (a, b, bias))
    y64 = 2.0 * t.bmm(a64, b64) + c64[:, None, :]
    y64.backward(gy.double())
    for name, got, w in (("y", y, y64), ("da", a.grad, a64.grad), ("db", b.grad, b64.grad), ("dbias", bias.grad, c64.grad)):
        exact(got.detach(), w.detach(), ("bmm", name))
    assert dev.stats()["detected"] == 0


# ------------------------------------------------------------------ GPU 4: seeded exact fuzz
@pytest.mark.gpu
@pytest.mark.parametrize("seed", range(40))
def test_exact_fuzz(cuda, ft, dev, seed):
    """Random shapes, variants, layouts, dyadic alpha / beta, entry points and decomposition knobs: the plain and the ABFT
    id of the variant are exact, the ABFT checks close with zero residual."""
    t = cuda
    p = fuzz_case(seed)
    M, N, K, amax = p["M"], p["N"], p["K"], p["amax"]
    g = t.Generator(device="cuda").manual_seed(9000 + seed)
    tag = str(p)
    with knobs(ft, **p["knobs"]):
        if p["entry"] == "batched":
            Bt = 3
            A, B = ints(g, (Bt, M, K), amax, "cuda", p["garbage"]), ints(g, (Bt, N, K), amax, "cuda", p["garbage"])
            C0 = ints(g, (Bt, M, N), p["cmax"], "cuda")
            mode = (NONE, ROW, COL)[seed // 5 % 3]
            bias = ints(g, (Bt, M if mode == ROW else N), p["bias_max"], "cuda") if mode else None
            want = batched_reference(A, B, p["alpha"], p["beta"], C0, bias, mode)
        else:
            A, B = ints(g, (M, K), amax, "cuda", p["garbage"]), ints(g, (N, K), amax, "cuda", p["garbage"])
            C0 = ints(g, (M, N), p["cmax"], "cuda")
            mode = {"run_bias_row": ROW, "run_bias_col": COL}.get(p["entry"], NONE)
            bias = ints(g, (M if mode == ROW else N,), p["bias_max"], "cuda") if mode else None
            want = reference(A, B, p["alpha"], p["beta"], C0, bias, mode)
            if p["entry"] == "run_act_relu":
                want = t.relu(want)
            prod = Prod(t, A, B)
        for kid in (ft.SGEMM_IDS[p["name"]], ft.ABFT_IDS[p["name"]]):
            dev.stats()
            if p["entry"] == "batched":
                got, _ = run_batched(t, dev, kid, A, B, p["alpha"], p["beta"], C0, bias, mode, la=p["la"], lb=p["lb"],
                                     pad=p["pad"])
            else:
                got, _ = prod.run(dev, kid, p["la"], p["lb"], p["pad"], M + 4 if p["pad"] else None, p["alpha"], p["beta"],
                                  C0, bias, mode, RELU if p["entry"] == "run_act_relu" else None)
            st = dev.stats()
            exact(got, want, (kid, tag))
            zero_residual(st, kid, ft, (kid, tag))


# ------------------------------------------------------------------ GPU 5: exact repairs at the tile geometry
def odd_ints(g, M, N, K, amax, batch=()):
    """A, B with every element of A~ B~^T odd (so nonzero: a sign or exponent upset anywhere changes it by >= 2 or to
    +-Inf): k = 0 holds 1 in both, A is even elsewhere"""
    A = 2 * ints(g, (*batch, M, K), amax // 2, "cuda")
    B = ints(g, (*batch, N, K), amax, "cuda")
    A[..., 0], B[..., 0] = 1.0, 1.0
    return A, B


def _upset(r, c, kind):
    if kind == "exp":
        return {"row": r, "col": c, "xor": 1 << 30}
    if kind == "sign":
        return {"row": r, "col": c, "xor": 1 << 31}
    return {"row": r, "col": c, "add": float(kind)}


@pytest.mark.gpu
@pytest.mark.parametrize("kid", [31, 16, 12])
def test_repairs_are_exact(cuda, ft, dev, kid):
    """Single upsets of integer size (add +-1, +-7, +-1000) and exponent / sign xors at column 0, BN - 1, the 32-column chunk
    edges, the epilogue-assist split BN/2 - 1 / BN/2, N - 1 of a ragged last tile; rows 0, 31 / 32, 127 / 128 and M - 1 of a
    ragged row tile: every corrected element equals the reference exactly, the event names it, nothing else changes.  Two
    upsets in one row: the recomputed row is exact.  A level-2 repair with beta != 0 is exact.  An upset in entry 2 of a
    batch is located there and repaired exactly."""
    t = cuda
    tm, bn = tiles(ft)[kid]
    M, N, K = 2 * tm + 4, 2 * bn + 4 if bn < 256 else bn + 132, 201
    g = t.Generator(device="cuda").manual_seed(41 + kid)
    # odd C everywhere, and garbage low bits, which the correction, the recompute of a row and level 2's chunk recompute
    # must all ignore
    A, B = odd_ints(g, M, N, K, 2)
    A, B = with_garbage(g, A), with_garbage(g, B)
    C0 = 2 * ints(g, (M, N), 32, "cuda")
    p = Prod(t, A, B)
    want = reference(A, B)
    assert bool((want.remainder(2) == 1).all())
    cols = [0, bn - 1, 31, 32, min(63, bn - 1), bn // 2 - 1, bn // 2, N - 1]
    rows = list(dict.fromkeys([0, 31, 32, 127, 128, M - 1, tm - 1, tm, 64, 200]))[:8]
    kinds = [1, -1, 7, -7, 1000, -1000, "exp", "sign"]
    for shift in range(3):
        faults, where = [], set()
        for i in range(8):
            r, c = rows[i], cols[(i + shift) % 8]
            faults.append(_upset(r, c, kinds[(i + 3 * shift) % 8]))
            where.add((r, c))
        for opts in ({}, dict(protect_epilogue=2)):
            dev.stats()
            got, _ = p.run(dev, kid, opts=ft.make_opts(faults=faults, **opts))
            st = dev.stats()
            exact(got, want, (kid, shift, faults, opts))
            assert st["detected"] == st["corrected"] == 8 and st["recomputed"] == 0, (kid, faults, st)
            assert {(e["row"], e["col"]) for e in st["events"]} == where and all(e["status"] == 1 for e in st["events"]), st
    # two upsets in one row: recomputed, exactly.  (Two upsets whose weighted mean column (d2 / d1) falls within 0.25 of a
    # column inside the tile are taken for one upset there, as the locate rule of DESIGN.md §3.3 allows: choose sizes that
    # keep it away from every integer.)
    v2 = next(v for v in (9.0, 100.0, 13.0, 250.0) if abs((4 * 7.0 + (bn - 1) * v) / (7.0 + v) % 1 - 0.5) < 0.2)
    for opts in ({}, dict(protect_epilogue=2)):
        dev.stats()
        got, _ = p.run(dev, kid, alpha=-0.5, beta=1.0, C0=C0,
                       opts=ft.make_opts(faults=[{"row": 33, "col": 3, "add": 7.0}, {"row": 33, "col": bn - 2, "add": v2}],
                                         **opts))
        st = dev.stats()
        exact(got, reference(A, B, -0.5, 1.0, C0), (kid, "two in a row", opts))
        assert st["detected"] == 1 and st["recomputed"] == 1, st
    # level 2 repairs an upset of the value about to be stored with beta != 0, at the last column of the ragged corner tile
    # (z = acc - 2 C0 is odd: flipping its top mantissa bit changes it by >= 0.5)
    w2 = reference(A, B, 1.0, -2.0, C0)
    dev.stats()
    got, _ = p.run(dev, kid, alpha=1.0, beta=-2.0, C0=C0, opts=ft.make_opts(
        faults=[{"row": M - 1, "col": N - 1, "xor": 1 << 22, "where": "epilogue_value"}], protect_epilogue=2))
    st = dev.stats()
    exact(got, w2, (kid, "level 2"))
    assert st["epilogue_faults"] == 1 and st["recomputed"] == 1, st
    # entry 2 of a batch
    Ab, Bb = odd_ints(g, M, N, K, 2, (3,))
    wb = batched_reference(Ab, Bb)
    r, c = 5, bn // 2
    dev.stats()
    got, _ = run_batched(t, dev, kid, Ab, Bb, opts=ft.make_opts(faults=[{"row": 2 * M + r, "col": c, "add": -1000.0}]))
    st = dev.stats()
    exact(got, wb, (kid, "batch"))
    assert st["corrected"] == 1 and [(e["row"], e["col"]) for e in st["events"]] == [(2 * M + r, c)], st


# ------------------------------------------------------------------ GPU 6: rounding tier
@pytest.mark.gpu
def test_rounding_tier_elementwise(cuda, ft, dev):
    """Standard-normal operands (and, for 3xTF32, operands with garbage low bits): every element within the worst-case bound
    of truncating FP32 accumulation, |C - ref| <= gamma * (|A~| |B~|^T)(m, n) + 2^-23 |beta C0|, gamma = (K + 8) 2^-22
    (3xTF32: + 2^-21, against the untruncated operands).  Rows the ABFT check flags on such data are repaired or recomputed
    and must meet the same bound.  Prints the largest measured fraction of the bound and the number of rows flagged."""
    t = cuda
    g = t.Generator(device="cuda").manual_seed(61)
    worst, flagged = {}, {}
    for M, N, K in ((260, 388, 201), (1024, 1024, 4096), (512, 512, 16384)):
        A = t.randn(M, K, generator=g, device="cuda")
        B = t.randn(N, K, generator=g, device="cuda")
        C0 = t.randn(M, N, generator=g, device="cuda")
        for precision in (0, 1):
            if precision:
                A, B = with_garbage(g, ints(g, (M, K), 8, "cuda")) * 0.37, with_garbage(g, ints(g, (N, K), 8, "cuda")) * 1.3
            trunc = precision == 0
            mag = (tf32(A) if trunc else A).double().abs() @ (tf32(B) if trunc else B).double().abs().T
            gamma = (K + 8) * 2.0 ** -22 + (2.0 ** -21 if precision else 0.0)
            for kid in (31, 16, 13):
                for beta in (0.0, 1.0):
                    want = reference(A, B, 1.0, beta, C0, truncate=trunc)
                    p = Prod(t, A, B)
                    dev.stats()
                    got, _ = p.run(dev, kid, beta=beta, C0=C0, opts=ft.make_opts(precision=precision))
                    key = ("3xTF32" if precision else "TF32", K)
                    flagged[key] = flagged.get(key, 0) + dev.stats()["detected"]
                    bound = gamma * mag + 2.0 ** -23 * (beta * C0.double()).abs()
                    err = (got.double() - want).abs()
                    ratio = float((err / bound).max())
                    assert ratio <= 1.0, (kid, M, N, K, precision, beta, ratio)
                    worst[key] = max(worst.get(key, 0.0), ratio)
    print("rounding tier: largest |C - ref| / bound:", {f"{k[0]} K={k[1]}": round(v, 5) for k, v in sorted(worst.items())},
          "rows flagged:", {f"{k[0]} K={k[1]}": v for k, v in sorted(flagged.items())})


# ------------------------------------------------------------------ GPU 7: sensitivity of the exact checks
@pytest.mark.gpu
def test_sensitivity_enc_rounding(cuda, ft, dev):
    """An encode that rounds B to TF32 instead of truncating it (debug knob enc_rounding = 1), on exact operands where two
    elements of B carry low bits that round up: nothing is detected -- the old assertion passes -- but the residual is no
    longer zero.  (With garbage bits in every element, as the other exact tests use them, the rounding encode is detected
    outright.)"""
    t = cuda
    g = t.Generator(device="cuda").manual_seed(71)
    M, N, K = 260, 388, 201
    A, B = ints(g, (M, K), 4, "cuda"), ints(g, (N, K), 4, "cuda")
    A[:, 17] = 1.0
    for n, k in ((3, 17), (300, 17)):
        B[n, k] = (t.tensor(3.0, device="cuda").view(dtype=t.int32) | 0x1FFF).view(dtype=t.float32)
    p = Prod(t, A, B)
    for kid in (31, 16):
        for rounding in (0, 1):
            with knobs(ft, enc_rounding=rounding, enc_front=0):
                dev.stats()
                got, _ = p.run(dev, kid)
                st = dev.stats()
            exact(got, reference(A, B), (kid, rounding))
            assert st["detected"] == 0, st
            assert (st["max_abs_residual"] > 0.0) == (rounding == 1), (kid, rounding, st)


@pytest.mark.gpu
def test_sensitivity_low_bit_epilogue_upset(cuda, ft, dev):
    """An unprotected upset of bit 3 of one accumulator value after the check (fault mode 2): the exact comparator reports
    exactly that element, while the norm-wise bound of the rest of the suite still passes."""
    t = cuda
    g = t.Generator(device="cuda").manual_seed(72)
    M, N, K = 1024, 1024, 256
    A, B = odd_ints(g, M, N, K, 4)   # every element odd, so nonzero: bit 3 of its mantissa is worth 8 ulp of it
    want = reference(A, B)
    r, c = 300, 77
    dev.stats()
    got, _ = Prod(t, A, B).run(dev, 31, opts=ft.make_opts(faults=[{"row": r, "col": c, "xor": 1 << 3, "where": "epilogue_tmem"}]))
    assert dev.stats()["detected"] == 0
    bad = ((got.double() != want)).nonzero().tolist()
    assert bad == [[r, c]], mismatch(got, want)
    rel_fro = float(t.linalg.norm(got.double() - want) / t.linalg.norm(want))
    assert 0.0 < rel_fro < TOL_MODEL
