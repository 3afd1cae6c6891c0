"""Exact, element-wise checks of the BF16 operand path (ftsgemm_run_typed / ftsgemm_run_batched_typed) against a float64
reference, held to the standard tests/test_exact.py holds the FP32 path to (DESIGN.md §3.1, §3.3, §4).

Every product of two BF16 values is exact in FP32.  With integer operands (or integers scaled by powers of two) whose
partial sums, tile row sums, expected row checksums, weighted column-block sums and stored values stay at or below 2^24
(test_bf16.exact_budget_ok), every correct path returns the float64 product of the BF16 values bit for bit, keeps the
padding of D and Z, leaves C's bytes alone when D != C, and closes every row check with a residual of exactly zero.

Covered here and nowhere else: the BF16 tile and stage edges (64 k per stage, 64-row A boxes, the BN/2 halves of the two
CTAs), more than one checksum tile-column (six checksum columns per N-tile straddle two of them), whole outputs at
production sizes, the planner knobs, batches past the encode's 65535 grid rows, the row and chunk recomputes in every
layout pair, and the BF16 value range (full 8-bit mantissas, wide exponent spreads, subnormals, column-block sums that
round to Inf in BF16).

With BF16 C, D and Z (ftsgemm_run_batched_mixed) the same checks hold against the float64 result rounded once to nearest
even (round_bf16, mismatch16); the tests that can take the output type do, and each of their BF16-output cases asserts that
its data needs that rounding (Rounding).  What only a BF16 output has is in tests/test_bf16_out_exact.py.
"""
import numpy as np
import pytest

from test_bf16 import exact_budget_ok, ld_bf16, pack16, pad8, run16, zero_residual
from test_exact import DYADIC, LIMIT, TOL_MODEL, _free, _upset, budget, knobs, mismatch, odd_ints, tiles

MN, KM = 0, 1
NONE, ROW, COL = 0, 1, 2
RELU = 1
PAIRS = {"256": (21, 31), "128": (3, 13), "128s": (22, 32), "auto": (20, 40)}   # plain and ABFT id of each BF16 tile
CUBLAS_BF16 = 7
F32, BF16 = 0, 1          # FTSGEMM_TYPE_*: the element type of C, D and Z
SENTINEL = -12345.5
Z_SENTINEL = 7777.25
SENTINEL16 = -12352.0     # the sentinels of a BF16 output: BF16 values (8 significant bits)
Z_SENTINEL16 = 7776.0
BF16_MAX = 2.0 ** 128 - 2.0 ** 120
CHK_PER_TILE = 6          # checksum columns per N-tile: e hi, mid, lo, w hi, mid, lo (DESIGN.md §3.1)


def _t():
    import torch
    return torch


# ------------------------------------------------------------------ exact-data helpers (no GPU)
def bf16_budget_ok(K, amax, bmax, alpha=1.0, beta=0.0, cmax=0.0, bias_max=0.0, BN=256):
    """exact_budget_ok, and every integer of [-amax, amax] and [-bmax, bmax] is a BF16 value (8 significant bits: up to 256)"""
    return max(amax, bmax) <= 256 and exact_budget_ok(K, amax, bmax, alpha, beta, cmax, bias_max, BN)


def pick_amax16(K, alpha=1.0, beta=0.0, cmax=0.0, bias_max=0.0, choices=(8, 4, 2, 1)):
    for a in choices:
        if bf16_budget_ok(K, a, a, alpha, beta, cmax, bias_max):
            return a
    raise ValueError((K, alpha, beta, cmax, bias_max))


def split3(x):
    """the encode's three BF16 terms of float64 totals x (store_split3): each the remainder after the ones before, rounded
    to nearest through FP32"""
    t = _t()
    terms, r = [], x
    for _ in range(3):
        h = r.float().to(t.bfloat16).double()
        terms.append(h)
        r = r - h
    return terms


def block_sums(B, BN):
    """float64 plain and weighted column-block sums of B (N x K) per N-tile: (tiles_n, K) each"""
    t = _t()
    N, K = B.shape
    tn = -(-N // BN)
    Bp = t.zeros(tn * BN, K, dtype=t.float64)
    Bp[:N] = B.double()
    Bp = Bp.reshape(tn, BN, K)
    w = t.arange(1, BN + 1, dtype=t.float64)[None, :, None]
    return Bp.sum(1), (Bp * w).sum(1)


def chk_geometry(BN, N):
    """plan_tiles for BF16: (tiles_n, tiles_c, the N-tiles whose six checksum columns straddle two checksum tile-columns)"""
    tiles_n = -(-N // BN)
    tiles_c = -(-CHK_PER_TILE * tiles_n // BN)
    straddle = [j for j in range(tiles_n) if CHK_PER_TILE * j // BN != (CHK_PER_TILE * j + CHK_PER_TILE - 1) // BN]
    return tiles_n, tiles_c, straddle


# ------------------------------------------------------------------ BF16 output: the reference rounded once (no GPU)
def _u32(x):
    """the FP32 bit patterns of float32 x as int64 in [0, 2^32)"""
    t = _t()
    return x.contiguous().view(t.int32).to(t.int64) & 0xFFFFFFFF


def round_bf16(want, double_round=False):
    """The BF16 bits (int64 in [0, 0xFFFF]) of float64 values rounded to nearest even from their FP32 bits u:
    (u + 0x7FFF + ((u >> 16) & 1)) >> 16, NaN as 0x7FC0 -- integer arithmetic, independent of torch's own cast, on want's
    device.  Every finite value must be an FP32 value: on exact data the kernels round once, at the store.  double_round
    declares a case whose results are not FP32 values (FP32 subnormals that lose bits): there the defined value is float64 ->
    FP32 (nearest even) -> BF16, the order the kernel rounds in."""
    t = _t()
    f = want.float()
    if not double_round:
        inexact = t.isfinite(want) & (f.double() != want)
        assert not bool(inexact.any()), f"{int(inexact.sum())} finite values are not FP32 values"
    u = _u32(f)
    r = (u + 0x7FFF + ((u >> 16) & 1)) >> 16
    return t.where(t.isnan(f), t.full_like(r, 0x7FC0), r)


def bits16(x):
    """the bits of a bfloat16 tensor as int64 in [0, 0xFFFF]"""
    t = _t()
    return x.contiguous().view(t.int16).to(t.int64) & 0xFFFF


def mismatch16(got, want_bits, show=4):
    """'' when the bfloat16 tensor got has the bits want_bits (round_bf16) at every element, with +0 == -0 and NaN == NaN
    (any payload); otherwise the count and the first few (index, got, want)"""
    if tuple(got.shape) != tuple(want_bits.shape):
        return f"shape {tuple(got.shape)} != {tuple(want_bits.shape)}"
    g, w = bits16(got), want_bits
    ng, nw = (g & 0x7FFF) > 0x7F80, (w & 0x7FFF) > 0x7F80
    zero = ((g | w) & 0x7FFF) == 0
    bad = (ng != nw) | (~ng & ~zero & (g != w))
    n = int(bad.sum())
    if n == 0:
        return ""
    val = lambda b: float(np.array([b << 16], np.uint32).view(np.float32)[0])
    out = []
    for i in bad.nonzero()[:show].tolist():
        gb, wb = int(g[tuple(i)]), int(w[tuple(i)])
        out.append(f"{tuple(i)}: got {val(gb)!r} (0x{gb:04x}) want {val(wb)!r} (0x{wb:04x})")
    return f"{n} elements differ, e.g. " + ", ".join(out)


class Rounding:
    """What the float64 references of one BF16-output test case asked of the rounding: elements that need more than 8
    significant bits, and exact ties rounded down (the even neighbour has the smaller magnitude) and up.  Data that needs no
    rounding proves nothing about it, so check() requires all three."""

    def __init__(self):
        self.wide = self.down = self.up = 0

    def add(self, want):
        t = _t()
        u = _u32(want[t.isfinite(want)].float())
        low, odd = u & 0xFFFF, ((u >> 16) & 1) == 1
        tie = low == 0x8000
        self.wide += int((low != 0).sum())
        self.down += int((tie & ~odd).sum())
        self.up += int((tie & odd).sum())

    def check(self, tag):
        assert self.wide > 0 and self.down > 0 and self.up > 0, (tag, "the data needs no rounding", vars(self))


def exact(got, want, tag, seen=None, double_round=False):
    """got equals the float64 want at every element: float32 bit for bit (NaN == NaN, +0 == -0), bfloat16 as want rounded
    once (round_bf16); seen (a Rounding) tallies what the rounding had to do"""
    if got.dtype == _t().bfloat16:
        msg = mismatch16(got, round_bf16(want, double_round))
        if seen is not None:
            seen.add(want)
    else:
        msg = mismatch(got, want)
    assert not msg, f"{tag}: {msg}"


TIE_A = 17.0


def tie_factors(alpha, most=63):
    """(v_down, v_up): the smallest integers v <= most for which alpha * 17 * v is an exact BF16 tie that rounds down, and
    one that rounds up"""
    t = _t()
    v = t.arange(1, most + 1, dtype=t.float64)
    u = _u32((alpha * TIE_A * v).float())
    tie, odd = (u & 0xFFFF) == 0x8000, ((u >> 16) & 1) == 1
    return float(v[tie & ~odd][0]), float(v[tie & odd][0])


def plant_ties(A, B, alpha, C0=None, bias=None, mode=NONE):
    """For the BF16-output cases whose small data would need no rounding: row 0 of A (of every entry) becomes 17 e_0 and four
    rows n of B become +-v e_0, so D(0, n) = alpha * 17 * (+-v) are exact ties of both signs, one pair rounded down and one
    up (tie_factors); C0 and the bias are zeroed where they are added to those four elements.  In place; returns the four
    columns.  The exactness budget holds: these rows only shrink, and a column-block sum grows by at most 4 * 63
    (plant_budget_ok)."""
    N = B.shape[-2]
    cols = sorted({0, N // 3, (2 * N) // 3, N - 1})
    assert len(cols) == 4, N
    vd, vu = tie_factors(alpha)
    A[..., 0, :] = 0.0
    A[..., 0, 0] = TIE_A
    for n, v in zip(cols, (vd, -vd, vu, -vu)):
        B[..., n, :] = 0.0
        B[..., n, 0] = v
    if C0 is not None:
        C0[..., 0, cols] = 0.0
    if bias is not None and mode == ROW:
        bias[..., 0] = 0.0
    elif bias is not None and mode == COL:
        bias[..., cols] = 0.0
    return cols


def plant_budget_ok(K, amax, BN=256):
    """bf16_budget_ok's checksum and weighted column-block sums with plant_ties' four rows of B (|v| <= 63) in one N-tile:
    only the k = 0 sums grow"""
    return K * amax * BN * amax + amax * 4 * 63 <= LIMIT and BN * (BN + 1) // 2 * amax + 4 * BN * 63 <= LIMIT


def with_cd(values, ids=None):
    """pytest params (value, F32) with the ids the F32 cases always had, then (value, BF16) with '-bf16' appended"""
    tup = lambda v: v if isinstance(v, tuple) else (v,)
    ids = ids or ["-".join(map(str, tup(v))) for v in values]
    return ([pytest.param(*tup(v), F32, id=i) for v, i in zip(values, ids)] +
            [pytest.param(*tup(v), BF16, id=f"{i}-bf16") for v, i in zip(values, ids)])


MULTI = ((128, 2816, 21), (128, 2944, 21), (256, 11008, 42))   # (BN, N, the straddling N-tile)

SWEEP_K = (1, 7, 8, 15, 16, 17, 63, 64, 65, 127, 129, 1000, 2088)
SWEEP_M = (4, 60, 64, 68, 124, 128, 132, 252, 256, 260, 516)
SWEEP_AB = ((1.0, 0.0), (0.5, 0.0), (-2.0, 1.0), (0.0, -0.5), (0.75, 2.0))


def sweep_n(BN):
    return (4, BN // 2 - 4, BN // 2, BN // 2 + 4, BN - 4, BN, BN + 4, BN + 28)


def sweep16(BN, seed):
    """a seeded pairwise subset of the BF16 tile-edge grid: every M, N and K value at least once, each with a layout pair,
    padded or tight leading dimensions, ldc > M or not, D != C in half the cases, a splitk setting and dyadic alpha / beta"""
    rng = np.random.default_rng(seed)
    Ms, Ns, Ks = SWEEP_M, sweep_n(BN), SWEEP_K
    n = max(len(Ms), len(Ns), len(Ks))
    off = int(rng.integers(0, 30))
    cols = [rng.permutation(np.resize(v, n)) for v in (Ms, Ns, Ks)]
    for j in range(n):
        i = j + off
        alpha, beta = SWEEP_AB[i % len(SWEEP_AB)]
        yield {"M": int(cols[0][j]), "N": int(cols[1][j]), "K": int(cols[2][j]), "la": i % 2, "lb": (i // 2) % 2,
               "pad": i % 3 != 0, "ldc": i % 2 == 1, "splitk": (-1, 0, 2)[i % 3], "alpha": alpha, "beta": beta,
               "out_of_place": (j // 2) % 2 == 0}


FUZZ_ENTRIES = ("plain", "bias_row", "bias_col", "relu_z", "out_of_place", "batched")


def fuzz16(seed, cd=F32):
    """the parameters of one seeded BF16 fuzz case (no GPU): shape, tile, layouts, padding, alpha / beta, entry point, knobs.
    With a BF16 output an alpha of 0 becomes 1 (the result must have ties to round: plant_ties)."""
    rng = np.random.default_rng(17000 + seed)
    p = {"seed": seed, "M": int(rng.integers(1, 200)) * 4, "N": int(rng.integers(1, 200)) * 4,
         "K": int(rng.choice([int(rng.integers(1, 130)), int(rng.integers(1, 1500))])),
         "pair": list(PAIRS)[seed % len(PAIRS)], "la": int(rng.integers(0, 2)), "lb": int(rng.integers(0, 2)),
         "pad": bool(rng.integers(0, 2)), "alpha": float(rng.choice(DYADIC)), "beta": float(rng.choice([0.0, 1.0, -0.5, 2.0])),
         "entry": FUZZ_ENTRIES[seed % len(FUZZ_ENTRIES)],
         "knobs": {"splitk": int(rng.choice([-1, 0, 2, 3])), "wave_sync": int(rng.choice([0, 1])), "pdl": int(rng.choice([0, 1])),
                   "epi_assist": int(rng.choice([0, 1])), "chk_slices": int(rng.choice([1, 2, 3])),
                   "enc_front": int(rng.choice([0, 1]))}}
    if cd == BF16 and p["alpha"] == 0.0:
        p["alpha"] = 1.0
    p["cmax"] = 0 if p["beta"] == 0.0 else 64
    p["bias_max"] = 64 if p["entry"] in ("bias_row", "bias_col", "batched") else 0
    p["amax"] = pick_amax16(p["K"], p["alpha"], p["beta"], p["cmax"], p["bias_max"])
    return p


# ------------------------------------------------------------------ CPU tests
def test_budgets_of_every_parameter_set():
    # full 8-bit mantissas against +-1, in both operand roles, K <= 256: exact, with one k of room left at BN = 256
    for amax, bmax in ((255, 1), (1, 255)):
        assert bf16_budget_ok(256, amax, bmax) and bf16_budget_ok(257, amax, bmax)
        assert not bf16_budget_ok(258, amax, bmax)
    assert budget(256, 256, 255, 1)["rowsum"] == 256 * 256 * 255 <= LIMIT
    assert not bf16_budget_ok(8, 257, 1)                           # 257 is not a BF16 value
    # the sweep, the multi-column shapes, the repairs, the batches and the value-range sets
    for K in SWEEP_K:
        for alpha, beta in SWEEP_AB:
            assert bf16_budget_ok(K, pick_amax16(K, alpha, beta, 64), pick_amax16(K, alpha, beta, 64), alpha, beta, 64)
    assert pick_amax16(2088) == 4 and pick_amax16(256) == 8
    # the ties planted in the BF16-output sets keep them exact
    for K in SWEEP_K:
        for alpha, beta in SWEEP_AB:
            assert plant_budget_ok(K, pick_amax16(K, alpha, beta, 64))
            if alpha != 0.0:
                assert max(tie_factors(alpha)) <= 63
    assert plant_budget_ok(200, 2) and plant_budget_ok(129, 4) and tie_factors(-1.0) == tie_factors(1.0) == (17.0, 19.0)
    assert bf16_budget_ok(200, 4, 4) and bf16_budget_ok(201, 2, 2, -0.5, 1.0, 64) and bf16_budget_ok(201, 2, 2, 1.0, -2.0, 64)
    assert bf16_budget_ok(6, 8, 8, bias_max=64) and bf16_budget_ok(201, 4, 4, -1.0, 0.5, 64, 64)
    assert bf16_budget_ok(301, 8, 8, -0.5) and bf16_budget_ok(256, 4, 4) and bf16_budget_ok(256, 8, 8)
    # production sizes: 4096^3 / 8192^3 / 16384^3 at |a| <= 2 (the last with no room left), K = 65536 at 1
    assert bf16_budget_ok(4096, 2, 2) and bf16_budget_ok(8192, 2, 2, 1.0, -1.0, 64) and bf16_budget_ok(16384, 2, 2)
    assert budget(16384, 256, 2, 2)["rowsum"] == LIMIT and budget(65536, 256, 1, 1)["rowsum"] == LIMIT
    assert bf16_budget_ok(65536, 1, 1) and bf16_budget_ok(32768, 1, 1) and not bf16_budget_ok(32768, 2, 2)


def test_full_mantissas_fill_all_three_checksum_planes():
    """On the full-mantissa data (B in [-255, 255]) the weighted column-block sums need all three BF16 terms, and the three
    terms hold every total exactly: the check of such data leans on every plane."""
    t = _t()
    g = t.Generator().manual_seed(5)
    for BN in (128, 256):
        B = t.randint(-255, 256, (388, 256), generator=g).float()
        for total in block_sums(B, BN):
            hi, mid, lo = split3(total)
            assert t.equal((hi + mid) + lo, total)
        hi, mid, lo = split3(block_sums(B, BN)[1])
        assert bool((lo != 0).any()) and bool((mid != 0).any())
    # between the largest BF16 value and FLT_MAX the hi term rounds to Inf (the check then cannot verify the row)
    x = t.tensor([BF16_MAX, 2.0 ** 128 - 2.0 ** 118], dtype=t.float64)
    assert float(x[1]) < float(np.finfo(np.float32).max) and BF16_MAX == float(t.tensor(BF16_MAX).to(t.bfloat16))
    hi = split3(x)[0]
    assert float(hi[0]) == BF16_MAX and hi[1].item() == float("inf")
    # a BF16 subnormal of the value-range test is a BF16 value, and its products with the scaled B are normal FP32
    v = t.tensor([2.0 ** -130 * k for k in range(1, 16)], dtype=t.float64)
    assert t.equal(v.float().to(t.bfloat16).double(), v) and float(v.max()) < 2.0 ** -126
    assert float(v.min()) * 2.0 ** 40 > 2.0 ** -126


def test_multi_column_shapes_straddle():
    for BN, N, tile in MULTI:
        tiles_n, tiles_c, straddle = chk_geometry(BN, N)
        assert tiles_c >= 2 and straddle == [tile], (BN, N, tiles_n, tiles_c, straddle)
        first = CHK_PER_TILE * tile
        assert first // BN == 0 and (first + CHK_PER_TILE - 1) // BN == 1
    assert [c for c in range(126, 132)] == list(range(CHK_PER_TILE * 21, CHK_PER_TILE * 22))
    assert [c for c in range(252, 258)] == list(range(CHK_PER_TILE * 42, CHK_PER_TILE * 43))
    # the smallest N with a straddling tile: 2689 at BN = 128, 10753 at BN = 256; FP32's four columns never straddle
    for BN, N in ((128, 2689), (256, 10753)):
        assert chk_geometry(BN, N)[2] and not chk_geometry(BN, N - 1)[2]
    assert all(4 * j // BN == (4 * j + 3) // BN for BN in (128, 256) for j in range(4096))


def test_sweep_covers_every_value():
    for BN in (128, 256):
        for seed in range(200, 204):
            cases = list(sweep16(BN, seed))
            assert {c["M"] for c in cases} == set(SWEEP_M)
            assert {c["N"] for c in cases} == set(sweep_n(BN))
            assert {c["K"] for c in cases} == set(SWEEP_K)
            assert {(c["la"], c["lb"]) for c in cases} == {(0, 0), (0, 1), (1, 0), (1, 1)}
            assert {c["splitk"] for c in cases} == {-1, 0, 2} and {c["out_of_place"] for c in cases} == {False, True}
            assert any(c["pad"] for c in cases) and any(c["ldc"] for c in cases)
            assert all(c["N"] % 4 == 0 and c["M"] % 4 == 0 for c in cases)


def test_fuzz_cases_are_within_budget():
    for seed in range(40):
        for cd in (F32, BF16):
            p = fuzz16(seed, cd)
            assert bf16_budget_ok(p["K"], p["amax"], p["amax"], p["alpha"], p["beta"], p["cmax"], p["bias_max"]), p
            assert p["M"] % 4 == 0 and p["N"] % 4 == 0 and p["K"] >= 1
            if cd == BF16:
                assert plant_budget_ok(p["K"], p["amax"]) and p["alpha"] != 0.0, p
                vd, vu = tie_factors(p["alpha"])
                assert max(vd, vu) <= 63
    cases = [fuzz16(s) for s in range(40)]
    assert {c["entry"] for c in cases} == set(FUZZ_ENTRIES) and {c["pair"] for c in cases} == set(PAIRS)
    for knob in ("splitk", "wave_sync", "pdl", "epi_assist", "chk_slices", "enc_front"):
        assert len({c["knobs"][knob] for c in cases}) > 1, knob


# ------------------------------------------------------------------ GPU harness
@pytest.fixture(scope="module")
def dev(cuda, ft):
    cuda.cuda.set_device(0)
    h = ft.FtSgemm()
    yield h
    h.close()


def ints(t, g, shape, amax):
    return t.randint(-amax, amax + 1, shape, generator=g, device="cuda", dtype=t.int32).float()


def reference(A, B, alpha=1.0, beta=0.0, C0=None, bias=None, mode=NONE):
    """float64 alpha * A B^T + beta * C0 (+ bias) of the BF16 values; A (..., M, K), B (..., N, K), bias (..., len)"""
    t = _t()
    out = alpha * (A.to(t.bfloat16).double() @ B.to(t.bfloat16).double().transpose(-1, -2))
    if beta != 0.0:
        out = out + beta * C0.double()
    if mode == ROW:
        out = out + bias.double()[..., :, None]
    elif mode == COL:
        out = out + bias.double()[..., None, :]
    return out


def out_buffers(t, cd):
    """(dtype, D sentinel, Z sentinel) of an output of type cd"""
    return (t.bfloat16, SENTINEL16, Z_SENTINEL16) if cd == BF16 else (t.float32, SENTINEL, Z_SENTINEL)


def run1(t, ft, dev, kid, A, B, la=KM, lb=KM, pad=False, ldc=None, alpha=1.0, beta=0.0, C0=None, bias=None, mode=NONE,
         act=0, z=False, out_of_place=False, opts=None, cd=F32):
    """run16 with Z's padding checked too: one run_typed call (cd = BF16: one run_batched_mixed call with BF16 C, D and Z,
    ldc rounded up to a multiple of 8; C0 must hold BF16 values); returns (D, Z) as M x N views"""
    M, K = A.shape
    N = B.shape[0]
    lda, ldb, ldc = ld_bf16(la, M, K, pad), ld_bf16(lb, N, K, pad), ldc or M
    typ, sent, zsent = out_buffers(t, cd)
    if cd == BF16:
        ldc = pad8(ldc)
        assert C0 is None or t.equal(C0.to(t.bfloat16).float(), C0.float())
    cbuf = t.full((N, ldc), sent, device="cuda", dtype=typ)
    cbuf[:, :M] = 0.0 if C0 is None else C0.T
    c_before = cbuf.clone()
    dbuf = t.full((N, ldc), sent, device="cuda", dtype=typ) if out_of_place else cbuf
    zbuf = t.full((N, ldc), zsent, device="cuda", dtype=typ) if z else None
    dA, dB = pack16(t, A, la, lda), pack16(t, B, lb, ldb)
    if cd == BF16:
        dev.run_batched_mixed(kid, M, N, K, dA, la, lda, 0, dB, lb, ldb, 0, ft.TYPE_BF16, cbuf, ldc, 0, dbuf, ft.TYPE_BF16, 1,
                              alpha, beta, bias, mode, 0, act, zbuf, opts)
    else:
        dev.run_typed(kid, M, N, K, dA, la, lda, dB, lb, ldb, ft.TYPE_BF16, cbuf, ldc, dbuf, alpha, beta, bias, mode, act, zbuf,
                      opts)
    t.cuda.synchronize()
    if out_of_place:
        assert t.equal(cbuf.view(t.int16), c_before.view(t.int16)), "C was written"
    if ldc > M:
        assert bool((dbuf[:, M:].float() == sent).all()), "D's padding was written"
        if z:
            assert bool((zbuf[:, M:].float() == zsent).all()), "Z's padding was written"
    return dbuf[:, :M].t(), (zbuf[:, :M].t() if z else None)


def pack_batch16(t, X, layout, ld, gap=0):
    """(Bt, rows, K) -> (flat BF16 buffer, entry stride): each entry packed as pack16 packs it, followed by `gap` elements;
    all padding NaN"""
    Bt, rows, K = X.shape
    lines, width = (K, rows) if layout == MN else (rows, K)
    buf = t.full((Bt, lines * ld + gap), float("nan"), device="cuda")
    view = buf[:, :lines * ld].view(Bt, lines, ld)
    view[:, :, :width] = X.transpose(1, 2) if layout == MN else X
    return buf.reshape(-1).to(t.bfloat16), lines * ld + gap


def batch16(t, ft, dev, kid, A, B, la=KM, lb=KM, pad=False, gap=0, alpha=1.0, beta=0.0, C0=None, bias=None, mode=NONE,
            act=0, z=False, out_of_place=False, opts=None, cd=F32):
    """one run_batched_typed call: A (Bt, M, K), B (Bt, N, K), C column-major per entry, one bias per entry (Bt, len) or
    None (cd = BF16: one run_batched_mixed call with BF16 C, D and Z, each entry's columns padded to pad8(M) with the
    sentinel).  Returns (D, Z) as (Bt, M, N) views; checks that C kept its bytes when D != C and that no padding was
    written."""
    Bt, M, K = A.shape
    N = B.shape[1]
    lda, ldb = ld_bf16(la, M, K, pad), ld_bf16(lb, N, K, pad)
    dA, sa = pack_batch16(t, A, la, lda, gap)
    dB, sb = pack_batch16(t, B, lb, ldb, gap)
    typ, sent, zsent = out_buffers(t, cd)
    ldc = pad8(M) if cd == BF16 else M
    dC = t.full((Bt, N, ldc), sent, device="cuda", dtype=typ)
    dC[:, :, :M] = 0.0 if C0 is None else C0.transpose(1, 2)
    c_before = dC.clone()
    dD = t.full((Bt, N, ldc), sent, device="cuda", dtype=typ) if out_of_place else dC
    dZ = t.full((Bt, N, ldc), zsent, device="cuda", dtype=typ) if z else None
    sbias = 0 if bias is None else bias.shape[1]
    if cd == BF16:
        dev.run_batched_mixed(kid, M, N, K, dA, la, lda, sa, dB, lb, ldb, sb, ft.TYPE_BF16, dC, ldc, ldc * N, dD, ft.TYPE_BF16,
                              Bt, alpha, beta, bias, mode, sbias, act, dZ, opts)
    else:
        dev.run_batched_typed(kid, M, N, K, dA, la, lda, sa, dB, lb, ldb, sb, ft.TYPE_BF16, dC, M, M * N, dD, Bt, alpha, beta,
                              bias, mode, sbias, act, dZ, opts)
    t.cuda.synchronize()
    if out_of_place:
        assert t.equal(dC.view(t.int16), c_before.view(t.int16)), "C was written"
    if ldc > M:
        assert bool((dD[:, :, M:].float() == sent).all()), "D's padding was written"
        if z:
            assert bool((dZ[:, :, M:].float() == zsent).all()), "Z's padding was written"
    return dD[:, :, :M].transpose(1, 2), (dZ[:, :, :M].transpose(1, 2) if z else None)


def events(st):
    return {(e["row"], e["col"]) for e in st["events"]}


def statuses(st):
    return [e["status"] for e in st["events"]]


# ------------------------------------------------------------------ GPU 1: tile and stage edges
@pytest.mark.gpu
@pytest.mark.parametrize("name,cd", with_cd(list(PAIRS)))
def test_tile_edges_exact(cuda, ft, dev, name, cd):
    """Ids 21 / 31, 3 / 13, 22 / 32 and 20 / 40 at K around the 16-k wgmma step and the 64-k stage, M around the 64-row A
    boxes and the tile, N around the BN/2 halves the two CTAs multicast and the tile: all four layout pairs, NaN-padded
    leading dimensions, ldc > M (sentinel untouched), D != C in half the cases (C untouched), splitk -1 / 0 / 2, dyadic
    alpha / beta with an integer C0.  D equals the float64 product at every element, every row check closes exactly.  With
    BF16 C / D: D equals the float64 product rounded once, the BF16 padding sentinel (rows of M % 8 = 4 end mid-sector)
    untouched; ties are planted where alpha != 0."""
    t = cuda
    seen = Rounding()
    plain, abft = PAIRS[name]
    BN = tiles(ft)[31 if name == "auto" else abft][1]
    g = t.Generator(device="cuda").manual_seed(300 + list(PAIRS).index(name))
    for c in sweep16(BN, 200 + list(PAIRS).index(name)):
        M, N, K, alpha, beta = c["M"], c["N"], c["K"], c["alpha"], c["beta"]
        amax = pick_amax16(K, alpha, beta, 64)
        A, B = ints(t, g, (M, K), amax), ints(t, g, (N, K), amax)
        C0 = ints(t, g, (M, N), 64)
        if cd == BF16 and alpha != 0.0:
            plant_ties(A, B, alpha, C0)
        want = reference(A, B, alpha, beta, C0)
        for kid in (plain, abft):
            tag = (kid, cd, c)
            with knobs(ft, splitk=c["splitk"]):
                dev.stats()
                got, _ = run1(t, ft, dev, kid, A, B, c["la"], c["lb"], c["pad"], M + 8 if c["ldc"] else None, alpha, beta, C0,
                              out_of_place=c["out_of_place"], cd=cd)
                st = dev.stats()
            exact(got, want, tag, seen)
            zero_residual(st, kid, tag)
    if cd == BF16:
        seen.check(name)


# ------------------------------------------------------------------ GPU 2: more than one checksum tile-column
@pytest.mark.gpu
@pytest.mark.parametrize("BN,N,tile,cd", with_cd(MULTI))
def test_multi_column_checksums(cuda, ft, dev, BN, N, tile, cd):
    """N wide enough for two checksum tile-columns, where the six checksum columns of one N-tile straddle both (BN = 128,
    tile 21: e hi / mid in columns 126..127, e lo and w in 128..131; BN = 256, tile 42: e and w hi in 252..255, w mid / lo in
    256..257).  Both layouts of B, the encode in the front phase and in the pre-pass, a single product and a 2-entry batch:
    exact with zero residuals, and single upsets in several rows and columns of the straddling tile are each corrected
    exactly, the event naming that element.  With BF16 C / D the same, each corrected element rounded once (ties planted in
    row 0)."""
    t = cuda
    seen = Rounding()
    pairs = [(p, a) for p, a in (PAIRS["256"], PAIRS["128"], PAIRS["128s"]) if tiles(ft)[a][1] == BN]
    assert pairs and chk_geometry(BN, N)[1] >= 2
    M, K = 260, 200
    g = t.Generator(device="cuda").manual_seed(N)
    A, B = odd_ints(g, M, N, K, 2)     # (|acc| small enough that an upset of 1 is located: 6 thr < 1)
    Ab, Bb = odd_ints(g, M, N, K, 2, (2,))
    if cd == BF16:
        plant_ties(A, B, 1.0)
        plant_ties(Ab, Bb, 1.0)
    want = reference(A, B)
    wantb = reference(Ab, Bb)
    n0 = tile * BN
    cols = [n0, n0 + 1, n0 + BN // 2 - 1, n0 + BN // 2, n0 + BN - 2, n0 + BN - 1]
    rows = [0, 37, 130, 255, 256, M - 1]
    adds = [1.0, -7.0, 1000.0, -1.0, 7.0, -1000.0]
    for plain, abft in pairs:
        for lb in (MN, KM):
            la = 1 - lb
            for front in (0, 1):
                tag = (abft, BN, N, lb, front)
                with knobs(ft, enc_front=front):
                    for kid in (plain, abft):
                        dev.stats()
                        got, _ = run1(t, ft, dev, kid, A, B, la, lb, pad=True, cd=cd)
                        exact(got, want, (kid,) + tag, seen)
                        zero_residual(dev.stats(), kid, (kid,) + tag)
                    for shift in range(2):
                        faults = [{"row": rows[i], "col": cols[(i + shift) % 6], "add": adds[i]} for i in range(6)]
                        dev.stats()
                        got, _ = run1(t, ft, dev, abft, A, B, la, lb, pad=True, opts=ft.make_opts(faults=faults), cd=cd)
                        st = dev.stats()
                        exact(got, want, tag + (faults,))
                        assert st["detected"] == st["corrected"] == 6 and st["recomputed"] == 0, (tag, st)
                        assert events(st) == {(f["row"], f["col"]) for f in faults} and set(statuses(st)) == {1}, (tag, st)
                    # a 2-entry batch: exact, and upsets in entry 1's straddling tile
                    faults = [{"row": M + rows[i], "col": cols[i], "add": adds[i]} for i in range(0, 6, 2)]
                    for kid, opts in ((plain, None), (abft, None), (abft, ft.make_opts(faults=faults))):
                        dev.stats()
                        got, _ = batch16(t, ft, dev, kid, Ab, Bb, la, lb, pad=True, opts=opts, cd=cd)
                        st = dev.stats()
                        exact(got, wantb, (kid, "batch") + tag, seen)
                        if opts is None:
                            zero_residual(st, kid, (kid, "batch") + tag)
                        else:
                            assert st["detected"] == st["corrected"] == 3, (tag, st)
                            assert events(st) == {(f["row"], f["col"]) for f in faults}, (tag, st)
    if cd == BF16:
        seen.check((BN, N))


# ------------------------------------------------------------------ GPU 3: production sizes, whole output
def within_one_ulp16(t, got, want):
    """bfloat16 got within one BF16 ulp of want rounded once (cuBLAS sums in another order and may round partial sums)"""
    w = (round_bf16(want) << 16).to(t.int32).view(t.float32).double()
    ulp = (w.abs() * 2.0 ** -7).clamp_min(2.0 ** -133)
    return bool(((got.double() - w).abs() <= ulp).all())


def _whole16(t, ft, dev, M, N, K, ids, amax, seed, layouts=((MN, MN),), beta=0.0, saturate=False, cd=F32, seen=None):
    g = t.Generator(device="cuda").manual_seed(seed)
    A, B = ints(t, g, (M, K), amax), ints(t, g, (N, K), amax)
    if saturate:  # row 0 of A and the first 256 rows of B all amax: acc(0, n < 256) = K * amax^2, r1 = s1 = 2^24 there
        A[0, :] = amax
        B[:256, :] = amax
    want = B.double() @ A.double().T                              # (N, M): column-major D
    C0 = None
    if beta != 0.0:
        C0 = ints(t, g, (N, M), 64)
        want += beta * C0.double()
    for la, lb in layouts:
        dA = (A.T if la == MN else A).contiguous().to(t.bfloat16)
        dB = (B.T if lb == MN else B).contiguous().to(t.bfloat16)
        lda, ldb = (M if la == MN else K), (N if lb == MN else K)
        for kid in ids:
            tag = (kid, M, N, K, la, lb, beta, cd)
            dev.stats()
            if cd == BF16:
                dD = t.full((N, M), SENTINEL16, device="cuda", dtype=t.bfloat16)
                c16 = None if C0 is None else C0.to(t.bfloat16)
                c_before = None if C0 is None else c16.clone()
                dev.run_batched_mixed(kid, M, N, K, dA, la, lda, 0, dB, lb, ldb, 0, ft.TYPE_BF16, c16 if C0 is not None else dD,
                                      M, 0, dD, ft.TYPE_BF16, 1, 1.0, beta)
                t.cuda.synchronize()
                if kid == CUBLAS_BF16:
                    assert within_one_ulp16(t, dD, want), tag
                else:
                    exact(dD, want, tag, seen)
                if C0 is not None:
                    assert t.equal(c16.view(t.int16), c_before.view(t.int16)), tag
            else:
                dD = t.full((N, M), SENTINEL, device="cuda")
                c_before = None if C0 is None else C0.clone()
                dev.run_typed(kid, M, N, K, dA, la, lda, dB, lb, ldb, ft.TYPE_BF16, C0 if C0 is not None else dD, M, dD, 1.0,
                              beta)
                t.cuda.synchronize()
                bad = int((dD.double() != want).sum())
                assert bad == 0, (tag, mismatch(dD.T, want.T))
                if C0 is not None:
                    assert t.equal(C0.view(t.int32), c_before.view(t.int32)), tag
            st = dev.stats()
            zero_residual(st, kid, tag)
            del dD, c_before
        del dA, dB
        _free(t)
    del A, B, C0, want
    _free(t)


@pytest.mark.gpu
@pytest.mark.slow
def test_production_sizes_whole_output(cuda, ft, dev):
    """Every output element against float64 at the sizes the project is measured at: 4096^3 (ids 21, 31, 13, 32, 40, with
    cuBLAS BF16 as witness), 8192^3 (21 and 31 in MN,MN and K,K, and beta = -1 with D != C), 16384^3 (id 31: the wave
    re-synchronisation), 256 x 256 x 65536 (1024 k-blocks of 64) with a row checksum of exactly 2^24 (31, 40, cuBLAS BF16)
    and 512 x 1024 x 32768.  Then all of it again with BF16 C and D: every element the float64 product rounded once (values
    up to 2^24, ties of both kinds by the million), cuBLAS with BF16 C in place within one BF16 ulp.  Peak device memory
    ~12 GB."""
    t = cuda
    both = ((MN, MN), (KM, KM))
    for cd in (F32, BF16):
        seen = Rounding()
        _whole16(t, ft, dev, 4096, 4096, 4096, (21, 31, 13, 32, 40, CUBLAS_BF16), 2, 1, both, cd=cd, seen=seen)
        _whole16(t, ft, dev, 8192, 8192, 8192, (21, 31), 2, 3, both, cd=cd, seen=seen)
        _whole16(t, ft, dev, 8192, 8192, 8192, (31,), 2, 4, ((MN, KM),), beta=-1.0, cd=cd, seen=seen)
        _whole16(t, ft, dev, 16384, 16384, 16384, (31,), 2, 5, cd=cd, seen=seen)
        _whole16(t, ft, dev, 256, 256, 65536, (31, 40, CUBLAS_BF16), 1, 6, both, saturate=True, cd=cd, seen=seen)
        _whole16(t, ft, dev, 512, 1024, 32768, (31, 40), 1, 7, ((KM, MN),), cd=cd, seen=seen)
        if cd == BF16:
            seen.check("production sizes")


# ------------------------------------------------------------------ GPU 4: batch edges
@pytest.mark.gpu
def test_batched_ragged_entries_exact(cuda, ft, dev):
    """Strided BF16 batches with M not a multiple of the tile (rows past M must not leak into the next entry), a per-entry
    ROW / COL bias, ReLU with Z, NaN gaps between entries, every layout pair: every entry exact.  Then the same with BF16 C,
    D and Z (entries' columns padded to 8 with the sentinel, ties planted in row 0 of every entry): rounded once."""
    t = cuda
    for cd in (F32, BF16):
        _batched_ragged(t, ft, dev, cd)


def _batched_ragged(t, ft, dev, cd):
    seen = Rounding()
    g = t.Generator(device="cuda").manual_seed(23)
    i = 0
    for kid in (31, 13, 32):
        for Bt, (M, N, K) in ((2, (132, 260, 96)), (7, (260, 132, 129)), (3, (68, 388, 65))):
            A, B = ints(t, g, (Bt, M, K), 4), ints(t, g, (Bt, N, K), 4)
            C0 = ints(t, g, (Bt, M, N), 64)
            for mode, L in ((ROW, M), (COL, N)):
                la, lb = i % 2, (i // 2) % 2
                i += 1
                bias = ints(t, g, (Bt, L), 64)
                if cd == BF16:
                    A, B, C0 = A.clone(), B.clone(), C0.clone()
                    plant_ties(A, B, -1.0, C0, bias, mode)
                want = reference(A, B, -1.0, 0.5, C0, bias, mode)
                dev.stats()
                c, z = batch16(t, ft, dev, kid, A, B, la, lb, pad=True, gap=8, alpha=-1.0, beta=0.5, C0=C0, bias=bias,
                               mode=mode, act=RELU, z=True, out_of_place=i % 2 == 0, cd=cd)
                tag = (kid, Bt, M, N, K, mode, la, lb, cd)
                zero_residual(dev.stats(), kid, tag)
                exact(z, want, tag + ("Z",), seen)
                exact(c, t.relu(want), tag + ("D",))
    if cd == BF16:
        seen.check("batched ragged")


@pytest.mark.gpu
@pytest.mark.slow
def test_batch_of_65537_entries(cuda, ft, dev):
    """65537 tiny entries (4 x 4 x 6, NaN padding inside and between entries), past the 65535 grid rows of the BF16 encode
    pre-pass (B below 8 MB, enc_front = 0) and through the front-phase encode (enc_front = 1): every entry exact in both
    layouts of B, every row of every entry checked with zero residual.  Then with BF16 C / D (each entry's 4 rows padded to
    8 with the sentinel): every entry rounded once -- results up to 448 with a bias, ties of both kinds among them."""
    t = cuda
    g = t.Generator(device="cuda").manual_seed(65537)
    Bt, M, N, K = 65537, 4, 4, 6
    assert 2 * N * K * Bt < 8 << 20
    A, B = ints(t, g, (Bt, M, K), 8), ints(t, g, (Bt, N, K), 8)
    bias = ints(t, g, (Bt, N), 64)
    want = reference(A, B, 1.0, 0.0, None, bias, COL)
    for cd in (F32, BF16):
        seen = Rounding()
        for kid in (31, 13):
            for la, lb in ((KM, KM), (MN, MN), (KM, MN)):
                for front in (0, 1):
                    tag = (kid, la, lb, front, cd)
                    with knobs(ft, enc_front=front):
                        dev.stats()
                        c, _ = batch16(t, ft, dev, kid, A, B, la, lb, pad=True, gap=8, bias=bias, mode=COL, cd=cd)
                        st = dev.stats()
                    zero_residual(st, kid, tag)
                    assert st["rows_checked"] >= Bt * M, (tag, st)
                    exact(c, want, tag, seen)
        if cd == BF16:
            seen.check("65537 entries")
    del A, B, bias, want
    _free(t)


# ------------------------------------------------------------------ GPU 5: seeded exact fuzz
@pytest.mark.gpu
@pytest.mark.parametrize("seed,cd", with_cd(list(range(40))))
def test_exact_fuzz(cuda, ft, dev, seed, cd):
    """Random shapes, BF16 tiles, layouts, padding, dyadic alpha / beta, entry points (plain, ROW / COL bias, ReLU with Z,
    D != C, batched with a per-entry bias) and planner knobs (splitk, wave_sync, pdl, epi_assist, chk_slices, enc_front): the
    plain and the ABFT id of the tile are exact, the ABFT checks close with zero residual.  With BF16 C / D / Z (fuzz16 with
    BF16, ties planted in row 0): rounded once."""
    t = cuda
    seen = Rounding()
    p = fuzz16(seed, cd)
    M, N, K, amax = p["M"], p["N"], p["K"], p["amax"]
    g = t.Generator(device="cuda").manual_seed(19000 + seed)
    tag = str(p)
    entry = p["entry"]
    with knobs(ft, **p["knobs"]):
        if entry == "batched":
            Bt = 3
            A, B = ints(t, g, (Bt, M, K), amax), ints(t, g, (Bt, N, K), amax)
            C0 = ints(t, g, (Bt, M, N), p["cmax"])
            mode = (ROW, COL)[seed // 6 % 2]
            bias = ints(t, g, (Bt, M if mode == ROW else N), p["bias_max"])
        else:
            A, B = ints(t, g, (M, K), amax), ints(t, g, (N, K), amax)
            C0 = ints(t, g, (M, N), p["cmax"])
            mode = {"bias_row": ROW, "bias_col": COL}.get(entry, NONE)
            bias = ints(t, g, (M if mode == ROW else N,), p["bias_max"]) if mode else None
        if cd == BF16:
            plant_ties(A, B, p["alpha"], C0, bias, mode)
        want = reference(A, B, p["alpha"], p["beta"], C0, bias, mode)
        for kid in PAIRS[p["pair"]]:
            dev.stats()
            z = None
            if entry == "batched":
                got, _ = batch16(t, ft, dev, kid, A, B, p["la"], p["lb"], p["pad"], 8 if p["pad"] else 0, p["alpha"], p["beta"],
                                 C0, bias, mode, cd=cd)
            else:
                got, z = run1(t, ft, dev, kid, A, B, p["la"], p["lb"], p["pad"], M + 4 if p["pad"] else None, p["alpha"],
                              p["beta"], C0, bias, mode, RELU if entry == "relu_z" else 0, entry == "relu_z",
                              entry == "out_of_place", cd=cd)
            st = dev.stats()
            if entry == "relu_z":
                exact(z, want, (kid, tag, "Z"), seen)
                exact(got, t.relu(want), (kid, tag))
            else:
                exact(got, want, (kid, tag), seen)
            zero_residual(st, kid, (kid, tag))
    if cd == BF16:
        seen.check(tag)


# ------------------------------------------------------------------ GPU 6: exact repairs in every layout pair
def _apart(bn):
    """an upset size v for which two upsets (7 at column 3, v at column bn - 2) of one row do not look like one: their
    weighted mean column stays away from every integer (DESIGN.md §4)"""
    return next(v for v in (9.0, 100.0, 13.0, 250.0) if abs((4 * 7.0 + (bn - 1) * v) / (7.0 + v) % 1 - 0.5) < 0.2)


@pytest.mark.gpu
@pytest.mark.parametrize("la,lb", [(MN, MN), (MN, KM), (KM, MN), (KM, KM)])
@pytest.mark.parametrize("kid,cd", with_cd([31, 32]))
def test_repairs_are_exact(cuda, ft, dev, kid, cd, la, lb):
    """test_exact.test_repairs_are_exact on BF16 operands, in every layout pair with padded leading dimensions.  Single upsets
    at columns 0, 31 / 32, BN/2 - 1 / BN/2, BN - 1 and N - 1 of a ragged tile and rows around the 32-row slabs and the row
    tile: each corrected exactly.  Two upsets in one row: the BF16 row recompute (status 5) is exact.  Level 2 with beta != 0
    and an upset of the value about to be stored: the chunk recompute (status 6) is exact.  Level 1 with D != C and beta != 0:
    the segment is recomputed into D (status 6), exactly.  Two upsets in entry 2 of a batch: recomputed exactly there (the
    entry offset in BF16 elements).  With BF16 C / D every repaired element is stored rounded once; C0 is then 16 times as
    large (BF16 values up to 512), so the recomputed rows hold ties at half-integers and the level 1 / 2 results at odd
    integers."""
    t = cuda
    seen = Rounding()
    tm, bn = tiles(ft)[kid]
    M, N, K = 2 * tm + 4, 2 * bn + 4 if bn < 256 else bn + 132, 201
    g = t.Generator(device="cuda").manual_seed(41 + kid + 2 * la + lb)
    A, B = odd_ints(g, M, N, K, 2)
    C0 = (16 if cd == BF16 else 2) * ints(t, g, (M, N), 32)
    want = reference(A, B)
    assert bool((want.remainder(2) == 1).all())
    kw = dict(la=la, lb=lb, pad=True, ldc=M + 8, cd=cd)
    cols = [0, 31, 32, bn // 2 - 1, bn // 2, bn - 1, N - 1, min(63, bn - 1)]
    rows = [0, 31, 32, 127, 128, M - 1, tm - 1, tm]
    kinds = [1, -1, 7, -7, 1000, -1000, "exp", "sign"]
    for shift in range(2):
        faults, where = [], set()
        for i in range(8):
            r, c = rows[i], cols[(i + shift) % 8]
            faults.append(_upset(r, c, kinds[(i + 3 * shift) % 8]))
            where.add((r, c))
        for opts in ({}, dict(protect_epilogue=2)):
            dev.stats()
            got, _ = run1(t, ft, dev, kid, A, B, opts=ft.make_opts(faults=faults, **opts), **kw)
            st = dev.stats()
            exact(got, want, (kid, la, lb, shift, faults, opts), seen)
            assert st["detected"] == st["corrected"] == 8 and st["recomputed"] == 0, (kid, la, lb, faults, st)
            assert events(st) == where and set(statuses(st)) == {1}, st
    # two upsets in one row: the row recompute, from A and B in BF16
    v2 = _apart(bn)
    two = [{"row": 33, "col": 3, "add": 7.0}, {"row": 33, "col": bn - 2, "add": v2}]
    for opts in ({}, dict(protect_epilogue=2)):
        dev.stats()
        got, _ = run1(t, ft, dev, kid, A, B, alpha=-0.5, beta=1.0, C0=C0, opts=ft.make_opts(faults=two, **opts), **kw)
        st = dev.stats()
        exact(got, reference(A, B, -0.5, 1.0, C0), (kid, la, lb, "two in a row", opts), seen)
        assert st["detected"] == 1 and st["recomputed"] == 1 and statuses(st) == [5], st
    # level 2: an upset of the value about to be stored, beta != 0, at the last column of the ragged corner tile (the chunk
    # recompute)
    w2 = reference(A, B, 1.0, -2.0, C0)
    dev.stats()
    got, _ = run1(t, ft, dev, kid, A, B, alpha=1.0, beta=-2.0, C0=C0, opts=ft.make_opts(
        faults=[{"row": M - 1, "col": N - 1, "xor": 1 << 22, "where": "epilogue_value"}], protect_epilogue=2), **kw)
    st = dev.stats()
    exact(got, w2, (kid, la, lb, "level 2"), seen)
    assert st["epilogue_faults"] == 1 and st["recomputed"] == 1 and statuses(st) == [6], st
    # level 1 with D != C and beta != 0: the failed segment is recomputed into D from A, B and the intact C
    dev.stats()
    got, _ = run1(t, ft, dev, kid, A, B, alpha=1.0, beta=-2.0, C0=C0, out_of_place=True, opts=ft.make_opts(
        faults=[{"row": 37, "col": 40, "xor": 1 << 27, "where": "epilogue_value"}], protect_epilogue=1), **kw)
    st = dev.stats()
    exact(got, w2, (kid, la, lb, "level 1, D != C"), seen)
    assert st["epilogue_faults"] == 1 and st["recomputed"] == 1 and statuses(st) == [6], st
    # two upsets in one row of entry 2 of a batch
    Ab, Bb = odd_ints(g, M, N, K, 2, (3,))
    r = 5
    dev.stats()
    got, _ = batch16(t, ft, dev, kid, Ab, Bb, la, lb, pad=True, gap=8, opts=ft.make_opts(
        faults=[{"row": 2 * M + r, "col": 3, "add": 7.0}, {"row": 2 * M + r, "col": bn - 2, "add": v2}]), cd=cd)
    st = dev.stats()
    exact(got, reference(Ab, Bb), (kid, la, lb, "batch"), seen)
    assert st["recomputed"] == 1 and [(e["row"], e["status"]) for e in st["events"]] == [(2 * M + r, 5)], st
    if cd == BF16:
        seen.check((kid, la, lb))


# ------------------------------------------------------------------ GPU 7: the BF16 value range
@pytest.mark.gpu
@pytest.mark.parametrize("role", ["a", "b"])
def test_full_mantissas_exact(cuda, ft, dev, role):
    """Integers of 8 significant bits (|x| <= 255) against {-1, 0, 1}, in either operand role, K = 256: every layout pair,
    exact, and every row check closes with zero residual -- with B in [-255, 255] the weighted checksums fill all three BF16
    planes, which must add up exactly (cuBLAS BF16 witnesses the data)."""
    t = cuda
    g = t.Generator(device="cuda").manual_seed(255 + (role == "b"))
    M, N, K = 260, 388, 256
    A = ints(t, g, (M, K), 255 if role == "a" else 1)
    B = ints(t, g, (N, K), 1 if role == "a" else 255)
    assert bf16_budget_ok(K, float(A.abs().max()), float(B.abs().max()))
    want = reference(A, B)
    for i, (la, lb) in enumerate(((MN, MN), (MN, KM), (KM, MN), (KM, KM))):
        for kid in (21, 31, 13, 32, 40, CUBLAS_BF16):
            dev.stats()
            got, _ = run1(t, ft, dev, kid, A, B, la, lb, pad=i % 2 == 1)
            exact(got, want, (kid, role, la, lb))
            zero_residual(dev.stats(), kid, (kid, role, la, lb))


def scale_rows(t, g, x, spread):
    """x with row i multiplied by 2^e_i, e_i uniform in [-spread, spread] (exact: BF16 has FP32's exponent range)"""
    e = t.randint(-spread, spread + 1, (x.shape[0], 1), generator=g, device="cuda", dtype=t.int32)
    return t.ldexp(x, e.float()).float()


@pytest.mark.gpu
def test_power_of_two_scaling_exact(cuda, ft, dev):
    """Rows of A scaled by 2^r, r in [-60, 60]: every term of D(m, n) has the same scale, so D is exact and every row check
    closes with zero residual.

    Rows of A and of B scaled together (2^(r_m + s_n), r, s in [-40, 40]): D is still exact, but the encode's FP32 groups of 8
    mix scales and round, and so does a tile row's sum.  The plain ids and detect_only are exact; the rows the check flags
    with mixed-sign operands are counted and printed, and with repairs on nothing but flagged rows may change (at most one
    element each).  With operands of one sign nothing is flagged.  All of it again with BF16 C / D: rounded once."""
    t = cuda
    for cd in (F32, BF16):
        _power_of_two_scaling(t, ft, dev, cd)


def _power_of_two_scaling(t, ft, dev, cd):
    seen = Rounding()
    g = t.Generator(device="cuda").manual_seed(52)
    M, N, K = 516, 388, 301
    A = scale_rows(t, g, ints(t, g, (M, K), 8), 60)
    B = ints(t, g, (N, K), 8)
    want = reference(A, B, -0.5)
    for kid in (21, 31, 3, 13, 32):
        for la, lb in ((MN, KM), (KM, MN)):
            dev.stats()
            got, _ = run1(t, ft, dev, kid, A, B, la, lb, alpha=-0.5, cd=cd)
            exact(got, want, (kid, la, lb, "2^r", cd), seen)
            zero_residual(dev.stats(), kid, (kid, la, lb, "2^r"))
    A2 = scale_rows(t, g, ints(t, g, (M, K), 2), 40)
    B2 = scale_rows(t, g, ints(t, g, (N, K), 2), 40)
    want = reference(A2, B2)
    flagged, changed = {}, {}
    for plain, kid in ((21, 31), (3, 13), (22, 32)):
        for la, lb in ((MN, MN), (KM, KM)):
            got, _ = run1(t, ft, dev, plain, A2, B2, la, lb, cd=cd)
            exact(got, want, (plain, la, lb, "2^r 2^s", cd), seen)
            dev.stats()
            got, _ = run1(t, ft, dev, kid, A2, B2, la, lb, opts=ft.make_opts(detect_only=True), cd=cd)
            st = dev.stats()
            exact(got, want, (kid, la, lb, "2^r 2^s, detect_only", cd))
            flagged[kid] = flagged.get(kid, 0) + st["detected"]
            got, _ = run1(t, ft, dev, kid, A2, B2, la, lb, cd=cd)
            st2 = dev.stats()
            bad = int((bits16(got) != round_bf16(want)).sum() if cd == BF16 else (got.double() != want).sum())
            assert st2["detected"] == st["detected"] and bad <= st2["detected"], (kid, la, lb, bad, st2)
            changed[kid] = changed.get(kid, 0) + bad
    print("bf16 2^r 2^s scaling, mixed signs, output", ("F32", "BF16")[cd], ": rows flagged", flagged,
          "elements changed by a repair", changed)
    A3 = scale_rows(t, g, ints(t, g, (M, K), 2).abs() + 1.0, 40)
    B3 = scale_rows(t, g, ints(t, g, (N, K), 2).abs() + 1.0, 40)
    want = reference(A3, B3)
    for kid in (31, 13, 32):
        for la, lb in ((MN, MN), (KM, KM)):
            dev.stats()
            got, _ = run1(t, ft, dev, kid, A3, B3, la, lb, cd=cd)
            st = dev.stats()
            exact(got, want, (kid, la, lb, "2^r 2^s, one sign", cd), seen)
            assert st["detected"] == 0 and st["rows_checked"] > 0, (kid, la, lb, st)
    if cd == BF16:
        seen.check("power-of-two scaling")


@pytest.mark.gpu
@pytest.mark.parametrize("role,cd", with_cd(["a", "b"]))
def test_subnormal_operands_exact(cuda, ft, dev, role, cd):
    """BF16 subnormals (2^-130 times integers of at most 15) in one operand against integers scaled by 2^40 in the other, so
    every product is a normal FP32 value: the tensor core keeps the subnormals, and D equals the float64 product in every
    layout pair (cuBLAS BF16 witnesses it), with zero residuals.  The CUDA-core row recompute (two upsets in a row) reads the
    same values and is exact too.  With BF16 C / D (cuBLAS: BF16 C in place, within one BF16 ulp): rounded once."""
    t = cuda
    seen = Rounding()
    g = t.Generator(device="cuda").manual_seed(130 + (role == "b"))
    M, N, K = 260, 388, 201
    tiny = lambda shape: ints(t, g, shape, 15) * 2.0 ** -130
    big = lambda shape: ints(t, g, shape, 8) * 2.0 ** 40
    A, B = (tiny((M, K)), big((N, K))) if role == "a" else (big((M, K)), tiny((N, K)))
    sub = A if role == "a" else B
    assert bool(((sub != 0) & (sub.abs() < 2.0 ** -126)).float().mean() > 0.9)
    assert t.equal(sub.to(t.bfloat16).float(), sub)
    want = reference(A, B)
    for la, lb in ((MN, MN), (MN, KM), (KM, MN), (KM, KM)):
        for kid in (21, 31, 13, CUBLAS_BF16):
            dev.stats()
            got, _ = run1(t, ft, dev, kid, A, B, la, lb, pad=True, cd=cd)
            assert bool((got != 0).any()), (kid, role, la, lb, "the tensor core flushed the BF16 subnormals")
            if kid == CUBLAS_BF16 and cd == BF16:
                assert within_one_ulp16(t, got, want), (kid, role, la, lb)
            else:
                exact(got, want, (kid, role, la, lb, cd), seen)
            zero_residual(dev.stats(), kid, (kid, role, la, lb))
        for kid in (31, 13):
            # (upsets far above the data: the threshold's absolute term, tau_abs = 1e-3, dwarfs these products)
            bn = tiles(ft)[kid][1]
            two = [{"row": 33, "col": 3, "add": 7.0}, {"row": 33, "col": bn - 2, "add": _apart(bn)}]
            dev.stats()
            got, _ = run1(t, ft, dev, kid, A, B, la, lb, pad=True, opts=ft.make_opts(faults=two), cd=cd)
            st = dev.stats()
            exact(got, want, (kid, role, la, lb, "recompute", cd), seen)
            assert st["detected"] == 1 and st["recomputed"] == 1 and statuses(st) == [5], (kid, role, st)
    if cd == BF16:
        seen.check(role)


@pytest.mark.gpu
def test_column_block_sum_past_bf16_range(cuda, ft, dev):
    """A column-block sum of B whose elements are all finite and whose total, 2^128 - 2^118, lies between the largest BF16
    value and FLT_MAX: the encode's hi term rounds to Inf in BF16, so the expected checksums of that N-tile are not finite
    and its rows cannot be verified (DESIGN.md §3.3).  They are not flagged and are stored bit for bit as the plain id
    stores them; every other N-tile is checked as usual.  A product term that overflows FP32 (2 x the largest BF16 value)
    lands as Inf where the float64 product rounded to FP32 does."""
    t = cuda
    g = t.Generator(device="cuda").manual_seed(128)
    M, N, K = 260, 388, 201
    A, B = ints(t, g, (M, K), 2), ints(t, g, (N, K), 2)
    k0, n1, n2 = 17, 5, 6                       # in N-tile 0 of every tile width
    B[:, k0] = 0.0
    B[n1, k0], B[n2, k0] = BF16_MAX, 2.0 ** 128 - BF16_MAX - 2.0 ** 118
    assert t.equal(B.to(t.bfloat16).float(), B) and float(B[n2, k0]) == 3 * 2.0 ** 118
    A[:4, k0] = t.tensor([2.0, -2.0, 1.0, 0.0], device="cuda")
    want = reference(A, B).float()             # FP32 rounding of the float64 product: Inf past FLT_MAX
    assert want[0, n1].item() == float("inf") and want[1, n1].item() == float("-inf") and want[2, n1].item() == BF16_MAX
    for plain, kid in ((21, 31), (3, 13), (22, 32)):
        for la, lb in ((MN, MN), (KM, KM), (MN, KM)):
            got_plain, _ = run1(t, ft, dev, plain, A, B, la, lb)
            exact(got_plain, want.double(), (plain, la, lb))
            for front in (0, 1):
                with knobs(ft, enc_front=front):
                    dev.stats()
                    got, _ = run1(t, ft, dev, kid, A, B, la, lb)
                    st = dev.stats()
                tag = (kid, la, lb, front, st)
                assert st["detected"] == 0 and st["recomputed"] == 0 and not st["events"], tag
                assert t.equal(got.contiguous().view(t.int32), got_plain.contiguous().view(t.int32)), tag
                # the other N-tiles' rows are still checked
                assert st["rows_checked"] > 0, tag


# ------------------------------------------------------------------ GPU 8: sensitivity of the exact comparator
@pytest.mark.gpu
def test_sensitivity_low_bit_epilogue_upset(cuda, ft, dev):
    """An unprotected upset of bit 3 of one accumulator value after the check (fault mode 2) on BF16 odd-integer data: the
    exact comparator names exactly that element, while the norm-wise bound of the rest of the suite still passes."""
    t = cuda
    g = t.Generator(device="cuda").manual_seed(73)
    M, N, K = 1024, 1024, 256
    A, B = odd_ints(g, M, N, K, 4)
    want = reference(A, B)
    r, c = 300, 77
    dev.stats()
    got, _ = run16(t, dev, 31, A, B, MN, KM, opts=ft.make_opts(
        faults=[{"row": r, "col": c, "xor": 1 << 3, "where": "epilogue_tmem"}]))
    assert dev.stats()["detected"] == 0
    bad = (got.double() != want).nonzero().tolist()
    assert bad == [[r, c]], mismatch(got, want)
    rel_fro = float(t.linalg.norm(got.double() - want) / t.linalg.norm(want))
    assert 0.0 < rel_fro < TOL_MODEL
