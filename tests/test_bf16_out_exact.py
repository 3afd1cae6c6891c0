"""BF16 results (ftsgemm_run_batched_mixed with BF16 C / D / Z; FtSgemm.matmul / bmm / linear with bfloat16 results) against
a float64 reference rounded once, element by element (DESIGN.md §3.6, §4).

tests/test_bf16_out.py holds every path to its definition: the FP32-output call of the same library, rounded by
.to(torch.bfloat16).  That is only as good as the FP32 call.  Here the reference is independent: the float64 product of the
BF16 values, which on exact data is an FP32 value, rounded to nearest even by round_bf16's integer arithmetic.  The exact
BF16-output paths shared with FP32 output are parametrized in tests/test_bf16_exact.py; this file holds what only a BF16
output has: its 32 kernel instantiations, the rounding edges (ties, the overflow boundary, double rounding through an FP32
subnormal) through every store path, GELU, and the torch layer's BF16 plan branches and gradients.  Every case asserts that
its data needs the rounding: values of more than 8 significant bits and exact ties rounded both ways."""
import math

import numpy as np
import pytest

from test_bf16_exact import (BF16, BF16_MAX, KM, LIMIT, MN, PAIRS, Rounding, _apart, _u32, batch16, bf16_budget_ok, bits16,
                             block_sums, exact, ints, mismatch16, reference, round_bf16, run1, split3, tiles)
from test_bf16_out import LAYOUTS, quiet
from test_exact import GELU_ULP, knobs

NONE, ROW, COL = 0, 1, 2
RELU, GELU = 1, 2
TIES = np.arange(257, 512, 2, dtype=np.float64)   # every odd integer of [257, 511]: an exact BF16 tie (511 -> 512 carries)
# the tie data's targets: the ties, values between ties (257.25 -> 258: more than 8 bits, no tie), exact small integers
TARGETS = np.concatenate([TIES, TIES + 0.25, np.arange(1.0, 33.0)])
SCALES = (1.0, -1.0, 2.0, -0.5)                 # +-2^j keeps a tie a tie
OVER_ALPHA = 2.0 ** 118
SUB_ALPHA = 2.0 ** -126
GELU_WINDOW = 2 * GELU_ULP                     # FP32 ulps of max(|z|, |GELU(z)|) the device's FP32 GELU may be off


def _t():
    import torch
    return torch


# ------------------------------------------------------------------ the three data kinds (no GPU)
def tie_data(M, N, beta=0.0, device="cpu"):
    """A (M, 5), B (N, 5), C0 (M, N) with A B^T + beta C0 = s_m t_n exactly: t_n runs through TARGETS with alternating
    signs (the column-block sums stay small), its three BF16 terms in k = 0..2; s_m through SCALES; C0(m, n) = c_n, BF16
    values up to 48, and k = 3 holds -beta c_n, so the old values are read and the result is still s_m t_n."""
    t = _t()
    n = t.arange(N, dtype=t.float64)
    tn = t.from_numpy(TARGETS)[t.arange(N) % len(TARGETS)] * (1 - 2 * ((n // 2) % 2))
    c = ((n % 7) - 3) * 16
    s = t.tensor(SCALES, dtype=t.float64)[t.arange(M) % len(SCALES)]
    one, zero = t.ones(M, dtype=t.float64), t.zeros(M, dtype=t.float64)
    A = t.stack([s, s, s, one, zero], 1)
    B = t.stack(split3(tn) + [-beta * c, t.zeros(N, dtype=t.float64)], 1)
    C0 = c[None, :].expand(M, N).clone()
    return A.float().to(device), B.float().to(device), C0.float().to(device)


def overflow_data(M, N, device="cpu"):
    """A (M, 2), B (N, 2): accumulators 1020..1023 (1024 - 4 .. 1024 - 1, by 32-column chunk) at columns n = 0 mod 32 and
    their negatives at n = 16 mod 32, zero elsewhere, rows of sign +-1.  Times OVER_ALPHA = 2^118 they are FP32 values and
    round to BF16_MAX, BF16_MAX, Inf (the tie goes to even) and Inf; every 32-column chunk sums to zero, so the checks stay
    finite."""
    t = _t()
    n = t.arange(N)
    v = 1020.0 + ((n // 32) % 4).double()
    sign = t.where(n % 32 == 0, 1.0, t.where(n % 32 == 16, -1.0, 0.0)).double()
    B = t.stack([1024.0 * sign, (v - 1024.0) * sign], 1)
    s = 1.0 - 2.0 * (t.arange(M) % 2).double()
    A = t.stack([s, s], 1)
    return A.float().to(device), B.float().to(device)


def subnormal_data(M, N, device="cpu"):
    """A (M, 3), B (N, 3): accumulators q 2^-7 + 2^-8 +- 2^-25 (q = 0..3), rows of sign +-1.  Times SUB_ALPHA = 2^-126 they
    are (q 2^16 + 2^15 +- 1/4) 2^-149: FP32 subnormals that are not FP32 values.  The kernel rounds them to FP32 first --
    onto the BF16 ties (q 2^16 + 2^15) 2^-149 -- and then to BF16: float64 -> FP32 -> BF16 is the definition here."""
    t = _t()
    n = t.arange(N)
    q = (n % 4).double()
    e = t.where((n // 4) % 2 == 0, 1.0, -1.0).double()
    B = t.stack([q * 2.0 ** -7, t.full((N,), 2.0 ** -8, dtype=t.float64), e * 2.0 ** -25], 1)
    s = 1.0 - 2.0 * (t.arange(M) % 2).double()
    A = t.stack([s, s, s], 1)
    return A.float().to(device), B.float().to(device)


def kind_case(kind, M, N, beta, device):
    """(A, B, C0, alpha, double_round) of one data kind; C0 None where it is zero"""
    if kind == "ties":
        A, B, C0 = tie_data(M, N, beta, device)
        return A, B, C0, 1.0, False
    if kind == "overflow":
        A, B = overflow_data(M, N, device)
        return A, B, None, OVER_ALPHA, False
    A, B = subnormal_data(M, N, device)
    return A, B, None, SUB_ALPHA, True


def gelu64(z):
    return 0.5 * z * (1.0 + _t().erf(z / math.sqrt(2.0)))


def _value16(bits):
    return (bits << 16).to(_t().int32).view(_t().float32).double()


def gelu_mismatch(got, z):
    """(elements that differ, elements whose window holds a BF16 midpoint).  The device's GELU is z 0.5 (1 + erff(z / sqrt 2))
    in FP32: within GELU_WINDOW FP32 ulps of max(|z|, |g|) of the float64 GELU g of the exact z.  Ulps of z, not of g: for
    negative z, 1 + erff cancels, and the error is a few ulps of z but thousands of ulps of the small result.  got must be
    the BF16 rounding of a value in that window: g rounded once wherever the window holds no BF16 midpoint, and otherwise
    one of the (few) BF16 values the window rounds to."""
    t = _t()
    g = gelu64(z)
    e = t.frexp(t.maximum(z.abs(), g.abs()).clamp_min(2.0 ** -126))[1].double()
    win = GELU_WINDOW * t.exp2(e - 24)
    lo, hi = _value16(round_bf16(g - win, double_round=True)), _value16(round_bf16(g + win, double_round=True))
    v = got.double()
    ok = (v >= lo) & (v <= hi)
    return int((~ok).sum()), int((lo != hi).sum())


# ------------------------------------------------------------------ CPU tests
def test_round_bf16_table():
    """round_bf16 on the edges the kernels must get right, and torch's CPU cast agrees"""
    t = _t()
    table = [(257.0, 256.0), (259.0, 260.0), (511.0, 512.0), (-257.0, -256.0), (-259.0, -260.0), (258.0, 258.0),
             (257.25, 258.0), (2.0 ** 128 - 2.0 ** 119, math.inf), (-(2.0 ** 128 - 2.0 ** 119), -math.inf),
             (2.0 ** 128 - 2.0 ** 119 - 2.0 ** 104, BF16_MAX), (510 * 2.0 ** 119, BF16_MAX), (BF16_MAX, BF16_MAX),
             (2.0 ** -133, 2.0 ** -133), (3 * 2.0 ** -134, 2.0 ** -132), (2.0 ** -134, 0.0), (5 * 2.0 ** -134, 2.0 ** -132),
             (7 * 2.0 ** -134, 2.0 ** -131), (2.0 ** -126 - 2.0 ** -133, 2.0 ** -126 - 2.0 ** -133), (-0.0, -0.0),
             (math.inf, math.inf)]
    x = t.tensor([a for a, _ in table], dtype=t.float64)
    want = t.tensor([b for _, b in table], dtype=t.float32).to(t.bfloat16)
    assert mismatch16(want, round_bf16(x)) == ""
    assert t.equal(bits16(x.float().to(t.bfloat16)), round_bf16(x))
    assert t.equal(bits16(want), round_bf16(x))                                        # (the sign of zero too)
    assert int(round_bf16(t.tensor([math.nan], dtype=t.float64))[0]) == 0x7FC0
    # a value that is not an FP32 value is refused unless declared
    with pytest.raises(AssertionError):
        round_bf16(t.tensor([1.0 + 2.0 ** -30], dtype=t.float64))
    assert int(round_bf16(t.tensor([1.0 + 2.0 ** -30], dtype=t.float64), double_round=True)[0]) == 0x3F80


def test_round_bf16_random_bit_patterns():
    """4 million random FP32 bit patterns (every exponent, NaNs, Infs, subnormals): round_bf16 equals torch's CPU cast,
    NaN for NaN"""
    t = _t()
    rng = np.random.default_rng(16)
    u = rng.integers(0, 2 ** 32, 4 << 20, dtype=np.uint64).astype(np.uint32)
    u[:65536] = (u[:65536] & 0xFFFF0000) | 0x8000        # exact ties, every BF16 value below them
    f = t.from_numpy(u.view(np.float32).copy())
    got = round_bf16(f.double())
    want = bits16(f.to(t.bfloat16))
    nan = t.isnan(f)
    assert t.equal(got[~nan], want[~nan])
    assert bool(((want[nan] & 0x7FFF) > 0x7F80).all()) and bool((got[nan] == 0x7FC0).all())


def test_comparator_and_tally():
    t = _t()
    want = t.tensor([257.0, 259.0, 1.0, 0.0, math.nan], dtype=t.float64)
    got = t.tensor([256.0, 260.0, 1.0, -0.0, math.nan]).to(t.bfloat16)
    assert mismatch16(got, round_bf16(want)) == ""
    bad = got.clone()
    bad.view(t.int16)[1] ^= 1
    assert mismatch16(bad, round_bf16(want)).startswith("1 elements differ")
    seen = Rounding()
    seen.add(want)
    assert (seen.wide, seen.down, seen.up) == (2, 1, 1)
    seen.check("table")
    with pytest.raises(AssertionError):
        s2 = Rounding()
        s2.add(t.tensor([1.0, 256.0, 300.0], dtype=t.float64))
        s2.check("no ties")


def test_rounding_edge_data():
    """The three data kinds are what they claim, and a kernel that rounded ties away from zero (cvt.rna) or truncated would
    fail on the tie data in many elements: the comparator is sensitive to the rounding mode."""
    t = _t()
    M, N = 260, 292
    for beta in (0.0, -2.0, 1.0):
        A, B, C0 = tie_data(M, N, beta)
        assert t.equal(A.to(t.bfloat16).float(), A) and t.equal(B.to(t.bfloat16).float(), B)
        assert t.equal(C0.to(t.bfloat16).float(), C0)
        want = reference(A, B, 1.0, beta, C0)
        target = t.from_numpy(TARGETS)[t.arange(N) % len(TARGETS)] * (1 - 2 * ((t.arange(N) // 2) % 2)).double()
        s = t.tensor(SCALES, dtype=t.float64)[t.arange(M) % 4]
        assert t.equal(want, s[:, None] * target[None, :])
        seen = Rounding()
        seen.add(want)
        seen.check(beta)
        assert seen.down > 1000 and seen.up > 1000
        # the column-block sums (plain and weighted) of this B stay exact in the encode's three BF16 terms
        for BN in (128, 256):
            assert max(float(x.abs().max()) for x in block_sums(B, BN)) <= LIMIT
    # the carry 511 -> 512 and both signs
    r = round_bf16(want)
    assert set(r[want == 511.0].tolist()) == {0x4400} and set(r[want == -511.0].tolist()) == {0xC400}     # +-512
    assert bool((want == 511.0).any()) and bool((want == -511.0).any())
    # sensitivity: ties away from zero, and truncation, differ from nearest even
    u = _u32(want.float())
    rna = (u + 0x8000) >> 16
    trunc = u >> 16
    got_rna = (rna << 16).to(t.int32).view(t.float32).to(t.bfloat16)
    got_trunc = (trunc << 16).to(t.int32).view(t.float32).to(t.bfloat16)
    n_rna = int(mismatch16(got_rna, r).split()[0])
    n_trunc = int(mismatch16(got_trunc, r).split()[0])
    assert n_rna > 1000 and n_trunc > 1000, (n_rna, n_trunc)
    # overflow: 1020, 1021 -> BF16_MAX, 1022 (a tie) and 1023 -> Inf, negatives alike; every FP32 product finite
    A, B = overflow_data(4, 128)
    want = reference(A, B, OVER_ALPHA)
    assert bool(t.isfinite(want.float()).all())
    r = round_bf16(want)
    assert [int(r[0, n]) for n in (0, 32, 64, 96)] == [0x7F7F, 0x7F7F, 0x7F80, 0x7F80]
    assert [int(r[0, n]) for n in (16, 48, 80, 112)] == [0xFF7F, 0xFF7F, 0xFF80, 0xFF80]
    assert [int(r[1, n]) for n in (0, 96)] == [0xFF7F, 0xFF80]
    assert float(t.tensor(BF16_MAX)) == 255 * 2.0 ** 120 == 1020 * OVER_ALPHA
    # double rounding: the results are FP32 subnormals that FP32 rounds onto BF16 ties; rounding float64 once would differ
    A, B = subnormal_data(4, 64)
    want = reference(A, B, SUB_ALPHA)
    assert bool((want.abs() < 2.0 ** -126).all()) and bool((want.float().double() != want).all())
    twice = round_bf16(want, double_round=True)
    units = want / 2.0 ** -149
    once = t.round(units / 65536.0) * 65536.0 * 2.0 ** -149            # float64 straight to BF16 (no ties in float64)
    differ = (twice != round_bf16(once)) & (once != 0)
    assert int(differ.sum()) >= 8, int(differ.sum())


def test_instantiation_and_gelu_sets_are_within_budget():
    assert bf16_budget_ok(768, 4, 4, -0.5, 2.0, 64, 64)
    assert 768 // 64 // 3 >= 4                      # splitk 3: three pieces of at least 4 k-blocks of 64
    assert bf16_budget_ok(96, 4, 4, 2.0 ** -6, 0.0, 0.0, 64)
    # the GELU comparator: an FP32 GELU passes, one BF16 ulp off does not, and where 1 + erf cancels (z < -4) its window is
    # a few BF16 ulps of the small result
    t = _t()
    z = t.linspace(-6.0, 6.0, 20001, dtype=t.float64).float().double()
    z32 = z.float()
    d16 = (z32 * 0.5 * (1.0 + t.erf(z32 * 0.70710678118654752))).to(t.bfloat16)
    bad, near = gelu_mismatch(d16, z)
    assert bad == 0 and 0 < near < len(z) // 3, (bad, near)
    off = (d16.view(t.int16) + 1).view(t.bfloat16)
    keep = z.abs() < 3.0
    assert gelu_mismatch(off[keep], z[keep])[0] > 0.9 * int(keep.sum())


# ------------------------------------------------------------------ GPU harness
@pytest.fixture(scope="module")
def dev(cuda, ft):
    cuda.cuda.set_device(0)
    h = ft.FtSgemm()
    yield h
    h.close()


def _kinds(dev):
    return {it["kind"] for unit in dev.debug_trace() for it in unit}


# ------------------------------------------------------------------ GPU 1: every BF16-output instantiation
@pytest.mark.gpu
def test_every_bf16_output_instantiation(cuda, ft, dev):
    """Each of the 32 BF16-output kernels (tile width 256 / 128, plain / ABFT, seeded / not, four layout pairs) on exact
    data with beta != 0, D != C and a COL bias, at levels 0 / 1 / 2 on the ABFT ones, with splitk 0, 2 and 3: D is the
    float64 result rounded once and bit-identical across splitk.  Which kernel ran is read from the work items of the
    launch (debug_set("trace", 1), FtSgemm.debug_trace): with splitk 0 every item is a whole tile (kind 0), so the unseeded
    kernel ran; with splitk 2 / 3 there are last pieces (kind 2), and with 3 middle pieces (kind 3), which only the seeded
    kernel runs."""
    t = cuda
    M, K = 260, 768
    ran = set()
    seen = Rounding()
    for plain, abft in (PAIRS["256"], PAIRS["128"]):
        bn = tiles(ft)[abft][1]
        N = 2 * bn + 36
        g = t.Generator(device="cuda").manual_seed(bn)
        A, B = ints(t, g, (M, K), 4), ints(t, g, (N, K), 4)
        C0, bias = ints(t, g, (M, N), 64), ints(t, g, (N,), 64)
        want = reference(A, B, -0.5, 2.0, C0, bias, COL)
        for kid, fault_tolerant in ((plain, False), (abft, True)):
            for la, lb in LAYOUTS:
                for level in ((0, 1, 2) if fault_tolerant else (0,)):
                    first = None
                    for sk in (0, 2, 3):
                        tag = (kid, bn, la, lb, level, sk)
                        with knobs(ft, splitk=sk, trace=1):
                            dev.stats()
                            got, _ = run1(t, ft, dev, kid, A, B, la, lb, pad=True, alpha=-0.5, beta=2.0, C0=C0, bias=bias,
                                          mode=COL, out_of_place=True, opts=ft.make_opts(protect_epilogue=level), cd=BF16)
                            kinds = _kinds(dev)
                            st = dev.stats()
                        quiet(st, tag)
                        exact(got, want, tag, seen)
                        if sk == 0:
                            assert kinds == {0}, (tag, kinds)
                        else:
                            assert 2 in kinds and (3 in kinds) == (sk == 3), (tag, kinds)
                        if first is None:
                            first = bits16(got)
                        assert t.equal(bits16(got), first), tag
                        ran.add((bn, fault_tolerant, sk > 0, (la, lb)))
    print("BF16-output instantiations run (BN, ft, seed, layouts):", sorted(ran))
    assert len(ran) == 32
    seen.check("instantiations")


# ------------------------------------------------------------------ GPU 2: rounding edges through every store path
PATHS = ("full N, beta != 0", "full N, beta = 0", "ragged N", "level 1", "level 1, repair", "level 2", "level 2, repair",
         "ReLU with Z", "row recompute")


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["ties", "overflow", "double"])
def test_rounding_edges_every_store_path(cuda, ft, dev, kind):
    """Ties of both parities and signs with the carry 511 -> 512 ("ties"), alpha = 2^118 on accumulators 1020..1023
    ("overflow": BF16_MAX, BF16_MAX, Inf, Inf and negatives, no alarm at any level) and FP32-subnormal results rounded
    float64 -> FP32 -> BF16 ("double"), each through every store path: store_tile over full N-tiles with beta != 0 (the
    pipelined old values) and beta = 0, the ragged-N element loop, level 1 and level 2 clean and repairing (level 1's segment
    recompute into D; level 2's chunk recompute at the last column of the ragged corner), ReLU with Z, and the row recompute
    (two upsets in one row).  Ids 31 (BN 256) and 13 (BN 128); D != C except in place on the first path.  The overflow data
    skips the two epilogue repairs: every chunk holds a value near 2^128, so the level 1 / 2 tolerance of the chunk is not
    finite and an upset there cannot be told from rounding (the non-finite rules of DESIGN.md §3.6)."""
    t = cuda
    seen = Rounding()
    M = 260
    for kid in (31, 13):
        bn = tiles(ft)[kid][1]
        for path in PATHS:
            if kind == "overflow" and path.endswith("repair"):
                continue
            N = 2 * bn if path.startswith("full") else bn + 36
            beta = 0.0 if path == "full N, beta = 0" else -2.0
            A, B, C0, alpha, dr = kind_case(kind, M, N, beta, "cuda")
            want = reference(A, B, alpha, beta, t.zeros(M, N, device="cuda") if C0 is None else C0)
            level = 2 if path.startswith("level 2") else 1 if path.startswith("level 1") else 0
            faults = None
            if path == "level 1, repair":
                faults = [{"row": 37, "col": 40, "xor": 1 << 30, "where": "epilogue_value"}]
            elif path == "level 2, repair":
                faults = [{"row": M - 1, "col": N - 1, "xor": 1 << 30, "where": "epilogue_value"}]
            elif path == "row recompute":
                faults = [{"row": 33, "col": 3, "add": 7.0}, {"row": 33, "col": bn - 2, "add": _apart(bn)}]
            act = RELU if path == "ReLU with Z" else 0
            tag = (kind, kid, path)
            dev.stats()
            got, z = run1(t, ft, dev, kid, A, B, MN if kid == 13 else KM, KM, pad=True, alpha=alpha, beta=beta, C0=C0,
                          act=act, z=act != 0, out_of_place=path != "full N, beta != 0",
                          opts=ft.make_opts(protect_epilogue=level, faults=faults), cd=BF16)
            st = dev.stats()
            if faults:
                assert st["uncorrectable"] == 0 and st["recomputed"] >= 1, (tag, st)
            else:
                quiet(st, tag)
            if act:
                exact(z, want, tag + ("Z",), seen, dr)
                exact(got, t.relu(want), tag, None, dr)
            else:
                exact(got, want, tag, seen, dr)
            if kind == "overflow":
                assert bool(t.isinf(got).any()) and bool((got.float() == BF16_MAX).any()), tag
    if kind == "ties":
        seen.check(kind)


# ------------------------------------------------------------------ GPU 3: GELU against float64
@pytest.mark.gpu
def test_gelu_against_float64(cuda, ft, dev):
    """GELU with Z, BF16 output: Z16 is the exact z rounded once, and D16 the float64 GELU of that exact z rounded once,
    except where the device's FP32 GELU may lie on either side of a BF16 midpoint (gelu_mismatch: within GELU_WINDOW FP32
    ulps; their number is printed).  Levels 0 / 1 / 2 on id 31, ragged N, and a batch with a per-entry bias on ids 31 and
    13."""
    t = cuda
    g = t.Generator(device="cuda").manual_seed(2)
    M, N, K = 260, 300, 96
    alpha = 2.0 ** -6                         # z of order 1, where GELU bends
    A, B = ints(t, g, (M, K), 4), ints(t, g, (N, K), 4)
    bias = ints(t, g, (N,), 64) * 2.0 ** -6
    z = reference(A, B, alpha, 0.0, None, bias, COL)
    seen = Rounding()
    near = {}
    for level in (0, 1, 2):
        dev.stats()
        got, z16 = run1(t, ft, dev, 31, A, B, KM, MN, pad=True, alpha=alpha, bias=bias, mode=COL, act=GELU, z=True,
                        opts=ft.make_opts(protect_epilogue=level), cd=BF16)
        quiet(dev.stats(), ("gelu", level))
        exact(z16, z, ("Z", level), seen)
        bad, near[level] = gelu_mismatch(got, z)
        assert bad == 0, (level, bad)
    Bt = 3
    Ab, Bb = ints(t, g, (Bt, M, K), 4), ints(t, g, (Bt, N, K), 4)
    pb = ints(t, g, (Bt, N), 64) * 2.0 ** -6
    zb = reference(Ab, Bb, alpha, 0.0, None, pb, COL)
    for kid in (31, 13):
        dev.stats()
        got, z16 = batch16(t, ft, dev, kid, Ab, Bb, KM, KM, pad=True, gap=8, alpha=alpha, bias=pb, mode=COL, act=GELU, z=True,
                           out_of_place=True, cd=BF16)
        quiet(dev.stats(), ("gelu batch", kid))
        exact(z16, zb, ("Z batch", kid), seen)
        bad, near[("batch", kid)] = gelu_mismatch(got, zb)
        assert bad == 0, (kid, bad)
    print(f"GELU, BF16 output: elements within {GELU_WINDOW} FP32 ulps of a BF16 midpoint (of {M * N}, {Bt * M * N}):", near)
    seen.check("gelu")


# ------------------------------------------------------------------ GPU 4: the torch layer, exact
def _bf_ints(t, g, shape, amax):
    return t.randint(-amax, amax + 1, shape, generator=g, device="cuda", dtype=t.int32).to(t.bfloat16)


@pytest.mark.gpu
def test_torch_layer_exact(cuda, ft, dev):
    """matmul / bmm / linear with bfloat16 results on integer bfloat16 data, against float64 rounded once, through every plan
    branch: a row-major out in place; a column-major out (a .t() view: no swap, the bias per kernel row); a copied out (a
    leading stride that is not a multiple of 8 at a base that is not 16-byte aligned, the bytes around it untouched); a bmm
    out whose batch stride is not a multiple of 8; a c with strides other than the destination's; beta != 0 with out as C;
    an expanded operand; a per-entry bias; 3-D linear with a bfloat16 residual and bias; ReLU with preact."""
    t = cuda
    g = t.Generator(device="cuda").manual_seed(12)
    seen = Rounding()
    M, N, K = 192, 264, 200
    a, b = _bf_ints(t, g, (M, K), 4), _bf_ints(t, g, (K, N), 4)
    bias = _bf_ints(t, g, (N,), 64)
    prod = a.double() @ b.double()
    want = prod + bias.double()

    def check(got, ref, tag):
        assert got.dtype == t.bfloat16, tag
        exact(got, ref, tag, seen)

    out = t.empty(M, N, device="cuda", dtype=t.bfloat16)
    dev.matmul(a, b, out, bias=bias)
    check(out, want, "row-major out")
    colmajor = t.empty(N, M, device="cuda", dtype=t.bfloat16).t()
    dev.matmul(a, b, colmajor, bias=bias)
    check(colmajor, want, "column-major out")
    wide = t.full((M, N + 4), 7.0, device="cuda", dtype=t.bfloat16)
    out = wide[:, 2:N + 2]
    dev.matmul(a, b, out, bias=bias)
    check(out, want, "copied out")
    assert bool((wide[:, :2] == 7).all()) and bool((wide[:, N + 2:] == 7).all())
    c = _bf_ints(t, g, (M, N), 64)
    ccol = c.t().contiguous().t()                                  # column-major: not out's strides
    y = dev.matmul(a, b, t.empty(M, N, device="cuda", dtype=t.bfloat16), c=ccol, beta=-2.0)
    check(y, prod - 2.0 * c.double(), "c with other strides")
    out = c.clone()
    dev.matmul(a, b, out, beta=-2.0)
    check(out, prod - 2.0 * c.double(), "beta != 0, out as C")
    z16 = t.empty(M, N, device="cuda", dtype=t.bfloat16)
    out = t.empty(M, N, device="cuda", dtype=t.bfloat16)
    dev.matmul(a, b, out, bias=bias, activation="relu", preact=z16)
    check(z16, want, "preact")
    check(out, t.relu(want), "relu")
    # bmm
    Bt = 3
    ab, bb = _bf_ints(t, g, (Bt, M, K), 4), _bf_ints(t, g, (Bt, K, N), 4)
    pb = _bf_ints(t, g, (Bt, N), 64).float()
    wantb = ab.double() @ bb.double() + pb.double()[:, None, :]
    check(dev.bmm(ab, bb, bias=pb, out_dtype=t.bfloat16), wantb, "per-entry bias")
    flat = t.full((Bt, M * N + 4), 7.0, device="cuda", dtype=t.bfloat16)
    out = flat[:, :M * N].view(Bt, M, N)
    assert out.stride(0) % 8 == 4
    dev.bmm(ab, bb, out, bias=pb)
    check(out, wantb, "batch stride not a multiple of 8")
    assert bool((flat[:, M * N:] == 7).all())
    a1 = _bf_ints(t, g, (1, M, K), 4).expand(Bt, M, K)
    check(dev.bmm(a1, bb, out_dtype=t.bfloat16), a1.double() @ bb.double(), "expanded a")
    b1 = _bf_ints(t, g, (1, K, N), 4).expand(Bt, K, N)
    check(dev.bmm(ab, b1, out_dtype=t.bfloat16), ab.double() @ b1.double(), "expanded b")
    # 3-D linear with a residual and a bias
    x, W = _bf_ints(t, g, (2, 96, K), 4), _bf_ints(t, g, (N, K), 4)
    r = _bf_ints(t, g, (2, 96, N), 64)
    y = dev.linear(x, W, bias, residual=r, out_dtype=t.bfloat16)
    check(y, x.double() @ W.double().t() + r.double() + bias.double(), "linear, residual, bias")
    quiet(dev.stats(), "torch layer")
    seen.check("torch layer")


@pytest.mark.gpu
def test_torch_layer_gradients_exact(cuda, ft, dev):
    """With integer bfloat16 data and an integer grad_y, the bfloat16 gradients of linear (no activation with a residual,
    and ReLU) and of bmm with c are the float64 products rounded once, bit for bit: x.grad, W.grad, bias.grad, r.grad and
    c.grad."""
    t = cuda
    g = t.Generator(device="cuda").manual_seed(13)
    seen = Rounding()
    T, N, K = 256, 192, 128
    x = _bf_ints(t, g, (T, K), 4).requires_grad_()
    W = _bf_ints(t, g, (N, K), 4).requires_grad_()
    bias = _bf_ints(t, g, (N,), 16).requires_grad_()
    r = _bf_ints(t, g, (T, N), 16).requires_grad_()
    gy = _bf_ints(t, g, (T, N), 4)
    for act, res in ((None, r), ("relu", None)):
        y = dev.linear(x, W, bias, activation=act, residual=res, out_dtype=t.bfloat16)
        y.backward(gy)
        gz = gy.double()
        if act == "relu":
            gz = gz * (y.detach().double() > 0)
        else:
            assert r.grad.dtype == t.bfloat16 and t.equal(r.grad, gy)
        exact(x.grad, gz @ W.detach().double(), (act, "x.grad"), seen)
        exact(W.grad, gz.t() @ x.detach().double(), (act, "W.grad"), seen)
        exact(bias.grad, gz.sum(0), (act, "bias.grad"), seen)
        for p in (x, W, bias, r):
            p.grad = None
    Bt = 2
    a = _bf_ints(t, g, (Bt, 64, K), 4).requires_grad_()
    bm = _bf_ints(t, g, (Bt, K, 96), 4).requires_grad_()
    c = _bf_ints(t, g, (Bt, 64, 96), 16).requires_grad_()
    y = dev.bmm(a, bm, c=c, beta=0.5)
    gyb = _bf_ints(t, g, (Bt, 64, 96), 4)
    y.backward(gyb)
    gd = gyb.double()
    exact(a.grad, gd @ bm.detach().double().transpose(1, 2), "a.grad", seen)
    exact(bm.grad, a.detach().double().transpose(1, 2) @ gd, "b.grad", seen)
    exact(c.grad, 0.5 * gd, "c.grad")
    dev.stats()
    seen.check("gradients")
