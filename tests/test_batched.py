"""Strided-batched fault-tolerant GEMM (ftsgemm_run_batched, FtSgemm.run_batched / bmm).

Entry i of a batched call is exactly the ftsgemm_run_bias product on A + i*stride_a, B + i*stride_b, C + i*stride_c: every
tensor-core kernel gives each entry bit for bit what run_bias gives on that entry alone, writes nothing between the entries
or in C's padding, and never lets an operand entry's neighbour into its tiles (the operands' gaps hold NaN).  The CPU tests
check the ABI's NULL-handle answer, the torch stride mapping of bmm and the batched work plan; the rest run on the GPU.
"""
import numpy as np
import pytest

TOL_NORM = 1e-3
TOL_MODEL = 5e-5
MN, KM = 0, 1
NAMES = ["small", "medium", "large", "tall", "wide", "huge", "giant", "pair128"]


# ------------------------------------------------------------------ CPU
def test_run_batched_null_handle(ft):
    assert ft.lib().ftsgemm_run_batched(None, 40, 128, 128, 128, None, 0, 128, 0, None, 0, 128, 0, None, 128, 0, 2, 1.0, 0.0,
                                        None, 0, None) == -4


def _st(rows, cols, rm, pad=0):
    return (cols + pad, 1) if rm else (1, rows + pad)


@pytest.mark.parametrize("a_rm", [True, False])
@pytest.mark.parametrize("b_rm", [True, False])
@pytest.mark.parametrize("o_rm", [True, False])
def test_bmm_plan_strides(ft, a_rm, b_rm, o_rm):
    Bt, M, N, K = 5, 64, 96, 40
    for pad, extra in ((0, 0), (4, 8)):
        sa = (M * K if a_rm else K * M) + pad * (M if a_rm else K) + extra
        sb = (K * N if b_rm else N * K) + pad * (K if b_rm else N) + extra
        so = M * N + pad * (M if o_rm else N) + extra
        p = ft.bmm_plan((Bt, M, K), (sa,) + _st(M, K, a_rm, pad), (Bt, K, N), (sb,) + _st(K, N, b_rm, pad),
                        (so,) + _st(M, N, o_rm, pad), 256, 512, 1024)
        m = ft.matmul_plan((M, K), _st(M, K, a_rm, pad), (K, N), _st(K, N, b_rm, pad), _st(M, N, o_rm, pad), 256, 512, 1024)
        assert not (p["copy_a"] or p["copy_b"] or p["copy_out"]), p
        for k in ("M", "N", "K", "layout_a", "lda", "layout_b", "ldb", "ldc", "swap"):
            assert p[k] == m[k], k
        assert p["batch"] == Bt and p["stride_c"] == so
        assert (p["stride_a"], p["stride_b"]) == ((sb, sa) if o_rm else (sa, sb))


def test_bmm_plan_marks_copies(ft):
    Bt, M, N, K = 4, 64, 96, 40
    rm = lambda r, c: (r * c, c, 1)  # noqa: E731  contiguous row-major (Bt, r, c)
    # contiguous bmm operands and q @ k.transpose(-1, -2): nothing copied
    p = ft.bmm_plan((Bt, M, K), rm(M, K), (Bt, K, N), rm(K, N), rm(M, N))
    assert not (p["copy_a"] or p["copy_b"] or p["copy_out"])
    p = ft.bmm_plan((Bt, M, K), rm(M, K), (Bt, K, N), (N * K, 1, K), rm(M, N))  # k (Bt, N, K) transposed
    assert not (p["copy_a"] or p["copy_b"] or p["copy_out"]) and p["layout_a"] == KM and p["layout_b"] == KM
    # expand()ed operand (batch stride 0)
    p = ft.bmm_plan((Bt, M, K), (0, K, 1), (Bt, K, N), rm(K, N), rm(M, N))
    assert p["copy_a"] and not p["copy_b"] and p["stride_b"] == M * K  # swapped: the copy of a is kernel B
    # batch stride not a multiple of 4 floats
    p = ft.bmm_plan((Bt, M, K), (M * K + 2, K, 1), (Bt, K, N), rm(K, N), rm(M, N))
    assert p["copy_a"] and not p["copy_b"]
    # misaligned base, non-unit stride
    p = ft.bmm_plan((Bt, M, K), rm(M, K), (Bt, K, N), rm(K, N), rm(M, N), a_ptr=260)
    assert p["copy_a"]
    p = ft.bmm_plan((Bt, M, K), rm(M, K), (Bt, K, N), (2 * K * N, 2 * N, 2), rm(M, N))
    assert p["copy_b"] and not p["copy_a"]
    # out entries overlapping / not a multiple of 4 apart
    p = ft.bmm_plan((Bt, M, K), rm(M, K), (Bt, K, N), rm(K, N), (M * N - 4, N, 1))
    assert p["copy_out"] and p["stride_c"] == M * N
    # one entry: batch strides do not matter
    p = ft.bmm_plan((1, M, K), (0, K, 1), (1, K, N), (3, N, 1), (1, N, 1))
    assert not (p["copy_a"] or p["copy_b"] or p["copy_out"])
    with pytest.raises(ValueError):
        ft.bmm_plan((Bt, M, K), rm(M, K), (Bt + 1, K, N), rm(K, N), rm(M, N))


def _simulate_batched(hdr, segs):
    """tests/test_schedule.py's circular-wait simulation, with a data tile of entry i waiting for entry i's checksum tiles"""
    units = hdr["units"]
    per_unit = [[] for _ in range(units)]
    for s in segs:
        per_unit[s["unit"]].append(s)
    chk_done, piece_at, tiles_c = {}, {}, 0
    for u, lst in enumerate(per_unit):
        for i, s in enumerate(lst):
            if s["is_chk"]:
                chk_done[(s["batch"], s["m_blk"], s["n_blk"], s["slice"])] = False
                tiles_c = max(tiles_c, s["n_blk"] + 1)
            if s["kind"] in (1, 2, 3):
                piece_at[(s["tile"], s["slice"])] = (u, i)
    mma, epi, done = [0] * units, [0] * units, set()
    progress = True
    while progress:
        progress = False
        for u, lst in enumerate(per_unit):
            while mma[u] < len(lst) and mma[u] - epi[u] < 1:
                s = lst[mma[u]]
                if s["kind"] in (2, 3) and piece_at[(s["tile"], s["slice"] - 1)] not in done:
                    break
                mma[u] += 1
                progress = True
            while epi[u] < mma[u]:
                s = lst[epi[u]]
                if hdr["n_chk_tiles"] and not s["is_chk"] and s["kind"] in (0, 2):
                    if not all(chk_done[(s["batch"], s["m_blk"], c, sl)] for c in range(tiles_c)
                               for sl in range(max(1, hdr["chk_slices"]))):
                        break
                done.add((u, epi[u]))
                if s["is_chk"]:
                    chk_done[(s["batch"], s["m_blk"], s["n_blk"], s["slice"])] = True
                epi[u] += 1
                progress = True
    return all(epi[u] == len(per_unit[u]) for u in range(units))


@pytest.mark.parametrize("kid", [6, 21, 13, 14, 16, 15, 31, 40])
@pytest.mark.parametrize("shape", [(1024, 1024, 128), (1024, 128, 1024), (260, 388, 201), (2048, 2048, 2048), (128, 4096, 512)])
@pytest.mark.parametrize("batch", [1, 3, 64])
@pytest.mark.parametrize("splitk", [-1, 2])
def test_batched_schedule_covers_and_cannot_deadlock(ft, kid, shape, batch, splitk):
    M, N, K = shape
    num_sms = 132
    try:
        ft.debug_set("splitk", splitk)
        hdr, segs = ft.debug_schedule_batched(kid, M, N, K, batch, num_sms)
        if batch == 1:
            h1, s1 = ft.debug_schedule(kid, M, N, K, num_sms)
            assert hdr == h1 and [{k: v for k, v in s.items() if k != "batch"} for s in segs] == s1
            assert all(s["batch"] == 0 for s in segs)
    finally:
        ft.debug_set("splitk", -1)
    num_kb = hdr["num_kb"]
    cover = {}
    for s in segs:
        assert 0 <= s["batch"] < batch
        cover.setdefault(s["tile"], []).append((s["kb_begin"], s["kb_end"], s["batch"], s["m_blk"], s["n_blk"], s["is_chk"]))
    assert sorted(cover) == list(range(hdr["num_tiles"]))
    S = max(1, hdr["chk_slices"])
    keys = set()
    for t, pieces in cover.items():
        pieces.sort()
        assert len({p[2:] for p in pieces}) == 1  # all pieces of a tile name the same (entry, tile)
        key = pieces[0][2:] + ((t // (hdr["n_chk_tiles"] // S)) if t < hdr["n_chk_tiles"] else 0,)
        assert key not in keys
        keys.add(key)
        if t < hdr["n_chk_tiles"] and S > 1:
            continue
        assert pieces[0][0] == 0 and pieces[-1][1] == num_kb
        assert all(a[1] == b[0] for a, b in zip(pieces, pieces[1:]))  # every k-block once
    data = {(s["batch"], s["m_blk"], s["n_blk"]) for s in segs if not s["is_chk"]}
    assert len(data) == hdr["num_tiles"] - hdr["n_chk_tiles"]
    assert len(data) % batch == 0 and len({d[0] for d in data}) == batch
    if splitk == 2 and hdr["sk_tiles"] == 0:
        pytest.skip("too few k-blocks to cut")
    assert _simulate_batched(hdr, segs), "circular wait in the batched schedule"


# ------------------------------------------------------------------ GPU helpers
def _rand(rng, shape):
    return (rng.integers(0, 10, shape) * 0.1 * rng.choice([-1.0, 1.0], shape)).astype(np.float32)


def _ints(rng, shape):
    """small integers: every product and sum is exact, so a corrected element equals the clean one bit for bit"""
    return rng.integers(-4, 5, shape).astype(np.float32)


def _pack(X, layout, ld):
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


def _stack(parts, stride, fill):
    """entries (flat arrays) at multiples of `stride` floats, gaps filled with `fill`"""
    buf = np.full(stride * (len(parts) - 1) + parts[-1].size, fill, np.float32)
    for i, p in enumerate(parts):
        buf[i * stride:i * stride + p.size] = p
    return buf


class _Batch:
    """Bt products on the GPU: A[i] (M x K), B[i] (N x K), C0[i] (M x N)"""

    def __init__(self, cuda, dev, A, B, C0):
        self.cuda, self.dev, self.A, self.B, self.C0 = cuda, dev, A, B, C0
        self.Bt, self.M, self.K = A.shape
        self.N = B.shape[1]

    def _c_entry(self, i, ldc):
        cbuf = np.full((self.N, ldc), SENTINEL, np.float32)
        cbuf[:, :self.M] = self.C0[i].T
        return cbuf.reshape(-1)

    def one(self, i, kid, la, lda, lb, ldb, ldc, alpha, beta, bias=None, mode=0, opts=None):
        """run_bias on entry i alone"""
        t = self.cuda
        dA = t.from_numpy(_pack(self.A[i], la, lda)).cuda()
        dB = t.from_numpy(_pack(self.B[i], lb, ldb)).cuda()
        dC = t.from_numpy(self._c_entry(i, ldc)).cuda()
        db = t.from_numpy(bias).cuda() if bias is not None else None
        self.dev.run_bias(kid, self.M, self.N, self.K, dA, la, lda, dB, lb, ldb, dC, ldc, alpha, beta, db, mode, opts)
        t.cuda.synchronize()
        return dC.cpu().numpy().reshape(self.N, ldc)[:, :self.M].T

    def batched(self, kid, la, lda, lb, ldb, ldc, alpha, beta, bias=None, mode=0, opts=None, gap=8):
        """run_batched on all entries, `gap` floats (NaN in A / B, SENTINEL in C) between them"""
        t = self.cuda
        pa = [_pack(self.A[i], la, lda) for i in range(self.Bt)]
        pb = [_pack(self.B[i], lb, ldb) for i in range(self.Bt)]
        pc = [self._c_entry(i, ldc) for i in range(self.Bt)]
        sa, sb, sc = pa[0].size + gap, pb[0].size + gap, pc[0].size + gap
        dA = t.from_numpy(_stack(pa, sa, np.nan)).cuda()
        dB = t.from_numpy(_stack(pb, sb, np.nan)).cuda()
        dC = t.from_numpy(_stack(pc, sc, SENTINEL)).cuda()
        db = t.from_numpy(bias).cuda() if bias is not None else None
        self.dev.run_batched(kid, self.M, self.N, self.K, dA, la, lda, sa, dB, lb, ldb, sb, dC, ldc, sc, self.Bt, alpha, beta,
                             db, mode, opts)
        t.cuda.synchronize()
        out = dC.cpu().numpy()
        res = []
        for i in range(self.Bt):
            e = out[i * sc:i * sc + pc[0].size].reshape(self.N, ldc)
            assert np.all(e[:, self.M:] == SENTINEL), "C's padding was written"
            if i + 1 < self.Bt:
                assert np.all(out[i * sc + pc[0].size:(i + 1) * sc] == SENTINEL), "a gap between C entries was written"
            res.append(e[:, :self.M].T)
        return np.stack(res)


def _rel(ref, x):
    ref, x = ref.astype(np.float64), x.astype(np.float64)
    return float(np.linalg.norm(ref - x) / np.linalg.norm(ref))


@pytest.fixture(scope="module")
def dev(cuda, ft):
    cuda.cuda.set_device(0)
    h = ft.FtSgemm()
    yield h
    h.close()


def _case(cuda, dev, seed, Bt=3, M=260, N=388, K=201, scales=None, gen=_rand):
    rng = np.random.default_rng(seed)
    A = np.stack([gen(rng, (M, K)) for _ in range(Bt)])
    if scales is not None:  # (powers of two: the entries stay exact)
        A *= np.asarray(scales, np.float32)[:, None, None]
    B = np.stack([gen(rng, (N, K)) for _ in range(Bt)])
    C0 = (gen(rng, (Bt, M, N)) if gen is _ints else rng.standard_normal((Bt, M, N))).astype(np.float32)
    return _Batch(cuda, dev, A, B, C0)


# ------------------------------------------------------------------ GPU: bit-identity
@pytest.mark.gpu
@pytest.mark.parametrize("splitk", [0, 2])
def test_batched_bit_identical_to_run_bias(cuda, ft, dev, splitk):
    """Every named variant, plain and fault-tolerant, cut tiles off and forced, all four layout pairs with padded lds and
    entry gaps, ragged M, N and K: entry i equals run_bias on entry i alone, bit for bit."""
    case = _case(cuda, dev, 31)
    M, N = case.M, case.N
    try:
        ft.debug_set("splitk", splitk)
        for name in NAMES:
            for kid in (ft.SGEMM_IDS[name], ft.ABFT_IDS[name]):
                dev.stats()
                for la in (MN, KM):
                    for lb in (MN, KM):
                        lda, ldb = _ld(la, M, case.K), _ld(lb, case.N, case.K)
                        got = case.batched(kid, la, lda, lb, ldb, M + 8, 0.75, -1.5)
                        for i in range(case.Bt):
                            assert np.array_equal(got[i], case.one(i, kid, la, lda, lb, ldb, M + 8, 0.75, -1.5)), (kid, la, lb, i)
                if kid >= 10:
                    assert dev.stats()["detected"] == 0, kid
    finally:
        ft.debug_set("splitk", -1)


@pytest.mark.gpu
def test_batched_bias_beta_and_options(cuda, ft, dev):
    """beta 0 / -1.5 with and without a ROW / COL bias, 3xTF32 and check_segments = 4: entry by entry as run_bias."""
    case = _case(cuda, dev, 32, Bt=3, M=256, N=132, K=300)
    rng = np.random.default_rng(33)
    biases = {1: rng.standard_normal(case.M).astype(np.float32), 2: rng.standard_normal(case.N).astype(np.float32)}
    for kid in (ft.ABFT_IDS["giant"], ft.ABFT_IDS["small"], ft.SGEMM_IDS["large"]):
        for beta in (0.0, -1.5):
            for mode in (0, 1, 2):
                b = biases.get(mode)
                got = case.batched(kid, KM, case.K + 4, MN, case.N, case.M, 1.25, beta, b, mode)
                for i in range(case.Bt):
                    assert np.array_equal(got[i], case.one(i, kid, KM, case.K + 4, MN, case.N, case.M, 1.25, beta, b, mode)), (kid, beta, mode)
    for opts in (dict(precision=1), dict(check_segments=4)):
        o = ft.make_opts(**opts)
        got = case.batched(31, MN, case.M, KM, case.K + 4, case.M, 1.0, -1.5, biases[2], 2, o)
        for i in range(case.Bt):
            assert np.array_equal(got[i], case.one(i, 31, MN, case.M, KM, case.K + 4, case.M, 1.0, -1.5, biases[2], 2, o)), opts
    assert dev.stats()["detected"] == 0


@pytest.mark.gpu
def test_cublas_batched_agrees(cuda, ft, dev):
    case = _case(cuda, dev, 34, Bt=4, M=256, N=384, K=300)
    ref = case.batched(31, MN, 256, KM, 304, 256, 0.75, -1.5)
    got = case.batched(7, MN, 256, KM, 304, 256, 0.75, -1.5)
    assert _rel(ref, got) < TOL_NORM  # (cuBLAS rounds its TF32 operands, the wgmma kernels truncate them)
    assert _rel(ref, case.batched(0, MN, 256, KM, 304, 256, 0.75, -1.5)) < TOL_NORM


# ------------------------------------------------------------------ GPU: ABFT in entries other than 0
@pytest.mark.gpu
def test_batched_abft_corrects_in_entry_two(cuda, ft, dev):
    """Bit flips in entry 2 are corrected and reported with stacked rows; two upsets in one row are recomputed from entry 2's
    own A and B; the other entries stay clean, also with entry magnitudes 2^10 apart."""
    case = _case(cuda, dev, 35, Bt=4, M=512, N=512, K=256, scales=[1.0, 1024.0, 1.0, 1.0 / 1024], gen=_ints)
    M = case.M
    clean = case.batched(31, KM, 256, KM, 256, M, 1.0, 0.0)
    st = dev.stats()
    assert st["detected"] == 0, st
    # (on nonzero elements: a flipped bit of 0 is a denormal, below any threshold)
    faults = [{"row": 2 * M + 10 + 40 * j, "col": next(c for c in range(3 + 70 * j, case.N) if clean[2, 10 + 40 * j, c] != 0),
               "xor": 1 << bit} for j, bit in enumerate((22, 25, 30, 31))]
    got = case.batched(31, KM, 256, KM, 256, M, 1.0, 0.0, opts=ft.make_opts(faults=faults))
    st = dev.stats()
    assert st["corrected"] == 4 and st["detected"] == 4, st
    assert sorted(e["row"] for e in st["events"]) == sorted(f["row"] for f in faults)
    assert np.array_equal(got, clean)
    two = [{"row": 2 * M + 77, "col": 5, "add": 50.0}, {"row": 2 * M + 77, "col": 100, "add": -30.0}]
    got = case.batched(31, KM, 256, KM, 256, M, 1.0, 0.0, opts=ft.make_opts(faults=two))
    st = dev.stats()
    assert st["recomputed"] == 1 and st["events"][0]["row"] == 2 * M + 77, st
    assert np.array_equal(got, clean)


@pytest.mark.gpu
def test_batched_protect_epilogue(cuda, ft, dev):
    case = _case(cuda, dev, 36, Bt=3, M=256, N=256, K=128, gen=_ints)
    M = case.M
    for beta in (0.0, -1.5):
        clean = case.batched(31, KM, 128, KM, 128, M, 1.0, beta, opts=ft.make_opts(protect_epilogue=True))
        assert dev.stats()["epilogue_faults"] == 0
        col = next(c for c in range(5, case.N) if clean[2, 9, c] != 0)  # (a flipped exponent bit of 0 is 2^-111)
        f = [{"row": 2 * M + 9, "col": col, "xor": 1 << 27, "where": "epilogue_value"}]
        got = case.batched(31, KM, 128, KM, 128, M, 1.0, beta, opts=ft.make_opts(faults=f, protect_epilogue=True))
        st = dev.stats()
        assert st["epilogue_faults"] == 1 and st["events"][0]["row"] == 2 * M + 9, st
        assert st["events"][0]["status"] == (6 if beta == 0.0 else 7)
        if beta == 0.0:
            assert np.array_equal(got, clean)
        for i in (0, 1):
            assert np.array_equal(got[i], clean[i])


@pytest.mark.gpu
def test_batched_faults_with_ragged_m(cuda, ft, dev):
    """M = 260: the last 256-row tile of entry i reaches past M into rows whose stacked index belongs to entry i+1.  A fault
    listed in entry 1 or 2 is injected there once -- not also into the previous entry's padding rows -- so every count and
    event is the fault's own: accumulator flips, and upsets after the check under protect_epilogue."""
    case = _case(cuda, dev, 41, Bt=3, M=260, N=256, K=128, gen=_ints)
    M = case.M
    clean = case.batched(31, KM, 128, KM, 128, M, 1.0, 0.0)
    assert dev.stats()["detected"] == 0
    rows = [(1, 5), (2, 3)]  # (entry, row): stacked rows 265 and 523 fall inside entries 0 / 1's last row tile
    cols = [next(c for c in range(7, case.N) if clean[e, r, c] != 0) for e, r in rows]
    faults = [{"row": e * M + r, "col": c, "xor": 1 << 27} for (e, r), c in zip(rows, cols)]
    got = case.batched(31, KM, 128, KM, 128, M, 1.0, 0.0, opts=ft.make_opts(faults=faults))
    st = dev.stats()
    assert st["detected"] == st["corrected"] == len(faults) and len(st["events"]) == len(faults), st
    assert sorted((e["row"], e["col"]) for e in st["events"]) == sorted((f["row"], f["col"]) for f in faults)
    assert np.array_equal(got, clean)
    for where in ("epilogue_value", "epilogue_tmem"):
        f = [{"row": M + 5, "col": cols[0], "xor": 1 << 27, "where": where}]
        got = case.batched(31, KM, 128, KM, 128, M, 1.0, 0.0, opts=ft.make_opts(faults=f, protect_epilogue=True))
        st = dev.stats()
        assert st["epilogue_faults"] == 1 and st["recomputed"] == 1 and len(st["events"]) == 1, (where, st)
        assert st["events"][0]["row"] == M + 5
        assert np.array_equal(got, clean), where


@pytest.mark.gpu
def test_bmm_empty_batch(cuda, ft, dev):
    t = cuda
    a, b = t.zeros(0, 64, 32, device="cuda"), t.zeros(0, 32, 16, device="cuda")
    out = dev.bmm(a, b)
    assert out.shape == (0, 64, 16)


@pytest.mark.gpu
def test_batched_selftest_hits_every_entry(cuda, ft, dev):
    case = _case(cuda, dev, 37, Bt=3, M=256, N=256, K=128, gen=_ints)
    clean = case.batched(16, KM, 128, KM, 128, 256, 1.0, 0.0)
    dev.stats()
    got = case.batched(16, KM, 128, KM, 128, 256, 1.0, 0.0, opts=ft.make_opts(selftest=(10000.0, 17, 5)))
    st = dev.stats()
    tiles = 3 * 2 * 2  # entries x 128-row tiles x 128-column tiles
    assert st["corrected"] == tiles and st["tiles"] >= tiles, st
    assert np.array_equal(got, clean)


@pytest.mark.gpu
def test_batched_encode_paths_and_launch_count(cuda, ft, dev):
    """A small B uses the pre-pass (2 launches for the whole batch), a batch whose B exceeds 8 MB the front phase (1)."""
    t = cuda
    # a row-major out runs swapped: the kernel's B is a -- 1 MB / 16 MB of it over the batch
    for Bt, M, K, launches in ((4, 256, 256, 2), (8, 1024, 512, 1)):
        rng = np.random.default_rng(38)
        a = t.from_numpy(_rand(rng, (Bt, M, K))).cuda()
        b = t.from_numpy(_rand(rng, (Bt, K, 256))).cuda()
        ref = t.bmm(a.double(), b.double()).float()
        n0 = dev.launch_count()
        out = dev.bmm(a, b, kernel_id=31)
        t.cuda.synchronize()
        assert dev.launch_count() - n0 == launches, (Bt, M, K)
        assert _rel(ref.cpu().numpy(), out.cpu().numpy()) < TOL_NORM
        st = dev.stats()
        assert st["detected"] == 0 and st["tiles"] > 0


@pytest.mark.gpu
def test_batched_reuse_b_checksums_keys(cuda, ft, dev):
    """reuse_b_checksums is not fooled by the same B pointer with another stride_b or batch."""
    t = cuda
    rng = np.random.default_rng(39)
    M = N = K = 256
    A = t.from_numpy(_rand(rng, (4 * M * K,))).cuda()
    B = t.from_numpy(_rand(rng, (8 * N * K,))).cuda()
    C = t.zeros(4 * M * N, device="cuda")
    reuse = ft.make_opts(reuse_b_checksums=True)
    dev.run_batched(31, M, N, K, A, KM, K, M * K, B, KM, K, N * K, C, M, M * N, 4, 1.0, 0.0)
    for sb, bt in ((2 * N * K, 4), (N * K, 2)):
        dev.run_batched(31, M, N, K, A, KM, K, M * K, B, KM, K, sb, C, M, M * N, bt, 1.0, 0.0, opts=reuse)
        st = dev.stats()
        assert st["detected"] == 0, (sb, bt, st)


@pytest.mark.gpu
def test_run_batched_argument_checks(cuda, ft, dev):
    t = cuda
    M = N = K = 128
    A = t.zeros(2 * M * K, device="cuda")
    B = t.zeros(2 * N * K, device="cuda")
    C = t.zeros(2 * M * N, device="cuda")
    L = ft.lib()

    def run(kid=31, sa=M * K, sb=N * K, sc=M * N, batch=2, bias=None, mode=0):
        return L.ftsgemm_run_batched(dev._h, kid, M, N, K, A.data_ptr(), KM, K, sa, B.data_ptr(), KM, K, sb, C.data_ptr(), M, sc,
                                     batch, 1.0, 0.0, bias, mode, None)
    assert run() == 0
    assert run(batch=0) == -1
    for kw in (dict(sa=0), dict(sb=-4), dict(sc=M * N + 2), dict(sa=6)):
        assert run(**kw) == -1, kw
    assert run(sc=M * N - 4) == -1  # overlapping C entries
    assert run(kid=10) == -2 and run(kid=30) == -2
    assert run(kid=7, bias=C.data_ptr(), mode=2) == -2
    assert run(kid=7) == 0
    assert run(sa=0, batch=1) == 0  # one entry: strides ignored
    t.cuda.synchronize()


@pytest.mark.gpu
def test_bmm_matches_torch_and_copies_nothing(cuda, ft, dev):
    t = cuda
    g = t.Generator(device="cuda").manual_seed(40)
    q = t.randn(8, 256, 64, device="cuda", generator=g)
    k = t.randn(8, 256, 64, device="cuda", generator=g)
    v = t.randn(8, 256, 64, device="cuda", generator=g)
    bias = t.randn(64, device="cuda", generator=g)
    t.backends.cuda.matmul.allow_tf32 = False
    try:
        for a, b, bi in ((q, k.transpose(-1, -2), None), (q @ k.transpose(-1, -2), v, bias)):
            ref = t.bmm(a.double(), b.double()) + (bi.double() if bi is not None else 0)
            plan = ft.bmm_plan(tuple(a.shape), a.stride(), tuple(b.shape), b.stride(), (a.shape[1] * b.shape[2], b.shape[2], 1),
                               a.data_ptr(), b.data_ptr(), 0)
            assert not (plan["copy_a"] or plan["copy_b"] or plan["copy_out"])
            n0 = dev.launch_count()
            out = dev.bmm(a, b, bias=bi)
            t.cuda.synchronize()
            assert dev.launch_count() - n0 <= 2
            assert _rel(ref.cpu().numpy(), out.cpu().numpy()) < TOL_NORM
        # baddbmm semantics, with an expanded (shared) operand that bmm copies once
        c0 = t.randn(8, 256, 64, device="cuda", generator=g)
        w = t.randn(1, 64, 64, device="cuda", generator=g).expand(8, 64, 64)
        ref = t.baddbmm(c0.double(), q.double(), w.double(), beta=-1.5, alpha=0.5)
        out = dev.bmm(q, w, c0.clone(), alpha=0.5, beta=-1.5)
        assert _rel(ref.cpu().numpy(), out.cpu().numpy()) < TOL_NORM
    finally:
        t.backends.cuda.matmul.allow_tf32 = True
    assert dev.stats()["detected"] == 0
