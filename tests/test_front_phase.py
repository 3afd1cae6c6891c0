"""The kernel's front phase: the transposer of MN-major operands (64-row x 32-k items, 16-byte copies in and out) and the
in-kernel encode of B beside it.

A transpose only moves values, so every product whose operands the front phase transposes must give C bit for bit as the
same product with K-major operands, which the main loop reads in place.  The shapes put the item edges everywhere: M and N
at +-4 around multiples of 32, 64, 128 and 256 (M % 4 == 0 is required), K at +-1 around multiples of 32, padded leading
dimensions, one operand of each layout, strided batches with padded entry strides, beta = 0 and beta != 0.  With the encode
forced into the front phase, injected single-bit flips are still located and corrected.
"""
import numpy as np
import pytest

MN, KM = 0, 1
SHAPES = [(252, 260, 255), (124, 388, 257), (516, 132, 129), (260, 508, 33), (68, 60, 31), (132, 252, 96)]


def _rand(rng, shape):
    return (rng.integers(0, 10, shape) * 0.1 * rng.choice([-1.0, 1.0], shape)).astype(np.float32)


def _pack(X, layout, ld, entry=None):
    """rows x K matrix X -> flat buffer in the layout (MN: X[r, k] at r + k*ld; KM: at k + r*ld), padding = NaN; with
    `entry` the buffer is that many floats long (a strided-batch entry)"""
    rows, K = X.shape
    if layout == MN:
        buf = np.full((K, ld), np.nan, np.float32)
        buf[:, :rows] = X.T
    else:
        buf = np.full((rows, ld), np.nan, np.float32)
        buf[:, :K] = X
    flat = buf.reshape(-1)
    if entry is not None:
        flat = np.concatenate([flat, np.full(entry - flat.size, np.nan, np.float32)])
    return flat


@pytest.fixture(scope="module")
def dev(cuda, ft):
    cuda.cuda.set_device(0)
    h = ft.FtSgemm()
    yield h
    h.close()


def _run_ex(t, dev, kid, A, B, C0, la, lda, lb, ldb, alpha, beta, opts=None):
    M, K = A.shape
    N = B.shape[0]
    dA = t.from_numpy(_pack(A, la, lda)).cuda()
    dB = t.from_numpy(_pack(B, lb, ldb)).cuda()
    dC = t.from_numpy(np.ascontiguousarray(C0.T).reshape(-1)).cuda()
    dev.run_ex(kid, M, N, K, dA, la, lda, dB, lb, ldb, dC, M, alpha, beta, opts)
    t.cuda.synchronize()
    return dC.cpu().numpy().reshape(N, M).T


@pytest.mark.gpu
@pytest.mark.parametrize("shape", SHAPES)
def test_transposed_operands_bit_identical_to_k_major(cuda, ft, dev, shape):
    M, N, K = shape
    rng = np.random.default_rng(M * 7 + N * 3 + K)
    A, B = _rand(rng, (M, K)), _rand(rng, (N, K))
    C0 = rng.standard_normal((M, N)).astype(np.float32)
    kk = (K + 3) // 4 * 4
    for kid in (31, 16, 21):
        for alpha, beta in ((1.0, 0.0), (0.75, -1.5)):
            dev.stats()
            ref = _run_ex(cuda, dev, kid, A, B, C0, KM, kk, KM, kk, alpha, beta)
            for la, lda, lb, ldb in ((MN, M, MN, N), (MN, M + 4, MN, N + 12), (MN, M + 8, KM, kk + 4), (KM, kk, MN, N + 4)):
                got = _run_ex(cuda, dev, kid, A, B, C0, la, lda, lb, ldb, alpha, beta)
                assert np.array_equal(ref, got), (kid, shape, la, lda, lb, ldb, beta)
            if kid != 21:
                assert dev.stats()["detected"] == 0, (kid, shape)


@pytest.mark.gpu
@pytest.mark.parametrize("beta", [0.0, -1.5])
def test_batched_padded_entries_bit_identical_to_k_major(cuda, ft, dev, beta):
    t = cuda
    rng = np.random.default_rng(31)
    batch, M, N, K = 3, 196, 132, 161
    As = [_rand(rng, (M, K)) for _ in range(batch)]
    Bs = [_rand(rng, (N, K)) for _ in range(batch)]
    C0 = [rng.standard_normal((M, N)).astype(np.float32) for _ in range(batch)]
    kk = (K + 3) // 4 * 4

    def run(kid, la, lda, lb, ldb):
        sa = (lda * (K if la == MN else M)) + 24  # padded entry strides (multiples of 4 floats)
        sb = (ldb * (K if lb == MN else N)) + 40
        sc = M * N + 8
        dA = t.from_numpy(np.concatenate([_pack(a, la, lda, sa) for a in As])).cuda()
        dB = t.from_numpy(np.concatenate([_pack(b, lb, ldb, sb) for b in Bs])).cuda()
        cbuf = np.zeros((batch, sc), np.float32)
        for i in range(batch):
            cbuf[i, :M * N] = np.ascontiguousarray(C0[i].T).reshape(-1)
        dC = t.from_numpy(cbuf.reshape(-1)).cuda()
        dev.run_batched(kid, M, N, K, dA, la, lda, sa, dB, lb, ldb, sb, dC, M, sc, batch, 0.75, beta)
        t.cuda.synchronize()
        return dC.cpu().numpy().reshape(batch, sc)
    for kid in (31, 21):
        dev.stats()
        ref = run(kid, KM, kk, KM, kk)
        for la, lda, lb, ldb in ((MN, M + 4, MN, N + 4), (MN, M, KM, kk + 4), (KM, kk + 8, MN, N)):
            assert np.array_equal(ref, run(kid, la, lda, lb, ldb)), (kid, la, lb, beta)
        if kid == 31:
            assert dev.stats()["detected"] == 0


@pytest.mark.gpu
@pytest.mark.parametrize("kid", [31, 16])
@pytest.mark.parametrize("shape", [(260, 512, 255), (132, 768, 96), (260, 516, 257)])
def test_front_phase_encode_matches_prepass(cuda, ft, dev, kid, shape):
    """The checksum operand the front phase encodes (fused with the transpose of B where the N-tiles are whole, after it
    otherwise) gives the same fault-free residuals, bit for bit, as the stand-alone encode pre-pass: the checksum product
    and hence the residuals depend on nothing else.  Dense and padded ldb (the pre-pass groups a K tail differently
    there), C unchanged."""
    M, N, K = shape
    rng = np.random.default_rng(M + N + K)
    A, B = _rand(rng, (M, K)), _rand(rng, (N, K))
    C0 = rng.standard_normal((M, N)).astype(np.float32)
    for ldb in (N, N + 4):
        res = {}
        try:
            for ef in (0, 1):
                ft.debug_set("enc_front", ef)
                dev.stats()
                c = _run_ex(cuda, dev, kid, A, B, C0, MN, M, MN, ldb, 0.75, -1.5)
                st = dev.stats()
                assert st["detected"] == 0, (ef, st)
                res[ef] = (c, st["max_abs_residual"], st["max_rel_residual"])
        finally:
            ft.debug_set("enc_front", -1)
        assert np.array_equal(res[0][0], res[1][0])
        assert res[0][1:] == res[1][1:], (kid, shape, ldb, res[0][1:], res[1][1:])


@pytest.mark.gpu
def test_front_phase_encode_corrects_flips(cuda, ft, dev):
    """enc_front forced on for a small B: the checksum operand comes from the front phase, next to the transposes of both
    operands.  No false alarms, C as with K-major operands, and single-bit flips in the exponent, sign and top mantissa bit
    of four elements (one per row and N-tile) are located and corrected."""
    rng = np.random.default_rng(32)
    M, N, K = 516, 772, 383
    A, B = _rand(rng, (M, K)), _rand(rng, (N, K))
    C0 = rng.standard_normal((M, N)).astype(np.float32)
    kk = (K + 3) // 4 * 4
    kid = 31
    try:
        ft.debug_set("enc_front", 1)
        dev.stats()
        clean = _run_ex(cuda, dev, kid, A, B, C0, MN, M + 4, MN, N + 4, 1.0, 0.0)
        assert dev.stats()["detected"] == 0
        assert np.array_equal(clean, _run_ex(cuda, dev, kid, A, B, C0, KM, kk, KM, kk, 1.0, 0.0))
        assert dev.stats()["detected"] == 0
        cand = np.argwhere(np.abs(clean) >= 2.0)
        faults, seen = [], set()
        for r, c in rng.permutation(cand):
            if r in {f["row"] for f in faults} or (c // 256) in seen:
                continue
            seen.add(c // 256)
            faults.append({"row": int(r), "col": int(c), "xor": 1 << [22, 25, 30, 31][len(faults)]})
            if len(faults) == 4:
                break
        assert len(faults) == 4
        got = _run_ex(cuda, dev, kid, A, B, C0, MN, M + 4, MN, N + 4, 1.0, 0.0, ft.make_opts(faults=faults))
        st = dev.stats()
        assert st["detected"] == 4 == st["corrected"], st
        assert {(e["row"], e["col"]) for e in st["events"]} == {(f["row"], f["col"]) for f in faults}
        assert np.abs(got - clean).max() < 2e-2
    finally:
        ft.debug_set("enc_front", -1)
