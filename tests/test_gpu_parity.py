"""GPU parity tests proper (run on an H100 with -m gpu): the CUDA path, called through the C ABI, against the
CPU oracle on the same seeded inputs, against the committed golden fixtures, and -- at BASELINE.json's full sizes --
through size-independent properties.

Tolerances (stated once, used everywhere):
  * TOL_NORM = 1e-3: Frobenius-norm relative error against the FP32 sequential-k oracle -- the north_star's
    "within 1e-3 rel of the reference's CPU SGEMM".  The main contraction is single-pass TF32 (operands truncated to
    10 mantissa bits by the tensor core, FP32 accumulate).
  * TOL_MODEL = 5e-5: norm-wise against a float64 product of TF32-TRUNCATED operands (what the tensor core computes up
    to FP32 accumulation order); measured 1.5e-7 (K=64) .. 2e-5 (K=8192).
  * the reference comparator verify_matrix (utils/utils.cu:61-77; fail iff rel>1e-2 AND abs>1e-2) is applied too; with
    single-pass TF32 a ~1e-5 fraction of near-zero elements of a K>=1024 product can exceed it (SURVEY.md section 7,
    hard part 1), so the assertion is on the failing FRACTION (< 1e-4), and exactly zero against the TF32 model.
"""
import json
from pathlib import Path

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

TOL_NORM = 1e-3
TOL_MODEL = 5e-5
GOLD = json.loads((Path(__file__).parent / "golden" / "ref_cpu_gemm.json").read_text())


def _fail_fraction(ref, x):
    d = np.abs(ref.astype(np.float64) - x.astype(np.float64))
    with np.errstate(divide="ignore", invalid="ignore"):
        bad = ((d / np.abs(ref.astype(np.float64))) > 0.01) & (d > 0.01)
    return float(bad.mean())


@pytest.fixture(scope="module")
def dev(cuda, ft):
    cuda.cuda.set_device(0)
    h = ft.FtSgemm()
    yield h
    h.close()


def _run(cuda, dev, kid, M, N, K, A, B, C0, alpha=1.0, beta=0.0, opts=None):
    dA, dB = cuda.from_numpy(A).cuda(), cuda.from_numpy(B).cuda()
    dC = cuda.from_numpy(C0.copy()).cuda()
    dev.run(kid, M, N, K, dA, dB, dC, alpha, beta, opts)
    cuda.cuda.synchronize()
    return dC.cpu().numpy()


def _rand(rng, count):
    return (rng.integers(0, 10, count) * 0.1 * rng.choice([-1.0, 1.0], count)).astype(np.float32)


# ------------------------------------------------------------------ golden fixtures (reference inputs, END = n)
@pytest.mark.parametrize("n", [256, 512, 1024])
@pytest.mark.parametrize("name", ["small", "medium", "large", "tall", "wide", "huge", "giant", "pair128"])
def test_reference_inputs_vs_golden_and_oracle(cuda, ft, dev, oracle, n, name):
    import hashlib
    A, B, C0 = oracle.make_inputs(n)
    want = oracle.sgemm_nt(n, n, n, 1.0, A, B, 0.0, C0.copy())
    assert hashlib.sha256(want.tobytes()).hexdigest() == GOLD[str(n)]["sha256"]["C"]  # oracle == reference cpu_gemm
    model = oracle.sgemm_nt_tf32_model(n, n, n, 1.0, A, B, 0.0, C0, "trunc")
    for kid in (ft.SGEMM_IDS[name], ft.ABFT_IDS[name]):
        got = _run(cuda, dev, kid, n, n, n, A, B, C0)
        em = oracle.error_metrics(want, got)
        assert em["rel_fro"] < TOL_NORM, (kid, em)
        assert oracle.error_metrics(model, got)["rel_fro"] < TOL_MODEL
        assert _fail_fraction(want, got) < 1e-4
        assert oracle.verify_matrix(model, got, n, n) == -1
        # golden scalars: C[0], C[1], C[n], C[n*n-1] and the sum, to the TF32 norm-wise tolerance
        scale = float(np.sqrt(np.mean(want.astype(np.float64) ** 2)))
        for idx, v in GOLD[str(n)]["C_sel"].items():
            assert abs(float(got[int(idx)]) - v) < 5e-3 * scale
    if name in ("huge", "giant"):  # fault-free FT run must not flag anything
        st = dev.stats()
        assert st["detected"] == 0 and st["rows_checked"] > 0


def test_ft_equals_plain_bitwise_when_fault_free(cuda, ft, dev):
    """The ABFT kernel must not perturb a single bit of a fault-free product -- whatever the planner cuts: a cut tile is
    a seeded chain that accumulates in exactly the k order of an uncut tile."""
    rng = np.random.default_rng(3)
    M, N, K = 512, 768, 640
    A, B = _rand(rng, M * K), _rand(rng, N * K)
    C0 = np.zeros(M * N, np.float32)
    ref = {}
    for splitk in (0, -1, 2, 3):
        try:
            ft.debug_set("splitk", splitk)
            for name in ("medium", "huge", "wide", "giant"):
                a = _run(cuda, dev, ft.SGEMM_IDS[name], M, N, K, A, B, C0)
                b = _run(cuda, dev, ft.ABFT_IDS[name], M, N, K, A, B, C0)
                assert np.array_equal(a, b), (name, splitk)
                assert np.array_equal(ref.setdefault(name, a), a), (name, splitk)
        finally:
            ft.debug_set("splitk", -1)


def test_prepass_encode_and_cached_checksums_agree(cuda, ft, dev, oracle):
    """The checksum vectors of B come from the encode pre-pass in front of the GEMM kernel; back-to-back launches reuse the
    flags / epochs, and the cached-checksum path (reuse_b_checksums) must give the same results and verdicts.  Also the
    ragged N / K tail and the narrow-tile (scalar) encode path, all FT tile widths, and a long odd K (129 k-blocks)."""
    rng = np.random.default_rng(5)
    M, N, K = 1024, 1280, 768
    A, B = _rand(rng, M * K), _rand(rng, N * K)
    C0 = rng.standard_normal(M * N).astype(np.float32)
    faults = [{"row": 77, "col": 300, "xor": 1 << 29}, {"row": 900, "col": 1279, "add": -55.0}]
    dev.stats()
    for rep in range(3):
        got = _run(cuda, dev, 31, M, N, K, A, B, C0, 1.0, -1.5, opts=ft.make_opts(faults=faults))
    st = dev.stats()
    assert st["detected"] == 6 and st["corrected"] == 6 and st["uncorrectable"] == 0
    dA, dB = cuda.from_numpy(A).cuda(), cuda.from_numpy(B).cuda()
    dC = cuda.from_numpy(C0.copy()).cuda()
    dev.run(31, M, N, K, dA, dB, dC, 1.0, -1.5, ft.make_opts(faults=faults))
    dC2 = cuda.from_numpy(C0.copy()).cuda()
    dev.run(31, M, N, K, dA, dB, dC2, 1.0, -1.5, ft.make_opts(faults=faults, reuse_b_checksums=True))
    cuda.cuda.synchronize()
    assert cuda.equal(dC, dC2) and np.array_equal(dC.cpu().numpy(), got)
    for (M2, N2, K2) in ((260, 388, 72), (260, 416, 200)):  # N % 32 != 0; ragged last tile, K tail
        A2, B2 = _rand(rng, M2 * K2), _rand(rng, N2 * K2)
        C2 = np.zeros(M2 * N2, np.float32)
        model = oracle.sgemm_nt_tf32_model(M2, N2, K2, 1.0, A2, B2, 0.0, C2, "trunc")
        for kid in (11, 12, 16, 15, 31, 32):
            dev.stats()
            res = _run(cuda, dev, kid, M2, N2, K2, A2, B2, C2, 1.0, 0.0, opts=ft.make_opts(selftest=(10000.0, 17, 5)))
            st = dev.stats()
            assert st["detected"] == st["corrected"] > 0 and st["uncorrectable"] == 0, (kid, st)
            assert oracle.error_metrics(model, res)["rel_fro"] < TOL_MODEL, kid
    M, N, K = 512, 768, 4128
    A, B = _rand(rng, M * K), _rand(rng, N * K)
    C0 = rng.standard_normal(M * N).astype(np.float32)
    model = oracle.sgemm_nt_tf32_model(M, N, K, 1.0, A, B, 0.5, C0, "trunc")
    faults = [{"row": 300, "col": 5, "xor": 1 << 30}, {"row": 511, "col": 767, "add": 123.0}]
    for kid in (31, 16):
        dev.stats()
        got = _run(cuda, dev, kid, M, N, K, A, B, C0, 1.0, 0.5, opts=ft.make_opts(faults=faults))
        st = dev.stats()
        assert st["detected"] == 2 and st["corrected"] == 2 and st["uncorrectable"] == 0, (kid, st)
        assert oracle.error_metrics(model, got)["rel_fro"] < TOL_MODEL, kid


@pytest.mark.parametrize("seed", range(10))
def test_random_shapes_and_knobs(cuda, ft, dev, oracle, seed):
    """Seeded fuzz over ragged shapes, kernel variants, alpha/beta and every decomposition knob (cut pieces, encode
    variants, wave re-synchronisation): results against the TF32 model, the ABFT variant bit-equal to its plain twin when
    fault-free, an injected fault corrected."""
    rng = np.random.default_rng(1000 + seed)
    M = int(rng.integers(1, 380)) * 4
    N = int(rng.integers(1, 380)) * 4
    K = int(rng.integers(1, 1100))
    name = ["small", "medium", "huge", "wide", "giant", "pair128"][seed % 6]
    alpha = float(rng.choice([1.0, 0.75, -2.0]))
    beta = float(rng.choice([0.0, -1.5, 1.0]))
    knobs = {"splitk": int(rng.choice([-1, 0, 2, 3])), 
             "wave_sync": int(rng.choice([0, 1])), "pdl": int(rng.choice([0, 1])), "epi_assist": int(rng.choice([0, 1])),
             "chk_slices": int(rng.choice([1, 2, 3])), "enc_front": int(rng.choice([0, 1]))}
    A, B = rng.standard_normal(M * K).astype(np.float32), rng.standard_normal(N * K).astype(np.float32)
    C0 = rng.standard_normal(M * N).astype(np.float32)
    model = oracle.sgemm_nt_tf32_model(M, N, K, alpha, A, B, beta, C0, "trunc")
    fr, fc = int(rng.integers(0, M)), int(rng.integers(0, N))
    try:
        for k, v in knobs.items():
            ft.debug_set(k, v)
        plain = _run(cuda, dev, ft.SGEMM_IDS[name], M, N, K, A, B, C0, alpha, beta)
        dev.stats()
        abft = _run(cuda, dev, ft.ABFT_IDS[name], M, N, K, A, B, C0, alpha, beta)
        st = dev.stats()
        assert st["detected"] == 0 and st["rows_checked"] > 0, (knobs, st)
        assert np.array_equal(plain, abft), (name, M, N, K, knobs)
        assert oracle.error_metrics(model, abft)["rel_fro"] < TOL_MODEL, (name, M, N, K, knobs)
        fixed = _run(cuda, dev, ft.ABFT_IDS[name], M, N, K, A, B, C0, alpha, beta,
                     opts=ft.make_opts(faults=[{"row": fr, "col": fc, "xor": 1 << 30}]))
        st = dev.stats()
        assert st["detected"] == 1 and st["corrected"] == 1, (name, M, N, K, knobs, st)
        diff = np.flatnonzero(fixed != abft)
        assert set(diff) <= {fr + fc * M}
        assert oracle.error_metrics(model, fixed)["rel_fro"] < TOL_MODEL
    finally:
        for k in knobs:
            ft.debug_set(k, -1)


def test_epilogue_assist_is_neutral(cuda, ft, dev):
    """The helper-assisted epilogue splits the columns of a final data-tile epilogue between the epilogue warp and the helper
    warp of the same 32-row quadrant (row sums exchanged through shared memory): results bit-identical with it on and
    off, injected faults in both column halves and on the split corrected."""
    rng = np.random.default_rng(13)
    M, N, K = 640, 1024, 352
    A, B = _rand(rng, M * K), _rand(rng, N * K)
    C0 = rng.standard_normal(M * N).astype(np.float32)
    faults = [{"row": 5, "col": 3, "xor": 1 << 29}, {"row": 300, "col": 127, "add": 77.0}, {"row": 301, "col": 128, "add": -9.0},
              {"row": 639, "col": 1023, "xor": 1 << 31}, {"row": 129, "col": 700, "add": 1e30}]
    for kid, plain in ((31, 21), (16, 6), (15, 5), (12, 2), (32, 22)):
        outs = []
        for on in (1, 0):
            try:
                ft.debug_set("epi_assist", on)
                a = _run(cuda, dev, plain, M, N, K, A, B, C0, 1.0, -1.5)
                dev.stats()
                b = _run(cuda, dev, kid, M, N, K, A, B, C0, 1.0, -1.5)
                assert np.array_equal(a, b) and dev.stats()["detected"] == 0, (kid, on)
                c = _run(cuda, dev, kid, M, N, K, A, B, C0, 1.0, -1.5, opts=ft.make_opts(faults=faults))
                st = dev.stats()
                assert st["detected"] == 5 and st["corrected"] == 5 and st["uncorrectable"] == 0, (kid, on, st)
                assert np.count_nonzero(c != b) <= 5 and np.allclose(c, b, rtol=1e-4, atol=1e-3)
                outs.append((a, c))
            finally:
                ft.debug_set("epi_assist", -1)
        assert np.array_equal(outs[0][0], outs[1][0]), kid
        assert np.allclose(outs[0][1], outs[1][1], rtol=1e-5, atol=1e-4), kid


def test_wave_sync_is_bitwise_neutral(cuda, ft, dev):
    """The wave re-synchronisation of large problems (a barrier among the leader producers at whole-tile boundaries) only
    delays loads: forced on a multi-wave shape, with and without cut tiles / ABFT, the results must not change a bit."""
    rng = np.random.default_rng(11)
    M, N, K = 2048, 2304, 288   # 72 tiles of 256x256 on 66 two-CTA units is just over one wave: use the 128-wide two-CTA tile as well
    A, B = _rand(rng, M * K), _rand(rng, N * K)
    C0 = rng.standard_normal(M * N).astype(np.float32)
    for kid in (6, 16, 22, 32, 21, 31):
        outs = []
        for sync in (0, 1):
            try:
                ft.debug_set("wave_sync", sync)
                dev.stats()
                outs.append(_run(cuda, dev, kid, M, N, K, A, B, C0, 0.5, 2.0, opts=ft.make_opts(selftest=(10000.0, 33, 7)) if kid in (16, 31, 32) else None))
                if kid in (16, 31, 32):
                    st = dev.stats()
                    assert st["detected"] == st["corrected"] > 0 and st["uncorrectable"] == 0, (kid, sync, st)
            finally:
                ft.debug_set("wave_sync", -1)
        assert np.array_equal(outs[0], outs[1]), kid


@pytest.mark.parametrize("slices", [2, 3, 5])
def test_split_k_head_forced(cuda, ft, dev, oracle, slices):
    """Force cut tiles (pieces park their accumulator, the next piece seeds its accumulator with it) on shapes where the
    planner would not cut, with and without ABFT + injected faults."""
    rng = np.random.default_rng(slices)
    M, N, K = 768, 1024, 1600
    A, B = _rand(rng, M * K), _rand(rng, N * K)
    C0 = rng.standard_normal(M * N).astype(np.float32)
    model = oracle.sgemm_nt_tf32_model(M, N, K, 1.0, A, B, -1.5, C0, "trunc")
    try:
        ft.debug_set("splitk", slices)
        for kid in (6, 21, 16, 31):
            got = _run(cuda, dev, kid, M, N, K, A, B, C0, 1.0, -1.5)
            assert oracle.error_metrics(model, got)["rel_fro"] < TOL_MODEL, kid
        dev.stats()
        got = _run(cuda, dev, 31, M, N, K, A, B, C0, 1.0, -1.5, opts=ft.make_opts(selftest=(10000.0, 17, 5)))
        st = dev.stats()
        assert st["detected"] == st["corrected"] == st["tiles"] == 6 * 4  # one upset per 128-row CTA tile
        assert oracle.error_metrics(model, got)["rel_fro"] < TOL_MODEL
    finally:
        ft.debug_set("splitk", -1)


@pytest.mark.parametrize("shape", [(128, 128, 8), (128, 32, 40), (200, 136, 100), (260, 388, 72), (1024, 256, 2048),
                                   (4, 4, 1), (132, 36, 33)])
def test_ragged_shapes_alpha_beta(cuda, ft, dev, oracle, shape):
    M, N, K = shape
    rng = np.random.default_rng(M * 7 + N)
    A, B = rng.standard_normal(M * K).astype(np.float32), rng.standard_normal(N * K).astype(np.float32)
    C0 = rng.standard_normal(M * N).astype(np.float32)
    want = oracle.sgemm_nt(M, N, K, 0.75, A, B, -1.5, C0.copy())
    model = oracle.sgemm_nt_tf32_model(M, N, K, 0.75, A, B, -1.5, C0, "trunc")
    for kid in (1, 2, 6, 5, 11, 12, 16, 15):
        got = _run(cuda, dev, kid, M, N, K, A, B, C0, 0.75, -1.5)
        assert oracle.error_metrics(model, got)["rel_fro"] < TOL_MODEL, kid
        assert oracle.error_metrics(want, got)["rel_fro"] < 2 * TOL_NORM, kid  # beta*C term dilutes; K tiny
    assert dev.stats()["detected"] == 0


def test_unsupported_and_invalid_args(cuda, ft, dev):
    t = cuda.zeros(64 * 64, device="cuda")
    with pytest.raises(ft.FtsgemmError) as e:
        dev.run(16, 62, 64, 64, t, t, t)  # M % 4 != 0 -> TMA stride not 16B
    assert e.value.code == -2
    with pytest.raises(ft.FtsgemmError) as e:
        dev.run(99, 64, 64, 64, t, t, t)
    assert e.value.code == -1
    with pytest.raises(ft.FtsgemmError) as e:
        dev.run(16, 64, 64, 0, t, t, t)
    assert e.value.code == -1
    # options: a zero-initialised struct (struct_size 0) is rejected, not read as "all defaults on the default stream";
    # negative self-test coordinates are rejected instead of indexing outside the tile's tensor-memory columns
    o = ft.Opts()
    with pytest.raises(ft.FtsgemmError) as e:
        dev.run(16, 64, 64, 64, t, t, t, 1.0, 0.0, o)
    assert e.value.code == -1
    for sel in ((10000.0, -1, 0), (10000.0, 0, -5)):
        with pytest.raises(ft.FtsgemmError) as e:
            dev.run(16, 64, 64, 64, t, t, t, 1.0, 0.0, ft.make_opts(selftest=sel))
        assert e.value.code == -1
    dev.run(16, 64, 64, 64, t, t, t, 1.0, 0.0, ft.make_opts(selftest=(10000.0, 17, 5)))  # (valid options still run)
    cuda.cuda.synchronize()
    dev.stats()


def test_handle_is_bound_to_its_device_and_scaled_inputs(cuda, ft, dev, oracle):
    """(1) A second handle (its own workspace, shared-memory attribute cached per handle) gives the same result.
    (2) Detection threshold and operand scale: thr = tau_abs + tau_rel * sum|acc| with tau_abs calibrated for operands of
    magnitude ~1 (include/ftsgemm.h); for operands scaled by s the caller scales tau_abs by s^2 -- with that, an upset of
    the same RELATIVE size is detected and repaired at 1e-3 and 1e3 times the reference magnitude."""
    rng = np.random.default_rng(77)
    M, N, K = 512, 512, 512
    A, B = _rand(rng, M * K), _rand(rng, N * K)
    C0 = np.zeros(M * N, np.float32)
    base = _run(cuda, dev, 31, M, N, K, A, B, C0)
    h2 = ft.FtSgemm()
    try:
        assert np.array_equal(_run(cuda, h2, 31, M, N, K, A, B, C0), base)
    finally:
        h2.close()
    for s in (1e-3, 1e3):
        As, Bs = (A * np.float32(s)).astype(np.float32), (B * np.float32(s)).astype(np.float32)
        clean = _run(cuda, dev, 31, M, N, K, As, Bs, C0, opts=ft.make_opts(tau_abs=1e-3 * s * s))
        dev.stats()
        fixed = _run(cuda, dev, 31, M, N, K, As, Bs, C0,
                     opts=ft.make_opts(tau_abs=1e-3 * s * s, faults=[{"row": 100, "col": 200, "add": 50.0 * s * s}]))
        st = dev.stats()
        assert st["detected"] == 1 and st["corrected"] == 1, (s, st)
        assert np.allclose(fixed, clean, rtol=0, atol=2e-3 * s * s)


# ------------------------------------------------------------------ cuBLAS rows and the non-fused baseline
def test_cublas_rows_and_baseline(cuda, ft, dev, oracle):
    n = 512
    A, B, C0 = oracle.make_inputs(n)
    want = oracle.sgemm_nt(n, n, n, 1.0, A, B, 0.0, C0.copy())
    got = _run(cuda, dev, ft.ID_CUBLAS, n, n, n, A, B, C0)
    assert oracle.error_metrics(want, got)["rel_fro"] < 1e-6 and oracle.verify_matrix(want, got, n, n) == -1
    got = _run(cuda, dev, ft.ID_CUBLAS_TF32, n, n, n, A, B, C0)
    assert oracle.error_metrics(want, got)["rel_fro"] < TOL_NORM
    for kid, tol in ((ft.ID_ABFT_BASELINE, 1e-6), (ft.ID_ABFT_BASELINE_TF32, TOL_NORM)):
        got = _run(cuda, dev, kid, n, n, n, A, B, C0)
        assert oracle.error_metrics(want, got)["rel_fro"] < tol
    # residual of the baseline's separate checksum pass (detection only, like the reference)
    dA, dB = cuda.from_numpy(A).cuda(), cuda.from_numpy(B).cuda()
    dC, res = cuda.zeros(n * n, device="cuda"), cuda.zeros(2, device="cuda")
    dev.baseline(n, n, n, dA, dB, dC, 1.0, 0.0, False, None, res)
    cuda.cuda.synchronize()
    assert float(res.abs().max()) < 0.5  # sum of 512 row/col residuals of an FP32 product


# ------------------------------------------------------------------ fault injection: detect + correct
def test_reference_selftest_every_tile_corrected(cuda, ft, dev, oracle):
    """The reference's always-on injector (+10000 into one accumulator of every CTA tile, ft_sgemm_huge.cuh:324-327):
    'FT kernel passes verify_matrix' <=> 'detect + correct worked'."""
    n = 1024
    A, B, C0 = oracle.make_inputs(n)
    want = oracle.sgemm_nt(n, n, n, 1.0, A, B, 0.0, C0.copy())
    for name in ("small", "medium", "tall", "huge", "wide"):
        clean = _run(cuda, dev, ft.ABFT_IDS[name], n, n, n, A, B, C0)
        dev.stats()
        got = _run(cuda, dev, ft.ABFT_IDS[name], n, n, n, A, B, C0, opts=ft.make_opts(selftest=(10000.0, 17, 5)))
        st = dev.stats()
        tiles = st["tiles"]
        assert tiles == (n // 128) * -(-n // [k for k in ft.kernel_table() if k["id"] == ft.ABFT_IDS[name]][0]["tile"][1])
        assert st["detected"] == tiles and st["corrected"] == tiles and st["uncorrectable"] == 0
        diff = np.flatnonzero(got != clean)
        assert len(diff) <= tiles  # only injected elements may differ (most are restored bit-exactly)
        assert np.abs(got - clean).max() < 5e-3  # corrected from the FP32 checksum: ~ulp(1e4)
        assert oracle.error_metrics(want, got)["rel_fro"] < TOL_NORM
        # without correction the same fault is fatal for the reference comparator
        bad = _run(cuda, dev, ft.ABFT_IDS[name], n, n, n, A, B, C0,
                   opts=ft.make_opts(selftest=(10000.0, 17, 5), detect_only=True))
        st = dev.stats()
        assert st["detected"] == tiles and st["corrected"] == 0
        assert oracle.verify_matrix(clean, bad, n, n) != -1


@pytest.mark.parametrize("bit", [31, 30, 27, 23, 22, 21, 20])
def test_single_bit_flips_detected_and_corrected(cuda, ft, dev, bit):
    """Config 4 of BASELINE.json in miniature: flip one bit of one FP32 accumulator.  Elements with
    |value| in [8, 64) are chosen so that every listed bit moves the value by >= 1 (bit 20 of an element in [8,16));
    the per-bit detection/correction RATES over random elements are measured by scripts/fault_campaign.py."""
    rng = np.random.default_rng(bit)
    M = N = 512
    K = 2048
    A, B = _rand(rng, M * K), _rand(rng, N * K)
    C0 = np.zeros(M * N, np.float32)
    clean = _run(cuda, dev, 16, M, N, K, A, B, C0)
    cand = np.flatnonzero((np.abs(clean) >= 8) & (np.abs(clean) < 64))
    faults, seen = [], set()
    for idx in rng.permutation(cand):
        r, c = int(idx % M), int(idx // M)
        if (r, c // 128) in seen:
            continue
        seen.add((r, c // 128))  # one fault per (row, tile)
        faults.append({"row": r, "col": c, "xor": 1 << bit})
        if len(faults) == 6:
            break
    dev.stats()
    got = _run(cuda, dev, 16, M, N, K, A, B, C0, opts=ft.make_opts(faults=faults))
    st = dev.stats()
    assert st["detected"] == len(faults) == st["corrected"], st
    located = {(e["row"], e["col"]) for e in st["events"]}
    assert located == {(f["row"], f["col"]) for f in faults}
    assert np.abs(got - clean).max() < 2e-2
    for f in faults:  # everything except the faulty elements is bit-identical to the fault-free run
        idx = f["row"] + f["col"] * M
        got[idx] = clean[idx]
    assert np.array_equal(got, clean)


def test_low_order_flip_below_threshold_is_harmless(cuda, ft, dev):
    rng = np.random.default_rng(9)
    M = N = 256
    K = 1024
    A, B = _rand(rng, M * K), _rand(rng, N * K)
    C0 = np.zeros(M * N, np.float32)
    clean = _run(cuda, dev, 16, M, N, K, A, B, C0)
    got = _run(cuda, dev, 16, M, N, K, A, B, C0, opts=ft.make_opts(faults=[{"row": 3, "col": 9, "xor": 1 << 2}]))
    assert np.abs(got - clean).max() < 1e-4  # an undetected flip is below the rounding floor by construction


def test_two_faults_in_one_row_are_recomputed(cuda, ft, dev):
    """Two upsets in one row of one tile cannot be repaired from the two checksums.  Default: the row segment is recomputed
    from A and B on CUDA cores (status 5) -- nothing detected is stored as computed; opts.no_recompute restores the
    round-1 behaviour (reported uncorrectable, left as computed).  All tile shapes, alpha / beta, helper-assisted halves."""
    rng = np.random.default_rng(11)
    M, N, K = 512, 768, 512
    A, B = _rand(rng, M * K), _rand(rng, N * K)
    C0 = rng.standard_normal(M * N).astype(np.float32)
    for kid in (16, 31, 15, 12, 32):
        clean = _run(cuda, dev, kid, M, N, K, A, B, C0, 0.75, -1.5)
        faults = [{"row": 40, "col": 10, "add": 100.0}, {"row": 40, "col": 25, "add": -37.0},     # same row, same tile
                  {"row": 300, "col": 520, "xor": 1 << 30}, {"row": 300, "col": 530, "xor": 1 << 28},
                  {"row": 511, "col": 767, "add": 55.0}]                                        # (a single one: corrected)
        dev.stats()
        got = _run(cuda, dev, kid, M, N, K, A, B, C0, 0.75, -1.5, opts=ft.make_opts(faults=faults))
        st = dev.stats()
        assert st["detected"] == 3 and st["corrected"] == 1 and st["recomputed"] == 2 and st["uncorrectable"] == 0, (kid, st)
        assert sorted(e["status"] for e in st["events"]) == [1, 5, 5]
        scale = float(np.abs(clean).max())
        assert np.abs(got - clean).max() <= 1e-4 * scale, (kid, np.abs(got - clean).max(), scale)
        # only the two recomputed row segments and the corrected element may differ from the fault-free run at all
        diff = np.flatnonzero(got != clean)
        rows = set((diff % M).tolist())
        assert rows <= {40, 300, 511}, (kid, rows)
        got2 = _run(cuda, dev, kid, M, N, K, A, B, C0, 0.75, -1.5, opts=ft.make_opts(faults=faults[:2], no_recompute=True))
        st = dev.stats()
        assert st["detected"] == 1 and st["corrected"] == 0 and st["uncorrectable"] == 1 and st["recomputed"] == 0
        assert np.abs(got2 - clean).max() > 10.0  # (left as computed)


def test_protected_epilogue(cuda, ft, dev):
    """opts.protect_epilogue (the reference's epilogue, ft_sgemm_huge.cuh:573-690, and the window between its last check and
    the store are unprotected): the store pass re-derives the verified row sums from what it re-reads out of the accumulator
    and checks the sum of what it stores.  Fault-free: bit-identical to the unprotected kernel, nothing flagged.  An upset of
    the accumulator AFTER the accumulator check (fault mode 2) or of the value being stored (mode 3) goes unnoticed without
    the option, is detected with it, and with beta == 0 the row segment is recomputed."""
    rng = np.random.default_rng(17)
    M, N, K = 640, 1024, 352
    A, B = _rand(rng, M * K), _rand(rng, N * K)
    C0 = rng.standard_normal(M * N).astype(np.float32)
    for kid in (31, 16, 15, 12, 14):
        for (alpha, beta) in ((0.75, 0.0), (1.0, -1.5)):
            clean = _run(cuda, dev, kid, M, N, K, A, B, C0, alpha, beta)
            dev.stats()
            prot = _run(cuda, dev, kid, M, N, K, A, B, C0, alpha, beta, opts=ft.make_opts(protect_epilogue=True))
            st = dev.stats()
            assert np.array_equal(clean, prot) and st["epilogue_faults"] == 0 and st["detected"] == 0, (kid, beta, st)
            if beta != 0.0:  # Inf / NaN already in the old C (the reference's timing phase lets C diverge): not an upset
                Cx = C0.copy()
                Cx[[5, 77777, M * N - 1]] = [np.inf, np.nan, -np.inf]
                a_ = _run(cuda, dev, kid, M, N, K, A, B, Cx, alpha, beta)
                dev.stats()
                b_ = _run(cuda, dev, kid, M, N, K, A, B, Cx, alpha, beta, opts=ft.make_opts(protect_epilogue=True))
                assert np.array_equal(a_, b_, equal_nan=True) and dev.stats()["epilogue_faults"] == 0
            # pre-check upsets are still corrected as usual in the protected kernel (a repaired row skips the bit-compare)
            pre = [{"row": 7, "col": 33, "xor": 1 << 29}, {"row": 600, "col": 1000, "add": 50.0}]
            got = _run(cuda, dev, kid, M, N, K, A, B, C0, alpha, beta, opts=ft.make_opts(faults=pre, protect_epilogue=True))
            st = dev.stats()
            assert st["detected"] == 2 and st["corrected"] == 2 and st["epilogue_faults"] == 0, (kid, beta, st)
            assert np.abs(got - clean).max() <= 1e-4 * float(np.abs(clean).max())
            for where, (r, c) in (("epilogue_tmem", (37, 5)), ("epilogue_tmem", (300, 900)), ("epilogue_value", (511, 130)),
                                  ("epilogue_value", (2, 1023))):
                f = [{"row": r, "col": c, "xor": 1 << 27, "where": where}]
                if where == "epilogue_tmem":  # unprotected: lands in C unnoticed
                    bad = _run(cuda, dev, kid, M, N, K, A, B, C0, alpha, beta, opts=ft.make_opts(faults=f))
                    st = dev.stats()
                    assert st["detected"] == 0 and st["epilogue_faults"] == 0
                    assert bad[r + c * M] != clean[r + c * M] and np.count_nonzero(bad != clean) == 1
                got = _run(cuda, dev, kid, M, N, K, A, B, C0, alpha, beta, opts=ft.make_opts(faults=f, protect_epilogue=True))
                st = dev.stats()
                assert st["epilogue_faults"] == 1 and st["detected"] == 0, (kid, beta, where, st)
                if beta == 0.0:
                    assert st["recomputed"] == 1 and st["uncorrectable"] == 0 and [e["status"] for e in st["events"]] == [6]
                    assert np.abs(got - clean).max() <= 1e-4 * float(np.abs(clean).max()), (kid, where)
                    assert set((np.flatnonzero(got != clean) % M).tolist()) <= {r}
                else:  # the old values of C are gone: reported, not repaired
                    assert st["recomputed"] == 0 and st["uncorrectable"] == 1 and [e["status"] for e in st["events"]] == [7]
                    assert st["events"][0]["row"] == r


def test_fault_campaign_floors(cuda, ft, dev):
    """BASELINE.json configs[3] in miniature at the real size (M=N=K=8192, the bench kernel id 31): single-bit flips of
    tensor-memory accumulators.  Floors: bits >= 22 (exponent, sign, top mantissa bit) detected 100 % and repaired
    (corrected or recomputed) 100 %, error left <= 1e-4 * max|C|; lower bits: whatever is detected is repaired -- no
    detected fault is stored as computed -- and what stays undetected is below the detection threshold
    (tau_abs + tau_rel * sum|acc| ~ 0.05 at K = 8192, i.e. < 5e-4 * max|C|)."""
    torch = cuda
    n, kid = 8192, 31
    g = torch.Generator(device="cuda").manual_seed(7)
    dA = (torch.randint(0, 10, (n * n,), generator=g, device="cuda").float() * 0.1) * \
        (torch.randint(0, 2, (n * n,), generator=g, device="cuda").float() * 2 - 1)
    dB = (torch.randint(0, 10, (n * n,), generator=g, device="cuda").float() * 0.1) * \
        (torch.randint(0, 2, (n * n,), generator=g, device="cuda").float() * 2 - 1)
    clean = torch.zeros(n * n, device="cuda")
    dev.stats()
    dev.run(kid, n, n, n, dA, dB, clean, 1.0, 0.0, None)
    torch.cuda.synchronize()
    assert dev.stats()["detected"] == 0
    scale = float(clean.abs().max())
    rng = np.random.default_rng(0)
    dC = torch.zeros(n * n, device="cuda")
    for bit in (31, 30, 29, 27, 25, 23, 22, 21, 20, 19, 18, 17, 16, 14, 10):
        inj = det = rep = 0
        worst = 0.0
        for _ in range(2):
            faults, seen = [], set()
            while len(faults) < ft.MAX_FAULTS:
                r, c = int(rng.integers(n)), int(rng.integers(n))
                if (r, c // 256) in seen:
                    continue
                seen.add((r, c // 256))
                faults.append({"row": r, "col": c, "xor": 1 << bit})
            dC.zero_()
            dev.run(kid, n, n, n, dA, dB, dC, 1.0, 0.0, ft.make_opts(faults=faults))
            torch.cuda.synchronize()
            st = dev.stats()
            inj += len(faults)
            det += st["detected"]
            rep += st["corrected"] + st["recomputed"]
            assert st["uncorrectable"] == 0 and st["checksum_faults"] == 0, (bit, st)
            worst = max(worst, float((dC - clean).abs().max()))
        assert rep == det, (bit, det, rep)
        assert worst <= 5e-4 * scale, (bit, worst, scale)
        if bit >= 22:
            assert det == inj and worst <= 1e-4 * scale, (bit, det, inj, worst, scale)


# ------------------------------------------------------------------ 3xTF32: FP32-grade accuracy mode
def test_3xtf32_elementwise_fp32_parity(cuda, ft, dev, oracle):
    """opts.precision = 1: hi/lo split of A and B, three fault-tolerant passes.  ELEMENT-wise parity with the FP32
    oracle (the reference's kernels are true FP32 FFMA): |got - want| <= 1e-3 * |want| + 1e-5 * rms(want) for every
    element, zero failures of the reference's own comparator, norm-wise < 5e-6 (measured 2.7e-6; single-pass TF32: 6e-4); alpha / beta;
    an injected fault in the main pass is still detected and repaired."""
    for n in (512, 1024):
        A, B, C0 = oracle.make_inputs(n)
        want = oracle.sgemm_nt(n, n, n, 1.0, A, B, 0.0, C0.copy())
        rms = float(np.sqrt(np.mean(want.astype(np.float64) ** 2)))
        for kid in (31, 16, 21, ft.ID_ABFT_AUTO):
            dev.stats()
            got = _run(cuda, dev, kid, n, n, n, A, B, C0, opts=ft.make_opts(precision=1))
            d = np.abs(got.astype(np.float64) - want.astype(np.float64))
            assert np.all(d <= 1e-3 * np.abs(want) + 1e-5 * rms), (kid, n, float(d.max()))
            assert oracle.verify_matrix(want, got, n, n) == -1
            assert oracle.error_metrics(want, got)["rel_fro"] < 5e-6, (kid, oracle.error_metrics(want, got))
            if kid != 21:
                st = dev.stats()
                assert st["detected"] == 0 and st["rows_checked"] >= 3 * n * (n // 256)  # three checked passes
    rng = np.random.default_rng(2)
    M, N, K = 384, 640, 1000
    A, B = rng.standard_normal(M * K).astype(np.float32), rng.standard_normal(N * K).astype(np.float32)
    C0 = rng.standard_normal(M * N).astype(np.float32)
    want = oracle.sgemm_nt(M, N, K, 0.75, A, B, -1.5, C0.copy())
    dev.stats()
    got = _run(cuda, dev, 31, M, N, K, A, B, C0, 0.75, -1.5,
               opts=ft.make_opts(precision=1, faults=[{"row": 100, "col": 300, "xor": 1 << 30}]))
    st = dev.stats()
    assert st["detected"] == 1 and st["corrected"] + st["recomputed"] == 1, st
    assert oracle.error_metrics(want, got)["rel_fro"] < 5e-6
    x1 = _run(cuda, dev, 31, M, N, K, A, B, C0, 0.75, -1.5)
    assert oracle.error_metrics(want, x1)["rel_fro"] > 1e-4  # (single-pass TF32 for comparison)


def test_intra_k_check_segments(cuda, ft, dev, oracle):
    """opts.check_segments = S: the product is verified K-segment by K-segment (the reference checks its accumulators
    every K/20 iterations, ft_sgemm_huge.cuh:324).  Same result as the one-shot product up to the FP32 rounding of the S - 1
    intermediate stores; S x the row checks; an upset is repaired inside its segment; 3xTF32 composes with it."""
    rng = np.random.default_rng(8)
    M, N, K = 512, 768, 2048 + 40
    A, B = _rand(rng, M * K), _rand(rng, N * K)
    C0 = rng.standard_normal(M * N).astype(np.float32)
    model = oracle.sgemm_nt_tf32_model(M, N, K, 0.5, A, B, -1.5, C0, "trunc")
    for kid in (31, 16):
        one = _run(cuda, dev, kid, M, N, K, A, B, C0, 0.5, -1.5)
        dev.stats()
        for S in (4, 20):
            got = _run(cuda, dev, kid, M, N, K, A, B, C0, 0.5, -1.5, opts=ft.make_opts(check_segments=S))
            st = dev.stats()
            tile_n = 256 if kid == 31 else 128
            assert st["detected"] == 0 and st["rows_checked"] == S * M * (N // tile_n), (kid, S, st)
            assert oracle.error_metrics(model, got)["rel_fro"] < TOL_MODEL
            assert np.allclose(got, one, rtol=0, atol=2e-5 * float(np.abs(one).max()))
        got = _run(cuda, dev, kid, M, N, K, A, B, C0, 0.5, -1.5,
                   opts=ft.make_opts(check_segments=4, faults=[{"row": 77, "col": 300, "xor": 1 << 30}]))
        st = dev.stats()
        assert st["detected"] == 1 and st["corrected"] + st["recomputed"] == 1, st
        assert np.allclose(got, one, rtol=0, atol=2e-4 * float(np.abs(one).max()))
    want = oracle.sgemm_nt(M, N, K, 0.5, A, B, -1.5, C0.copy())
    got = _run(cuda, dev, 31, M, N, K, A, B, C0, 0.5, -1.5, opts=ft.make_opts(check_segments=3, precision=1))
    assert oracle.error_metrics(want, got)["rel_fro"] < 5e-6


def test_auto_ids_resolve_and_run(cuda, ft, dev, oracle):
    """ids 20 / 40 pick the variant per shape (ftsgemm_select_kernel) and give bit-for-bit the result of that variant."""
    rng = np.random.default_rng(4)
    for (M, N, K) in ((512, 768, 256), (2304, 2304, 128)):
        A, B = _rand(rng, M * K), _rand(rng, N * K)
        C0 = np.zeros(M * N, np.float32)
        for auto, is_ft in ((ft.ID_SGEMM_AUTO, False), (ft.ID_ABFT_AUTO, True)):
            kid = ft.select_kernel(M, N, K, is_ft)
            assert np.array_equal(_run(cuda, dev, auto, M, N, K, A, B, C0), _run(cuda, dev, kid, M, N, K, A, B, C0))
    assert dev.stats()["detected"] == 0


# ------------------------------------------------------------------ host-buffer (e2e) entry point
def test_run_host_matches_device_path(cuda, ft, dev, oracle):
    n = 384
    A, B, C0 = oracle.make_inputs(n)
    C0 = np.random.default_rng(0).standard_normal(n * n).astype(np.float32)
    want = _run(cuda, dev, 16, n, n, n, A, B, C0, 1.0, -1.5)
    hC = C0.copy()
    dev.run_host(16, n, n, n, A, B, hC, 1.0, -1.5, None)
    assert np.array_equal(hC, want)
    # the panel pipeline (4 column panels from N = 4096 on; forced here on a ragged N): upload | GEMM | download per panel,
    # bit-identical to the one-shot device path, with and without the C upload (beta = 0), pinned and pageable memory
    rng = np.random.default_rng(3)
    M, N, K = 512, 1000, 320
    A, B = _rand(rng, M * K), _rand(rng, N * K)
    C0 = rng.standard_normal(M * N).astype(np.float32)
    for kid in (31, 16):
        for beta in (-1.5, 0.0):
            want = _run(cuda, dev, kid, M, N, K, A, B, C0, 0.5, beta)
            for panels in (3, 4, 1):
                try:
                    ft.debug_set("host_panels", panels)
                    hC = C0.copy()
                    dev.run_host(kid, M, N, K, A, B, hC, 0.5, beta, None)
                    assert np.array_equal(hC, want), (kid, beta, panels)
                    pA, pB = cuda.from_numpy(A).pin_memory(), cuda.from_numpy(B).pin_memory()
                    pC = cuda.from_numpy(C0.copy()).pin_memory()
                    dev.run_host(kid, M, N, K, pA, pB, pC, 0.5, beta, None)
                    assert np.array_equal(pC.numpy(), want), (kid, beta, panels, "pinned")
                finally:
                    ft.debug_set("host_panels", -1)
    assert dev.stats()["detected"] == 0


# ------------------------------------------------------------------ BASELINE.json full sizes: properties
@pytest.mark.parametrize("n,kid", [(4096, 16), (4096, 15), (8192, 16), (4096, 31), (8192, 31), (16384, 31), (16384, 16)])
def test_full_size_properties(cuda, ft, dev, oracle, n, kid):
    """Size-independent checks at the metric's sizes: (1) sampled rows against the CPU oracle, (2) the checksum of
    checksums e^T C e = (e^T A)(B^T e) in float64, (3) linearity in alpha, (4) injected faults are repaired in place."""
    torch = cuda
    g = torch.Generator(device="cuda").manual_seed(n)
    dA = (torch.randint(0, 10, (n * n,), generator=g, device="cuda").float() * 0.1) * \
        (torch.randint(0, 2, (n * n,), generator=g, device="cuda").float() * 2 - 1)
    dB = (torch.randint(0, 10, (n * n,), generator=g, device="cuda").float() * 0.1) * \
        (torch.randint(0, 2, (n * n,), generator=g, device="cuda").float() * 2 - 1)
    dC = torch.zeros(n * n, device="cuda")
    dev.stats()
    dev.run(kid, n, n, n, dA, dB, dC, 1.0, 0.0, None)
    torch.cuda.synchronize()
    st = dev.stats()
    assert st["detected"] == 0 and st["rows_checked"] >= n * (n // 256)
    # (1) sampled rows x all columns on the host cores (the kernel the bench times, ids 31 / 21, included; 16384 runs the
    #     wave re-synchronisation path that is on by default from 24 waves)
    rows = np.random.default_rng(n).choice(n, 16 if n <= 8192 else 8, replace=False)
    A, B = dA.cpu().numpy(), dB.cpu().numpy()
    want = oracle.sgemm_nt_rows(n, n, n, 1.0, A, B, 0.0, None, rows)
    got = dC.view(n, n).t()[torch.from_numpy(rows).cuda()].cpu().numpy()  # C is column-major
    assert np.linalg.norm(want - got) / np.linalg.norm(want) < TOL_NORM
    # (2) checksum of checksums (TF32-truncated operands, float64 reference)
    At = (dA.view(torch.int32) & -8192).view(torch.float32).view(n, n)  # [k][m]
    Bt = (dB.view(torch.int32) & -8192).view(torch.float32).view(n, n)  # [k][n]
    sa, sb = At.sum(1, dtype=torch.float64), Bt.sum(1, dtype=torch.float64)
    ref_total = float((sa * sb).sum())
    got_total = float(dC.sum(dtype=torch.float64))
    denom = float((At.abs().sum(1, dtype=torch.float64) * Bt.abs().sum(1, dtype=torch.float64)).sum())
    del At, Bt
    assert abs(ref_total - got_total) / denom < 1e-6
    # (3) linearity: alpha = 2 gives exactly twice the result (power-of-two scaling is exact in FP32)
    dC2 = torch.zeros(n * n, device="cuda")
    dev.run(kid, n, n, n, dA, dB, dC2, 2.0, 0.0, None)
    torch.cuda.synchronize()
    assert torch.equal(dC2, dC * 2)
    # (4) faults in distinct tiles are repaired; all other elements stay bit-identical
    faults = [{"row": 1234, "col": 4000, "xor": 1 << 30}, {"row": 17, "col": 5, "add": 10000.0},
              {"row": n - 1, "col": n - 1, "xor": 1 << 31}]
    dC3 = torch.zeros(n * n, device="cuda")
    dev.run(kid, n, n, n, dA, dB, dC3, 1.0, 0.0, ft.make_opts(faults=faults))
    torch.cuda.synchronize()
    st = dev.stats()
    assert st["detected"] == 3 and st["corrected"] == 3
    delta = (dC3 - dC).abs()
    assert int((delta > 0).sum()) <= 3 and float(delta.max()) < 2e-2
