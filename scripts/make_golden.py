"""Generate tests/golden/* from the reference's OWN code (oracle/_ref/libref_utils.so = the reference's utils/utils.cu
compiled unmodified, oracle/_ref/libref_kernels_cpu.so = its generated kernels under a CPU thread shim).  Run where the
reference checkout exists (`make -C oracle REF=<path>`); the fixtures are committed, so the tests need neither.

For END in {64,128,256,512,1024}: srand(10); A,B,C = generate_random_matrix(END); C=0 (sgemm.cu:12,52-56);
C = cpu_gemm(1, 0, B^T-buffer, A-buffer) which is the kernels' column-major NT result
(SURVEY.md section 8c oracle 1).  Stored: leading elements of A/B/C, selected C entries, sums, and a
sha256 of the raw float32 bytes of A, B and C.
"""
import hashlib, json, sys
from pathlib import Path
import numpy as np
sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from oracle import oracle as O

out_dir = Path(__file__).resolve().parents[1] / "tests" / "golden"
out_dir.mkdir(parents=True, exist_ok=True)
r = O.ref_utils()
assert r is not None, "needs oracle/_ref (run `make -C oracle`)"
gold = {}
for n in (64, 128, 256, 512, 1024):
    A, B, C = O.ref_make_inputs(n)
    # cpu_gemm is row-major square: Z = X*Y.  With X := B-buffer read row-major = B^T ... see SURVEY 8c:
    # kernels' C buffer == cpu_gemm(alpha, beta, B^T_buffer, A_buffer).  B^T_buffer: row-major (K x N)^T
    # Concretely Cbuf[m + n*M] = sum_k A[m+k*M]*B[n+k*N]; as row-major Z[i=n][j=m] = sum_k X[n][k] Y[k][m]
    # with X[n][k] = B[n + k*N] (i.e. X = transpose of the B buffer read row-major) and Y = A buffer row-major.
    X = np.ascontiguousarray(B.reshape(n, n).T)
    Z = np.zeros(n * n, np.float32)
    r.ref_cpu_gemm(1.0, 0.0, O._p(X.reshape(-1)), O._p(A), n, O._p(Z))
    gold[str(n)] = {
        "A_head": [float(x) for x in A[:8]], "B_head": [float(x) for x in B[:8]],
        "C_sel": {"0": float(Z[0]), "1": float(Z[1]), str(n): float(Z[n]), str(n * n - 1): float(Z[n * n - 1])},
        "C_sum": float(Z.astype(np.float64).sum()), "C_abs_sum": float(np.abs(Z.astype(np.float64)).sum()),
        "sha256": {"A": hashlib.sha256(A.tobytes()).hexdigest(), "B": hashlib.sha256(B.tobytes()).hexdigest(),
                   "C": hashlib.sha256(Z.tobytes()).hexdigest()},
    }
    print(n, gold[str(n)]["C_sel"], gold[str(n)]["C_sum"], gold[str(n)]["C_abs_sum"])
(out_dir / "ref_cpu_gemm.json").write_text(json.dumps(gold, indent=1))

# Host-code pins at END = 160 (tests/test_oracle.py::test_oracle_equals_reference_host_code): the reference's inputs, its
# cpu_gemm result and its verify_matrix verdicts on an exact and a perturbed copy.
n = 160
A, B, _ = O.ref_make_inputs(n)
X = np.ascontiguousarray(B.reshape(n, n).T).reshape(-1)
Z = np.zeros(n * n, np.float32)
r.ref_cpu_gemm(1.0, 0.0, O._p(X), O._p(A), n, O._p(Z))
bad = Z.copy(); bad[77] += 5.0
host = {"n": n, "sha256": {"A": hashlib.sha256(A.tobytes()).hexdigest(), "B": hashlib.sha256(B.tobytes()).hexdigest(),
                           "C": hashlib.sha256(Z.tobytes()).hexdigest()},
        "verify_exact": int(r.ref_verify_matrix(O._p(Z), O._p(Z.copy()), n, n)),
        "verify_perturbed_77": int(r.ref_verify_matrix(O._p(Z), O._p(bad), n, n))}
(out_dir / "ref_host_code.json").write_text(json.dumps(host, indent=1))

# The reference's generated kernels executed on the CPU (oracle/_ref/libref_kernels_cpu.so): their C for the inputs
# tests/test_oracle.py::test_reference_kernels_on_cpu builds (seed 2), one .npy per case (<= 64 KiB each).
rk = O.ref_kernels()
assert rk is not None, "needs oracle/_ref/libref_kernels_cpu.so"
for kid, variant, K in ((6, "huge", 160), (16, "huge", 160), (13, "large", 160), (11, "small", 480)):
    ms, ns, _, _, _ = O.VARIANTS[variant]
    M, N = ms, ns
    rng = np.random.default_rng(2)
    pad = 4096
    A = np.zeros(M * K + pad, np.float32); B = np.zeros(N * K + pad, np.float32)
    A[:M * K] = (rng.integers(-9, 10, M * K) * 0.1).astype(np.float32)
    B[:N * K] = (rng.integers(-9, 10, N * K) * 0.1).astype(np.float32)
    C = np.zeros(M * N, np.float32)
    assert rk.ref_kernel_run(kid, M, N, K, O._p(A), O._p(B), O._p(C), 1.0, 0.0) == 0
    np.save(out_dir / f"ref_kernel_{kid}_{variant}_K{K}.npy", C)
