"""Strided-batched fault-tolerant GEMM against a loop of single products, cuBLAS strided-batched and torch.bmm.

Arms, alternated over 5 rounds (medians): run_batched with id 40 (one launch for the batch), a Python loop of run_ex with
id 40 over the entries, id 7 (cublasSgemmStridedBatched, TF32) and torch.bmm with TF32 allowed.  Both operands K-major
(contiguous torch tensors, q @ k^T form).  Prints one JSON line; also checks that C of the batched and the loop arm is
bit-identical and records the library launches per call.
"""
import json
import subprocess
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import __graft_entry__ as ge  # noqa: E402

SHAPES = [  # (name, batch, M, N, K) of C_i = A_i B_i^T
    ("attn_qk", 128, 1024, 1024, 128),
    ("attn_pv", 128, 1024, 128, 1024),
    ("cube1024", 32, 1024, 1024, 1024),
    ("cube2048", 8, 2048, 2048, 2048),
]


def _time(fn, reps):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    fn()
    torch.cuda.synchronize()
    s.record()
    for _ in range(reps):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / reps * 1e-3


def main():
    ft = ge.load_package()
    dev = ft.FtSgemm()
    torch.backends.cuda.matmul.allow_tf32 = True
    try:
        gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True).stdout.strip()
    except OSError:
        gpu = torch.cuda.get_device_name()
    res = {"gpu": gpu, "rounds": 5, "shapes": {}}
    for name, Bt, M, N, K in SHAPES:
        g = torch.Generator(device="cuda").manual_seed(1)
        A = torch.randn(Bt, M, K, device="cuda", generator=g)
        B = torch.randn(Bt, N, K, device="cuda", generator=g)  # K-major B: C_i = A_i B_i^T
        Cb = torch.zeros(Bt, N, M, device="cuda")  # column-major C_i (ldc = M)
        Cl = torch.zeros_like(Cb)
        Cc = torch.zeros_like(Cb)
        o = ft.make_opts(stream=torch.cuda.current_stream().cuda_stream)
        arms = {
            "batched": lambda: dev.run_batched(40, M, N, K, A, 1, K, M * K, B, 1, K, N * K, Cb, M, M * N, Bt, 1.0, 0.0, opts=o),
            "loop": lambda: [dev.run_ex(40, M, N, K, A[i], 1, K, B[i], 1, K, Cl[i], M, 1.0, 0.0, o) for i in range(Bt)],
            "cublas_tf32": lambda: dev.run_batched(7, M, N, K, A, 1, K, M * K, B, 1, K, N * K, Cc, M, M * N, Bt, 1.0, 0.0, opts=o),
            "torch_bmm": lambda: torch.bmm(A, B.transpose(1, 2)),
        }
        launches = {}
        for k in ("batched", "loop"):
            n0 = dev.launch_count()
            arms[k]()
            launches[k] = dev.launch_count() - n0
        torch.cuda.synchronize()
        times = {k: [] for k in arms}
        reps = max(2, int(2e11 / (2.0 * Bt * M * N * K)))
        for _ in range(5):
            for k, fn in arms.items():
                times[k].append(_time(fn, reps))
        st = dev.stats()
        flop = 2.0 * Bt * M * N * K
        med = {k: sorted(v)[2] for k, v in times.items()}
        res["shapes"][name] = {
            "batch": Bt, "M": M, "N": N, "K": K,
            "tflops": {k: round(flop / t * 1e-12, 1) for k, t in med.items()},
            "ms": {k: round(t * 1e3, 3) for k, t in med.items()},
            "launches_per_call": launches,
            "batched_vs_loop": round(med["loop"] / med["batched"], 3),
            "bit_identical_to_loop": bool(torch.equal(Cb, Cl)),
            "faults_detected": st["detected"],
        }
    dev.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
