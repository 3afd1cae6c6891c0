"""Cost of the fused residual: FtSgemm.linear(x, W, b, residual=r) (y = (x @ W^T + r) + b from one launch, r read in place of
the old output) against the ways a caller could form a residual layer without it.

usage: residual_bench.py [shapes=8192x4096x4096,8192x4096x16384,8192x16384x4096,4096x4096x4096] [id=40] [steps=20]
                         [rounds=5] [out=PATH]
A shape is tokens M x in_features K x out_features N; x (M, K), W (N, K), b (N,) and r (M, N) are row-major float32 tensors
(the linear_bench.py shapes).  Arms:
  fused        linear(x, W, b, residual=r)                       one launch, r read by the store pass, y written
  add          linear(x, W, b) + r                               torch's add reads y and r and writes a new y
  clone        y = r.clone(); matmul(x, W^T, out=y, bias=b, beta=1)   an extra copy, then the in-place biased product
  no_residual  linear(x, W, b)                                   the biased product alone: fused - no_residual is the cost
  torch        F.linear(x, W, b) + r, TF32 allowed               cuBLASLt and torch's add, no fault tolerance
Per shape and round the arms run in an order that rotates from round to round: 3 warm-up calls, then CUDA events around
`steps` back-to-back calls.  Reported per arm: median and range over the rounds of the time per call, and TFLOP/s at the
median (2MNK).  The fused output is compared bit for bit with the clone arm's.  One JSON line on stdout (and in `out`), with
the GPU name and its power limit.
"""
import json
import statistics
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402
import __graft_entry__ as ge  # noqa: E402
from scripts.layout_bench import gpu_identity  # noqa: E402


def main():
    pkg = ge.load_package()
    kv = dict(a.split("=", 1) for a in sys.argv[1:])
    shapes = [tuple(int(v) for v in s.split("x"))
              for s in kv.get("shapes", "8192x4096x4096,8192x4096x16384,8192x16384x4096,4096x4096x4096").split(",")]
    kid = int(kv.get("id", 40))
    steps, rounds = int(kv.get("steps", 20)), int(kv.get("rounds", 5))
    torch.backends.cuda.matmul.allow_tf32 = True
    ft = pkg.FtSgemm()
    g = torch.Generator(device="cuda").manual_seed(13)
    gpu, power = gpu_identity()
    result = {"what": "fused residual, us per call", "gpu": gpu, "power_limit_w": power, "id": kid, "steps": steps,
              "rounds": rounds, "shapes": {}}
    for M, K, N in shapes:
        x = torch.randn(M, K, device="cuda", generator=g)
        W = torch.randn(N, K, device="cuda", generator=g) * K ** -0.5
        b = torch.randn(N, device="cuda", generator=g)
        r = torch.randn(M, N, device="cuda", generator=g)

        def clone():
            y = r.clone()
            return ft.matmul(x, W.t(), y, bias=b, beta=1.0, kernel_id=kid)
        arms = {
            "fused": lambda: ft.linear(x, W, b, residual=r, kernel_id=kid),
            "add": lambda: ft.linear(x, W, b, kernel_id=kid) + r,
            "clone": clone,
            "no_residual": lambda: ft.linear(x, W, b, kernel_id=kid),
            "torch": lambda: F.linear(x, W, b) + r,
        }
        names = list(arms)
        us = {k: [] for k in names}
        ft.stats()
        with torch.no_grad():
            for rd in range(rounds):
                for i in range(len(names)):
                    name = names[(i + rd) % len(names)]
                    for _ in range(3):
                        arms[name]()
                    torch.cuda.synchronize()
                    time.sleep(0.02)
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    for _ in range(steps):
                        arms[name]()
                    e1.record()
                    torch.cuda.synchronize()
                    us[name].append(e0.elapsed_time(e1) / steps * 1e3)
            fused, ref = arms["fused"](), clone()
            torch.cuda.synchronize()
        row = {}
        for name, v in us.items():
            med = statistics.median(v)
            row[name] = {"median_us": round(med, 1), "range_us": [round(min(v), 1), round(max(v), 1)],
                         "tflops": round(2.0 * M * N * K / med * 1e-6, 1)}
        med = {k: row[k]["median_us"] for k in names}
        row["residual_cost_pct"] = round(100.0 * (med["fused"] / med["no_residual"] - 1.0), 2)
        row["gain_over_add_pct"] = round(100.0 * (med["add"] / med["fused"] - 1.0), 2)
        row["gain_over_clone_pct"] = round(100.0 * (med["clone"] / med["fused"] - 1.0), 2)
        row["fused_equals_clone"] = bool(torch.equal(fused.view(torch.int32), ref.view(torch.int32)))
        row["detected"] = ft.stats()["detected"]
        result["shapes"][f"{M}x{K}x{N}"] = row
        del x, W, b, r, fused, ref
        torch.cuda.empty_cache()
    ft.close()
    line = json.dumps(result)
    print(line)
    if "out" in kv:
        Path(kv["out"]).parent.mkdir(parents=True, exist_ok=True)
        Path(kv["out"]).write_text(line + "\n")


if __name__ == "__main__":
    main()
