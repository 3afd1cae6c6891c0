"""Cost of the fused bias: FtSgemm.linear (x @ W^T + b, the bias added in the kernel's store pass) against the unfused form
and against torch's own F.linear.

usage: linear_bench.py [shapes=8192x4096x4096,8192x4096x16384,8192x16384x4096,4096x4096x4096] [id=40] [steps=20]
                       [rounds=5] [out=PATH]
A shape is tokens M x in_features K x out_features N; x (M, K), W (N, K) and b (N,) are row-major float32 tensors.  Arms:
  fused       linear(x, W, b)                          one launch, the bias in the store pass
  unfused     matmul(x, W^T) then out += b             the separate torch add reads and writes all of out once more
  protected   linear(x, W, b) with protect_epilogue    the store pass checked as well
  no_bias     matmul(x, W^T)                           the product alone: fused - no_bias is the cost of the bias
  torch       F.linear(x, W, b), TF32 allowed          cuBLASLt with its own bias epilogue, no fault tolerance
  train       forward + backward of linear             (and train_torch: the same step with F.linear)
Per shape and round the arms run in an order that rotates from round to round: 3 warm-up calls, then CUDA events around
`steps` back-to-back calls.  Reported per arm: median and range over the rounds of the time per call, and TFLOP/s at the
median (2MNK per forward, 6MNK per training step).  The fused and unfused outputs are compared bit for bit.  One JSON line on
stdout (and in `out`), with the GPU name and its power limit.
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
    prot = pkg.make_opts(protect_epilogue=True)
    g = torch.Generator(device="cuda").manual_seed(12)
    gpu, power = gpu_identity()
    result = {"what": "fused bias, us per call", "gpu": gpu, "power_limit_w": power, "id": kid, "steps": steps,
              "rounds": rounds, "shapes": {}}
    for M, K, N in shapes:
        x = torch.randn(M, K, device="cuda", generator=g)
        W = torch.randn(N, K, device="cuda", generator=g)
        b = torch.randn(N, device="cuda", generator=g)
        out = torch.empty(M, N, device="cuda")
        xg, Wg, bg = (t.clone().requires_grad_() for t in (x, W, b))
        gy = torch.randn(M, N, device="cuda", generator=g)

        def unfused():
            ft.matmul(x, W.t(), out, kernel_id=kid)
            out.add_(b)

        def train(fn):
            def step():
                xg.grad = Wg.grad = bg.grad = None
                fn(xg, Wg, bg).backward(gy)
            return step
        arms = {
            "fused": lambda: ft.matmul(x, W.t(), out, bias=b, kernel_id=kid),
            "unfused": unfused,
            "protected": lambda: ft.matmul(x, W.t(), out, bias=b, kernel_id=kid, opts=prot),
            "no_bias": lambda: ft.matmul(x, W.t(), out, kernel_id=kid),
            "torch": lambda: F.linear(x, W, b),
            "train": train(lambda a, w, c: ft.linear(a, w, c, kernel_id=kid)),
            "train_torch": train(F.linear),
        }
        names = list(arms)
        us = {k: [] for k in names}
        ft.stats()
        for r in range(rounds):
            for i in range(len(names)):
                name = names[(i + r) % len(names)]
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
        row = {}
        for name, v in us.items():
            med = statistics.median(v)
            flop = (6.0 if name.startswith("train") else 2.0) * M * N * K
            row[name] = {"median_us": round(med, 1), "range_us": [round(min(v), 1), round(max(v), 1)],
                         "tflops": round(flop / med * 1e-6, 1)}
        row["bias_cost_pct"] = round(100.0 * (row["fused"]["median_us"] / row["no_bias"]["median_us"] - 1.0), 2)
        row["fusion_gain_pct"] = round(100.0 * (row["unfused"]["median_us"] / row["fused"]["median_us"] - 1.0), 2)
        fused = ft.matmul(x, W.t(), bias=b, kernel_id=kid)
        unf = ft.matmul(x, W.t(), kernel_id=kid).add_(b)
        torch.cuda.synchronize()
        row["fused_equals_unfused"] = bool(torch.equal(fused, unf))
        row["detected"] = ft.stats()["detected"]
        result["shapes"][f"{M}x{K}x{N}"] = row
        del x, W, b, out, xg, Wg, bg, gy, fused, unf
        torch.cuda.empty_cache()
    ft.close()
    line = json.dumps(result)
    print(line)
    if "out" in kv:
        Path(kv["out"]).parent.mkdir(parents=True, exist_ok=True)
        Path(kv["out"]).write_text(line + "\n")


if __name__ == "__main__":
    main()
