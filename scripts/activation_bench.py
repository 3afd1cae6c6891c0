"""Cost of the fused activation: FtSgemm.linear(..., activation=) (act(x @ W^T + b), the activation applied in the kernel's
store pass) against the unfused form and against torch.

usage: activation_bench.py [shapes=8192x4096x4096,8192x4096x16384,8192x16384x4096,4096x4096x4096] [id=40] [steps=20]
                           [rounds=5] [out=PATH]
A shape is tokens M x in_features K x out_features N; x (M, K), W (N, K) and b (N,) are row-major float32 tensors.  The
forward arms run under torch.no_grad() (no pre-activation output is written).  Arms:
  relu_fused      linear(x, W, b, activation="relu")      one launch, ReLU in the store pass
  relu_unfused    F.relu(linear(x, W, b))                  a separate torch kernel reads and writes all of y once more
  gelu_fused      linear(x, W, b, activation="gelu")
  gelu_unfused    F.gelu(linear(x, W, b))
  no_act          linear(x, W, b)                          the biased product alone: fused - no_act is the activation's cost
  torch_gelu      F.gelu(F.linear(x, W, b)), TF32 allowed  cuBLASLt and torch's GELU, no fault tolerance
  train_fused     forward + backward of linear(..., activation="gelu")   (z written for the backward)
  train_unfused   forward + backward of F.gelu(linear(...))
Per shape and round the arms run in an order that rotates from round to round: 3 warm-up calls, then CUDA events around
`steps` back-to-back calls.  Reported per arm: median and range over the rounds of the time per call, and TFLOP/s at the
median (2MNK per forward, 6MNK per training step).  Fused and unfused outputs are compared: bit for bit for ReLU, max ulp
for GELU.  One JSON line on stdout (and in `out`), with the GPU name and its power limit.
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


def max_ulp(a, b):
    def key(x):
        i = x.contiguous().view(torch.int32).long()
        return torch.where(i < 0, -(i & 0x7FFFFFFF), i)
    return int((key(a) - key(b)).abs().max())


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
    result = {"what": "fused activation, us per call", "gpu": gpu, "power_limit_w": power, "id": kid, "steps": steps,
              "rounds": rounds, "shapes": {}}
    for M, K, N in shapes:
        x = torch.randn(M, K, device="cuda", generator=g)
        W = torch.randn(N, K, device="cuda", generator=g) * K ** -0.5
        b = torch.randn(N, device="cuda", generator=g)
        xg, Wg, bg = (t.clone().requires_grad_() for t in (x, W, b))
        gy = torch.randn(M, N, device="cuda", generator=g)

        def lin(act=None):
            return ft.linear(x, W, b, activation=act, kernel_id=kid)

        def fwd(fn):
            def call():
                with torch.no_grad():
                    return fn()
            return call

        def train(fn):
            def step():
                xg.grad = Wg.grad = bg.grad = None
                fn(xg, Wg, bg).backward(gy)
            return step
        arms = {
            "relu_fused": fwd(lambda: lin("relu")),
            "relu_unfused": fwd(lambda: F.relu(lin())),
            "gelu_fused": fwd(lambda: lin("gelu")),
            "gelu_unfused": fwd(lambda: F.gelu(lin())),
            "no_act": fwd(lin),
            "torch_gelu": fwd(lambda: F.gelu(F.linear(x, W, b))),
            "train_fused": train(lambda a, w, c: ft.linear(a, w, c, activation="gelu", kernel_id=kid)),
            "train_unfused": train(lambda a, w, c: F.gelu(ft.linear(a, w, c, kernel_id=kid))),
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
        for act in ("relu", "gelu"):
            row[f"{act}_fusion_gain_pct"] = round(
                100.0 * (row[f"{act}_unfused"]["median_us"] / row[f"{act}_fused"]["median_us"] - 1.0), 2)
            row[f"{act}_cost_pct"] = round(100.0 * (row[f"{act}_fused"]["median_us"] / row["no_act"]["median_us"] - 1.0), 2)
        row["train_fusion_gain_pct"] = round(
            100.0 * (row["train_unfused"]["median_us"] / row["train_fused"]["median_us"] - 1.0), 2)
        with torch.no_grad():
            y = lin()
            relu_f, gelu_f = lin("relu"), lin("gelu")
            torch.cuda.synchronize()
            row["relu_fused_equals_unfused"] = bool(torch.equal(relu_f, F.relu(y)))
            row["gelu_max_ulp_vs_unfused"] = max_ulp(gelu_f, F.gelu(y))
        row["detected"] = ft.stats()["detected"]
        result["shapes"][f"{M}x{K}x{N}"] = row
        del x, W, b, xg, Wg, bg, gy, y, relu_f, gelu_f
        torch.cuda.empty_cache()
    ft.close()
    line = json.dumps(result)
    print(line)
    if "out" in kv:
        Path(kv["out"]).parent.mkdir(parents=True, exist_ok=True)
        Path(kv["out"]).write_text(line + "\n")


if __name__ == "__main__":
    main()
