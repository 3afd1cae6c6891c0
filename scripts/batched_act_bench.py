"""Cost of the fused batched activation and per-entry bias: FtSgemm.bmm(x, W^T, bias=b, activation="gelu") (one launch,
the bias of each expert and GELU in the store pass) against the unfused forms and torch, and FtSgemm.bmm as the two
attention products, forward and backward.

usage: batched_act_bench.py [id=40] [steps=20] [rounds=5] [out=PATH]
Expert FFN shapes (experts x tokens x in -> out): 8 x 1024 x 4096 -> 4096 and 8 x 2048 x 4096 -> 14336; x (E, T, in),
W (E, out, in) and b (E, out) are contiguous float32 tensors.  Arms (forward arms under torch.no_grad()):
  fused         bmm(x, W^T, bias=b, activation="gelu")        one launch
  unfused       F.gelu(bmm(x, W^T, bias=b))                    the batched product, then torch's GELU
  loop          [linear(x[e], W[e], b[e], activation="gelu")]   one fused single product per expert
  torch         F.gelu(baddbmm(b, x, W^T)), TF32 allowed       cuBLAS and torch's GELU, no fault tolerance
  train_fused   forward + backward of the fused arm            (z written for the backward)
  train_torch   forward + backward of the torch arm
Attention shapes (batch x M x N x K): 128 x 1024 x 1024 x 128 (q k^T) and 128 x 1024 x 128 x 1024 (p v), no bias or
activation.  Arms: ft (bmm), torch (torch.bmm, TF32), train_ft and train_torch (forward + backward).
Per shape and round the arms run in an order that rotates from round to round: 3 warm-up calls, then CUDA events around
`steps` back-to-back calls.  Reported per arm: median and range over the rounds of the time per call, and TFLOP/s at the
median (2 flop per multiply-add forward, 3x that per training step).  The fused and unfused expert outputs are compared (max
ulp; the pre-activation values bit for bit), and the library's fault counters must stay at 0.  One JSON line on stdout (and
in `out`), with the GPU name and its power limit, read in the same run.
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

EXPERTS = [(8, 1024, 4096, 4096), (8, 2048, 4096, 14336)]
ATTENTION = [("qk", 128, 1024, 1024, 128), ("pv", 128, 1024, 128, 1024)]


def max_ulp(a, b):
    def key(x):
        i = x.contiguous().view(torch.int32).long()
        return torch.where(i < 0, -(i & 0x7FFFFFFF), i)
    return int((key(a) - key(b)).abs().max())


def measure(arms, steps, rounds):
    names = list(arms)
    us = {k: [] for k in names}
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
    return us


def summarise(us, flop):
    row = {}
    for name, v in us.items():
        med = statistics.median(v)
        f = (3.0 if name.startswith("train") else 1.0) * flop
        row[name] = {"median_us": round(med, 1), "range_us": [round(min(v), 1), round(max(v), 1)],
                     "tflops": round(f / med * 1e-6, 1)}
    return row


def main():
    pkg = ge.load_package()
    kv = dict(a.split("=", 1) for a in sys.argv[1:])
    kid = int(kv.get("id", 40))
    steps, rounds = int(kv.get("steps", 20)), int(kv.get("rounds", 5))
    torch.backends.cuda.matmul.allow_tf32 = True
    ft = pkg.FtSgemm()
    g = torch.Generator(device="cuda").manual_seed(17)
    gpu, power = gpu_identity()
    result = {"what": "batched activation and per-entry bias, us per call", "gpu": gpu, "power_limit_w": power, "id": kid,
              "steps": steps, "rounds": rounds, "experts": {}, "attention": {}}
    for E, T, K, N in EXPERTS:
        x = torch.randn(E, T, K, device="cuda", generator=g)
        W = torch.randn(E, N, K, device="cuda", generator=g) * K ** -0.5
        b = torch.randn(E, N, device="cuda", generator=g)
        xg, Wg, bg = (t.clone().requires_grad_() for t in (x, W, b))
        gy = torch.randn(E, T, N, device="cuda", generator=g)

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

        def ft_fused(a, w, c):
            return ft.bmm(a, w.transpose(1, 2), bias=c, activation="gelu", kernel_id=kid)

        def torch_ffn(a, w, c):
            return F.gelu(torch.baddbmm(c.unsqueeze(1), a, w.transpose(1, 2)))
        arms = {
            "fused": fwd(lambda: ft_fused(x, W, b)),
            "unfused": fwd(lambda: F.gelu(ft.bmm(x, W.transpose(1, 2), bias=b, kernel_id=kid))),
            "loop": fwd(lambda: [ft.linear(x[e], W[e], b[e], activation="gelu", kernel_id=kid) for e in range(E)]),
            "torch": fwd(lambda: torch_ffn(x, W, b)),
            "train_fused": train(ft_fused),
            "train_torch": train(torch_ffn),
        }
        ft.stats()
        row = summarise(measure(arms, steps, rounds), 2.0 * E * T * N * K)
        row["fusion_gain_pct"] = round(100.0 * (row["unfused"]["median_us"] / row["fused"]["median_us"] - 1.0), 2)
        row["train_vs_torch_pct"] = round(100.0 * (row["train_torch"]["median_us"] / row["train_fused"]["median_us"] - 1.0), 2)
        with torch.no_grad():
            launches = ft.launch_count()
            z = torch.empty(E, T, N, device="cuda")
            y = ft.bmm(x, W.transpose(1, 2), bias=b, activation="gelu", preact=z, kernel_id=kid)
            row["fused_launches"] = ft.launch_count() - launches
            plain = ft.bmm(x, W.transpose(1, 2), bias=b, kernel_id=kid)
            loop = torch.stack([ft.linear(x[e], W[e], b[e], activation="gelu", kernel_id=kid) for e in range(E)])
            torch.cuda.synchronize()
            row["preact_equals_unfused"] = bool(torch.equal(z, plain))
            row["gelu_max_ulp_vs_unfused"] = max_ulp(y, F.gelu(plain))
            row["fused_equals_loop"] = bool(torch.equal(y, loop))
        row["detected"] = ft.stats()["detected"]
        result["experts"][f"{E}x{T}x{K}->{N}"] = row
        del x, W, b, xg, Wg, bg, gy, z, y, plain, loop
        torch.cuda.empty_cache()
    for name, Bt, M, N, K in ATTENTION:
        a = torch.randn(Bt, M, K, device="cuda", generator=g)
        # q @ k^T: k row-major (Bt, N, K) read transposed; p @ v: v row-major (Bt, K, N)
        bt = (torch.randn(Bt, K, N, device="cuda", generator=g) if name == "pv" else
              torch.randn(Bt, N, K, device="cuda", generator=g).transpose(1, 2))
        ag, bg = a.clone().requires_grad_(), bt.detach().clone().requires_grad_()
        gy = torch.randn(Bt, M, N, device="cuda", generator=g)

        def train(fn):
            def step():
                ag.grad = bg.grad = None
                fn(ag, bg).backward(gy)
            return step

        def ft_bmm(p, q):
            return ft.bmm(p, q, kernel_id=kid)
        arms = {
            "ft": lambda: ft.bmm(a, bt, kernel_id=kid),
            "torch": lambda: torch.bmm(a, bt),
            "train_ft": train(ft_bmm),
            "train_torch": train(torch.bmm),
        }
        ft.stats()
        row = summarise(measure(arms, steps, rounds), 2.0 * Bt * M * N * K)
        row["detected"] = ft.stats()["detected"]
        result["attention"][f"{name} {Bt}x{M}x{N}x{K}"] = row
        del a, bt, ag, bg, gy
        torch.cuda.empty_cache()
    ft.close()
    line = json.dumps(result)
    print(line)
    if "out" in kv:
        Path(kv["out"]).parent.mkdir(parents=True, exist_ok=True)
        Path(kv["out"]).write_text(line + "\n")


if __name__ == "__main__":
    main()
