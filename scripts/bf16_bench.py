"""BF16 operands against FP32: run_typed id 31 with BF16 A and B against the FP32 id 31 in the same layout pairs, cuBLAS BF16
(id 7), and FtSgemm.linear with BF16 x and W at the F.linear shapes against the FP32 layer and torch's BF16 F.linear.

usage: bf16_bench.py [sizes=4096,8192] [shapes=8192x4096x4096,8192x4096x16384,8192x16384x4096,4096x4096x4096] [steps=20]
                     [rounds=5] [out=PATH]
Products (alpha = 1, beta = -1.5, C reset before every burst): per size the arms run in an order that rotates from round to
round, 3 warm-up launches, then CUDA events around `steps` back-to-back launches:
  fp32_31_MN,MN / fp32_31_K,K    run_ex id 31 on FP32 operands (the MN-major pair runs the front-phase transposes)
  bf16_31_MN,MN / bf16_31_K,K    run_typed id 31 on BF16 operands (both layouts read in place)
  bf16_7_K,K                     run_typed id 7: cuBLAS with BF16 A / B, FP32 C, compute 32F
Layers (x (M, K), W (N, K) row-major, tokens M x in K x out N, no bias):
  fp32_linear   FtSgemm.linear(x, W) on FP32 tensors (id 40)
  bf16_linear   FtSgemm.linear(x, W) on BF16 tensors (id 40): FP32 out
  torch_bf16    F.linear(x, W) on BF16 tensors (cuBLAS, BF16 out, no fault tolerance)
Every arm allocates its output per call, as the layers do.
Reported per arm: median and range over the rounds of the time per call, and TFLOP/s at the median (2MNK).  The BF16 outputs
of the four layout pairs are compared bit for bit, and the ABFT counters are reported.  One JSON line on
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


def timed(arms, steps, rounds, reset=None):
    us = {k: [] for k in arms}
    names = list(arms)
    for r in range(rounds):
        for i in range(len(names)):
            name = names[(i + r) % len(names)]
            fn = arms[name]
            if reset:
                reset()
            for _ in range(3):
                fn()
            if reset:
                reset()
            torch.cuda.synchronize()
            time.sleep(0.02)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(steps):
                fn()
            e1.record()
            torch.cuda.synchronize()
            us[name].append(e0.elapsed_time(e1) / steps * 1e3)
    return us


def summary(us, flop):
    out = {}
    for k, v in us.items():
        med = statistics.median(v)
        out[k] = {"median_us": round(med, 1), "range_us": [round(min(v), 1), round(max(v), 1)],
                  "tflops": round(flop / med * 1e-6, 1)}
    return out


def main():
    pkg = ge.load_package()
    kv = dict(a.split("=", 1) for a in sys.argv[1:])
    sizes = [int(x) for x in kv.get("sizes", "4096,8192").split(",")]
    shapes = [tuple(int(v) for v in s.split("x"))
              for s in kv.get("shapes", "8192x4096x4096,8192x4096x16384,8192x16384x4096,4096x4096x4096").split(",")]
    steps, rounds = int(kv.get("steps", 20)), int(kv.get("rounds", 5))
    alpha, beta = 1.0, -1.5
    ft = pkg.FtSgemm()
    opts = pkg.make_opts(stream=torch.cuda.current_stream().cuda_stream)
    g = torch.Generator(device="cuda").manual_seed(13)
    gpu, power = gpu_identity()
    result = {"what": "BF16 operands against FP32, us per call", "gpu": gpu, "power_limit_w": power, "alpha": alpha,
              "beta": beta, "steps": steps, "rounds": rounds, "products": {}, "layers": {}}
    lay = {"MN": pkg.LAYOUT_MN_MAJOR, "K": pkg.LAYOUT_K_MAJOR}
    for n in sizes:
        A = torch.randn(n, n, device="cuda", generator=g)
        B = torch.randn(n, n, device="cuda", generator=g)
        f32 = {("A", "MN"): A.t().contiguous(), ("A", "K"): A, ("B", "MN"): B.t().contiguous(), ("B", "K"): B}
        b16 = {k: v.to(torch.bfloat16) for k, v in f32.items()}
        C0 = torch.randn(n * n, device="cuda", generator=g)
        dC = torch.empty_like(C0)

        def fp32(la, lb):
            return lambda: ft.run_ex(31, n, n, n, f32[("A", la)], lay[la], n, f32[("B", lb)], lay[lb], n, dC, n, alpha, beta, opts)

        def bf16(kid, la, lb):
            return lambda: ft.run_typed(kid, n, n, n, b16[("A", la)], lay[la], n, b16[("B", lb)], lay[lb], n, pkg.TYPE_BF16, dC,
                                        n, dC, alpha, beta, opts=opts)
        arms = {"fp32_31_MN,MN": fp32("MN", "MN"), "fp32_31_K,K": fp32("K", "K"), "bf16_31_MN,MN": bf16(31, "MN", "MN"),
                "bf16_31_K,K": bf16(31, "K", "K"), "bf16_7_K,K": bf16(7, "K", "K")}
        ft.stats()
        row = summary(timed(arms, steps, rounds, lambda: dC.copy_(C0)), 2.0 * n ** 3)
        st = ft.stats()
        outs = []
        for la, lb in (("MN", "MN"), ("K", "K"), ("MN", "K"), ("K", "MN")):
            dC.copy_(C0)
            bf16(31, la, lb)()
            outs.append(dC.clone())
        torch.cuda.synchronize()
        row["bf16_layouts_bit_identical"] = all(torch.equal(outs[0], o) for o in outs)
        row["detected"] = st["detected"]
        result["products"][str(n)] = row
        del A, B, f32, b16, C0, dC, outs
        torch.cuda.empty_cache()
    for M, K, N in shapes:
        x = torch.randn(M, K, device="cuda", generator=g)
        W = torch.randn(N, K, device="cuda", generator=g)
        xb, Wb = x.to(torch.bfloat16), W.to(torch.bfloat16)
        arms = {"fp32_linear": lambda: ft.linear(x, W), "bf16_linear": lambda: ft.linear(xb, Wb),
                "torch_bf16": lambda: F.linear(xb, Wb)}
        ft.stats()
        row = summary(timed(arms, steps, rounds), 2.0 * M * N * K)
        row["detected"] = ft.stats()["detected"]
        result["layers"][f"{M}x{K}x{N}"] = row
        del x, W, xb, Wb
        torch.cuda.empty_cache()
    ft.close()
    line = json.dumps(result)
    print(line)
    if "out" in kv:
        Path(kv["out"]).parent.mkdir(parents=True, exist_ok=True)
        Path(kv["out"]).write_text(line + "\n")


if __name__ == "__main__":
    main()
