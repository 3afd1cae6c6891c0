"""BF16 results against FP32 results on BF16 operands: run_batched_mixed id 31 with BF16 C / D against FP32 C / D (with and
without a separate cast to bfloat16), cuBLAS BF16 with BF16 C (id 7), and FtSgemm.linear with out_dtype=torch.bfloat16
against linear(...).to(torch.bfloat16) and torch's BF16 F.linear.

usage: bf16_out_bench.py [sizes=4096,8192] [shapes=8192x4096x4096,8192x4096x16384,8192x16384x4096,4096x4096x4096]
                         [steps=20] [rounds=5] [out=PATH]
Products (alpha = 1, beta = -1.5, D separate from C, so no reset is needed): per size and layout pair (MN,MN and K,K) the
arms run in an order that rotates from round to round, 3 warm-up launches, then CUDA events around `steps` back-to-back
calls:
  31_<pair>_bf16        run_batched_mixed id 31, BF16 C and D
  31_<pair>_fp32        the same call with FP32 C and D
  31_<pair>_fp32_cast   the FP32 call followed by D.to(torch.bfloat16) into a preallocated BF16 tensor
  7_K,K_bf16            cuBLAS with BF16 A / B / C, compute 32F, in place (no fault tolerance)
Layers (x (M, K), W (N, K) row-major, tokens M x in K x out N, a bias, each arm allocating its output):
  linear_bf16           FtSgemm.linear(x, W, b, out_dtype=torch.bfloat16)
  linear_cast           FtSgemm.linear(x, W, b).to(torch.bfloat16)
  torch_bf16            F.linear(x, W, b)
  gelu_bf16 / gelu_cast / torch_gelu          the same with activation="gelu" (torch: F.gelu(F.linear(...)))
  residual_bf16 / residual_cast / torch_residual   the same with residual=r (bf16 r, or its float32 upcast for the FP32 arm;
                        torch: F.linear(x, W, b) + r)
Training step (one BF16 linear at each shape, forward + backward with a bfloat16 grad_y, grad for x and W):
  step_fp32_out_cast    the parent's layer: float32 y, backward products written as float32 then cast to bfloat16
  step_fp32_out         float32 y, backward products written as bfloat16 by the kernels (this change)
  step_bf16_out         y = linear(..., out_dtype=torch.bfloat16), grad_y bfloat16
Reported per arm: median and range over the rounds of the time per call, and TFLOP/s at the median (2MNK; a training step
counts 3 products).  The outputs of the BF16 arms are checked against the FP32 arms rounded by .to(torch.bfloat16), and the
ABFT counters are reported.  One JSON line on stdout (and in `out`), with the GPU name and its power limit.
"""
import json
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402
import __graft_entry__ as ge  # noqa: E402
from scripts.bf16_bench import summary, timed  # noqa: E402
from scripts.layout_bench import gpu_identity  # noqa: E402


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
    g = torch.Generator(device="cuda").manual_seed(17)
    gpu, power = gpu_identity()
    result = {"what": "BF16 results against FP32 results on BF16 operands, us per call", "gpu": gpu, "power_limit_w": power,
              "alpha": alpha, "beta": beta, "steps": steps, "rounds": rounds, "products": {}, "layers": {}, "training": {}}
    lay = {"MN": pkg.LAYOUT_MN_MAJOR, "K": pkg.LAYOUT_K_MAJOR}
    F32, BF16 = pkg.TYPE_F32, pkg.TYPE_BF16
    for n in sizes:
        A = torch.randn(n, n, device="cuda", generator=g).to(torch.bfloat16)
        B = torch.randn(n, n, device="cuda", generator=g).to(torch.bfloat16)
        ops = {("A", "MN"): A.t().contiguous(), ("A", "K"): A, ("B", "MN"): B.t().contiguous(), ("B", "K"): B}
        C16 = torch.randn(n * n, device="cuda", generator=g).to(torch.bfloat16)
        C32 = C16.float()
        D16, D32, cast = torch.empty_like(C16), torch.empty_like(C32), torch.empty_like(C16)

        def call(kid, la, lb, cd):
            C, D = (C16, D16) if cd == BF16 else (C32, D32)
            ft.run_batched_mixed(kid, n, n, n, ops[("A", la)], lay[la], n, 0, ops[("B", lb)], lay[lb], n, 0, BF16, C, n, 0, D,
                                 cd, 1, alpha, beta, opts=opts)

        def cublas():
            ft.run_batched_mixed(7, n, n, n, ops[("A", "K")], lay["K"], n, 0, ops[("B", "K")], lay["K"], n, 0, BF16, D16, n, 0,
                                 D16, BF16, 1, alpha, 0.0, opts=opts)

        arms = {}
        for la, lb in (("MN", "MN"), ("K", "K")):
            p = f"31_{la},{lb}"
            arms[p + "_bf16"] = (lambda la=la, lb=lb: call(31, la, lb, BF16))
            arms[p + "_fp32"] = (lambda la=la, lb=lb: call(31, la, lb, F32))
            arms[p + "_fp32_cast"] = (lambda la=la, lb=lb: (call(31, la, lb, F32), cast.copy_(D32)))
        arms["7_K,K_bf16"] = cublas
        ft.stats()
        row = summary(timed(arms, steps, rounds), 2.0 * n ** 3)
        row["detected"] = ft.stats()["detected"]
        same = True
        for la, lb in (("MN", "MN"), ("K", "K")):
            call(31, la, lb, BF16)
            call(31, la, lb, F32)
            torch.cuda.synchronize()
            same = same and torch.equal(D16.view(torch.int16), D32.to(torch.bfloat16).view(torch.int16))
        row["bf16_equals_fp32_rounded"] = same
        result["products"][str(n)] = row
        del A, B, ops, C16, C32, D16, D32, cast
        torch.cuda.empty_cache()
    for M, K, N in shapes:
        x = torch.randn(M, K, device="cuda", generator=g).to(torch.bfloat16)
        W = (torch.randn(N, K, device="cuda", generator=g) * K ** -0.5).to(torch.bfloat16)
        b = torch.randn(N, device="cuda", generator=g).to(torch.bfloat16)
        r = torch.randn(M, N, device="cuda", generator=g).to(torch.bfloat16)
        r32 = r.float()
        bf = torch.bfloat16
        arms = {"linear_bf16": lambda: ft.linear(x, W, b, out_dtype=bf), "linear_cast": lambda: ft.linear(x, W, b).to(bf),
                "torch_bf16": lambda: F.linear(x, W, b),
                "gelu_bf16": lambda: ft.linear(x, W, b, activation="gelu", out_dtype=bf),
                "gelu_cast": lambda: ft.linear(x, W, b, activation="gelu").to(bf),
                "torch_gelu": lambda: F.gelu(F.linear(x, W, b)),
                "residual_bf16": lambda: ft.linear(x, W, b, residual=r, out_dtype=bf),
                "residual_cast": lambda: ft.linear(x, W, b, residual=r32).to(bf),
                "torch_residual": lambda: F.linear(x, W, b) + r}
        ft.stats()
        row = summary(timed(arms, steps, rounds), 2.0 * M * N * K)
        row["detected"] = ft.stats()["detected"]
        checks = (("linear_bf16", "linear_cast"), ("gelu_bf16", "gelu_cast"), ("residual_bf16", "residual_cast"))
        row["bf16_equals_cast"] = all(torch.equal(arms[u]().view(torch.int16), arms[v]().view(torch.int16)) for u, v in checks)
        result["layers"][f"{M}x{K}x{N}"] = row
        # one training step of a BF16 linear
        xg, Wg = x.clone().requires_grad_(), W.clone().requires_grad_()
        gy16 = torch.randn(M, N, device="cuda", generator=g).to(bf)
        gy32 = gy16.float()

        def step_cast():  # the parent's backward: float32 products, then a cast
            y = ft.linear(x, W)
            g16 = gy32.to(bf)
            ft.matmul(g16, W).to(bf)
            ft.matmul(g16.t(), x).to(bf)
            return y

        def step_fp32_out():
            ft.linear(xg, Wg).backward(gy32)
            xg.grad = Wg.grad = None

        def step_bf16_out():
            ft.linear(xg, Wg, out_dtype=bf).backward(gy16)
            xg.grad = Wg.grad = None

        t_arms = {"step_fp32_out_cast": step_cast, "step_fp32_out": step_fp32_out, "step_bf16_out": step_bf16_out}
        result["training"][f"{M}x{K}x{N}"] = summary(timed(t_arms, max(steps // 2, 1), rounds), 6.0 * M * N * K)
        del x, W, b, r, r32, xg, Wg, gy16, gy32
        torch.cuda.empty_cache()
    ft.close()
    line = json.dumps(result)
    print(line)
    if "out" in kv:
        Path(kv["out"]).parent.mkdir(parents=True, exist_ok=True)
        Path(kv["out"]).write_text(line + "\n")


if __name__ == "__main__":
    main()
