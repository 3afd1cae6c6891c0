"""Host overhead a CUDA graph removes: an eager loop of fault-tolerant GEMM calls against replays of the same calls captured
once with torch.cuda.graph.

usage: graph_bench.py [steps=50] [rounds=7] [out=PATH]
Workloads:
  linear4   four FtSgemm.linear layers (bias fused), 256 tokens, 1024 -> 4096 -> 1024 -> 4096 -> 1024, forward only;
            tau_abs = 1e-2: the fault-free residuals of the K = 4096 layers reach a few 1e-3 on these unit-variance
            activations, above the default floor, and every row flagged by it would be recomputed on CUDA cores
  qk        attention scores of 128 heads through FtSgemm.bmm: q (128, 1024, 128) @ k^T, 1024 x 1024 x 128 per head
  run31     one ftsgemm_run_ex, id 31, 4096^3, the reference (MN-major) layout: the launch dominates, the arms should tie
Arms: eager (the calls themselves) and graph (one replay of the captured calls), both on one handle.  Per workload and round
the two arms run in an order that alternates from round to round: 3 warm-up steps, then CUDA events around `steps`
back-to-back steps.  Reported per arm: median and range over the rounds of the time per step, and the eager / graph ratio.
The outputs of the two arms are compared bit for bit.  One JSON line on stdout (and in `out`), with the GPU name and its
power limit.
"""
import json
import statistics
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
import torch  # noqa: E402
import __graft_entry__ as ge  # noqa: E402
from scripts.layout_bench import gpu_identity  # noqa: E402


def workloads(pkg, ft, g):
    """name -> (step(out) -> None, out for the eager arm, out for the graph arm)"""
    # linear4
    dims = [1024, 4096, 1024, 4096, 1024]
    x = torch.randn(256, dims[0], device="cuda", generator=g)
    ws = [torch.randn(dims[i + 1], dims[i], device="cuda", generator=g) * dims[i] ** -0.5 for i in range(4)]
    bs = [torch.randn(dims[i + 1], device="cuda", generator=g) for i in range(4)]

    lin_opts = pkg.make_opts(tau_abs=1e-2)

    def linear4(out):
        h = x
        for w, b in zip(ws, bs):
            h = ft.linear(h, w, b, opts=lin_opts)
        out.copy_(h)

    # qk
    q = torch.randn(128, 1024, 128, device="cuda", generator=g)
    k = torch.randn(128, 1024, 128, device="cuda", generator=g)

    def qk(out):
        ft.bmm(q, k.transpose(1, 2), out)

    # run31
    n = 4096
    A = torch.randn(n * n, device="cuda", generator=g)
    B = torch.randn(n * n, device="cuda", generator=g)

    def run31(out):
        ft.run_ex(31, n, n, n, A, pkg.LAYOUT_MN_MAJOR, n, B, pkg.LAYOUT_MN_MAJOR, n, out, n, 1.0, 0.0,
                  pkg.make_opts(stream=torch.cuda.current_stream().cuda_stream))

    def outs(*shape):
        return torch.empty(*shape, device="cuda"), torch.empty(*shape, device="cuda")

    return {"linear4": (linear4, *outs(256, dims[-1])), "qk": (qk, *outs(128, 1024, 1024)),
            "run31": (run31, *outs(n * n))}


def timed(fn, steps):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    time.sleep(0.02)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps * 1e3


def main():
    pkg = ge.load_package()
    kv = dict(a.split("=", 1) for a in sys.argv[1:])
    steps, rounds = int(kv.get("steps", 50)), int(kv.get("rounds", 7))
    ft = pkg.FtSgemm()
    g = torch.Generator(device="cuda").manual_seed(21)
    gpu, power = gpu_identity()
    result = {"what": "eager loop vs CUDA graph replay, us per step", "gpu": gpu, "power_limit_w": power, "steps": steps,
              "rounds": rounds, "workloads": {}}
    for name, (step, out_e, out_g) in workloads(pkg, ft, g).items():
        step(out_e)  # first call of the shape: plan and workspaces, outside the capture (graphs replay, they do not warm up)
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            step(out_g)
        arms = {"eager": lambda: step(out_e), "graph": graph.replay}
        us = {"eager": [], "graph": []}
        for r in range(rounds):
            for a in (("eager", "graph") if r % 2 == 0 else ("graph", "eager")):
                us[a].append(timed(arms[a], steps))
        row = {a: {"median_us": round(statistics.median(v), 1), "range_us": [round(min(v), 1), round(max(v), 1)]}
               for a, v in us.items()}
        row["eager_over_graph"] = round(row["eager"]["median_us"] / row["graph"]["median_us"], 3)
        row["bit_identical"] = bool(torch.equal(out_e, out_g))
        row["detected"] = ft.stats()["detected"]
        result["workloads"][name] = row
        del graph
    ft.close()
    line = json.dumps(result)
    print(line)
    if "out" in kv:
        Path(kv["out"]).parent.mkdir(parents=True, exist_ok=True)
        Path(kv["out"]).write_text(line + "\n")


if __name__ == "__main__":
    main()
