"""Cost of the operand layouts: the same product with A and B MN-major (the reference's layout: the kernel's front phase
transposes both), K-major (x @ W.T: read in place, no transpose), and the two mixed cases.

usage: layout_bench.py [sizes=4096,8192] [ids=31,21,7] [steps=20] [rounds=5] [out=PATH]
Per size, id and round, the four layouts are timed in an order that rotates from round to round: 3 warm-up launches, then
CUDA events around `steps` back-to-back launches (alpha = 1, beta = -1.5, C reset before every burst).  Reported per layout:
median and range over the rounds of the time per launch, and TFLOP/s at the median.  For the tensor-core ids the C of every
layout is compared bit for bit with the reference layout's.  One JSON line on stdout (and in `out`), with the GPU name and
its power limit read the way bench.py reads them.
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

LAYOUTS = [("MN", "MN"), ("K", "K"), ("MN", "K"), ("K", "MN")]


def gpu_identity():
    name, limit = torch.cuda.get_device_name(0), None
    try:
        import pynvml
        pynvml.nvmlInit()
        h = pynvml.nvmlDeviceGetHandleByIndex(torch.cuda.current_device())
        nm = pynvml.nvmlDeviceGetName(h)
        name = nm.decode() if isinstance(nm, bytes) else str(nm)
        limit = pynvml.nvmlDeviceGetPowerManagementLimit(h) / 1000.0
    except Exception:
        pass
    return name, limit


def main():
    pkg = ge.load_package()
    kv = dict(a.split("=", 1) for a in sys.argv[1:])
    sizes = [int(x) for x in kv.get("sizes", "4096,8192").split(",")]
    ids = [int(x) for x in kv.get("ids", "31,21,7").split(",")]
    steps, rounds = int(kv.get("steps", 20)), int(kv.get("rounds", 5))
    alpha, beta = 1.0, -1.5
    ft = pkg.FtSgemm()
    opts = pkg.make_opts(stream=torch.cuda.current_stream().cuda_stream)
    g = torch.Generator(device="cuda").manual_seed(11)
    gpu, power = gpu_identity()
    result = {"what": "operand layouts, us per launch", "gpu": gpu, "power_limit_w": power, "alpha": alpha, "beta": beta,
              "steps": steps, "rounds": rounds, "sizes": {}}
    for n in sizes:
        A = torch.randn(n, n, device="cuda", generator=g)  # A[m, k]
        B = torch.randn(n, n, device="cuda", generator=g)  # B[n, k]
        # MN-major: element (r, k) at r + k*n, i.e. the row-major storage of the transpose; K-major: the row-major storage
        ops = {("A", "MN"): A.t().contiguous(), ("A", "K"): A, ("B", "MN"): B.t().contiguous(), ("B", "K"): B}
        C0 = torch.randn(n * n, device="cuda", generator=g)
        dC = torch.empty_like(C0)
        lay = {"MN": pkg.LAYOUT_MN_MAJOR, "K": pkg.LAYOUT_K_MAJOR}

        def launch(kid, la, lb):
            ft.run_ex(kid, n, n, n, ops[("A", la)], lay[la], n, ops[("B", lb)], lay[lb], n, dC, n, alpha, beta, opts)

        per_size = {}
        for kid in ids:
            us = {f"{la},{lb}": [] for la, lb in LAYOUTS}
            ft.stats()  # (resets the counters: "detected" below covers every launch of this id)
            for r in range(rounds):
                for i in range(len(LAYOUTS)):
                    la, lb = LAYOUTS[(i + r) % len(LAYOUTS)]
                    dC.copy_(C0)
                    for _ in range(3):
                        launch(kid, la, lb)
                    dC.copy_(C0)
                    torch.cuda.synchronize()
                    time.sleep(0.02)
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    for _ in range(steps):
                        launch(kid, la, lb)
                    e1.record()
                    torch.cuda.synchronize()
                    us[f"{la},{lb}"].append(e0.elapsed_time(e1) / steps * 1e3)
            row = {}
            for key, v in us.items():
                med = statistics.median(v)
                row[key] = {"median_us": round(med, 1), "range_us": [round(min(v), 1), round(max(v), 1)],
                            "tflops": round(2.0 * n ** 3 / med * 1e-6, 1)}
            if kid != 7:  # one launch per layout from the same C: bit-identical to the reference layout's
                outs = {}
                for la, lb in LAYOUTS:
                    dC.copy_(C0)
                    launch(kid, la, lb)
                    outs[(la, lb)] = dC.clone()
                torch.cuda.synchronize()
                row["bit_identical"] = all(torch.equal(outs[("MN", "MN")], o) for o in outs.values())
                st = ft.stats()
                row["detected"] = st["detected"]
            per_size[str(kid)] = row
        result["sizes"][str(n)] = per_size
        del A, B, ops, C0, dC
        torch.cuda.empty_cache()
    ft.close()
    line = json.dumps(result)
    print(line)
    if "out" in kv:
        Path(kv["out"]).parent.mkdir(parents=True, exist_ok=True)
        Path(kv["out"]).write_text(line + "\n")


if __name__ == "__main__":
    main()
