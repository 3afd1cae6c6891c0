"""Cost of the protected store pass: opts.protect_epilogue = 0 (unprotected), 1 (checked, judged per row segment) and 2
(every chunk verified before it is written, repairable with any beta).

usage: protect_repair_bench.py [ids=31,16] [sizes=2048,4096,8192] [linear=8188x4096x4096] [steps=20] [rounds=5] [out=PATH]
Square products run through run_ex (both operands MN-major) with alpha = 1, beta = -1.5; the old C is restored before each
arm's warm-up, outside the timed window.  The linear shape is tokens x in_features x out_features through
FtSgemm.linear(x, W, b) (id 40, row-major operands, fused bias, beta = 0); a token count that is not a multiple of the tile
width leaves a last tile column ragged in N, which only level 2 covers.  Per cell and round the three levels run in an order
that rotates from round to round: 3 warm-up calls, then CUDA events around `steps` back-to-back calls.  Reported per level:
median and range over the rounds of the time per call, TFLOP/s at the median, and the cost over level 0 in percent; the C of
levels 1 and 2 is bit-compared with level 0's and the store-pass alarms are counted (both must be 0 / true).  One JSON line
on stdout (and in `out`), with the GPU name and its power limit read in the same process.
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

LEVELS = (0, 1, 2)


def time_levels(ft, arms, reset, steps, rounds, flop):
    """arms: level -> call; reset() restores the inputs.  Returns the per-level summary."""
    us = {lv: [] for lv in arms}
    for r in range(rounds):
        for i in range(len(LEVELS)):
            lv = LEVELS[(i + r) % len(LEVELS)]
            reset()
            for _ in range(3):
                arms[lv]()
            torch.cuda.synchronize()
            time.sleep(0.02)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(steps):
                arms[lv]()
            e1.record()
            torch.cuda.synchronize()
            us[lv].append(e0.elapsed_time(e1) / steps * 1e3)
    row = {}
    for lv, v in us.items():
        med = statistics.median(v)
        row[f"level{lv}"] = {"median_us": round(med, 1), "range_us": [round(min(v), 1), round(max(v), 1)],
                             "tflops": round(flop / med * 1e-6, 1)}
    base = statistics.median(us[0])
    for lv in (1, 2):
        row[f"level{lv}_cost_pct"] = round(100.0 * (statistics.median(us[lv]) / base - 1.0), 2)
    return row


def main():
    pkg = ge.load_package()
    kv = dict(a.split("=", 1) for a in sys.argv[1:])
    ids = [int(v) for v in kv.get("ids", "31,16").split(",")]
    sizes = [int(v) for v in kv.get("sizes", "2048,4096,8192").split(",")]
    linear = [tuple(int(v) for v in s.split("x")) for s in kv.get("linear", "8188x4096x4096").split(",") if s]
    steps, rounds = int(kv.get("steps", 20)), int(kv.get("rounds", 5))
    ft = pkg.FtSgemm()
    g = torch.Generator(device="cuda").manual_seed(17)
    gpu, power = gpu_identity()
    if power is None:  # (no pynvml: ask nvidia-smi, read-only)
        try:
            import subprocess
            q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i",
                                str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
            gpu, power = (s.strip() for s in q.stdout.strip().split(","))
            power = float(power)
        except Exception:
            pass
    result = {"what": "protected store pass levels 0 / 1 / 2, us per call", "gpu": gpu, "power_limit_w": power,
              "beta": -1.5, "steps": steps, "rounds": rounds, "square": {}, "linear": {}}
    opts = {lv: pkg.make_opts(protect_epilogue=lv) for lv in LEVELS}
    for n in sizes:
        dA = torch.randn(n * n, device="cuda", generator=g)
        dB = torch.randn(n * n, device="cuda", generator=g)
        C0 = torch.randn(n * n, device="cuda", generator=g)
        dC = C0.clone()
        for kid in ids:
            def call(lv, out=dC):
                ft.run_ex(kid, n, n, n, dA, pkg.LAYOUT_MN_MAJOR, n, dB, pkg.LAYOUT_MN_MAJOR, n, out, n, 1.0, -1.5, opts[lv])
            ft.stats()
            outs = {}
            for lv in LEVELS:
                outs[lv] = C0.clone()
                call(lv, outs[lv])
            torch.cuda.synchronize()
            st = ft.stats()
            row = time_levels(ft, {lv: (lambda lv=lv: call(lv)) for lv in LEVELS}, lambda: dC.copy_(C0), steps, rounds,
                              2.0 * n ** 3)
            row["bit_identical"] = all(torch.equal(outs[0].view(torch.int32), outs[lv].view(torch.int32)) for lv in (1, 2))
            row["epilogue_faults"] = st["epilogue_faults"] + ft.stats()["epilogue_faults"]
            row["detected"] = st["detected"]
            result["square"][f"id{kid}_{n}"] = row
            del outs
        del dA, dB, C0, dC
        torch.cuda.empty_cache()
    for M, K, N in linear:
        x = torch.randn(M, K, device="cuda", generator=g)
        W = torch.randn(N, K, device="cuda", generator=g) * K ** -0.5
        b = torch.randn(N, device="cuda", generator=g)
        ft.stats()
        with torch.no_grad():
            outs = {lv: ft.linear(x, W, b, opts=opts[lv]) for lv in LEVELS}
            torch.cuda.synchronize()
            st = ft.stats()

            def lin(lv):
                ft.linear(x, W, b, opts=opts[lv])
            row = time_levels(ft, {lv: (lambda lv=lv: lin(lv)) for lv in LEVELS}, lambda: None, steps, rounds, 2.0 * M * N * K)
        row["bit_identical"] = all(torch.equal(outs[0].view(torch.int32), outs[lv].view(torch.int32)) for lv in (1, 2))
        row["epilogue_faults"] = st["epilogue_faults"] + ft.stats()["epilogue_faults"]
        row["detected"] = st["detected"]
        result["linear"][f"{M}x{K}x{N}"] = row
        del x, W, b, outs
        torch.cuda.empty_cache()
    ft.close()
    line = json.dumps(result)
    print(line)
    if "out" in kv:
        Path(kv["out"]).parent.mkdir(parents=True, exist_ok=True)
        Path(kv["out"]).write_text(line + "\n")


if __name__ == "__main__":
    main()
