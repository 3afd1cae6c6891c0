"""BASELINE.json config 4: single-bit fault injection into the FP32 accumulator tile of the fused
ABFT kernel, M=N=K=8192 by default; detection / location / correction rate per flipped bit position, plus the
run-time overhead of the always-on self-test.  Writes out/fault_campaign_<n>_id<k>.json.

usage: python scripts/fault_campaign.py [n=8192] [kernel_id=31] [trials_per_bit=6]
"""
import json
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
import torch  # noqa: E402
import __graft_entry__ as ge  # noqa: E402

pkg = ge.load_package()
n = int(sys.argv[1]) if len(sys.argv) > 1 else 8192
kid = int(sys.argv[2]) if len(sys.argv) > 2 else 31
trials = int(sys.argv[3]) if len(sys.argv) > 3 else 6
info = [k for k in pkg.kernel_table() if k["id"] == kid][0]
TM, TN = info["tile"][0], info["tile"][1]
torch.cuda.set_device(0)
g = torch.Generator(device="cuda").manual_seed(7)


def ref_dist(count):
    return (torch.randint(0, 10, (count,), generator=g, device="cuda").float() * 0.1) * \
           (torch.randint(0, 2, (count,), generator=g, device="cuda").float() * 2 - 1)


dA, dB = ref_dist(n * n), ref_dist(n * n)
clean = torch.zeros(n * n, device="cuda")
ft = pkg.FtSgemm()
ft.run(kid, n, n, n, dA, dB, clean, 1.0, 0.0, None)
torch.cuda.synchronize()
base_stats = ft.stats()
scale = float(clean.abs().max())
rng = np.random.default_rng(0)
out = {"n": n, "kernel": info["name"], "tile": [TM, TN], "fault_free": {k: base_stats[k] for k in
       ("tiles", "rows_checked", "detected", "max_abs_residual", "max_rel_residual")}, "bits": {}}
dC = torch.zeros(n * n, device="cuda")
for bit in range(31, -1, -1):
    inj = det = cor = unc = located = rec = 0
    worst_left = 0.0
    for _ in range(trials):
        faults, seen = [], set()
        while len(faults) < pkg.MAX_FAULTS:
            r, c = int(rng.integers(n)), int(rng.integers(n))
            key = (r, c // TN)
            if key in seen:
                continue
            seen.add(key)
            faults.append({"row": r, "col": c, "xor": 1 << bit})
        dC.zero_()
        ft.run(kid, n, n, n, dA, dB, dC, 1.0, 0.0, pkg.make_opts(faults=faults))
        torch.cuda.synchronize()
        st = ft.stats()
        inj += len(faults)
        det += st["detected"]
        cor += st["corrected"]
        unc += st["uncorrectable"]
        rec += st["recomputed"]
        want = {(f["row"], f["col"]) for f in faults}
        located += sum(1 for e in st["events"] if (e["row"], e["col"]) in want)
        worst_left = max(worst_left, float((dC - clean).abs().max()))
    out["bits"][str(bit)] = {"injected": inj, "detected": det, "corrected": cor, "recomputed": rec, "uncorrectable": unc,
                             "located_ok": located, "max_abs_error_left": worst_left,
                             "max_abs_error_left_over_maxC": worst_left / scale}
    print(bit, out["bits"][str(bit)], flush=True)

# overhead of fault handling itself: fault-free vs reference self-test (one upset in EVERY tile)
def timed(opts, reps=5):
    for _ in range(2):
        ft.run(kid, n, n, n, dA, dB, dC, 1.0, 0.0, opts)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(reps):
        ft.run(kid, n, n, n, dA, dB, dC, 1.0, 0.0, opts)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


t_clean = timed(None)
t_self = timed(pkg.make_opts(selftest=(10000.0, 17, 5)))
st = ft.stats()
out["timing_ms"] = {"fault_free": t_clean, "selftest_every_tile": t_self,
                    "selftest_overhead_pct": 100.0 * (t_self / t_clean - 1.0)}
out["maxC"] = scale
(ROOT / "out").mkdir(exist_ok=True)
p = ROOT / "out" / f"fault_campaign_{n}_id{kid}.json"
p.write_text(json.dumps(out, indent=1))
print("wrote", p)
