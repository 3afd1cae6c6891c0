"""Burst-regime comparison of debug-knob settings inside ONE process (same box, same clock state).

usage: knob_matrix.py sizes=2048,4096 id=31 steps=20 rounds=3 -- "splitk=0" "splitk=0,epi_assist=0" ...
Every setting is a comma-separated list of key=value debug knobs ("" = defaults); per size and round the settings (and
cuBLAS-TF32, id 7) are interleaved.  One JSON line per size: median us per launch per setting, overhead vs id 7, and whether
each setting's C (beta = 0) is bit-identical to the first setting's.
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


def main():
    pkg = ge.load_package()
    argv = sys.argv[1:]
    cut = argv.index("--") if "--" in argv else len(argv)
    kv = dict(a.split("=", 1) for a in argv[:cut])
    settings = argv[cut + 1:] or [""]
    sizes = [int(x) for x in kv.get("sizes", "4096").split(",")]
    kid, steps, rounds = int(kv.get("id", 31)), int(kv.get("steps", 20)), int(kv.get("rounds", 3))
    big = max(sizes)
    g = torch.Generator(device="cuda").manual_seed(7)

    def ref_dist(count):
        return (torch.randint(0, 10, (count,), generator=g, device="cuda").float() * 0.1) * \
               (torch.randint(0, 2, (count,), generator=g, device="cuda").float() * 2 - 1)
    dA, dB = ref_dist(big * big), ref_dist(big * big)
    dC = torch.zeros(big * big, device="cuda")
    ft = pkg.FtSgemm()
    opts = pkg.make_opts(stream=torch.cuda.current_stream().cuda_stream)

    def apply(s, on):
        for item in filter(None, s.split(",")):
            k, v = item.split("=")
            pkg.debug_set(k, int(v) if on else -1)  # (-1 erases the knob)

    def burst(k, n, beta):
        for _ in range(3):
            ft.run(k, n, n, n, dA, dB, dC, 1.0, beta, opts)
        torch.cuda.synchronize()
        time.sleep(0.05)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(steps):
            ft.run(k, n, n, n, dA, dB, dC, 1.0, beta, opts)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / steps * 1e3

    for n in sizes:
        us = {s: [] for s in settings}
        cub = []
        same = {}
        ref = None
        for s in settings:  # correctness first: beta = 0, one launch
            apply(s, True)
            dC[: n * n].zero_()
            ft.run(kid, n, n, n, dA, dB, dC, 1.0, 0.0, opts)
            torch.cuda.synchronize()
            apply(s, False)
            if ref is None:
                ref = dC[: n * n].clone()
            else:
                same[s] = bool(torch.equal(ref, dC[: n * n]))
        for _ in range(rounds):
            cub.append(burst(7, n, -1.5))
            for s in settings:
                apply(s, True)
                us[s].append(burst(kid, n, -1.5))
                apply(s, False)
        c = statistics.median(cub)
        med = {s: statistics.median(v) for s, v in us.items()}
        print(json.dumps({"n": n, "id": kid, "cublas_tf32_us": round(c, 2), "us": {s or "default": round(v, 2) for s, v in med.items()},
                          "overhead_pct": {s or "default": round(100.0 * (v / c - 1.0), 2) for s, v in med.items()},
                          "bit_identical_to_first": same}), flush=True)
    st = ft.stats()
    print(json.dumps({"stats": {k: st[k] for k in ("tiles", "rows_checked", "detected", "uncorrectable", "max_rel_residual")}}))


if __name__ == "__main__":
    main()
