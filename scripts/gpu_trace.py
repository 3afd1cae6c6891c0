"""Device timeline of the persistent kernel (ftsgemm_debug_trace): per-item main-loop / epilogue durations and stalls.

usage: gpu_trace.py [ID N [key=value ...]] ...   writes out/trace_<id>_<n>[_tag].json (summary + raw timeline)
"""
import json
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "scripts"))
import __graft_entry__ as ge  # noqa: E402
import cuda_rt as cu  # noqa: E402

OUT = ROOT / "out"
OUT.mkdir(exist_ok=True)


def stats(xs):
    if not xs:
        return None
    a = np.asarray(xs, dtype=np.float64) / 1e3
    return {"n": len(xs), "mean_us": round(float(a.mean()), 2), "min_us": round(float(a.min()), 2),
            "p50_us": round(float(np.median(a)), 2), "max_us": round(float(a.max()), 2)}


def trace_case(pkg, kid, n, dbg=None, tag="", reuse=False, m=None, k=None):
    m = m or n
    k = k or n
    rng = np.random.default_rng(0)
    A = (rng.integers(-9, 10, m * k) * 0.1).astype(np.float32)
    B = (rng.integers(-9, 10, n * k) * 0.1).astype(np.float32)
    dA, dB, dC = cu.DevBuf.from_numpy(A), cu.DevBuf.from_numpy(B), cu.DevBuf(4 * m * n)
    dC.zero()
    dbg = dict(dbg or {})
    big_tau = dbg.pop("bigtau", 0)
    for key, v in dbg.items():
        pkg.debug_set(key, v)
    ft = pkg.FtSgemm()
    opts = pkg.make_opts(reuse_b_checksums=1) if reuse else None
    if big_tau:
        opts = pkg.make_opts(tau_abs=1e30)
    for _ in range(3):
        ft.run(kid, m, n, k, dA, dB, dC, 1.0, 0.0, opts)
    cu.sync()
    pkg.debug_set("trace", 1)
    ft.run(kid, m, n, k, dA, dB, dC, 1.0, 0.0, opts)
    cu.sync()
    tr = ft.debug_trace()
    pkg.debug_set("trace", -1)
    for key in (dbg or {}):
        pkg.debug_set(key, -1)
    hdr, segs = pkg.debug_schedule(kid, m, n, k)
    n_chk = hdr["n_chk_tiles"]
    t0 = min(it["prod_start"] for u in tr for it in u if it["prod_start"])
    t_end = max(it["epi_end"] for u in tr for it in u)
    main = {"chk": [], "whole": [], "contrib": [], "finish": [], "enc_tile": []}
    epi = {"chk": [], "whole": [], "contrib": [], "finish": [], "enc_tile": []}
    chk_wait = []
    mma_gap, acc_lag = [], []
    unit_end = []
    for u in tr:
        prev_end = None
        for it in u:
            cls = "chk" if it["tile"] < n_chk else {0: "whole", 1: "contrib", 2: "finish", 3: "contrib", 5: "enc_tile", 6: "enc_tile"}[it["kind"]]
            main[cls].append(it["mma_end"] - it["mma_start"])
            epi[cls].append(it["epi_end"] - it["acc_done"])
            if cls in ("whole", "finish", "enc_tile") and it["check_done"]:
                chk_wait.append(it["check_done"] - it["acc_done"])
            acc_lag.append(it["acc_done"] - it["mma_end"])
            if prev_end is not None:
                mma_gap.append(it["mma_start"] - prev_end)
            prev_end = it["mma_end"]
        if u:
            unit_end.append(u[-1]["epi_end"] - t0)
    res = {"id": kid, "M": m, "N": n, "K": k, "tag": tag, "hdr": hdr, "span_us": round((t_end - t0) / 1e3, 2),
           "mainloop": {c: stats(v) for c, v in main.items()}, "epilogue": {c: stats(v) for c, v in epi.items()},
           "check_phase": stats(chk_wait), "mma_gap_between_items": stats(mma_gap), "acc_done_after_last_issue": stats(acc_lag),
           "unit_end_us": {"min": round(min(unit_end) / 1e3, 2), "p50": round(float(np.median(unit_end)) / 1e3, 2),
                           "max": round(max(unit_end) / 1e3, 2)},
           "first_data_epilogue_start_us": round(min(it["acc_done"] for u in tr for it in u if it["tile"] >= n_chk) / 1e3 - t0 / 1e3, 2),
           "encode_end_us": (lambda e: None if not e else {"min": round(min(e) / 1e3, 2), "max": round(max(e) / 1e3, 2)})(
               [u[0]["enc_end"] - t0 for u in tr if u and u[0].get("enc_end")]),
           "encode_dur_us": (lambda e: None if not e else {"min": round(min(e) / 1e3, 2), "max": round(max(e) / 1e3, 2),
                                                              "mean": round(sum(e) / len(e) / 1e3, 2)})(
               [u[0]["enc_end"] - u[0]["enc_start"] for u in tr if u and u[0].get("enc_end")]),
           "encode_all_done_after_first_start_us": (lambda a, b: None if not a else round((max(a) - min(b)) / 1e3, 2))(
               [u[0]["enc_end"] for u in tr if u and u[0].get("enc_end")], [u[0]["enc_start"] for u in tr if u and u[0].get("enc_start")]),
           "enc_worker0_wait_work_us_slots": [(round(u[0]["enc_worker0"][0] / 1e3, 1), round(u[0]["enc_worker0"][1] / 1e3, 1), u[0]["enc_worker0"][2])
                                              for u in tr if u and u[0].get("enc_worker0") and u[0]["enc_worker0"][2]][:6],
           "chk_items_end_us": [round((it["epi_end"] - t0) / 1e3, 1) for u in tr for it in u if it["tile"] < n_chk][:40]}
    raw = [[{kk: (vv - t0 if kk not in ("tile", "kind", "enc_worker0") and vv else vv) for kk, vv in it.items()} for it in u] for u in tr]
    name = f"trace_{kid}_{n}{('_' + tag) if tag else ''}.json"
    (OUT / name).write_text(json.dumps({"summary": res, "timeline_ns": raw}))
    print(json.dumps(res))
    return res


def main():
    pkg = ge.load_package()
    cases = []
    args = sys.argv[1:]
    if not args:
        cases = [(31, 4096, {}, ""), (21, 4096, {}, ""), (31, 8192, {}, ""), (21, 8192, {}, "")]
    else:
        i = 0
        while i < len(args):
            kid, n = int(args[i]), int(args[i + 1])
            i += 2
            dbg, tag = {}, ""
            while i < len(args) and "=" in args[i]:
                kk, vv = args[i].split("=")
                if kk == "tag":
                    tag = vv
                else:
                    dbg[kk] = int(vv)
                i += 1
            cases.append((kid, n, dbg, tag))
    for kid, n, dbg, tag in cases:
        trace_case(pkg, kid, n, dbg, tag)


if __name__ == "__main__":
    main()
