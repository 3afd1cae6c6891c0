"""Device timeline of the persistent kernel (ftsgemm_debug_trace): per-item main-loop / epilogue durations and stalls, and
the front phase (operand transposes + in-kernel encode of B) against the card's device-to-device copy bandwidth.

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


def copy_bandwidth(mib=256, reps=20):
    """Device-to-device copy of a `mib` MiB buffer (torch copy_, CUDA events): bytes read + written per second, and the
    card it ran on -- the roofline the front phase is judged against."""
    import subprocess

    import torch
    n = mib * 1024 * 1024 // 4
    src = torch.randn(n, device="cuda")
    dst = torch.empty_like(src)
    for _ in range(3):
        dst.copy_(src)
    times = []
    for _ in range(5):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            dst.copy_(src)
        e1.record()
        e1.synchronize()
        times.append(e0.elapsed_time(e1) / reps * 1e-3)
    t = float(np.median(times))
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    return {"bytes": 2 * 4 * n, "us": round(t * 1e6, 2), "tb_s": round(2 * 4 * n / t / 1e12, 3), "gpu": q}


def front_bytes(m, n, k, ft, bn):
    """HBM bytes of the front phase of the reference layout (dense leading dimensions) from the shapes: each operand read
    once and its K-major copy (row stride ldk = K rounded up to 4) written once; with the in-kernel encode (ABFT, B >= 8 MiB)
    B is read once more, unless the encode is fused with B's transpose (128- or 256-wide tiles, N a multiple of the tile:
    front_phase in csrc/ftsgemm_kernel.cuh).  The checksum operand it writes (16 bytes per N-tile and k) is not counted."""
    ldk = (k + 3) // 4 * 4
    b = 4 * m * (k + ldk) + 4 * n * (k + ldk)
    fused = bn in (128, 256) and n % bn == 0
    enc = 4 * n * k if ft and 4 * n * k >= 8 * 1048576 and not fused else 0
    return b, enc


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
    # front phase: earliest CTA start to the latest CTA end (every producer waits for the latest)
    spans = [f for u in tr if u for f in u[0].get("front", [])]
    front = None
    if spans:
        f0, f1 = min(s for s, _ in spans), max(e for _, e in spans)
        bn = next(v["tile"][1] for v in pkg.kernel_table() if v["id"] == kid)
        tr_bytes, enc_bytes = front_bytes(m, n, k, hdr["n_chk_tiles"] > 0, bn)
        front = {"span_us": round((f1 - f0) / 1e3, 2), "transpose_bytes": tr_bytes, "encode_bytes": enc_bytes,
                 "tb_s": round((tr_bytes + enc_bytes) / ((f1 - f0) * 1e-9) / 1e12, 3),
                 "cta_end_us": {"min": round((min(e for _, e in spans) - f0) / 1e3, 2), "max": round((f1 - f0) / 1e3, 2)},
                 "first_producer_after_front_us": round((t0 - f1) / 1e3, 2)}
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
           "front_phase": front,
           "chk_items_end_us": [round((it["epi_end"] - t0) / 1e3, 1) for u in tr for it in u if it["tile"] < n_chk][:40]}
    raw = [[{kk: (vv - t0 if kk not in ("tile", "kind", "front") and vv else vv) for kk, vv in it.items()} for it in u] for u in tr]
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
    print(json.dumps({"copy_bandwidth": copy_bandwidth()}))


if __name__ == "__main__":
    main()
