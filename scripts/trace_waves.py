"""Per-wave main-loop times from a device timeline (out/trace_<id>_<n>.json): does the tile time grow with the wave?"""
import json, sys
import numpy as np
for path in sys.argv[1:]:
    d = json.load(open(path))
    tl = d["timeline_ns"]
    by_wave = {}
    starts = {}
    for u in tl:
        w = 0
        for it in u:
            if it["kind"] == 0 and it["mma_end"]:
                by_wave.setdefault(w, []).append((it["mma_end"] - it["mma_start"]) / 1e3)
                starts.setdefault(w, []).append(it["mma_start"] / 1e3)
                w += 1
    print(path, d["summary"]["span_us"])
    for w in sorted(by_wave):
        a = np.array(by_wave[w]); s = np.array(starts[w])
        if w % 4 == 0 or w == max(by_wave):
            print(f"  wave {w:3d}: n={len(a):3d} mainloop mean {a.mean():7.1f} min {a.min():7.1f} max {a.max():7.1f} us; start spread {s.max()-s.min():8.1f} us")
