"""CPU checks of the kernel's work decomposition (cut tiles computed as seeded chains + whole tiles + checksum
tile-columns), using the host-side enumeration of the SAME inline code the device runs (ftsgemm_debug_schedule):
  * every (tile, k-block) is computed exactly once, the pieces of a cut tile are contiguous and ordered first/middle/last;
  * every unit's list follows the global order [early first pieces][checksum][whole][late first pieces][2nd pieces]...;
  * no circular wait: with in-order roles, one accumulator per unit, a piece's main loop waiting for the
    previous piece's parked accumulator and ABFT data tiles waiting for their checksum tile-columns in the epilogue,
    every item completes."""
import itertools

import pytest

TILE_N = {1: 64, 2: 64, 3: 128, 4: 32, 6: 128, 5: 256, 21: 256, 22: 128, 11: 64, 12: 64, 13: 128, 14: 32, 16: 128, 15: 256, 31: 256,
          32: 128}
PAIR_IDS = (2, 3, 12, 13, 21, 22, 31, 32)  # 256-row tiles (two CTAs per work unit)


def _simulate(hdr, segs, acc_stages):
    units = hdr["units"]
    per_unit = [[] for _ in range(units)]
    for s in segs:
        per_unit[s["unit"]].append(s)
    tiles_c = 0
    chk_done = {}     # (m_blk, c) -> bool
    piece_at = {}     # (tile, piece) -> (unit, idx)
    for u, lst in enumerate(per_unit):
        for i, s in enumerate(lst):
            if s["is_chk"]:
                chk_done[(s["m_blk"], s["n_blk"], s["slice"])] = False
                tiles_c = max(tiles_c, s["n_blk"] + 1)
            if s["kind"] in (1, 2, 3):
                piece_at[(s["tile"], s["slice"])] = (u, i)
    mma_done = [0] * units   # number of items whose main loop finished
    epi_done = [0] * units
    done_epi = set()         # (unit, idx)
    progress = True
    while progress:
        progress = False
        for u, lst in enumerate(per_unit):
            # the main loop of item i needs the accumulator stage of item i - acc_stages drained and, for a seeded piece,
            # the previous piece parked (its epilogue done)
            while mma_done[u] < len(lst) and mma_done[u] - epi_done[u] < acc_stages:
                s = lst[mma_done[u]]
                if s["kind"] in (2, 3) and piece_at[(s["tile"], s["slice"] - 1)] not in done_epi:
                    break
                mma_done[u] += 1
                progress = True
            while epi_done[u] < mma_done[u]:
                i = epi_done[u]
                s = lst[i]
                ok = True
                if hdr["n_chk_tiles"] and not s["is_chk"] and s["kind"] in (0, 2):  # parking pieces are not checked
                    ok = all(chk_done[(s["m_blk"], c, sl)] for c in range(tiles_c) for sl in range(max(1, hdr.get("chk_slices", 1))))
                if not ok:
                    break
                epi_done[u] += 1
                done_epi.add((u, i))
                if s["is_chk"]:
                    chk_done[(s["m_blk"], s["n_blk"], s["slice"])] = True
                progress = True
    return all(epi_done[u] == len(per_unit[u]) for u in range(units))


@pytest.mark.parametrize("kid", [1, 4, 6, 5, 21, 22, 12, 13, 14, 16, 15, 31, 32])
@pytest.mark.parametrize("shape", [(4096, 4096, 4096), (2048, 2048, 2048), (1024, 1024, 1024), (8192, 8192, 512),
                                   (1536, 2560, 1000), (256, 256, 64), (128, 4096, 32), (5120, 384, 4096),
                                   (16384, 16384, 1024), (32768, 1024, 256)])
@pytest.mark.parametrize("num_sms", [148, 132, 16, 6])
def test_decomposition_covers_and_cannot_deadlock(ft, kid, shape, num_sms):
    M, N, K = shape
    hdr, segs = ft.debug_schedule(kid, M, N, K, num_sms)
    units, num_kb, H, S = hdr["units"], hdr["num_kb"], hdr["sk_tiles"], hdr["sk_slices"]
    assert hdr["num_kb"] == -(-K // 32)
    first_cut = hdr["num_tiles"] - H
    cover = {}
    for s in segs:
        assert 0 <= s["kb_begin"] < s["kb_end"] <= num_kb
        assert s["kind"] in (0, 1, 2, 3, 6)
        cover.setdefault(s["tile"], []).append((s["kb_begin"], s["kb_end"], s["kind"], s["slice"]))
        if s["kind"] in (1, 2, 3):
            assert not s["is_chk"]
    assert sorted(cover) == list(range(hdr["num_tiles"]))
    S_chk = max(1, hdr["chk_slices"])
    for t, pieces in cover.items():
        pieces.sort()
        if t < hdr["n_chk_tiles"] and S_chk > 1:  # a K-slice of a checksum tile: one item over its own k range
            sl = t // (hdr["n_chk_tiles"] // S_chk)
            assert pieces == [(num_kb * sl // S_chk, num_kb * (sl + 1) // S_chk, 0, sl)], (t, pieces)
            continue
        assert pieces[0][0] == 0 and pieces[-1][1] == num_kb
        for a, b in zip(pieces, pieces[1:]):
            assert a[1] == b[0]  # contiguous, no overlap
        if len(pieces) == 1:
            assert pieces[0][2] in (0, 6)
        else:
            assert 2 <= len(pieces) <= S
            assert [p[2] for p in pieces] == [1] + [3] * (len(pieces) - 2) + [2]
            assert [p[3] for p in pieces] == list(range(len(pieces)))
            assert all(p[1] - p[0] >= 4 for p in pieces)
    # global item order: [early first pieces][checksum tiles][whole tiles][late first pieces][2nd pieces]...;
    # every unit's list follows it (regular expression P* C* W* P* then later pieces by piece index), checksum and whole
    # tiles in raster order; the circular-wait simulation below is the actual safety check
    import re
    per_unit = {}
    for s_ in segs:
        per_unit.setdefault(s_["unit"], []).append(s_)
    for lst in per_unit.values():
        word = "".join("C" if s_["is_chk"] else "WPFM"[s_["kind"]] for s_ in lst)
        assert re.fullmatch(r"P*C*W*P*[FM]*", word), word
        later = [s_["slice"] for s_ in lst if s_["kind"] in (2, 3)]
        assert later == sorted(later)
        for cls in ("C", "W"):
            tiles = [s_["tile"] for s_, ch in zip(lst, word) if ch == cls]
            assert tiles == sorted(tiles)
        for s_ in lst:
            if s_["is_chk"]:
                assert s_["tile"] < hdr["n_chk_tiles"]
    # checksum tiles: n_chk_tiles of them, 8 columns per N-tile
    chk = {(s["m_blk"], s["n_blk"], s["slice"]) for s in segs if s["is_chk"]}
    assert len(chk) == hdr["n_chk_tiles"]
    assert all(s_["kind"] in (0, 1, 2, 3) for s_ in segs)
    if kid in (11, 12, 13, 14, 16, 15, 31, 32):
        tiles_n = -(-N // TILE_N[kid])
        assert hdr["n_chk_tiles"] == -(-M // (128 * hdr["cta_group"])) * -(-(tiles_n * 4) // TILE_N[kid]) * S_chk
        if S_chk > 1:  # slices only where every data tile and every slice get a unit of their own
            assert hdr["num_tiles"] <= units and num_kb // S_chk >= 8
    acc_stages = 1  # the next main loop of a unit starts once the previous epilogue has freed the ring
    assert _simulate(hdr, segs, acc_stages), "circular wait in the schedule"


def test_planner_levels_the_units(ft):
    """The list scheduler + cut tiles remove the wave-quantisation loss where that pays."""
    def makespan(kid, n):
        hdr, segs = ft.debug_schedule(kid, n, n, n, 132)
        work = [0.0] * hdr["units"]
        for s in segs:
            work[s["unit"]] += (0.58 if s["is_chk"] else 1.25 if s["kind"] == 6 else 1.0) * (s["kb_end"] - s["kb_begin"]) / hdr["num_kb"]
        return hdr, max(work), sum(work) / hdr["units"]
    hdr, t, ideal = makespan(21, 3072)   # 144 tiles on 66 units: 2.18 waves -> 3 waves uncut
    assert hdr["sk_tiles"] > 0 and hdr["sk_slices"] == 2 and t <= 2.5
    hdr, t, ideal = makespan(21, 1024)   # 16 tiles on 66 units: nothing to level
    assert hdr["sk_tiles"] == 0 and t == 1.0
    hdr, t, ideal = makespan(31, 4096)   # ABFT tiles are cut as well (seeded chains keep the checksum algebra exact); the
    assert hdr["sk_tiles"] > 0 and hdr["n_chk_tiles"] == 16 and t <= ideal * 1.05  # checksum product: one item per tile-row
    hdr, t, ideal = makespan(31, 8192)
    assert hdr["n_chk_tiles"] == 32 and t <= ideal * 1.03
