"""CPU-only checks of the drop-in boundary: libftsgemm.so loads, exports every symbol include/ftsgemm.h declares,
the kernel-variant table mirrors the reference's id/name table, and -- without a GPU -- compute entry points fail
loudly instead of falling back to the CPU."""
import ctypes as C
import re
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parents[1]


def test_header_symbols_all_exported(ft):
    hdr = (ROOT / "include" / "ftsgemm.h").read_text()
    declared = set(re.findall(r"\b(ftsgemm_[a-z_0-9]+)\s*\(", hdr))
    declared -= {"ftsgemm_handle_s"}
    assert declared == set(ft.EXPORTED_SYMBOLS), declared ^ set(ft.EXPORTED_SYMBOLS)
    lib = C.CDLL(str(ft.LIB_PATH))
    for sym in declared:
        assert hasattr(lib, sym), sym
    assert lib.ftsgemm_abi_version() == 2


def test_header_cites_reference_interfaces():
    hdr = (ROOT / "include" / "ftsgemm.h").read_text()
    for cite in ("sgemm.cu:13-19", "ft_sgemm_huge.cuh:11", "sgemm.cu:235-237", "code_gen/main.py:8-16",
                 "baseline_ft_sgemm.cuh:1", "utils/utils.cu:61-77"):
        assert cite in hdr, cite


def test_kernel_table_matches_reference_ids(ft):
    tab = {k["id"]: k for k in ft.kernel_table()}
    # reference rows (sgemm.cu:235-237), verbatim ids and labels
    ref_rows = {0: "cublas", 1: "kernel_sgemm_small", 2: "kernel_sgemm_medium", 3: "kernel_sgemm_large",
                4: "kernel_sgemm_tall", 5: "kernel_sgemm_wide", 6: "kernel_sgemm_huge", 10: "abft_baseline",
                11: "abft_kernel_small", 12: "abft_kernel_medium", 13: "abft_kernel_large", 14: "abft_kernel_tall",
                15: "abft_kernel_wide", 16: "abft_kernel_huge"}
    for kid, name in ref_rows.items():
        assert tab[kid]["name"] == name
        assert tab[kid]["fault_tolerant"] == (kid >= 10)
    # reference tiles (code_gen/main.py:8-16)
    ref_tiles = {"small": (16, 16, 16), "medium": (32, 32, 8), "large": (64, 64, 8), "tall": (128, 32, 8),
                 "wide": (32, 128, 8), "huge": (128, 128, 8)}
    for nm, tile in ref_tiles.items():
        assert tab[ft.SGEMM_IDS[nm]]["ref_tile"] == tile and tab[ft.ABFT_IDS[nm]]["ref_tile"] == tile
        assert tab[ft.SGEMM_IDS[nm]]["tile"] == tab[ft.ABFT_IDS[nm]]["tile"]  # FT and non-FT share the tiling
    # config 2 of BASELINE.json: the huge tile is literally 128 x 128 with MMA K = 8 steps
    assert tab[16]["tile"][:2] == (128, 128) and tab[14]["tile"][:2] == (128, 32)
    # six names, six DISTINCT sm_90a tiles (round 1 aliased small = tall and large = huge)
    tiles = {nm: tab[ft.SGEMM_IDS[nm]]["tile"][:2] for nm in ref_tiles}
    assert len(set(tiles.values())) == 6, tiles
    assert tiles == {"small": (128, 64), "medium": (256, 64), "large": (256, 128), "tall": (128, 32), "wide": (128, 256),
                     "huge": (128, 128)}
    # legality of every wgmma tile: M = 128 (one CTA) or 256 (two CTAs), N % 16 == 0, 16 <= N <= 256
    for k in tab.values():
        if k["engine"] == 1 and k["id"] not in (ft.ID_SGEMM_AUTO, ft.ID_ABFT_AUTO):
            m, n, kk = k["tile"]
            assert m in (128, 256) and n % 16 == 0 and 16 <= n <= 256 and kk % 8 == 0
    # AUTO ids resolve per shape to a concrete variant of the right kind (no GPU needed)
    for (M, N) in ((1024, 1024), (2048, 2048), (4096, 4096), (256, 16384), (16384, 16384)):
        a, b = ft.select_kernel(M, N, 1024, False), ft.select_kernel(M, N, 1024, True)
        assert tab[a]["engine"] == 1 and not tab[a]["fault_tolerant"] and tab[b]["fault_tolerant"]
    assert ft.select_kernel(4096, 4096, 4096, True) == 31 and ft.select_kernel(1024, 1024, 1024, False) == 3
    assert ft.select_kernel(1536, 1536, 1536, True) == 31 and ft.select_kernel(1536, 1536, 1536, False) == 3


def test_opts_struct_layout(ft):
    o = ft.default_opts()
    assert o.struct_size == C.sizeof(ft.Opts)
    assert o.selftest_value == 10000.0 and o.inject_mode == 0 and o.baseline_host_sync == 1
    assert o.precision == 0 and o.no_recompute == 0 and o.check_segments == 0
    o = ft.make_opts(faults=[{"row": 1, "col": 2, "xor": 1 << 30}, {"row": 3, "col": 4, "add": 2.5}])
    assert o.inject_mode == 2 and o.n_faults == 2 and o.faults[0].xor_mask == 1 << 30 and o.faults[1].add_value == 2.5


def test_no_silent_cpu_fallback(ft):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(ft.FtsgemmError) as ei:
        ft.FtSgemm()
    assert ei.value.code == -4  # FTSGEMM_ERR_NO_DEVICE
    # the raw ABI refuses a NULL handle as well
    assert ft.lib().ftsgemm_run(None, 16, 128, 128, 128, None, None, None, 1.0, 0.0, None) == -4


def test_product_never_imports_oracle():
    """Only tests/, __graft_entry__.smoke() and bench.py's CPU legs may touch oracle/."""
    pkg = ROOT / "fault-tolerant-sgemm-on-nvidia-gpus_b200"
    for p in list(pkg.rglob("*.py")) + list(pkg.rglob("*.cu")) + list(pkg.rglob("*.cuh")) + [ROOT / "include" / "ftsgemm.h"]:
        assert "oracle" not in p.read_text(), p
