"""The ft_sgemm driver keeps the reference's argv and stdout contract (kernel/ft_sgemm/sgemm.cu:13-19, :100, :214, :223,
:227, :231, :239-243, :248, :435)."""
import re

import pytest


@pytest.mark.gpu
def test_cli_stdout_contract(cuda, ft):
    p = ft.run_cli([256, 512, 256, 0, 16], timeout=300)
    assert p.returncode == 0, p.stderr
    lines = p.stdout.splitlines()
    assert lines[0] == "Start verification!"
    ids = list(range(0, 17))
    body = lines[1:1 + 2 * len(ids)]
    for i, kid in enumerate(ids):
        assert body[2 * i] == "[Kernel Completed Successfully]"
        assert body[2 * i + 1] == f"kernel {kid} finish verified!"
    assert "failed to pass" not in p.stdout
    k = 1 + 2 * len(ids)
    assert lines[k] == "################## Performance (GFLOPS) ########################"
    assert lines[k + 1] == "Matrix Size         |" + "%8d|%8d|" % (256, 512)
    labels = ["cublas", "kernel_sgemm_small", "kernel_sgemm_medium", "kernel_sgemm_large", "kernel_sgemm_tall",
              "kernel_sgemm_wide", "kernel_sgemm_huge", "abft_baseline", "abft_kernel_small", "abft_kernel_medium",
              "abft_kernel_large", "abft_kernel_tall", "abft_kernel_wide", "abft_kernel_huge"]
    rows = lines[k + 2:k + 2 + len(labels)]
    for lab, row in zip(labels, rows):
        assert re.fullmatch(re.escape("%-20s|" % lab) + r"( *\d+\|){2}", row), row
    # every fused ABFT id corrected the reference's always-on self-test fault in every tile
    for kid in range(11, 17):
        m = re.search(rf"\[abft\] kernel {kid}: tiles (\d+) detected (\d+) corrected (\d+) uncorrectable 0", p.stderr)
        assert m and m.group(1) == m.group(2) == m.group(3), p.stderr


@pytest.mark.gpu
def test_cli_config1_single_size_and_cpu_verify(cuda, ft):
    """BASELINE.json config 1: `ft_sgemm 1024 1024 0 0 0` (GAP = 0 loops forever in the reference)."""
    p = ft.run_cli([1024, 1024, 0, 0, 0], timeout=300)
    assert p.returncode == 0
    assert p.stdout.splitlines()[-2] == "Matrix Size         |" + "%8d|" % 1024
    assert "[cpu-verify] kernel 0" in p.stderr and ": pass" in p.stderr


def test_cli_refuses_without_gpu(ft):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    p = ft.run_cli([64, 64, 0, 0, 0], timeout=60)
    assert p.returncode == 1 and "no sm_90 CUDA device" in p.stderr
