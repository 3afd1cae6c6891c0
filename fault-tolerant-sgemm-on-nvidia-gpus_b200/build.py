"""In-tree build of libftsgemm.so and the ft_sgemm driver for sm_90a (nvcc cross-compiles without a GPU)."""
from __future__ import annotations

import os
import subprocess
import sys
import tempfile
from pathlib import Path

HERE = Path(__file__).resolve().parent
CSRC = HERE / "csrc"
ROOT = HERE.parent
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
COMMON = ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC", "-ccbin", "/usr/bin/g++"]
# ptxas compiles the library's kernels on several threads: the same machine code as a serial run (SASS identical), in about
# half the build time.  The units compiled at the same time share one budget of threads, which bounds the build's memory
# (~1 GB per thread): 3 x min(8, CPUs) in all, what three units of 8 threads took before the fourth unit existed.
PTXAS_BUDGET = 3 * max(1, min(8, os.cpu_count() or 1))

LIB = HERE / "libftsgemm.so"
CLI = HERE / "ft_sgemm"


def _stale(target: Path, sources) -> bool:
    if not target.exists():
        return True
    t = target.stat().st_mtime
    return any(Path(s).stat().st_mtime > t for s in sources)


def build(force: bool = False, verbose: bool = False) -> None:
    # four translation units compiled at the same time (their device compilation is single-threaded up to ptxas): the
    # library, the OUT kernels of ftsgemm_run_batched_out (ftsgemm_out.cu), the BF16 kernels of ftsgemm_run_batched_typed
    # (ftsgemm_bf16.cu) and their BF16-output twins of ftsgemm_run_batched_mixed (ftsgemm_bf16_cd.cu); then one link
    lib_src = [CSRC / "ftsgemm.cu", CSRC / "ftsgemm_out.cu", CSRC / "ftsgemm_bf16.cu", CSRC / "ftsgemm_bf16_cd.cu"]
    lib_dep = lib_src + sorted(CSRC.glob("*.cuh")) + sorted(CSRC.glob("*.h")) + [ROOT / "include" / "ftsgemm.h"]
    if force or _stale(LIB, lib_dep):
        threads = ["-Xptxas", f"--split-compile={max(1, PTXAS_BUDGET // len(lib_src))}"]
        with tempfile.TemporaryDirectory() as tmp:
            objs = [Path(tmp) / (src.stem + ".o") for src in lib_src]
            # (each unit's output goes to files: a full pipe would stall a unit until the slowest one is read)
            logs = [(Path(tmp) / (src.stem + ".out"), Path(tmp) / (src.stem + ".err")) for src in lib_src]
            procs = []
            for src, obj, (lo, le) in zip(lib_src, objs, logs):
                with open(lo, "w") as fo, open(le, "w") as fe:
                    procs.append(subprocess.Popen([NVCC, *ARCH, *COMMON, *threads, "-c", "-Xptxas", "-v", str(src), "-o", str(obj)],
                                                  stdout=fo, stderr=fe))
            for p in procs:
                p.wait()
            outs = [(lo.read_text(), le.read_text()) for lo, le in logs]
            err = "".join(e for _, e in outs)
            rc = max(p.returncode for p in procs)
            if rc == 0:
                link = subprocess.run([NVCC, *ARCH, "-ccbin", "/usr/bin/g++", "-shared", *map(str, objs), "-o", str(LIB),
                                       "-lcublas"], capture_output=True, text=True)
                err += link.stderr
                rc = link.returncode
        (HERE / "build_ptxas.log").write_text(err)
        if verbose or rc != 0:
            print("".join(o for o, _ in outs), err, file=sys.stderr)
        if rc != 0:
            raise RuntimeError("nvcc failed building libftsgemm.so")
    cli_src = CSRC / "ft_sgemm_main.cu"
    if cli_src.exists() and (force or _stale(CLI, [cli_src, LIB])):
        cmd = [NVCC, *ARCH, "-O3", "-std=c++17", "-ccbin", "/usr/bin/g++", str(cli_src), "-o", str(CLI),
               f"-L{HERE}", "-lftsgemm", "-Xlinker", "-rpath", "-Xlinker", "$ORIGIN"]
        out = subprocess.run(cmd, capture_output=True, text=True)
        if verbose or out.returncode != 0:
            print(out.stdout, out.stderr, file=sys.stderr)
        if out.returncode != 0:
            raise RuntimeError("nvcc failed building ft_sgemm")


if __name__ == "__main__":
    build(force="--force" in sys.argv, verbose=True)
