"""Build the in-tree native libraries (sm_90a only: H100).

    python -m flowgger_b200.build [--force]

Produces, under flowgger_b200/lib/:
  libflowgger_cuda.so   the C-ABI decoder (CUDA kernels + host pipeline), include/flowgger_cuda.h
  libflowgger_host.so   C++ mirror of the reference's Decoder/Record/Splitter interface on top of the C ABI
  libfg_gen.so          synthetic log generators for tests and bench (not product code)
The oracle (oracle/liboracle.so) is test infrastructure and is built by its own Makefile.
"""
from __future__ import annotations

import os
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent
REPO = ROOT.parent
CSRC = ROOT / "csrc"
LIB = ROOT / "lib"

NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC,-Wall,-O3",
    "--fmad=false",          # keep IEEE double semantics explicit (timestamp recipe)
    "-Xptxas", "-v",
]
CXX = os.environ.get("CXX", "g++")
CXX_FLAGS = ["-O3", "-std=c++17", "-fPIC", "-Wall", "-Wextra", "-pthread", "-march=x86-64-v3"]


def _newer(target: Path, sources: list[Path]) -> bool:
    if not target.exists():
        return True
    t = target.stat().st_mtime
    return any(s.stat().st_mtime > t for s in sources)


def _build(target: Path, sources: list[Path], cmd: list[str], force: bool) -> None:
    """Run `cmd` when `target` is missing, older than a source, or was built by another command line (a change of
    NVCC_FLAGS, e.g. the architecture, rebuilds even when no source changed).  The command line is kept next to the
    target in `<target>.cmd`."""
    stamp = target.with_name(target.name + ".cmd")
    line = " ".join(cmd).replace(str(REPO), ".")  # a moved or copied tree keeps its build
    if force or _newer(target, sources) or not stamp.exists() or stamp.read_text() != line:
        _run(cmd)
        stamp.write_text(line)


def _run(cmd: list[str]) -> None:
    print("+", " ".join(cmd), flush=True)
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    out = r.stdout
    if r.returncode != 0:
        sys.stdout.write(out)
        raise RuntimeError(f"build step failed: {' '.join(cmd)}")
    # keep the ptxas resource lines: they are the first thing to read before GPU time
    for line in out.splitlines():
        if "registers" in line or "spill" in line or "error" in line.lower():
            print("   ", line.strip())


def build_cuda(force: bool = False) -> Path:
    LIB.mkdir(exist_ok=True)
    target = LIB / "libflowgger_cuda.so"
    srcs = sorted(CSRC.glob("*.cu")) + sorted(CSRC.glob("*.cuh")) + sorted(CSRC.glob("*.h")) + [
        REPO / "include" / "flowgger_cuda.h"]
    cus = [str(p) for p in sorted(CSRC.glob("*.cu"))]
    _build(target, srcs, [NVCC, *NVCC_FLAGS, "-shared", "-o", str(target), *cus, "-I", str(REPO / "include")], force)
    return target


def build_host(force: bool = False) -> Path | None:
    hdir = CSRC / "host"
    if not hdir.exists():
        return None
    target = LIB / "libflowgger_host.so"
    srcs = sorted(hdir.glob("*.cpp")) + sorted(hdir.glob("*.hpp")) + [REPO / "include" / "flowgger_cuda.h"]
    _build(target, srcs, [CXX, *CXX_FLAGS, "-shared", "-o", str(target), *[str(p) for p in sorted(hdir.glob("*.cpp"))],
                          "-I", str(REPO / "include"), f"-L{LIB}", "-lflowgger_cuda", "-Wl,-rpath,$ORIGIN"], force)
    return target


def build_gen(force: bool = False) -> Path | None:
    gdir = CSRC / "gen"
    if not gdir.exists():
        return None
    target = LIB / "libfg_gen.so"
    srcs = sorted(gdir.glob("*.cpp")) + sorted(gdir.glob("*.hpp"))
    _build(target, srcs, [CXX, *CXX_FLAGS, "-shared", "-o", str(target), *[str(p) for p in sorted(gdir.glob("*.cpp"))]], force)
    return target


def build_oracle(force: bool = False) -> Path:
    odir = REPO / "oracle"
    target = odir / "liboracle.so"
    srcs = [odir / "oracle.cpp", odir / "capi.cpp", odir / "encoder.cpp", odir / "rfc3164.cpp", odir / "oracle.hpp"]
    if force or _newer(target, srcs):
        _run(["make", "-C", str(odir), "-B" if force else "-s", "liboracle.so"])
    return target


def build_all(force: bool = False) -> None:
    build_cuda(force)
    build_host(force)
    build_gen(force)
    build_oracle(force)


if __name__ == "__main__":
    build_all("--force" in sys.argv)
    print("ok")
