"""In-tree build of the native runtime (``adapcc_b200/_C/libadapcc.so``).

The reference builds ``communicator.so`` with a bare ``nvcc -shared`` and no arch flags. Here
every translation unit is compiled for sm_90a (H100: wgmma, TMA, clusters, setmaxnreg need the
arch-specific target) with -lineinfo so profilers map kernels to our source, and linked into ONE
shared object that Python loads with ctypes (and that exports the reference's six C symbols).

Usage: ``python -m adapcc_b200.build [--force] [--verbose]``
"""
from __future__ import annotations

import hashlib
import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

PKG = Path(__file__).resolve().parent
CSRC = PKG / "csrc"
OUT_DIR = PKG / "_C"
BUILD_DIR = PKG / "_C" / "obj"
LIB = OUT_DIR / "libadapcc.so"

GENCODE = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr",
              "-Xptxas", "-v"]
CXX_FLAGS = ["-O2", "-std=c++17", "-fPIC"]


def _nvcc() -> str:
    cand = os.environ.get("NVCC") or shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not Path(cand).exists():
        raise RuntimeError("nvcc not found; set NVCC or add /usr/local/cuda/bin to PATH")
    return cand


def sources() -> list[Path]:
    return sorted(list(CSRC.glob("*.cu")) + list(CSRC.glob("*.cpp")))


def tool_sources() -> list[Path]:
    """Stand-alone binaries (csrc/bin/*.cu -> _C/<name>), e.g. ``check_p2p``."""
    return sorted((CSRC / "bin").glob("*.cu"))


def _build_tool(src: Path) -> str:
    out = OUT_DIR / src.stem
    tmp = OUT_DIR / (src.stem + ".tmp")
    cmd = [_nvcc(), *GENCODE, "-O3", "-std=c++17", "-lineinfo", "-I", str(CSRC), str(src), "-o", str(tmp),
           "-cudart", "static", "-ldl", "-lpthread"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"tool build failed: {src.name}\n$ {' '.join(cmd)}\n{r.stdout}{r.stderr}")
    os.replace(tmp, out)
    return f"$ {' '.join(cmd)}\n{r.stdout}{r.stderr}"


def _digest(paths: list[Path]) -> str:
    h = hashlib.sha256()
    for p in sorted(paths):
        h.update(p.name.encode())
        h.update(p.read_bytes())
    h.update(" ".join(GENCODE + NVCC_FLAGS + CXX_FLAGS).encode())
    return h.hexdigest()


def _compile(src: Path, verbose: bool) -> tuple[Path, str]:
    obj = BUILD_DIR / (src.name + ".o")
    nvcc = _nvcc()
    if src.suffix == ".cu":
        cmd = [nvcc, *GENCODE, *NVCC_FLAGS, "-I", str(CSRC), "-c", str(src), "-o", str(obj)]
    else:
        cmd = [nvcc, "-O2", "-std=c++17", "-Xcompiler", "-fPIC", "-I", str(CSRC), "-x", "cu",
               *GENCODE, "-c", str(src), "-o", str(obj)]
    r = subprocess.run(cmd, capture_output=True, text=True)
    log = f"$ {' '.join(cmd)}\n{r.stdout}{r.stderr}"
    if r.returncode != 0:
        raise RuntimeError(f"compile failed: {src.name}\n{log}")
    if verbose:
        print(log)
    return obj, log


def build(force: bool = False, verbose: bool = False) -> Path:
    """Compile (if stale) and return the path of libadapcc.so."""
    srcs = sources()
    hdrs = list(CSRC.glob("*.h")) + list(CSRC.glob("*.cuh"))
    stamp = OUT_DIR / "build.stamp"
    tools = tool_sources()
    want = _digest(srcs + hdrs + tools)
    have_tools = all((OUT_DIR / t.stem).exists() for t in tools)
    if not force and LIB.exists() and have_tools and stamp.exists() and stamp.read_text().strip() == want:
        return LIB
    BUILD_DIR.mkdir(parents=True, exist_ok=True)
    with ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
        tool_logs = [ex.submit(_build_tool, t) for t in tools]
        results = list(ex.map(lambda s: _compile(s, verbose), srcs))
        tool_logs = [f.result() for f in tool_logs]
    objs = [str(o) for o, _ in results]
    (OUT_DIR / "build.log").write_text("\n".join([log for _, log in results] + tool_logs))
    tmp = LIB.with_suffix(".so.tmp")                 # link aside, then rename: a reader (or a snapshot of the
    cmd = [_nvcc(), "-shared", *GENCODE, "-o", str(tmp), *objs, "-cudart", "static", "-ldl", "-lpthread"]
    r = subprocess.run(cmd, capture_output=True, text=True)   # tree) never sees a half-written library
    if r.returncode != 0:
        raise RuntimeError(f"link failed\n$ {' '.join(cmd)}\n{r.stdout}{r.stderr}")
    os.replace(tmp, LIB)
    stamp.write_text(want)
    return LIB


if __name__ == "__main__":
    p = build(force="--force" in sys.argv, verbose="--verbose" in sys.argv)
    print(p)
