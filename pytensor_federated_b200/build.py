"""In-tree build of the native library (``libb200fed.so``) for sm_90a.

No torch headers and no pybind: the library is plain CUDA runtime + a C ABI, loaded with
``ctypes`` (see :mod:`pytensor_federated_b200.ops.native`).  That keeps a full rebuild at a
few seconds and lets the ``.so`` travel to the GPU box with the repository snapshot.
"""
from __future__ import annotations

import hashlib
import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path
from typing import List, Optional

PKG = Path(__file__).resolve().parent
CSRC = PKG / "csrc"
BUILD = CSRC / "build"
LIB = PKG / "libb200fed.so"

SOURCES = ["runtime.cu", "linreg.cu", "glm_simt.cu", "glm_tc.cu", "glm_fp8.cu", "glm_generic.cu", "ode.cu", "ode_generic.cu", "codec.cu"]
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr"]


def nvcc_path() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found (set NVCC=/path/to/nvcc)")


def _cudart_dir() -> Optional[str]:
    try:
        import nvidia.cuda_runtime as rt  # wheel that torch depends on

        cand = Path(list(rt.__path__)[0]) / "lib"
        return str(cand) if (cand / "libcudart.so.12").exists() else None
    except Exception:
        return None


def _digest(paths: List[Path]) -> str:
    h = hashlib.sha256()
    for p in sorted(paths):
        h.update(p.name.encode())
        h.update(p.read_bytes())
    h.update(" ".join(ARCH + NVCC_FLAGS).encode())
    return h.hexdigest()


def source_digest() -> str:
    return _digest([p for p in CSRC.iterdir() if p.suffix in (".cu", ".cuh", ".h")])


def is_current() -> bool:
    stamp = BUILD / "stamp.txt"
    return LIB.exists() and stamp.exists() and stamp.read_text().strip() == source_digest()


def build(force: bool = False, verbose: bool = False, ptxas_info: bool = False) -> Path:
    """Compiles every ``.cu`` under ``csrc/`` for sm_90a and links ``libb200fed.so``."""
    if not force and is_current():
        return LIB
    nvcc = nvcc_path()
    BUILD.mkdir(parents=True, exist_ok=True)
    flags = list(NVCC_FLAGS) + (["-Xptxas", "-v"] if ptxas_info else [])

    def compile_one(src: str) -> Path:
        obj = BUILD / (Path(src).stem + ".o")
        cmd = [nvcc, *ARCH, *flags, "-I", str(CSRC), "-c", str(CSRC / src), "-o", str(obj)]
        res = subprocess.run(cmd, capture_output=True, text=True)
        if verbose or ptxas_info or res.returncode != 0:
            sys.stderr.write(" ".join(cmd) + "\n" + res.stdout + res.stderr)
        if res.returncode != 0:
            raise RuntimeError(f"nvcc failed for {src}")
        return obj

    with ThreadPoolExecutor(max_workers=min(8, len(SOURCES))) as pool:
        objs = list(pool.map(compile_one, SOURCES))
    link = [nvcc, *ARCH, "-shared", "-o", str(LIB), *map(str, objs), "-lcudart"]
    rt = _cudart_dir()
    if rt:  # same libcudart.so.12 that torch loads; resolvable even without LD_LIBRARY_PATH
        link += ["-L", rt, "-Xlinker", f"-rpath={rt}"]
    res = subprocess.run(link, capture_output=True, text=True)
    if res.returncode != 0:
        sys.stderr.write(res.stdout + res.stderr)
        raise RuntimeError("link failed")
    (BUILD / "stamp.txt").write_text(source_digest())
    return LIB


def dump_sass(out_dir: Optional[Path] = None) -> Path:
    """Writes ``cuobjdump -sass`` of the library (HGMMA / UTMALDG / multimem instructions) to ``out_dir``."""
    out_dir = Path(out_dir or BUILD)
    out_dir.mkdir(parents=True, exist_ok=True)
    out = out_dir / "libb200fed.sass"
    res = subprocess.run(["cuobjdump", "-sass", str(LIB)], capture_output=True, text=True, check=True)
    out.write_text(res.stdout)
    return out


if __name__ == "__main__":
    path = build(force="--force" in sys.argv, verbose="-v" in sys.argv, ptxas_info="--ptxas" in sys.argv)
    print(path)
