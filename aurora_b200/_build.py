"""In-tree build of ``libaurora_b200.so`` (sm_90a only) with plain ``nvcc``.

The shared library lands next to the sources (``aurora_b200/csrc/libaurora_b200.so``) so that it
travels with a snapshot of the repository; objects go to ``build/`` (git-ignored).  Nothing here
imports torch: the library has a pure C ABI (``include/aurora_b200.h``).
"""

from __future__ import annotations

import concurrent.futures
import hashlib
import os
import shutil
import subprocess
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
CSRC = ROOT / "aurora_b200" / "csrc"
LIB_PATH = CSRC / "libaurora_b200.so"
OBJ_DIR = ROOT / "build" / "obj"

NVCC_FLAGS = [
    "-gencode",
    "arch=compute_90a,code=sm_90a",
    "-O3",
    "-std=c++17",
    "-lineinfo",
    "--expt-relaxed-constexpr",
    "-Xcompiler",
    "-fPIC",
]


def _nvcc() -> str:
    cand = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not Path(cand).exists():
        raise RuntimeError("nvcc not found; libaurora_b200.so cannot be built")
    return cand


def sources() -> list[Path]:
    return sorted(CSRC.glob("*.cu"))


HASH_PATH = CSRC / "libaurora_b200.srchash"  # git-ignored like the .so; travels with a snapshot


def _dep_files() -> list[Path]:
    files = list(CSRC.glob("*.cu")) + list(CSRC.glob("*.cuh")) + list(CSRC.glob("*.h"))
    files += list((ROOT / "include").glob("*.h"))
    return sorted(files)


def source_hash() -> str:
    """SHA-256 over every source / header the library is built from (and the compiler flags).  Content, not mtime:
    a snapshot copied to another machine keeps its library fresh whatever the copy did to the time stamps."""
    h = hashlib.sha256(" ".join(NVCC_FLAGS).encode())
    for f in _dep_files():
        h.update(f.name.encode())
        h.update(f.read_bytes())
    return h.hexdigest()


def is_stale() -> bool:
    if not LIB_PATH.exists() or not HASH_PATH.exists():
        return True
    return HASH_PATH.read_text().strip() != source_hash()


def build(force: bool = False, verbose: bool = False, ptxas_info: bool = False) -> Path:
    """Compile every ``csrc/*.cu`` for sm_90a and link ``libaurora_b200.so``."""
    if not force and not is_stale():
        return LIB_PATH
    nvcc = _nvcc()
    OBJ_DIR.mkdir(parents=True, exist_ok=True)
    digest = source_hash()
    headers_m = max(
        [f.stat().st_mtime for f in list(CSRC.glob("*.cuh")) + list(CSRC.glob("*.h"))]
        + [f.stat().st_mtime for f in (ROOT / "include").glob("*.h")]
    )

    def compile_one(src: Path) -> tuple[Path, str]:
        obj = OBJ_DIR / (src.stem + ".o")
        if not force and obj.exists() and obj.stat().st_mtime >= max(src.stat().st_mtime, headers_m):
            return obj, ""
        cmd = [nvcc, *NVCC_FLAGS, "-c", str(src), "-o", str(obj)]
        if ptxas_info:
            cmd[1:1] = ["-Xptxas", "-v"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed for {src.name}:\n{r.stdout}\n{r.stderr}")
        return obj, r.stderr

    workers = min(len(sources()), os.cpu_count() or 4)
    with concurrent.futures.ThreadPoolExecutor(max_workers=workers) as ex:
        results = list(ex.map(compile_one, sources()))
    if verbose or ptxas_info:
        for obj, log in results:
            if log.strip():
                print(f"--- {obj.name}\n{log}")
    objs = [str(o) for o, _ in results]
    tmp = LIB_PATH.with_suffix(".so.tmp")
    cmd = [nvcc, "-shared", *NVCC_FLAGS[:2], "-o", str(tmp), *objs]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    os.replace(tmp, LIB_PATH)
    HASH_PATH.write_text(digest + "\n")
    return LIB_PATH


if __name__ == "__main__":
    import sys

    p = build(force="--force" in sys.argv, verbose=True, ptxas_info="--ptxas" in sys.argv)
    print(p)
