"""Build libtgis_engine.so in-tree with nvcc for sm_90a (H100) (no torch extension machinery, no JIT cache).

The .so lands in vllm_tgis_adapter_b200/lib/, next to the package, so the package imports from the source tree.
"""
from __future__ import annotations

import concurrent.futures
import hashlib
import os
import subprocess
import sys
from pathlib import Path

CSRC = Path(__file__).resolve().parent
PKG = CSRC.parent
LIB_DIR = PKG / "lib"
OBJ_DIR = CSRC / "build"
LIB_PATH = LIB_DIR / "libtgis_engine.so"
SOURCES = ["gemm_wgmma.cu", "gemm_ref.cu", "elementwise.cu", "attention.cu", "sampler.cu", "lora.cu", "opt.cu", "engine.cu", "test_api.cu"]
HEADERS = ["ptx.cuh", "launch.cuh", "gemm_sched.cuh", "kernels.h", "../../include/tgis_engine.h", "../../include/tgis_kernels.h"]
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = [
    *ARCH,
    "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC", "-Xcompiler", "-pthread",
    # bounded mbarrier spins: a pipeline-protocol bug traps (sticky CUDA error) instead of hanging the GPU
    "-DTGIS_MBAR_TIMEOUT=1",
]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if cand and (cand == "nvcc" or Path(cand).exists()):
            return cand
    raise RuntimeError("nvcc not found")


def have_nvcc() -> bool:
    try:
        n = _nvcc()
    except RuntimeError:
        return False
    if n == "nvcc":
        import shutil

        return shutil.which("nvcc") is not None
    return True


def _digest() -> str:
    h = hashlib.sha256()
    for name in SOURCES + HEADERS + ["build.py"]:
        h.update((CSRC / name).read_bytes())
    h.update(" ".join(NVCC_FLAGS).encode())
    h.update(os.environ.get("TGIS_EXTRA_NVCC_FLAGS", "").encode())
    return h.hexdigest()


def build(force: bool = False, verbose: bool = False) -> Path:
    LIB_DIR.mkdir(exist_ok=True)
    OBJ_DIR.mkdir(exist_ok=True)
    stamp = LIB_DIR / "libtgis_engine.stamp"
    digest = _digest()
    if not force and LIB_PATH.exists() and stamp.exists() and stamp.read_text() == digest:
        return LIB_PATH
    nvcc = _nvcc()
    extra = os.environ.get("TGIS_EXTRA_NVCC_FLAGS", "").split()

    def compile_one(src: str) -> Path:
        obj = OBJ_DIR / (src.replace(".cu", ".o"))
        cmd = [nvcc, *NVCC_FLAGS, *extra, "-c", str(CSRC / src), "-o", str(obj)]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed for {src}:\n{r.stdout}\n{r.stderr}")
        if verbose and r.stderr:
            print(r.stderr, file=sys.stderr)
        return obj

    with concurrent.futures.ThreadPoolExecutor(max_workers=min(8, len(SOURCES))) as ex:
        objs = list(ex.map(compile_one, SOURCES))
    link = [nvcc, "-shared", *ARCH, "-o", str(LIB_PATH), *map(str, objs),
            "-Xcompiler", "-pthread", "-cudart", "static", "-lrt", "-ldl"]
    r = subprocess.run(link, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    stamp.write_text(digest)
    return LIB_PATH


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
