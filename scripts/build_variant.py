"""Build an alternative libtgis_engine_<name>.so from the same sources with extra nvcc flags (A/B experiments, debug
timeline builds):  python scripts/build_variant.py stl -DTGIS_STEP_TIMELINE     -> lib/libtgis_engine_stl.so
Use it with TGIS_ENGINE_LIB=<path>."""
import concurrent.futures
import subprocess
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from vllm_tgis_adapter_b200.csrc import build as b  # noqa: E402

name, extra = sys.argv[1], sys.argv[2:]
lib = b.LIB_DIR / f"libtgis_engine_{name}.so"
objdir = b.CSRC / f"build_{name}"
objdir.mkdir(exist_ok=True)
nvcc = b._nvcc()


def one(src: str) -> Path:
    obj = objdir / src.replace(".cu", ".o")
    r = subprocess.run([nvcc, *b.NVCC_FLAGS, *extra, "-c", str(b.CSRC / src), "-o", str(obj)], capture_output=True, text=True)
    if r.returncode != 0:
        raise SystemExit(f"nvcc failed for {src}:\n{r.stderr}")
    return obj


with concurrent.futures.ThreadPoolExecutor(8) as ex:
    objs = list(ex.map(one, b.SOURCES))
r = subprocess.run([nvcc, "-shared", *b.ARCH, "-o", str(lib), *map(str, objs),
                    "-Xcompiler", "-pthread", "-cudart", "static", "-lrt", "-ldl"], capture_output=True, text=True)
if r.returncode != 0:
    raise SystemExit(r.stderr)
print(lib)
