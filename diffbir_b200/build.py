"""In-tree build of libdiffbir_b200.so (sm_90a only; nvcc cross-compiles without a GPU).

    python -m diffbir_b200.build [--bf16] [--force] [-v]

Objects go to diffbir_b200/csrc/_build/, the library to diffbir_b200/libdiffbir_b200.so
(git-ignored). --bf16 builds the bf16-operand
variant into csrc/_build_bf16/ and libdiffbir_b200_bf16.so (loaded when DBIR_OPERANDS=bf16).
"""
from __future__ import annotations

import hashlib
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

HERE = Path(__file__).resolve().parent
CSRC = HERE / "csrc"
OUT = HERE / "libdiffbir_b200.so"
OUT_BF16 = HERE / "libdiffbir_b200_bf16.so"      # -DDBIR_OPERAND_BF16 variant, selected with DBIR_OPERANDS=bf16
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
FLAGS = ["-O3", "-lineinfo", "-std=c++17", "--expt-relaxed-constexpr", "-Xcompiler", "-fPIC",
         "-Xptxas", "-v"]


def _digest(paths, extra):
    h = hashlib.sha1()
    for p in sorted(paths):
        h.update(p.name.encode())
        h.update(p.read_bytes())
    h.update(" ".join(extra).encode())
    return h.hexdigest()


def build_library(bf16: bool = False, force: bool = False, verbose: bool = False) -> Path:
    srcs = sorted(CSRC.glob("*.cu"))
    hdrs = sorted(CSRC.glob("*.cuh")) + sorted((HERE.parent / "include").glob("*.h"))
    defs = ["-DDBIR_OPERAND_BF16"] if bf16 else []
    bdir = CSRC / ("_build_bf16" if bf16 else "_build")
    bdir.mkdir(exist_ok=True)
    out = OUT_BF16 if bf16 else OUT
    stamp = bdir / "stamp.txt"
    dig = _digest(srcs + hdrs, ARCH + FLAGS + defs)
    if out.exists() and stamp.exists() and stamp.read_text() == dig and not force:
        return out

    hdig = _digest(hdrs, ARCH + FLAGS + defs)

    def compile_one(src: Path) -> Path:
        obj = bdir / (src.stem + ".o")
        tag = bdir / (src.stem + ".tag")
        sd = hashlib.sha1(src.read_bytes()).hexdigest() + hdig
        if obj.exists() and tag.exists() and tag.read_text() == sd and not force:
            return obj
        cmd = [NVCC, *ARCH, *FLAGS, *defs, "-c", str(src), "-o", str(obj)]
        r = subprocess.run(cmd, capture_output=True, text=True)
        log = (r.stdout or "") + (r.stderr or "")
        (bdir / (src.stem + ".log")).write_text(log)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed for {src.name}:\n{log}")
        if verbose:
            print(log)
        tag.write_text(sd)
        return obj

    with ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
        objs = list(ex.map(compile_one, srcs))
    cmd = [NVCC, *ARCH, "-shared", "-o", str(out), *map(str, objs), "-lcudart"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"link failed:\n{r.stdout}{r.stderr}")
    stamp.write_text(dig)
    return out


if __name__ == "__main__":
    p = build_library(bf16="--bf16" in sys.argv, force="--force" in sys.argv, verbose="-v" in sys.argv)
    print(p)
