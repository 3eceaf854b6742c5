"""Build liboasr_b200.so in-tree with nvcc for sm_90a (H100; nvcc cross-compiles without a GPU).

    python -m olmoasr_b200.build [--force]

The .so lands next to the sources (olmoasr_b200/csrc/liboasr_b200.so) so that it travels with a
snapshot of the repository; nothing is cached outside the tree.
"""
from __future__ import annotations

import concurrent.futures as cf
import hashlib
import os
import shutil
import subprocess
import sys
from pathlib import Path

CSRC = Path(__file__).resolve().parent / "csrc"
LIB = CSRC / "liboasr_b200.so"
OBJ_DIR = CSRC / "_obj"

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-lineinfo", "-O3", "-std=c++17",
    "--expt-relaxed-constexpr",
    "-Xcompiler", "-fPIC",
    "-Xcompiler", "-fvisibility=hidden",
]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found (set NVCC=/path/to/nvcc)")


def _digest(paths) -> str:
    h = hashlib.sha256()
    for p in sorted(paths):
        h.update(p.name.encode())
        h.update(p.read_bytes())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def sources():
    return sorted(CSRC.glob("*.cu"))


def headers():
    return sorted(CSRC.glob("*.cuh")) + [CSRC.parent.parent / "include" / "oasr_b200.h"]


def build_variant(name: str, defines) -> Path:
    """A/B build: the whole library compiled with extra -D flags into csrc/_ab/<name>.so (select it at run time with
    OASR_B200_LIB; the default library is untouched)."""
    out_dir = CSRC / "_ab"
    obj_dir = out_dir / ("_obj_" + name)
    obj_dir.mkdir(parents=True, exist_ok=True)
    nvcc = _nvcc()

    def one(src: Path):
        obj = obj_dir / (src.stem + ".o")
        r = subprocess.run([nvcc, *NVCC_FLAGS, *defines, "-c", str(src), "-o", str(obj)], capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed for {src.name}:\n{r.stdout}\n{r.stderr}")
        return str(obj)

    with cf.ThreadPoolExecutor(max_workers=8) as ex:
        objs = list(ex.map(one, sources()))
    lib = out_dir / f"{name}.so"
    r = subprocess.run([nvcc, "-shared", "-o", str(lib), *objs], capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    shutil.rmtree(obj_dir, ignore_errors=True)
    return lib


def build(force: bool = False, verbose: bool = False) -> Path:
    srcs = sources()
    stamp = OBJ_DIR / "stamp.txt"
    OBJ_DIR.mkdir(exist_ok=True)
    hdr_digest = _digest(headers())
    nvcc = _nvcc()

    def compile_one(src: Path):
        obj = OBJ_DIR / (src.stem + ".o")
        tag = OBJ_DIR / (src.stem + ".tag")
        want = hashlib.sha256((hdr_digest + _digest([src])).encode()).hexdigest()
        if not force and obj.exists() and tag.exists() and tag.read_text() == want:
            return obj, ""
        cmd = [nvcc, *NVCC_FLAGS, "-c", str(src), "-o", str(obj)]
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed for {src.name}:\n{r.stdout}\n{r.stderr}")
        tag.write_text(want)
        return obj, r.stderr

    with cf.ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
        results = list(ex.map(compile_one, srcs))
    objs = [str(o) for o, _ in results]
    if verbose:
        for _, log in results:
            if log:
                print(log)
    link_want = _digest([Path(o) for o in objs])
    if force or not LIB.exists() or not stamp.exists() or stamp.read_text() != link_want:
        cmd = [nvcc, "-shared", "-o", str(LIB), *objs]  # cudart is linked statically (nvcc default)
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
        stamp.write_text(link_want)
    return LIB


if __name__ == "__main__":
    if "--variant" in sys.argv:     # python -m olmoasr_b200.build --variant attn_poly2 -DOASR_ATTN_POLY=2
        i = sys.argv.index("--variant")
        print(build_variant(sys.argv[i + 1], [a for a in sys.argv[i + 2:] if a.startswith("-D")]))
    else:
        out = build(force="--force" in sys.argv, verbose="-v" in sys.argv)
        print(out)
