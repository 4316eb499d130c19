"""Build the CUDA extension in-tree: sela_b200/libsela_b200.so (sm_90a only).

    python -m sela_b200.build [--force] [--verbose]

nvcc cross-compiles without a GPU.  Flags that matter for parity:
  -fmad=false     no FMA contraction anywhere in the translation unit (the double
                  front end additionally uses the *_rn intrinsics, which are never
                  contracted) -- SURVEY.md 7.3-H1;
  no --use_fast_math, ever.
"""
import pathlib
import subprocess
import sys

PKG = pathlib.Path(__file__).resolve().parent
CSRC = PKG / "csrc"
LIB = PKG / "libsela_b200.so"
SOURCES = [CSRC / "c_abi.cu"]
DEPS = list(CSRC.glob("*.cu")) + list(CSRC.glob("*.cuh")) + [PKG.parent / "include" / "sela_b200.h"]

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-lineinfo", "-std=c++17", "-fmad=false",
    "-Xcompiler", "-fPIC", "-shared", "--extended-lambda",
    "-Xptxas", "-v",
]


def needs_build():
    if not LIB.exists():
        return True
    t = LIB.stat().st_mtime
    return any(p.stat().st_mtime > t for p in DEPS + [pathlib.Path(__file__)])


def build(force=False, verbose=False):
    if not force and not needs_build():
        return LIB
    tmp = LIB.with_suffix(".so.tmp")           # built aside and renamed: a reader (or a snapshot) never sees half a library
    cmd = ["nvcc", *NVCC_FLAGS, "-o", str(tmp), *map(str, SOURCES)]
    proc = subprocess.run(cmd, capture_output=True, text=True)
    if verbose or proc.returncode != 0:
        sys.stderr.write(proc.stdout + proc.stderr)
    if proc.returncode != 0:
        tmp.unlink(missing_ok=True)
        raise RuntimeError("nvcc failed building %s" % LIB)
    tmp.replace(LIB)
    (PKG / "build_ptxas.log").write_text(proc.stdout + proc.stderr)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="--verbose" in sys.argv or True))
