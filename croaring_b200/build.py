"""Build recipe for libroaring_b200.so (in-tree, so the package imports from the repository).

    python -m croaring_b200.build [--force] [--verbose]

nvcc cross-compiles for sm_90a (H100) without a GPU.  cudart is linked statically so the library is
self-contained next to torch's own CUDA runtime.
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libroaring_b200.so")
SOURCES = ["rb200_kernels.cu", "rb200_compute.cu", "rb200_many.cu", "rb200_many2.cu", "rb200_convert.cu", "rb200_build.cu", "rb200_host.cu", "rb200_shard.cu",
           "rb200_fused.cu", "rb200_offset.cu", "rb200_query.cu", "rb200_range.cu"]
HEADERS = ["rb200_common.h", "rb200_device.cuh", "rb200_cells.cuh", "rb200_internal.h", "rb200_portable.h",
           os.path.join("..", "..", "include", "roaring_b200.h")]

ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]   # H100 (Hopper) only
NVCC_FLAGS = [
    "-O3", "-std=c++17",
    *ARCH,
    "-lineinfo",
    "-Xcompiler", "-fPIC,-fvisibility=hidden,-O3",
    "--expt-relaxed-constexpr",
    "-cudart", "static",
    "-DRB200_BUILDING_LIBRARY",   # include/roaring_b200.h: never pull an installed copy of the reference's headers
]
# The pairwise cell kernel writes results it never reads again: its global stores default to
# evict-first, so that they do not push the operands, which every cell reads, out of L2
# (rb200_compute.cu).
SOURCE_FLAGS = {"rb200_compute.cu": ["-Xptxas", "-dscm=cs"]}


def _newest(paths):
    return max(os.path.getmtime(p) for p in paths)


def needs_build():
    if not os.path.exists(LIB):
        return True
    deps = [os.path.join(CSRC, s) for s in SOURCES] + [os.path.join(CSRC, h) for h in HEADERS]
    deps.append(os.path.abspath(__file__))
    return _newest(deps) > os.path.getmtime(LIB)


WORKGEN_LIB = os.path.join(HERE, "libworkgen.so")


def build_workgen(force=False):
    """Host-only workload generators (plain C + pthreads; bench / test input builders)."""
    src = os.path.join(CSRC, "workgen.c")
    if not force and os.path.exists(WORKGEN_LIB) and os.path.getmtime(WORKGEN_LIB) >= os.path.getmtime(src):
        return WORKGEN_LIB
    subprocess.check_call([os.environ.get("CC", "gcc"), "-O3", "-fPIC", "-std=gnu11", "-shared",
                           "-fvisibility=hidden", "-ffp-contract=off", "-o", WORKGEN_LIB, src, "-lm", "-lpthread"])
    return WORKGEN_LIB


def build(force=False, verbose=False, defines=(), out=None):
    """defines / out: an experimental variant (-DNAME=VALUE ...) written to another .so (tuning
    runs load it through RB200_LIB); the default build is the product."""
    build_workgen(force)
    lib = out or LIB
    if not force and not out and not needs_build():
        return LIB
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    objs = []
    tag = "" if not out else "." + os.path.basename(out).replace(".so", "")
    for s in SOURCES:
        o = os.path.join(CSRC, s.replace(".cu", tag + ".o"))
        cmd = [nvcc] + NVCC_FLAGS + SOURCE_FLAGS.get(s, []) + ["-D" + d for d in defines] + (["-Xptxas", "-v"] if verbose else []) + \
              ["-c", os.path.join(CSRC, s), "-o", o]
        if verbose:
            print(" ".join(cmd), flush=True)
        subprocess.check_call(cmd)
        objs.append(o)
    cmd = [nvcc, "-shared", *ARCH, "-cudart", "static", "-o", lib] + objs + \
          ["-Xlinker", "-Bsymbolic", "-ldl", "-lpthread"]
    if verbose:
        print(" ".join(cmd), flush=True)
    subprocess.check_call(cmd)
    return lib


if __name__ == "__main__":
    defs = [a[2:] for a in sys.argv[1:] if a.startswith("-D")]
    outs = [a.split("=", 1)[1] for a in sys.argv[1:] if a.startswith("--out=")]
    print(build(force="--force" in sys.argv, verbose="--verbose" in sys.argv, defines=defs,
                out=os.path.abspath(outs[0]) if outs else None))
