"""Build the C-ABI CUDA library in-tree:  nabladft_b200/libnabla_b200.so  (sm_90a only: H100).

    python -m nabladft_b200.build [--force]

nvcc cross-compiles without a GPU.
"""
import glob
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libnabla_b200.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr",
] + os.environ.get("NB200_NVCC_EXTRA", "").split()
# per-source flags: the quasi-Newton line search rounds every float64 operation as Python does, so no FMA contraction there
SOURCE_FLAGS = {"quasinewton.cu": ["-fmad=false"]}


def sources():
    return sorted(glob.glob(os.path.join(CSRC, "*.cu")))


STAMP = os.path.join(HERE, "build", "stamp.txt")


def stamp_text() -> str:
    """What the library was built with: compiler, flags (architecture and NB200_NVCC_EXTRA included)."""
    return " ".join([NVCC, *FLAGS, repr(sorted(SOURCE_FLAGS.items()))])


def stale() -> bool:
    """Rebuild when the library is missing, was built with other flags / for another architecture, or any source is newer."""
    if not os.path.exists(LIB) or not os.path.exists(STAMP):
        return True
    with open(STAMP) as f:
        if f.read() != stamp_text():
            return True
    t = os.path.getmtime(LIB)
    deps = sources() + glob.glob(os.path.join(CSRC, "*.cuh")) + glob.glob(os.path.join(CSRC, "*.inc")) + \
        glob.glob(os.path.join(HERE, "..", "include", "*.h")) + [os.path.abspath(__file__)]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not stale():
        return LIB
    objs = []
    procs = []
    os.makedirs(os.path.join(HERE, "build"), exist_ok=True)
    for src in sources():
        obj = os.path.join(HERE, "build", os.path.basename(src)[:-3] + ".o")
        cmd = [NVCC, *FLAGS, *SOURCE_FLAGS.get(os.path.basename(src), []), "-c", src, "-o", obj] + (["-Xptxas", "-v"] if verbose else [])
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        objs.append(obj)
    for src, p in procs:
        out, _ = p.communicate()
        if verbose or p.returncode:
            print(out)
        if p.returncode:
            raise RuntimeError(f"nvcc failed on {src}")
    link = [NVCC, "-shared", "-o", LIB, *objs, "-gencode", "arch=compute_90a,code=sm_90a",
            "-L/usr/local/cuda/lib64", "-lcublas", "-Xlinker", "-rpath=/usr/local/cuda/lib64"]
    subprocess.check_call(link)
    with open(STAMP, "w") as f:
        f.write(stamp_text())
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
