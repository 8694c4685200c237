"""Build libunivl_b200.so (sm_90a) in-tree with nvcc.

The shared library is the C-ABI boundary (include/univl_b200.h); it links cudart statically and does
not link libcuda, so it loads on a GPU-less host (the CPU test-suite checks its exported symbols).
"""
import glob
import hashlib
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libunivl_b200.so")
STAMP = os.path.join(HERE, "csrc", ".build_stamp")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-lineinfo", "-std=c++17",
    "--use_fast_math",
    "-Xcompiler", "-fPIC",
    "--expt-relaxed-constexpr",
    "-cudart", "static",
]


def _sources():
    return sorted(glob.glob(os.path.join(CSRC, "*.cu")))


def _digest():
    h = hashlib.sha256()
    for f in _sources() + sorted(glob.glob(os.path.join(CSRC, "*.cuh"))):
        h.update(f.encode())
        with open(f, "rb") as fh:
            h.update(fh.read())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def build(force=False, verbose=False):
    """Compile every .cu under csrc/ into one shared library. Returns the library path."""
    digest = _digest()
    if not force and os.path.exists(LIB) and os.path.exists(STAMP):
        with open(STAMP) as fh:
            if fh.read().strip() == digest:
                return LIB
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    objs = []
    procs = []
    for src in _sources():
        obj = src[:-3] + ".o"
        cmd = [nvcc, *NVCC_FLAGS, "-I", CSRC, "-c", src, "-o", obj]
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
            print(" ".join(cmd), flush=True)
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        objs.append(obj)
    failed = False
    for src, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            failed = True
            sys.stderr.write("nvcc failed for %s:\n%s\n" % (src, out))
        elif verbose or "warning" in out:
            sys.stderr.write(out)
    if failed:
        raise RuntimeError("univl_b200: nvcc compilation failed")
    link = [nvcc, "-shared", "-cudart", "static", "-gencode", "arch=compute_90a,code=sm_90a",
            "-o", LIB, *objs]
    subprocess.check_call(link)
    with open(STAMP, "w") as fh:
        fh.write(digest)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
