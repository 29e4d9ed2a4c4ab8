"""Builds libmfr_b200.so (hand-written sm_90a CUDA behind a C ABI) in-tree with nvcc.

Usage: python map-free-reloc_b200/build.py [--force]
The .so and the object files are build products (git-ignored).
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, "libmfr_b200.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC", "-Xptxas", "-v",
]
# sift.cu restates OpenCV's float arithmetic operation by operation: no contraction into FMAs
FILE_FLAGS = {"sift.cu": ["-fmad=false"]}


def sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cu"))


def needs_build():
    if not os.path.exists(OUT):
        return True
    t = os.path.getmtime(OUT)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)]
    deps.append(os.path.join(HERE, "..", "include", "mfr_b200.h"))
    deps.append(os.path.abspath(__file__))
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=True):
    if not force and not needs_build():
        return OUT
    objs = []
    build_dir = os.path.join(HERE, "build")
    os.makedirs(build_dir, exist_ok=True)
    procs = []
    for src in sources():
        obj = os.path.join(build_dir, os.path.basename(src)[:-3] + ".o")
        objs.append(obj)
        cmd = [NVCC, *FLAGS, *FILE_FLAGS.get(os.path.basename(src), []), "-c", src, "-o", obj]
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    ok = True
    for src, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            ok = False
            sys.stderr.write(out)
        elif verbose:
            for line in out.splitlines():
                if "registers" in line or ("spill" in line and "0 bytes spill" not in line):
                    print(os.path.basename(src), line.strip())
    if not ok:
        raise RuntimeError("nvcc failed")
    cmd = [NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-shared", "-o", OUT, *objs, "-lcudart"]
    subprocess.check_call(cmd)
    return OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv))
