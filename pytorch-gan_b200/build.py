"""Build libb200gan.so (sm_90a only) in-tree with nvcc.  No torch headers, no -lcuda.

    python pytorch-gan_b200/build.py [--force] [--verbose]

The resulting shared library sits next to the Python package
(pytorch-gan_b200/b200gan/libb200gan.so) and is git-ignored.
"""
import argparse
import concurrent.futures as cf
import hashlib
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, "b200gan", "libb200gan.so")
OBJ = os.path.join(HERE, "build")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr",
    "-DB200GAN_BUILD",
]


def sources():
    return sorted(f for f in os.listdir(CSRC) if f.endswith(".cu"))


def digest():
    h = hashlib.sha256()
    for f in sorted(os.listdir(CSRC)) + ["../../include/b200gan.h"]:
        with open(os.path.join(CSRC, f), "rb") as fh:
            h.update(f.encode())
            h.update(fh.read())
    h.update(" ".join(FLAGS).encode())
    return h.hexdigest()


def build(force=False, verbose=False):
    os.makedirs(OBJ, exist_ok=True)
    stamp = os.path.join(OBJ, "stamp")
    dg = digest()
    if not force and os.path.exists(OUT) and os.path.exists(stamp) and open(stamp).read() == dg:
        return OUT
    if not os.path.exists(NVCC):
        if os.path.exists(OUT):
            return OUT  # no toolchain: use the library built earlier
        raise RuntimeError("nvcc not found and no prebuilt libb200gan.so")

    def compile_one(src):
        obj = os.path.join(OBJ, src.replace(".cu", ".o"))
        cmd = [NVCC, *FLAGS, "-c", os.path.join(CSRC, src), "-o", obj]
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
        r = subprocess.run(cmd, capture_output=True, text=True)
        return src, obj, r

    objs = []
    with cf.ThreadPoolExecutor(max_workers=min(8, os.cpu_count() or 1)) as ex:
        for src, obj, r in ex.map(compile_one, sources()):
            if r.returncode != 0:
                sys.stderr.write(r.stdout + r.stderr)
                raise RuntimeError(f"nvcc failed on {src}")
            if verbose:
                sys.stderr.write(f"== {src}\n{r.stderr}\n")
            objs.append(obj)
    link = [NVCC, "-shared", "-gencode", "arch=compute_90a,code=sm_90a", "-o", OUT, *objs, "-lcudart"]
    r = subprocess.run(link, capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout + r.stderr)
        raise RuntimeError("link failed")
    with open(stamp, "w") as fh:
        fh.write(dg)
    return OUT


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--force", action="store_true")
    ap.add_argument("--verbose", action="store_true")
    a = ap.parse_args()
    print(build(a.force, a.verbose))
