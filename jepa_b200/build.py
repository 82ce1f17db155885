"""Build the C-ABI shared library (libvjepa_b200.so) in-tree with nvcc for sm_90a (H100).

The built .so and objects are git-ignored build products.  No torch headers are involved: the
library is a plain C ABI over raw device pointers (include/vjepa_b200.h).
"""
import hashlib
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libvjepa_b200.so")
OBJ_DIR = os.path.join(HERE, "build")

NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
FLAGS = ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC",
         "-I" + os.path.join(ROOT, "include"), "-I" + CSRC]


def sources():
    return sorted(f for f in os.listdir(CSRC) if f.endswith(".cu"))


def _digest(paths):
    h = hashlib.sha256()
    for p in paths:
        with open(p, "rb") as f:
            h.update(f.read())
    h.update(" ".join(FLAGS + ARCH).encode())
    return h.hexdigest()


def build(force=False, verbose=False):
    """Compile every .cu under csrc/ and link libvjepa_b200.so.  Incremental per source."""
    os.makedirs(OBJ_DIR, exist_ok=True)
    headers = [os.path.join(CSRC, f) for f in sorted(os.listdir(CSRC)) if f.endswith((".cuh", ".h"))]
    headers.append(os.path.join(ROOT, "include", "vjepa_b200.h"))
    objs, procs = [], []
    for src in sources():
        sp = os.path.join(CSRC, src)
        obj = os.path.join(OBJ_DIR, src[:-3] + ".o")
        stamp = obj + ".sha"
        dig = _digest([sp] + headers)
        objs.append(obj)
        if not force and os.path.exists(obj) and os.path.exists(stamp) and open(stamp).read() == dig:
            continue
        cmd = [NVCC] + ARCH + FLAGS + ["-c", sp, "-o", obj]
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
        procs.append((src, stamp, dig, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)))
    relink = force or not os.path.exists(LIB)
    for src, stamp, dig, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            sys.stderr.write(out.decode())
            raise RuntimeError(f"nvcc failed on {src}")
        if verbose:
            sys.stderr.write(out.decode())
        with open(stamp, "w") as f:
            f.write(dig)
        relink = True
    if relink:
        cmd = [NVCC] + ARCH + ["-shared", "-o", LIB] + objs + ["-cudart", "static"]
        subprocess.check_call(cmd)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
