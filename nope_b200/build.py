"""Build libnope_b200.so in-tree with nvcc for sm_90a (no torch extension machinery:
the library is a plain C-ABI shared object, bound from Python with ctypes)."""
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
SRC = os.path.join(HERE, "csrc", "nope_b200.cu")
CSRC = os.path.join(HERE, "csrc")
DEPS = [os.path.join(CSRC, f) for f in sorted(os.listdir(CSRC)) if f.endswith((".cu", ".cuh", ".h"))] + \
       [os.path.join(ROOT, "include", "nope_b200.h")]
OUT_DIR = os.path.join(HERE, "lib")
OUT = os.path.join(OUT_DIR, "libnope_b200.so")


def nvcc_path():
    p = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(p):
        raise RuntimeError("nvcc not found; the CUDA library cannot be built")
    return p


def have_nvcc():
    return bool(shutil.which("nvcc")) or os.path.exists("/usr/local/cuda/bin/nvcc")


STAMP = OUT + ".srchash"


def source_hash():
    """Content hash of every source the library is built from (mtimes do not survive a copy of the
    tree to another box, contents do)."""
    import hashlib
    h = hashlib.sha256()
    for d in DEPS:
        h.update(os.path.basename(d).encode())
        with open(d, "rb") as f:
            h.update(f.read())
    return h.hexdigest()


def is_stale():
    if not os.path.exists(OUT) or not os.path.exists(STAMP):
        return True
    with open(STAMP) as f:
        return f.read().strip() != source_hash()


def build(force=False, verbose=False):
    if not force and not is_stale():
        return OUT
    os.makedirs(OUT_DIR, exist_ok=True)
    tmp = f"{OUT}.{os.getpid()}.tmp"       # several ranks may build at once: private temp, atomic rename
    cmd = [nvcc_path(), "-gencode", "arch=compute_90a,code=sm_90a", "-std=c++17", "-O3",
           "-lineinfo", "-Xcompiler", "-fPIC", "-shared", "-I", os.path.join(ROOT, "include"),
           "-o", tmp, SRC]
    if verbose:
        cmd.insert(1, "-Xptxas=-v")
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout + r.stderr)
        raise RuntimeError("nvcc failed building libnope_b200.so")
    if verbose:
        sys.stderr.write(r.stderr)
    os.replace(tmp, OUT)
    with open(f"{STAMP}.{os.getpid()}.tmp", "w") as f:
        f.write(source_hash())
    os.replace(f"{STAMP}.{os.getpid()}.tmp", STAMP)
    return OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
