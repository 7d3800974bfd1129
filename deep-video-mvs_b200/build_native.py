"""Builds libdvmvs_sm90.so (the C-ABI kernel library, include/dvmvs_b200.h) in-tree with nvcc for sm_90a (H100).

    python deep-video-mvs_b200/build_native.py [--force] [--verbose]

The .so lands in deep-video-mvs_b200/lib/ (git-ignored)."""
import hashlib
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB_DIR = os.path.join(HERE, "lib")
LIB = os.path.join(LIB_DIR, "libdvmvs_sm90.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
# IEEE division / sqrt / exp everywhere (no --use_fast_math)
FLAGS = ARCH + ["-lineinfo", "-O3", "-std=c++17", "-Xcompiler", "-fPIC"]


def sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cu"))


def _stamp():
    h = hashlib.sha256()
    headers = ["../../include/" + f for f in sorted(os.listdir(os.path.join(HERE, "..", "include")))]
    for f in sorted(os.listdir(CSRC)) + headers:
        with open(os.path.join(CSRC, f), "rb") as fh:
            h.update(f.encode() + b"\0" + fh.read())
    h.update(" ".join(FLAGS).encode())
    return h.hexdigest()


def build(force=False, verbose=False):
    os.makedirs(LIB_DIR, exist_ok=True)
    stamp_file = LIB + ".stamp"
    stamp = _stamp()
    if not force and os.path.isfile(LIB) and os.path.isfile(stamp_file) and open(stamp_file).read() == stamp:
        return LIB
    objs = []
    procs = []
    for src in sources():
        obj = os.path.join(LIB_DIR, os.path.basename(src)[:-3] + ".o")
        cmd = [NVCC] + FLAGS + ["-c", src, "-o", obj] + (["-Xptxas", "-v"] if verbose else [])
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        objs.append(obj)
    failed = False
    for src, pr in procs:
        out, _ = pr.communicate()
        if pr.returncode != 0 or verbose:
            print(out)
        if pr.returncode != 0:
            print("nvcc failed for", src)
            failed = True
    if failed:
        raise RuntimeError("libdvmvs_sm90.so: compilation failed")
    cmd = [NVCC, "-shared"] + ARCH + ["-o", LIB] + objs + ["-lcuda"]
    subprocess.check_call(cmd)
    with open(stamp_file, "w") as fh:
        fh.write(stamp)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="--verbose" in sys.argv))
