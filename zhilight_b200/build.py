"""In-tree build of libzhilight_b200.so (sm_90a only: H100).  nvcc cross-compiles without a GPU.

    python -m zhilight_b200.build [--force] [--verbose]
"""
import hashlib
import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ_DIR = os.path.join(HERE, "build")
LIB_PATH = os.path.join(HERE, "libzhilight_b200.so")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-lineinfo", "-std=c++17",
    "--expt-relaxed-constexpr",
    "-Xcompiler", "-fPIC",
    "-Xptxas", "-v",
    "-DZL_BUILD",
]


def _nvcc():
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", shutil.which("nvcc")):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found: the CUDA extension cannot be built (no CPU fallback exists)")


def _sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cu"))


def _headers():
    hs = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    hs.append(os.path.join(HERE, "..", "include", "zhilight_b200.h"))
    return sorted(hs)


def _digest(paths):
    h = hashlib.sha256()
    for p in paths:
        with open(p, "rb") as f:
            h.update(f.read())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def build(force=False, verbose=False):
    # fast path: the library already matches the sources
    all_digest = _digest(_sources() + _headers())
    dig_path = LIB_PATH + ".digest"
    if not force and os.path.exists(LIB_PATH) and os.path.exists(dig_path) and open(dig_path).read() == all_digest:
        return LIB_PATH
    os.makedirs(OBJ_DIR, exist_ok=True)
    nvcc = _nvcc()
    hdr_digest = _digest(_headers())
    jobs = []
    objs = []
    for src in _sources():
        name = os.path.splitext(os.path.basename(src))[0]
        obj = os.path.join(OBJ_DIR, name + ".o")
        stamp = obj + ".stamp"
        digest = _digest([src]) + hdr_digest
        objs.append(obj)
        if not force and os.path.exists(obj) and os.path.exists(stamp) and open(stamp).read() == digest:
            continue
        jobs.append((src, obj, stamp, digest))

    def compile_one(job):
        src, obj, stamp, digest = job
        cmd = [nvcc] + NVCC_FLAGS + ["-c", src, "-o", obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        log = r.stdout + r.stderr
        with open(obj + ".log", "w") as f:
            f.write(" ".join(cmd) + "\n" + log)
        if r.returncode != 0:
            raise RuntimeError("nvcc failed for %s:\n%s" % (src, log))
        with open(stamp, "w") as f:
            f.write(digest)
        return src, log

    if jobs:
        with ThreadPoolExecutor(max_workers=min(8, len(jobs))) as ex:
            for src, log in ex.map(compile_one, jobs):
                if verbose:
                    print("== %s\n%s" % (os.path.basename(src), log))
    if jobs or force or not os.path.exists(LIB_PATH):
        cmd = [nvcc, "-shared", "-o", LIB_PATH] + objs + ["-gencode", "arch=compute_90a,code=sm_90a",
                                                          "-lcudart", "-Xlinker", "--no-undefined"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("link failed:\n" + r.stdout + r.stderr)
    with open(dig_path, "w") as f:
        f.write(all_digest)
    return LIB_PATH


if __name__ == "__main__":
    path = build(force="--force" in sys.argv, verbose="--verbose" in sys.argv)
    print(path)
