"""Builds libaae_b200.so in-tree with nvcc for sm_90a (H100; the only target: no multi-arch, no fallbacks)."""
import hashlib
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libaae_b200.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17", "-Xcompiler", "-fPIC,-fvisibility=hidden",
         "--expt-relaxed-constexpr"]


def sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cu"))


def _newest(paths):
    return max(os.path.getmtime(p) for p in paths)


def _digest(paths):
    h = hashlib.sha256()
    for p in sorted(paths):
        h.update(os.path.basename(p).encode())
        h.update(open(p, "rb").read())
    h.update(" ".join(FLAGS).encode())
    return h.hexdigest()


def build(force: bool = False, verbose: bool = False) -> str:
    """Compile (if needed) and return the path of libaae_b200.so.  Staleness is decided by a content hash of the sources
    stored beside the library (file times do not survive every copy of the tree), and the library is replaced atomically
    so that other ranks may dlopen it while rank 0 is (re)building."""
    srcs = sources()
    deps = srcs + [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cuh")] + \
        [os.path.join(HERE, "..", "include", "aae_b200.h")]
    stamp = LIB + ".sha256"
    digest = _digest(deps)
    if not force and os.path.exists(LIB) and os.path.exists(stamp) and open(stamp).read().strip() == digest:
        return LIB
    objdir = os.path.join(HERE, "build")
    os.makedirs(objdir, exist_ok=True)
    wanted = {os.path.basename(src)[:-3] + ".o" for src in srcs}
    for f in os.listdir(objdir):                       # objects whose source is gone must neither be linked nor travel with the tree
        if f.endswith(".o") and f not in wanted:
            os.remove(os.path.join(objdir, f))

    def compile_one(src):
        obj = os.path.join(objdir, os.path.basename(src)[:-3] + ".o")
        hdrs = [p for p in deps if not p.endswith(".cu")]
        if not force and os.path.exists(obj) and os.path.getmtime(obj) >= max(os.path.getmtime(src), _newest(hdrs)):
            return obj
        cmd = [NVCC] + FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-c", src, "-o", obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("nvcc failed for %s:\n%s\n%s" % (src, r.stdout, r.stderr))
        if verbose:
            sys.stderr.write(r.stderr)
        return obj

    with ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
        objs = list(ex.map(compile_one, srcs))
    tmp = LIB + ".tmp.%d" % os.getpid()
    cmd = [NVCC, "-shared", "-o", tmp] + objs + ["-gencode", "arch=compute_90a,code=sm_90a", "-cudart", "static"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("link failed:\n%s\n%s" % (r.stdout, r.stderr))
    os.replace(tmp, LIB)
    with open(stamp, "w") as f:
        f.write(digest + "\n")
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
