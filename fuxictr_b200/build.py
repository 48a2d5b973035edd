"""In-tree build of the sm_90a (H100) C-ABI library (libfuxictr_b200.so) with plain nvcc.

The library has no torch / Python dependency: it is what a C, Go or Python (ctypes)
host binds.  `python -m fuxictr_b200.build` or `__graft_entry__.build()` runs this.
"""
import hashlib
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
INCLUDE = os.path.join(os.path.dirname(HERE), "include")
LIB = os.path.join(HERE, "libfuxictr_b200.so")
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-lineinfo", "-std=c++17",
    "--expt-relaxed-constexpr",
    "-Xcompiler", "-fPIC",
    "-Xcompiler", "-fvisibility=hidden",
]


def _nvcc():
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found; cannot build the sm_90a library")


def _digest():
    h = hashlib.sha256()
    for root in (CSRC, INCLUDE):
        for name in sorted(os.listdir(root)):
            with open(os.path.join(root, name), "rb") as fd:
                h.update(name.encode())
                h.update(fd.read())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def build(force=False, verbose=False):
    """Compile every .cu for sm_90a and link libfuxictr_b200.so next to this file."""
    stamp = os.path.join(HERE, "build", "stamp")
    digest = _digest()
    if not force and os.path.exists(LIB) and os.path.exists(stamp):
        with open(stamp) as fd:
            if fd.read().strip() == digest:
                return LIB
    nvcc = _nvcc()
    objdir = os.path.join(HERE, "build")
    os.makedirs(objdir, exist_ok=True)
    sources = [s for s in sorted(os.listdir(CSRC)) if s.endswith(".cu")]
    procs = []
    for src in sources:
        obj = os.path.join(objdir, src[:-3] + ".o")
        cmd = [nvcc] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + \
              ["-I", INCLUDE, "-c", os.path.join(CSRC, src), "-o", obj]
        procs.append((src, obj, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)))
    objs = []
    for src, obj, p in procs:
        out, _ = p.communicate()
        if verbose or p.returncode != 0:
            sys.stderr.write(out.decode())
        if p.returncode != 0:
            raise RuntimeError("nvcc failed on %s" % src)
        objs.append(obj)
    cmd = [nvcc, "-shared", "-o", LIB] + objs + ["-lcudart_static", "-lcuda", "-lpthread", "-ldl", "-lrt"]
    subprocess.check_call(cmd)
    with open(stamp, "w") as fd:
        fd.write(digest)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
