"""Builds libvalida_b200.so (all CUDA kernels + the C ABI + host code) in-tree for sm_90a (H100).

nvcc cross-compiles without a GPU.  The .so and the objects are build products and stay out of git.
Also builds the oracle (test infrastructure) via its own Makefile on request.
"""
import hashlib
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(HERE, "build")
LIB = os.path.join(HERE, "libvalida_b200.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
HOST_CXX = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"

GENCODE = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = GENCODE + [
    "-lineinfo", "-O3", "-std=c++17",
    "--expt-relaxed-constexpr", "--extended-lambda",
    "-ccbin", HOST_CXX, "-Xcompiler", "-fPIC,-fopenmp,-O3", "-I", os.path.join(ROOT, "include"),
]


def sources():
    out = []
    for d, _, files in os.walk(CSRC):
        for f in sorted(files):
            if f.endswith((".cu", ".cc")):
                out.append(os.path.join(d, f))
    return sorted(out)


def headers_digest():
    h = hashlib.sha256()
    for d, _, files in sorted(os.walk(CSRC)):
        for f in sorted(files):
            if f.endswith((".h", ".cuh", ".inc")):
                h.update(open(os.path.join(d, f), "rb").read())
    h.update(open(os.path.join(ROOT, "include", "valida_b200.h"), "rb").read())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def build(verbose=False, ptxas_info=False):
    os.makedirs(OBJ, exist_ok=True)
    hd = headers_digest()
    srcs = sources()
    jobs = []
    objs = []
    for s in srcs:
        key = hashlib.sha256((hd + open(s, "rb").read().hex()).encode()).hexdigest()[:16]
        o = os.path.join(OBJ, os.path.basename(s) + "." + key + ".o")
        objs.append(o)
        if not os.path.exists(o):
            cmd = [NVCC] + NVCC_FLAGS + (["-Xptxas", "-v"] if ptxas_info else []) + ["-x", "cu", "-c", s, "-o", o]
            jobs.append((s, cmd))

    def run(job):
        s, cmd = job
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("nvcc failed for %s:\n%s\n%s" % (s, r.stdout, r.stderr))
        if verbose or ptxas_info:
            sys.stderr.write(r.stderr)
        return s

    if jobs:
        with ThreadPoolExecutor(max_workers=min(8, len(jobs))) as ex:
            list(ex.map(run, jobs))
    stale = not os.path.exists(LIB) or any(os.path.getmtime(o) > os.path.getmtime(LIB) for o in objs)
    if jobs or stale:
        # the arch is named at the link too: nvcc's device-link stub is otherwise an (empty) cubin for its default sm_52
        cmd = [NVCC, "-shared"] + GENCODE + ["-o", LIB] + objs + ["-ccbin", HOST_CXX, "-Xcompiler", "-fopenmp", "-lgomp", "-lcudart"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("link failed:\n%s\n%s" % (r.stdout, r.stderr))
    # drop objects of older source revisions
    keep = set(objs)
    for f in os.listdir(OBJ):
        p = os.path.join(OBJ, f)
        if p.endswith(".o") and p not in keep:
            os.remove(p)
    return LIB


def build_oracle():
    r = subprocess.run(["make", "-C", os.path.join(ROOT, "oracle")], capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("oracle build failed:\n%s\n%s" % (r.stdout, r.stderr))
    return os.path.join(ROOT, "oracle", "liboracle.so")


if __name__ == "__main__":
    print(build(verbose="-v" in sys.argv, ptxas_info="--ptxas" in sys.argv))
    if "--oracle" in sys.argv:
        print(build_oracle())
