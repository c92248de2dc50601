"""Build libgdrn_b200.so in-tree with nvcc for sm_90a (no torch dependency in the library)."""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libgdrn_b200.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr",
]


def sources():
    return sorted(f for f in os.listdir(CSRC) if f.endswith(".cu"))


def _needs_rebuild(obj, src):
    if not os.path.exists(obj):
        return True
    t = os.path.getmtime(obj)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".h", ".cuh"))]
    deps += [src, os.path.join(HERE, "..", "include", "gdrn_b200.h")]
    return any(os.path.getmtime(d) > t for d in deps)


def build(verbose=False, force=False):
    objdir = os.path.join(CSRC, "build")
    os.makedirs(objdir, exist_ok=True)
    jobs = []
    for f in sources():
        src = os.path.join(CSRC, f)
        obj = os.path.join(objdir, f[:-3] + ".o")
        if force or _needs_rebuild(obj, src):
            jobs.append((src, obj))

    def compile_one(job):
        src, obj = job
        cmd = [NVCC] + FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-c", src, "-o", obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed for {src}:\n{r.stdout}\n{r.stderr}")
        if verbose:
            print(r.stderr)
        return obj

    with ThreadPoolExecutor(max_workers=min(8, max(1, len(jobs)))) as ex:
        list(ex.map(compile_one, jobs))
    objs = [os.path.join(objdir, f[:-3] + ".o") for f in sources()]
    if jobs or not os.path.exists(LIB):
        cmd = [NVCC, "-shared", "-gencode", "arch=compute_90a,code=sm_90a", "-o", LIB] + objs + ["-lcudart"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    return LIB


if __name__ == "__main__":
    print(build(verbose="-v" in sys.argv, force="-f" in sys.argv))
