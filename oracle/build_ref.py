"""ORACLE (test infrastructure): build the checker libraries.

  * oracle/liboracle_ops.so      -- our CPU restatement (ops_oracle.c), always built.
  * oracle/_ref/libfps_ref.so    -- the REFERENCE's own FPS C++ (core/csrc/fps/src/farthest_point_sampling.cpp)
                                    compiled where it lies with the flags of core/csrc/fps/setup.py:5-7.
  * oracle/_ref/libupnp_ceres_ref.so -- uncertainty-PnP solved with the REFERENCE's vendored Ceres 2.0 headers (Jet
                                    autodiff + TinySolver LM), see upnp_ceres_ref.cpp.
  * oracle/_ref/<mod>/<mod>.so   -- the REFERENCE's own CUDA extensions (ransac_voting, torch_nndistance_aten,
                                    flow_cuda) compiled unmodified for sm_90a: the GPU-side ground truth that
                                    tools/make_golden_ref.py turns into tests/golden/ fixtures.
The _ref outputs are only (re)built when GDRN_REFERENCE_SRC names a checkout of the reference project; they are
git-ignored.  The tests read the stored fixtures, never oracle/_ref.  No reference source is copied into the repo.
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ.get("GDRN_REFERENCE_SRC", "")
REFDIR = os.path.join(HERE, "_ref")


def run(cmd):
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("command failed: %s\n%s\n%s" % (" ".join(cmd), r.stdout, r.stderr))


def build_oracle_ops():
    out = os.path.join(HERE, "liboracle_ops.so")
    src = os.path.join(HERE, "ops_oracle.c")
    if not os.path.exists(out) or os.path.getmtime(out) < os.path.getmtime(src):
        run(["gcc", "-O2", "-ffp-contract=off", "-fopenmp", "-shared", "-fPIC", "-o", out, src, "-lm"])
    return out


def build_fps_ref():
    src = os.path.join(REF, "core/csrc/fps/src/farthest_point_sampling.cpp")
    if not REF or not os.path.exists(src):
        return None
    os.makedirs(REFDIR, exist_ok=True)
    out = os.path.join(REFDIR, "libfps_ref.so")
    if not os.path.exists(out):
        run(["g++", "-shared", src, "-o", out, "-fopenmp", "-fPIC", "-O2", "-std=c++11"])
    return out


def build_upnp_ceres_ref():
    """oracle/upnp_ceres_ref.cpp (our restatement of the reference's residual functor) on top of the REFERENCE's vendored
    Ceres 2.0 headers (jet.h autodiff, rotation.h, tiny_solver.h LM) and Eigen, included where they lie; glog is stubbed
    (oracle/stubs).  libceres.so itself is absent, so the reference's own uncertainty_pnp.cpp cannot be linked."""
    inc = os.path.join(REF, "core/csrc/uncertainty_pnp/include")
    if not REF or not os.path.isdir(inc):
        return None
    os.makedirs(REFDIR, exist_ok=True)
    out = os.path.join(REFDIR, "libupnp_ceres_ref.so")
    src = os.path.join(HERE, "upnp_ceres_ref.cpp")
    if not os.path.exists(out) or os.path.getmtime(out) < os.path.getmtime(src):
        run(["g++", "-O2", "-std=c++14", "-w", "-shared", "-fPIC", "-I", os.path.join(HERE, "stubs"), "-I", inc,
             "-I", os.path.join(inc, "eigen3"), src, "-o", out])
    return out


CUDA_EXTS = {
    "ransac_voting": ["core/csrc/ransac_voting/src/ransac_voting.cpp", "core/csrc/ransac_voting/src/ransac_voting_kernel.cu"],
    "torch_nndistance_aten": ["core/csrc/torch_nndistance/src/nnd_cuda.cpp", "core/csrc/torch_nndistance/src/nnd_cuda_kernel.cu"],
    "flow_cuda": ["core/csrc/flow/src/flow_cuda_kernel.cu", "core/csrc/flow/src/flow_cuda.cpp"],
}


def build_cuda_refs(names=None):
    if not REF or not os.path.isdir(REF):
        return {}
    os.environ.setdefault("TORCH_CUDA_ARCH_LIST", "9.0a")
    os.environ.setdefault("MAX_JOBS", "4")
    from torch.utils.cpp_extension import load

    built = {}
    for name, srcs in CUDA_EXTS.items():
        if names and name not in names:
            continue
        bdir = os.path.join(REFDIR, name)
        so = os.path.join(bdir, name + ".so")
        if os.path.exists(so):
            built[name] = so
            continue
        os.makedirs(bdir, exist_ok=True)
        extra_inc = [os.path.join(REF, os.path.dirname(srcs[0]))]
        try:
            load(name=name, sources=[os.path.join(REF, s) for s in srcs], extra_include_paths=extra_inc,
                 extra_cuda_cflags=["-gencode", "arch=compute_90a,code=sm_90a"], build_directory=bdir,
                 with_cuda=True, is_python_module=False, verbose=False)
        except Exception as e:  # loading a CUDA .so can fail on a CPU-only box after a successful build
            if not os.path.exists(so):
                raise
            print(f"[build_ref] {name}: built, load skipped ({type(e).__name__})")
        built[name] = so
    return built


if __name__ == "__main__":
    print(build_oracle_ops())
    print(build_fps_ref())
    print(build_upnp_ceres_ref())
    if "--cuda-refs" in sys.argv:
        print(build_cuda_refs())
