"""In-tree build of the CUDA extensions (libb200env.so, libb200nn.so) for sm_90a (H100).  nvcc cross-compiles
without a GPU."""
import os
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
SRCS = [os.path.join(HERE, "csrc", "b200env.cu"), os.path.join(HERE, "csrc", "b200env_v2p.cu")]
HDRS = [os.path.join(os.path.dirname(HERE), "include", h) for h in ("b200env.h", "b200env_v2p.h", "b200ball.h")] + [os.path.join(HERE, "csrc", f) for f in ("packed.cuh", "packed_t.cuh", "ballgen.cuh", "dyn_common.cuh", "counter_rng.cuh")]
LIB_DIR = os.path.join(HERE, "lib")
LIB = os.environ.get("B200ENV_LIB", os.path.join(LIB_DIR, "libb200env.so"))  # override: A/B kernel variants
# the network forwards of SURVEY.md 8f-1 (wgmma GEMMs): a library of their own, include/b200nn.h
SRCS_NN = [os.path.join(HERE, "csrc", "b200nn.cu")]
HDRS_NN = [os.path.join(os.path.dirname(HERE), "include", "b200nn.h"), os.path.join(HERE, "csrc", "counter_rng.cuh")]
LIB_NN = os.environ.get("B200NN_LIB", os.path.join(LIB_DIR, "libb200nn.so"))

NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17", "--shared",
              "-Xcompiler", "-fPIC", "-diag-suppress", "177,550"]


def needs_build(lib=None, deps=None):
    lib = LIB if lib is None else lib
    deps = SRCS + HDRS if deps is None else deps
    if not os.path.exists(lib):
        return True
    t = os.path.getmtime(lib)
    return any(os.path.getmtime(p) > t for p in deps)


def _nvcc(lib, srcs, verbose):
    os.makedirs(LIB_DIR, exist_ok=True)
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    cmd = [nvcc] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-o", lib] + srcs
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("nvcc failed:\n" + r.stdout + r.stderr)
    if verbose:
        print(r.stderr)


def build(force=False, verbose=False):
    """libb200env.so and libb200nn.so, both for sm_90a, in-tree"""
    if force or needs_build():
        _nvcc(LIB, SRCS, verbose)
    if force or needs_build(LIB_NN, SRCS_NN + HDRS_NN):
        _nvcc(LIB_NN, SRCS_NN, verbose)
    return LIB


if __name__ == "__main__":
    print(build(force=True, verbose=True))
