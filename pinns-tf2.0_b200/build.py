"""Build recipe for libpinn_b200.so (sm_90a only: H100; built in-tree, next to the package that loads it).

    python pinns-tf2.0_b200/build.py [--force]
"""
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB_DIR = os.path.join(HERE, "lib")
LIB = os.path.join(LIB_DIR, "libpinn_b200.so")
SOURCES = ["pinn_api.cu"]
HEADERS = ["pinn_common.cuh", "burgers_fused.cuh", "burgers_fused_v2.cuh", "nls_fused.cuh", "generic_fused.cuh", "optim_kernels.cuh",
           "navier_stokes_fused.cuh", "lhs_draw.cuh", "rad_sample.cuh", "source_terms.cuh",
           os.path.join("..", "..", "include", "pinn_b200.h")]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
              "-Xcompiler", "-fPIC", "-shared"]


def _nvcc():
    return shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"


def up_to_date():
    if not os.path.exists(LIB):
        return False
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, s) for s in SOURCES + HEADERS] + [os.path.abspath(__file__)]
    return all(os.path.getmtime(d) <= t for d in deps)


def build(force=False, verbose=False, out=None, extra_flags=None):
    """out / extra_flags: build a variant of the library next to the product one (kernel experiments)."""
    if out is None and not force and up_to_date():
        return LIB
    os.makedirs(LIB_DIR, exist_ok=True)
    extra = os.environ.get("PINN_EXTRA_NVCC_FLAGS", "").split() + list(extra_flags or [])
    out = out or LIB
    os.makedirs(os.path.dirname(out), exist_ok=True)
    cmd = [_nvcc()] + NVCC_FLAGS + extra + (["-Xptxas", "-v"] if verbose else []) + \
          ["-o", out] + [os.path.join(CSRC, s) for s in SOURCES] + ["-lcudart", "-ldl"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("nvcc failed:\n" + " ".join(cmd) + "\n" + r.stdout + r.stderr)
    if verbose:
        print(r.stderr)
    return out


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
