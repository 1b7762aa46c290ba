"""CPU: libpinn_b200.so builds for sm_90a, loads, and exports every symbol include/pinn_b200.h declares.
No compute calls here (they need no GPU)."""
import ctypes
import os
import re
import subprocess

import pytest

from conftest import ROOT


def header_functions():
    src = open(os.path.join(ROOT, "include", "pinn_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    names = re.findall(r"\b(pinn_[a-z0-9_]+)\s*\(", src)
    return sorted(set(n for n in names if n not in ("pinn_log_cb",)))


def test_header_declares_the_survey_contract():
    names = header_functions()
    for need in ("pinn_create", "pinn_set_collocation", "pinn_set_data", "pinn_set_boundary", "pinn_set_weights",
                 "pinn_get_weights", "pinn_loss_grad", "pinn_adam_step", "pinn_lbfgs", "pinn_predict", "pinn_residual",
                 "pinn_sync", "pinn_destroy", "pinn_last_error"):
        assert need in names


def test_library_exports_every_declared_symbol(lib_built):
    lib = ctypes.CDLL(lib_built)
    for name in header_functions():
        assert hasattr(lib, name), f"{name} declared in include/pinn_b200.h but not exported"


def test_binding_covers_header(lib_built):
    import pinn_cabi
    assert sorted(pinn_cabi.SIGNATURES) == header_functions()
    pinn_cabi.load()


def test_sass_is_sm90a_with_dmma_and_tma(lib_built):
    out = subprocess.run(["cuobjdump", "-sass", lib_built], capture_output=True, text=True).stdout
    assert "sm_90a" in out
    assert "DMMA.8x8x4" in out          # FP64 tensor-core MMA in the fused kernel
    assert "UBLKCP" in out              # TMA bulk copy staging the weights


def test_create_fails_loudly_without_gpu(lib_built):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    import pinn_cabi
    with pytest.raises(pinn_cabi.PinnError, match="no CUDA device|no CPU fallback"):
        pinn_cabi.Pinn(pinn_cabi.BURGERS_INF, [2] + [20] * 8 + [1], [-1, 0], [1, 1])


def test_header_is_plain_c_and_links_from_c(lib_built, tmp_path):
    """include/pinn_b200.h compiles as strict C99 (gcc -std=c99 -pedantic -Werror) and a C program linked against the shared
    library gets the version string and, on a box without a GPU, a clean error code + message from pinn_create."""
    import shutil
    import subprocess
    if shutil.which("gcc") is None:
        pytest.skip("no gcc")
    exe = str(tmp_path / "c99_caller")
    libdir = os.path.dirname(os.path.realpath(lib_built))
    r = subprocess.run(["gcc", "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", "-I", os.path.join(ROOT, "include"),
                        os.path.join(ROOT, "tests", "cabi", "c99_caller.c"), "-o", exe, "-L", libdir, "-lpinn_b200",
                        "-Wl,-rpath," + libdir], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    import torch
    if torch.cuda.is_available():
        return                                   # with a GPU the creation succeeds; the GPU tests cover that path
    r = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0 and "pinn_b200" in r.stdout and "no CUDA device" in r.stdout, r.stdout + r.stderr


def test_fused_and_tail_kernels_fit_their_resource_budget(lib_built):
    """cuobjdump -res-usage of the built library: the two DMMA kernels are designed for one 256-thread CTA per SM with every
    value in registers -- no stack (spill) frame, at most 255 registers; the default Burgers kernel must stay at <= 252 so that
    8 warps fit the 64 K register file.  A regression here is a silent 2x slow-down, so it is pinned on the CPU.  The
    stand-alone tail kernel (reduce_tail) and adam_update stay at <= 64 registers without a stack."""
    out = subprocess.run(["cuobjdump", "-res-usage", lib_built], capture_output=True, text=True).stdout
    usage = {}
    for m in re.finditer(r"Function (\S+?):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:(\d+)", out):
        usage[m.group(1)] = tuple(int(v) for v in m.groups()[1:])
    def find(*parts):
        keys = [k for k in usage if all(p in k for p in parts)]
        assert len(keys) == 1, (parts, keys)
        return usage[keys[0]]
    regs, stack, _ = find("burgers2", "fused_loss_grad")
    assert regs <= 252 and stack == 0
    regs, stack, _ = find("3nls", "fused_loss_grad")
    assert regs <= 255 and stack == 0
    for name in ("reduce_tail", "adam_update"):
        regs, stack, _ = find(name)
        assert regs <= 64 and stack == 0
    regs, stack, _ = find("lbfgs_iterate", "ILi12ELi256E")        # the Burgers-size L-BFGS keeps its P-vector slice in registers
    assert stack == 0
