"""CPU: the built library's Navier-Stokes fused kernel runs its GEMMs on Hopper's 16x8 FP64 MMA shape, keeps every value in
registers (no stack frame) and stays within the register bound of one 256-thread CTA per SM (__launch_bounds__(256, 1))."""
import re
import subprocess

NS_KERNEL = "_ZN4pinn4nsid15fused_loss_gradENS0_4ArgsE"


def _functions(out):
    parts = re.split(r"\n\s*Function : (\S+)\n", out)
    return {parts[i]: parts[i + 1] for i in range(1, len(parts), 2)}


def test_ns_kernel_uses_dmma_16x8(lib_built):
    out = subprocess.run(["cuobjdump", "-sass", "-fun", NS_KERNEL, lib_built], capture_output=True, text=True).stdout
    body = _functions(out)[NS_KERNEL]
    assert "DMMA.16x8x4" in body
    assert "DMMA.8x8x4" not in body


def test_ns_kernel_resources(lib_built):
    out = subprocess.run(["cuobjdump", "-res-usage", lib_built], capture_output=True, text=True).stdout
    m = re.search(r"Function " + NS_KERNEL + r":\s*\n\s*REG:(\d+) STACK:(\d+)", out)
    assert m, "NS fused kernel not found"
    regs, stack = int(m.group(1)), int(m.group(2))
    assert stack == 0 and regs <= 255
