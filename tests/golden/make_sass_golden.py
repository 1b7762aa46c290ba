"""Per-function digests of the SASS that libpinn_b200.so carries for sm_90a -> tests/golden/kernel_sass.json.

    python tests/golden/make_sass_golden.py [path/to/libpinn_b200.so]

tests/test_kernel_sass_cpu.py rebuilds the library and requires every function listed here to keep its SASS.  A change that alters
a kernel on purpose regenerates this file, so its diff names exactly the functions whose machine code changed; a change that
should leave a kernel alone (host code, a new kernel) leaves its digest in place.  The digests depend on the CUDA toolkit, which
is recorded with them: under another nvcc the comparison is skipped."""
import hashlib
import json
import os
import re
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "kernel_sass.json")


def nvcc_build():
    nvcc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "nvcc")
    out = subprocess.run([nvcc if os.path.exists(nvcc) else "nvcc", "--version"], capture_output=True, text=True).stdout
    return [ln.strip() for ln in out.splitlines() if ln.startswith(("Cuda compilation tools", "Build "))]


def sass_digests(lib):
    """{mangled function name: sha1 of its SASS}, with the instruction-address comments (which move when code before the function
    grows) removed; branch targets are offsets within the function and stay."""
    out = subprocess.run(["cuobjdump", "-sass", lib], capture_output=True, text=True, check=True).stdout
    d = {}
    for blk in re.split(r"\n\s*Function : ", out)[1:]:
        name, body = blk.split("\n", 1)
        lines = [re.sub(r"/\*[0-9a-f]{4,}\*/", "", ln).strip() for ln in body.splitlines()]
        d[name.strip()] = hashlib.sha1("\n".join(lines).encode()).hexdigest()
    return d


if __name__ == "__main__":
    lib = sys.argv[1] if len(sys.argv) > 1 else os.path.join(HERE, "..", "..", "pinns-tf2.0_b200", "lib", "libpinn_b200.so")
    with open(GOLDEN, "w") as f:
        json.dump({"nvcc": nvcc_build(), "arch": "sm_90a", "functions": dict(sorted(sass_digests(lib).items()))}, f, indent=1)
        f.write("\n")
    print(GOLDEN)
