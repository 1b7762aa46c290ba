"""Build compile-time variants of libpinn_b200.so (nvcc needs no GPU) and time them on the GPU.

    python profiles/kernel_variants.py build            # nvcc cross-compiles every variant into pinns-tf2.0_b200/lib/variants/
    python profiles/kernel_variants.py time [n_f ...]   # on the GPU: one subprocess per variant (PINN_LIB=...), JSON lines

Variants whose name starts with "abl_" are timing ablations (they compute wrong gradients on purpose).  "phase_clocks" prints
per-warp cycle counts per phase of the Burgers kernel (PINN_PHASE_CLOCKS in csrc/burgers_fused_v2.cuh); `time` reports their
mean over the reporting warps of the last launch (an Adam step at the last size) as "phase_cycles".  The first line of `time` is the GPU's name, power limit and
SM clock (read-only nvidia-smi query); every variant also reports the SM clock sampled while it was timed ("clocks")."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "pinns-tf2.0_b200")
VDIR = os.path.join(PKG, "lib", "variants")
VARIANTS = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "kernel_variants.json")))


def build():
    sys.path.insert(0, PKG)
    import build as pinn_build
    from concurrent.futures import ThreadPoolExecutor
    def one(kv):
        name, flags = kv
        out = os.path.join(VDIR, "libpinn_b200_%s.so" % name)
        pinn_build.build(out=out, extra_flags=flags)
        return name
    with ThreadPoolExecutor(4) as ex:
        for n in ex.map(one, VARIANTS.items()):
            print("built", n, flush=True)


WORKER = r'''
import json, os, sys
import numpy as np
ROOT = %r
for p in (ROOT, os.path.join(ROOT, "pinns-tf2.0_b200", "utils")):
    sys.path.insert(0, p)
import pinn_cabi, bench
name = sys.argv[1]
clocks = bench.ClockSampler(0)
out = {"variant": name}
g = np.load(os.path.join(ROOT, "tests", "golden", "burgers_inf.npz"))
p = pinn_cabi.Pinn(pinn_cabi.BURGERS_INF, bench.LAYERS, g["lb"], g["ub"])
p.set_pde_params([float(g["nu"])]); p.set_collocation(g["X_f"][:, 0], g["X_f"][:, 1]); p.set_data(g["X_u"], g["u"])
loss, grad, _ = p.loss_grad(w=g["w"])
out["rel_loss"] = abs(loss - float(g["loss"])) / abs(float(g["loss"]))
out["rel_grad"] = float(np.linalg.norm(grad - g["grad"]) / np.linalg.norm(g["grad"]))
p.close()
for n_f in [int(v) for v in sys.argv[2:]] or [100000]:
    X_f, X_u, u = bench.synthetic_problem(1234, n_f)
    p = pinn_cabi.Pinn(pinn_cabi.BURGERS_INF, bench.LAYERS, bench.LB, bench.UB)
    p.set_pde_params([bench.NU]); p.set_data(X_u, u); p.set_collocation(X_f[:, 0], X_f[:, 1]); p.set_weights(bench.init_weights())
    p.time_kernel_ms(5)
    with clocks:
        ks = [p.time_kernel_ms(20) / 20 for _ in range(5)]
    for _ in range(10):
        p.adam_step(1e-3, sync=False)
    p.sync()
    ss = []
    for _ in range(3):
        p.event_record(0)
        for _ in range(50):
            p.adam_step(1e-3, sync=False)
        p.event_record(1)
        ss.append(p.event_elapsed_ms(0, 1) / 50)
    out["n_f=%%d" %% n_f] = {"kernel_ms_min": min(ks), "kernel_ms_med": float(np.median(ks)), "adam_step_ms_min": min(ss),
                             "frac_fp64_peak": (n_f * bench.FLOP_PER_COLLOC + 100 * bench.FLOP_PER_DATA) / (min(ks) * 1e-3) / (bench.FP64_PEAK_TFLOPS_DATASHEET * 1e12)}
    out["kernel_info"] = p.kernel_info()
    p.close()
out["clocks"] = clocks.summary()
sys.stdout.flush()
import ctypes
ctypes.CDLL(None).fflush(None)      # device printf output (phase_clocks) goes through the C library's stdout buffer
print(json.dumps(out))
''' % ROOT


PHASES = ["fwd_gemm", "fwd_act", "out", "bwd_act", "bwd_gemm", "wait"]


def phase_summary(lines):
    """'phase <cta> <warp> <6 cycle counts>' lines -> mean cycles per launch and phase of chain (warps 0-3) and weight-gradient
    warps (4-7; phase fwd_gemm = their DMMA tasks); each (cta, warp) contributes its last launch"""
    last = {}
    for ln in lines:
        f = ln.split()
        last[(int(f[1]), int(f[2]))] = [int(v) for v in f[3:9]]
    out = {}
    for role, warps in (("chain", range(4)), ("wgrad", range(4, 8))):
        rows = [v for (cta, w), v in last.items() if w in warps]
        if rows:
            out[role] = {PHASES[k]: sum(r[k] for r in rows) / len(rows) for k in range(6)}
            out[role]["total"] = sum(out[role].values())
    return out


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader,nounits"], capture_output=True, text=True,
                           timeout=20).stdout.strip().splitlines()
        return [dict(zip(q.split(","), [v.strip() for v in ln.split(",")])) for ln in r]
    except Exception as e:
        return repr(e)


def time_all(argv):
    print(json.dumps({"gpu": gpu_info()}), flush=True)
    names = [n for n in VARIANTS]
    sizes = [a for a in argv if a.isdigit()]
    only = [a for a in argv if not a.isdigit()]
    if only:
        names = [n for n in names if n in only]
    for n in names:
        lib = os.path.join(VDIR, "libpinn_b200_%s.so" % n)
        if not os.path.exists(lib):
            print(json.dumps({"variant": n, "error": "not built"}), flush=True)
            continue
        env = dict(os.environ, PINN_LIB=lib)
        r = subprocess.run([sys.executable, "-c", WORKER, n] + sizes, env=env, capture_output=True, text=True, timeout=600)
        lines = r.stdout.strip().splitlines()
        res = [ln for ln in lines if ln.startswith("{")]
        if not res:
            print(json.dumps({"variant": n, "error": r.stderr[-400:]}), flush=True)
            continue
        out = json.loads(res[-1])
        phase = [ln for ln in lines if ln.startswith("phase ")]
        if phase:
            out["phase_cycles"] = phase_summary(phase)
        print(json.dumps(out), flush=True)


if __name__ == "__main__":
    if sys.argv[1] == "build":
        build()
    else:
        time_all(sys.argv[2:])
