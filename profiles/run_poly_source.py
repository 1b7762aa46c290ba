"""Source tables on the device (pinn_set_source_terms, DESIGN §4.8): what a forced user-defined PDE pays per redraw.

POLY_INF on the net [2, 20 x 8, 1] with the heat residual u_t - 0.5 u_xx and the manufactured forcing of u = sin(pi x) e^-t,
s = (0.5 pi^2 - 1) sin(pi x) e^-t, at N_f = 100 000 and 2 000 000:
  (a) resident: the Adam step on a set that stays on the device;
  (b) device:   an LHS draw, the device source (the table follows the new set) and the step;
  (c) host:     an LHS draw, the host round trip a callable source takes (pinn_get_collocation, s in numpy,
                pinn_set_source) and the step;
  (d) source:   the source kernel alone (pinn_set_source_terms on the stored set);
  (e) rad:      one pinn_draw_collocation_rad call with the table (N_f = 100 000 picks, k = 1, c = 1) from a pool of 100 000 and
                of 1 000 000 points, with its per-kernel split from torch.profiler in a process of its own.
(a), (b), (d) and (e) are device-event times around each call; (c) is a host clock around the call, which ends in a device
synchronisation (its read-back), so it counts the host's share too.  Every shape is warmed up first; each number is the median of
`--steps` calls, alternated in two rounds.  The card's name and power limit are read in the same run.  Run from the repository
root; prints one JSON object and, with --out DIR, writes it to DIR/run_poly_source_h100.json."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.getcwd()
sys.path[:0] = [ROOT, os.path.join(ROOT, "pinns-tf2.0_b200", "utils")]
import pinn_cabi  # noqa: E402
import poly_spec  # noqa: E402
from bench import init_weights  # noqa: E402
from oracle import lhs_draw as ld  # noqa: E402

NET = [2] + 8 * [20] + [1]
LB, UB = np.array([-1.0, 0.0]), np.array([1.0, 1.0])
K = 0.5
SOURCE = "(k*pi**2 - 1)*sin(pi*x)*exp(-t)"
LR = 1e-3
T0 = time.perf_counter()
KERNELS = {"pool_draw": ("lhs", "draw_kernel"), "pool_forward": ("mlp_forward_generic",),
           "pool_head": ("source", "pool_head_kernel"), "quantise": ("rad", "quantise_kernel"), "pick": ("rad", "pick_kernel"),
           "source_eval": ("source", "eval_kernel")}


def table():
    return poly_spec.parse_source(SOURCE, {"k": K}.get)


def host_source(x, t):
    return (K * np.pi ** 2 - 1) * np.sin(np.pi * x) * np.exp(-t)


def handle(n_f, with_table=True):
    x0 = np.linspace(-1, 1, 100)[:, None]
    p = pinn_cabi.Pinn(pinn_cabi.POLY_INF, NET, LB, UB)
    p.set_residual([(1.0, 0, (0, 0, 1, 0)), (-K, 0, (0, 0, 0, 1))])
    p.set_data(np.hstack([x0, 0 * x0]), np.sin(np.pi * x0))
    p.set_collocation(*ld.lhs_draw(3, 0, n_f, 0, n_f, LB, UB))
    if with_table:
        p.set_source_terms(table())
    p.set_weights(init_weights(NET))
    return p


def log(*msg):
    print("[run_poly_source %.0f s]" % (time.perf_counter() - T0), *msg, file=sys.stderr, flush=True)


def device_ms(p, steps, body):
    """Per-call device times (ms) of body(i), CUDA events on the handle's stream around each call."""
    for i in range(steps):
        p.event_record(2 * i)
        body(i)
        p.event_record(2 * i + 1)
    p.sync()
    return [p.event_elapsed_ms(2 * i, 2 * i + 1) for i in range(steps)]


def host_ms(p, steps, body):
    out = []
    for i in range(steps):
        p.sync()
        t0 = time.perf_counter()
        body(i)
        p.sync()
        out.append((time.perf_counter() - t0) * 1e3)
    return out


def stats(v):
    return {"median_ms": float(np.median(v)), "p10_p90_ms": [float(np.percentile(v, 10)), float(np.percentile(v, 90))]}


def measure(n_f, steps):
    p, q = handle(n_f), handle(n_f, with_table=False)
    step = lambda i: p.adam_step(LR, sync=False)                                           # noqa: E731

    def device(i):
        p.draw_collocation(7, 1 + i, n_f)
        p.adam_step(LR, sync=False)

    def host(i):
        q.draw_collocation(7, 1 + i, n_f)
        x, t = q.get_collocation()
        q.set_source(host_source(x, t))
        q.adam_step(LR, sync=False)

    src = lambda i: p.set_source_terms(table())                                             # noqa: E731
    timers = {"a_resident": (device_ms, p, step), "b_draw_device_source_step": (device_ms, p, device),
              "c_draw_host_round_trip_step": (host_ms, q, host), "d_source_kernel": (device_ms, p, src)}
    for fn, h, body in timers.values():
        fn(h, 10, body)
    got = {k: [] for k in timers}
    for _ in range(2):
        for k, (fn, h, body) in timers.items():
            got[k] += fn(h, steps, body)
    p.close(); q.close()
    row = {"n_f": n_f, "steps": steps}
    row.update({k: stats(v) for k, v in got.items()})
    a = row["a_resident"]["median_ms"]
    row["b_over_a"] = row["b_draw_device_source_step"]["median_ms"] / a
    row["c_over_a"] = row["c_draw_host_round_trip_step"]["median_ms"] / a
    return row


def measure_rad(n_pool, steps):
    n_f = 100000
    p = handle(n_f)
    rad = lambda i: p.draw_collocation_rad(7, 1000 + i, n_f, n_pool)                       # noqa: E731
    device_ms(p, 10, rad)
    v = device_ms(p, steps, rad) + device_ms(p, steps, rad)
    p.close()
    return dict(n_f=n_f, n_pool=n_pool, steps=steps, **{"e_rad_call": stats(v)})


def kernel_split(n_pool, calls=30):
    """Mean device time (ms) per RAD call of each of its kernels, from torch.profiler."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    n_f = 100000
    p = handle(n_f)
    for i in range(5):
        p.draw_collocation_rad(7, i, n_f, n_pool)
    p.sync()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for i in range(calls):
            p.draw_collocation_rad(7, 100 + i, n_f, n_pool)
        p.sync()
    p.close()
    out = {k: 0.0 for k in KERNELS}
    for e in prof.key_averages():
        total_us = getattr(e, "device_time_total", None)
        if total_us is None:
            total_us = e.cuda_time_total
        for k, parts in KERNELS.items():
            if all(s in e.key for s in parts):
                out[k] += total_us / 1e3 / calls
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--out", default=None)
    ap.add_argument("--split", type=int, default=None, help="(internal) print the kernel split of one pool size and exit")
    args = ap.parse_args()
    if args.split:
        print(json.dumps(kernel_split(args.split)))
        return
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip().splitlines()
    rows = []
    for n in (100000, 2000000):
        rows.append(measure(n, args.steps))
        log("cost", rows[-1])
    rad = []
    for n_pool in (100000, 1000000):
        rad.append(measure_rad(n_pool, args.steps))
        split = subprocess.run([sys.executable, os.path.abspath(__file__), "--split", str(n_pool)], capture_output=True,
                               text=True, check=True)
        rad[-1]["e_split_ms"] = json.loads(split.stdout.strip().splitlines()[-1])
        log("rad", rad[-1])
    out = {"card": card[0] if card else "unknown", "net": NET, "residual": "u_t - 0.5 u_xx", "source": SOURCE, "rows": rows,
           "rad": rad}
    print(json.dumps(out))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "run_poly_source_h100.json"), "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
