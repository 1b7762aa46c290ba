"""Multi-GPU parity check (run under torchrun on N GPUs; driven by tests/test_gpu_multi.py and by hand):
    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29511 tests/mgpu_check.py
Sharded loss/gradient/Adam/L-BFGS must match the single-GPU evaluation of the whole set -- through the fused NVLink push
exchange (exchange_block) AND through the NCCL path, for the Burgers and the Schrodinger kernels."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "pinns-tf2.0_b200", "utils")):
    sys.path.insert(0, p)
import pinn_cabi  # noqa: E402
import sharding  # noqa: E402


def rel(a, b):
    return float(np.linalg.norm(np.asarray(a) - np.asarray(b)) / np.linalg.norm(b))


def compare(tag, p, s, w, rank, world, adam=(1e-3, 0.9, 0.999, 1e-7), lbfgs_iters=8):
    l1, g1, _ = s.loss_grad(w=w)
    lN, gN, _ = p.loss_grad(w=w)
    assert abs(lN - l1) <= 1e-12 * abs(l1), (tag, lN, l1)
    assert rel(gN, g1) < 1e-12, (tag, rel(gN, g1))
    s.set_weights(w); p.set_weights(w)
    for _ in range(5):
        a1 = s.adam_step(*adam); aN = p.adam_step(*adam)
    assert abs(aN - a1) <= 1e-10 * abs(a1) and rel(p.get_weights(), s.get_weights()) < 1e-10, tag
    # asynchronous steps (no host sync between exchanges) give the same trajectory
    s.set_weights(w); p.set_weights(w); s.adam_reset(); p.adam_reset()
    for _ in range(20):
        s.adam_step(*adam, sync=False); p.adam_step(*adam, sync=False)
    assert abs(p.last_loss() - s.last_loss()) <= 1e-9 * abs(s.last_loss()) and rel(p.get_weights(), s.get_weights()) < 1e-9, tag
    s.set_weights(w); p.set_weights(w)
    eps = float(np.finfo(float).eps)
    r1 = s.lbfgs(lbfgs_iters, learning_rate=0.8, n_correction=50, tol_fun=eps, sync_every=3, want_x_final=True)
    rN = p.lbfgs(lbfgs_iters, learning_rate=0.8, n_correction=50, tol_fun=eps, sync_every=3, want_x_final=True)
    assert rN["n_iter"] == r1["n_iter"] and rN["n_eval"] == r1["n_eval"] and rel(rN["x_final"], r1["x_final"]) < 1e-8, tag
    # every rank holds identical weights (replicated optimiser state, no broadcast)
    wt = torch.from_numpy(p.get_weights())
    ws = [torch.empty_like(wt) for _ in range(world)]
    dist.all_gather(ws, wt)
    assert all(torch.equal(ws[0], x) for x in ws), tag
    return lN, rel(gN, g1), rN["n_iter"]


def burgers_case(rank, local_rank, world, uid):
    layers = [2] + [20] * 8 + [1]
    rng = np.random.default_rng(5)
    lb, ub = np.array([-1.0, 0.0]), np.array([1.0, 0.99])
    n_f = 40000
    X_f = lb + (ub - lb) * rng.random((n_f, 2))
    X_u = lb + (ub - lb) * rng.random((100, 2)); u = rng.uniform(-1, 1, (100, 1))
    w = np.load(os.path.join(ROOT, "tests", "golden", "burgers_inf.npz"))["w"]
    lo, hi = sharding.shard_rows(n_f, rank, world)
    p = pinn_cabi.Pinn(pinn_cabi.BURGERS_INF, layers, lb, ub, device=local_rank, rank=rank, world=world, nccl_uid=uid)
    used_p2p = sharding.connect_p2p(dist, p, world)
    p.set_pde_params([0.01 / np.pi])
    p.set_collocation(X_f[lo:hi, 0], X_f[lo:hi, 1], n_global=n_f)
    p.set_data(X_u, u, weight=sharding.data_weight(rank))
    s = pinn_cabi.Pinn(pinn_cabi.BURGERS_INF, layers, lb, ub, device=local_rank)      # the whole set on every rank's GPU
    s.set_pde_params([0.01 / np.pi]); s.set_collocation(X_f[:, 0], X_f[:, 1]); s.set_data(X_u, u)
    out = compare("burgers", p, s, w, rank, world)
    dist.barrier()
    p.close(); s.close()
    return used_p2p, out


def nls_case(rank, local_rank, world, uid):
    g = np.load(os.path.join(ROOT, "tests", "golden", "nls_inf.npz"))
    layers = [int(v) for v in g["layers"]]
    lb, ub = g["lb"], g["ub"]
    rng = np.random.default_rng(6)
    n_f = 6000
    X_f = lb + (ub - lb) * rng.random((n_f, 2))
    lo, hi = sharding.shard_rows(n_f, rank, world)
    p = pinn_cabi.Pinn(pinn_cabi.NLS_INF, layers, lb, ub, device=local_rank, rank=rank, world=world, nccl_uid=uid)
    used_p2p = sharding.connect_p2p(dist, p, world)
    p.set_collocation(X_f[lo:hi, 0], X_f[lo:hi, 1], n_global=n_f); p.set_boundary(g["tb"])
    p.set_data(g["x0"], g["uv0"], weight=sharding.data_weight(rank))
    s = pinn_cabi.Pinn(pinn_cabi.NLS_INF, layers, lb, ub, device=local_rank)
    s.set_collocation(X_f[:, 0], X_f[:, 1]); s.set_boundary(g["tb"]); s.set_data(g["x0"], g["uv0"])
    out = compare("nls", p, s, g["w"], rank, world, adam=(0.05, 0.99, 0.999, 0.1), lbfgs_iters=4)
    dist.barrier()
    p.close(); s.close()
    return used_p2p, out


def main():
    rank, local_rank, world = sharding.env_rank_world()
    torch.cuda.set_device(local_rank)
    dist.init_process_group("gloo")      # control plane only; the data-path NCCL communicator lives inside the library
    for mode in ("p2p", "nccl"):
        os.environ["PINN_COLLECTIVE"] = mode
        for case in (burgers_case, nls_case):
            uid = sharding.exchange_nccl_uid(dist, rank, pinn_cabi.nccl_unique_id)
            used_p2p, (loss, rg, its) = case(rank, local_rank, world, uid)
            if rank == 0:
                print(f"mgpu_check ok: {case.__name__} mode={mode} p2p={used_p2p} world={world} loss={loss:.12e} rel_grad={rg:.1e} "
                      f"lbfgs_iters={its}", flush=True)
            assert used_p2p == (mode == "p2p"), "the NVLink push exchange could not be set up"
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
