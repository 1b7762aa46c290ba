"""GPU: fused sm_90a Burgers kernel (through the C ABI) against the oracle golden vectors and, at full
BASELINE sizes, against the numpy Taylor oracle and size-independent properties.

Tolerances: the reference is fp64 and north_star asks 1e-5 (loss) / 1e-4 (u); the kernel computes in fp64 with a
different summation order, so single evaluations are held to 1e-10 and short optimiser trajectories to 1e-7."""
import numpy as np
import pytest

from conftest import assert_matches_reference_run, load_golden

pytestmark = pytest.mark.gpu

LAYERS = [2] + [20] * 8 + [1]


def rel(a, b):
    a, b = np.asarray(a, float), np.asarray(b, float)
    return np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300)


@pytest.fixture(scope="module")
def cabi():
    import pinn_cabi
    pinn_cabi.load()
    return pinn_cabi


def make_inf(cabi, g):
    p = cabi.Pinn(cabi.BURGERS_INF, LAYERS, g["lb"], g["ub"])
    p.set_pde_params([float(g["nu"])])
    p.set_collocation(g["X_f"][:, 0], g["X_f"][:, 1])
    p.set_data(g["X_u"], g["u"])
    p.set_weights(g["w"])
    return p


def test_loss_grad_matches_golden(cabi):
    g = load_golden("burgers_inf")
    p = make_inf(cabi, g)
    loss, grad, parts = p.loss_grad()
    assert abs(loss - g["loss"]) <= 1e-10 * abs(g["loss"])
    assert rel(grad, g["grad"]) < 1e-10
    assert np.allclose([parts[0], parts[2]], g["parts"], rtol=1e-10)
    assert_matches_reference_run(loss, grad, "burgers_inf_loss", "burgers_inf_grad")      # the reference's own code, executed
    # the closure form: pass the weights with the call (get_loss_and_flat_grad, neuralnetwork.py:91-103)
    loss2, grad2, _ = p.loss_grad(w=g["w"])
    assert loss2 == loss and np.array_equal(grad, grad2)       # deterministic reduction order
    assert p.launch_count() > 0


def test_derivative_probes_predict_residual(cabi):
    g = load_golden("burgers_inf")
    p = make_inf(cabi, g)
    U, Ux, Ut, Uxx = p.derivatives(g["X_f"][:64])
    assert rel(np.hstack([U, Ux, Ut, Uxx]), g["probes"]) < 1e-11
    assert rel(p.predict(g["X_star"]), g["predict"]) < 1e-12
    assert rel(p.residual(g["X_f"].shape[0]), g["residual"]) < 1e-10


def test_adam_trajectory(cabi):
    g = load_golden("burgers_inf")
    for k, lr in enumerate(g["adam_lr"]):
        p = make_inf(cabi, g)
        losses = [p.adam_step(float(lr)) for _ in range(5)]
        assert rel(losses, g["adam_losses"][k]) < 1e-8
        assert rel(p.get_weights(), g["adam_w"][k]) < 1e-8
        # async steps give the same trajectory as synchronous ones
        q = make_inf(cabi, g)
        for _ in range(5):
            q.adam_step(float(lr), sync=False)
        assert abs(q.last_loss() - losses[-1]) <= 1e-12 * abs(losses[-1])
        assert rel(q.get_weights(), p.get_weights()) < 1e-12


def test_lbfgs_trace_and_discarded_last_step(cabi):
    g = load_golden("burgers_inf")
    p = make_inf(cabi, g)
    logged = []
    r = p.lbfgs(6, learning_rate=0.8, n_correction=50, tol_fun=np.finfo(float).eps, tol_x=1e-19, sync_every=1,
                log_fn=lambda it, f: logged.append((it, f)), want_x_final=True)
    assert r["n_iter"] == int(g["lbfgs_n_iter"]) and r["n_eval"] == int(g["lbfgs_n_eval"])
    assert r["reason_str"] == "max iterations"
    assert [it for it, _ in logged] == [int(v) for v in g["lbfgs_logged"][:, 0]]
    assert rel([f for _, f in logged], g["lbfgs_logged"][:, 1]) < 1e-7
    assert rel(r["x_final"], g["lbfgs_x_final"]) < 1e-7
    # the model keeps the weights of the last EVALUATED point (custom_lbfgs.py:176-182, neuralnetwork.py:131-136)
    assert rel(p.get_weights(), g["lbfgs_x_eval"][-1]) < 1e-7
    # batched host sync gives the same result
    q = make_inf(cabi, g)
    r2 = q.lbfgs(6, learning_rate=0.8, n_correction=50, tol_fun=np.finfo(float).eps, sync_every=4, want_x_final=True)
    assert r2["n_iter"] == r["n_iter"] and rel(r2["x_final"], r["x_final"]) < 1e-12
    assert p.lbfgs(0)["n_iter"] == 0      # maxIter == 0 returns immediately (custom_lbfgs.py:43-44)


def test_identification_matches_golden(cabi):
    g = load_golden("burgers_ide")
    p = cabi.Pinn(cabi.BURGERS_IDE, LAYERS, g["lb"], g["ub"])
    assert p.P == 3023
    p.set_data(g["X_u"], g["u"])
    for wk, fk, gk in (("w", "loss", "grad"), ("w2", "loss2", "grad2")):
        loss, grad, _ = p.loss_grad(w=g[wk])
        assert abs(loss - g[fk]) <= 1e-10 * abs(g[fk])
        assert rel(grad, g[gk]) < 1e-10
        assert rel(grad[-2:], g[gk][-2:]) < 1e-9
        assert_matches_reference_run(loss, grad, "burgers_ide_" + fk, "burgers_ide_" + gk)
        assert np.allclose(p.get_params(), [g[wk][-2], np.exp(g[wk][-1])], rtol=1e-15)      # (lambda_1, exp(lambda_2))
    p.set_weights(g["w"])
    losses = [p.adam_step(1e-3) for _ in range(5)]
    assert rel(losses, g["adam_losses"]) < 1e-8 and rel(p.get_weights(), g["adam_w"]) < 1e-8
    p.set_weights(g["w"])
    r = p.lbfgs(5, learning_rate=0.8, n_correction=50, tol_fun=np.finfo(float).eps, want_x_final=True)
    assert r["n_iter"] == int(g["lbfgs_n_iter"]) and rel(r["x_final"], g["lbfgs_x_final"]) < 1e-7


@pytest.mark.parametrize("n_f,n_u", [(1, 1), (7, 3), (31, 0), (33, 100), (4736, 100), (10000, 100)])
def test_ragged_sizes_against_taylor_oracle(cabi, n_f, n_u):
    from oracle import taylor as ty
    rng = np.random.default_rng(n_f * 7 + n_u)
    lb, ub = np.array([-1.0, 0.0]), np.array([1.0, 0.99])
    X_f = lb + (ub - lb) * rng.random((n_f, 2))
    X_u = lb + (ub - lb) * rng.random((n_u, 2))
    u = rng.uniform(-1, 1, (n_u, 1))
    w = load_golden("burgers_inf")["w"]
    p = cabi.Pinn(cabi.BURGERS_INF, LAYERS, lb, ub)
    p.set_pde_params([0.01 / np.pi])
    p.set_collocation(X_f[:, 0], X_f[:, 1])
    p.set_data(X_u, u)
    loss, grad, _ = p.loss_grad(w=w)
    if n_u == 0:
        (U, Ux, Ut, Uxx), st = ty.forward(w, LAYERS, lb, ub, X_f)
        f = Ut + U * Ux - 0.01 / np.pi * Uxx
        c = 2 * f / n_f
        f2, g2 = float(np.sum(f * f) / n_f), ty.backward(w, LAYERS, st, (c * Ux, c * U, c, -c * 0.01 / np.pi))
    else:
        f2, g2, _ = ty.burgers_loss_grad(w, LAYERS, lb, ub, X_f, X_u, u, nu=0.01 / np.pi)
    assert abs(loss - f2) <= 1e-10 * abs(f2)
    assert rel(grad, g2) < 1e-10


def test_full_size_properties(cabi):
    """BASELINE configs[1] size (N_f = 100 000): parity with the numpy Taylor oracle, and the sharding property
    the multi-GPU path relies on: loss/grad of the whole set == sum over shards evaluated with n_global."""
    from oracle import taylor as ty
    rng = np.random.default_rng(99)
    lb, ub = np.array([-1.0, 0.0]), np.array([1.0, 0.99])
    n_f = 100000
    X_f = lb + (ub - lb) * rng.random((n_f, 2))
    X_u = lb + (ub - lb) * rng.random((100, 2)); u = rng.uniform(-1, 1, (100, 1))
    w = load_golden("burgers_inf")["w"]
    p = cabi.Pinn(cabi.BURGERS_INF, LAYERS, lb, ub)
    p.set_pde_params([0.01 / np.pi]); p.set_data(X_u, u)
    p.set_collocation(X_f[:, 0], X_f[:, 1])
    loss, grad, _ = p.loss_grad(w=w)
    f2, g2, _ = ty.burgers_loss_grad(w, LAYERS, lb, ub, X_f, X_u, u, nu=0.01 / np.pi)
    assert abs(loss - f2) <= 1e-10 * abs(f2) and rel(grad, g2) < 1e-10
    tot_l, tot_g = 0.0, np.zeros_like(grad)
    for r, (a, b) in enumerate([(0, 37000), (37000, 100000)]):
        p.set_collocation(X_f[a:b, 0], X_f[a:b, 1], n_global=n_f)
        p.set_data(X_u, u, weight=1.0 if r == 0 else 0.0)
        l, g, _ = p.loss_grad(w=w)
        tot_l += l; tot_g += g
    assert abs(tot_l - loss) <= 1e-12 * abs(loss) and rel(tot_g, grad) < 1e-12


def test_errors_are_reported_not_thrown(cabi):
    with pytest.raises(cabi.PinnError, match="1 network output"):
        cabi.Pinn(cabi.BURGERS_INF, [2, 10, 2], [-1, 0], [1, 1])
    with pytest.raises(cabi.PinnError, match="width out of range"):
        cabi.Pinn(cabi.BURGERS_INF, [2, 300, 1], [-1, 0], [1, 1])
    with pytest.raises(cabi.PinnError, match="input dimension"):
        cabi.Pinn(cabi.BURGERS_INF, [3, 10, 1], [-1, 0], [1, 1])
    p = cabi.Pinn(cabi.BURGERS_INF, LAYERS, [-1, 0], [1, 1])
    with pytest.raises(cabi.PinnError, match="expected 3021"):
        p.set_weights(np.zeros(5))
    with pytest.raises(cabi.PinnError, match="no points"):
        p.loss_grad()


def test_device_tanh_accuracy(cabi):
    """The kernels' branch-free tanh: <= 4 ulp against libm over the whole range, exact limits, odd symmetry."""
    xs = np.concatenate([np.linspace(-25, 25, 200001), np.logspace(-300, 1.4, 20001), -np.logspace(-300, 1.4, 20001),
                         [0.0, 1e300, -1e300, 5e-324]])
    got = cabi.device_tanh(xs)
    ref = np.tanh(xs)
    ulp = np.abs(got - ref) / np.spacing(np.maximum(np.abs(ref), 5e-324))
    assert ulp.max() <= 4.0
    assert got[-3] == 1.0 and got[-2] == -1.0 and got[-4] == 0.0
    assert np.array_equal(cabi.device_tanh(-xs), -got)
    # non-finite and edge inputs: quiet NaNs of both signs with payloads give NaN (libm's tanh), +-Inf and +-(20 +- ulp) give
    # exactly +-1, +-0 keeps its sign, the smallest denormal stays within 4 ulp
    nans = np.array([0x7FF8000000000000, 0xFFF8000000000000, 0x7FF800000000BEEF, 0xFFFC0000DEAD0001], dtype=np.uint64).view(np.float64)
    assert np.all(np.isnan(cabi.device_tanh(nans)))
    sat = np.array([np.inf, -np.inf, 20.0, -20.0, np.nextafter(20.0, 0), -np.nextafter(20.0, 0), np.nextafter(20.0, 30),
                    -np.nextafter(20.0, 30)])
    assert np.array_equal(cabi.device_tanh(sat), np.sign(sat))
    z = cabi.device_tanh(np.array([0.0, -0.0]))
    assert np.array_equal(z, [0.0, 0.0]) and not np.signbit(z[0]) and np.signbit(z[1])
    tiny = np.array([5e-324, -5e-324])
    assert np.all(np.abs(cabi.device_tanh(tiny) - np.tanh(tiny)) <= 4 * 5e-324)


def test_zero_copy_collocation_matches_copied_and_sees_host_updates(cabi):
    """pinn_set_collocation_mapped: the fused kernel reads the pinned batch over PCIe.  Same loss/gradient as the copied
    path, and a batch rewritten in place by the host is what the next launch sees (no stale device-side caching)."""
    import ctypes as C
    g = load_golden("burgers_inf")
    n = g["X_f"].shape[0]
    hx, hx_ptr = cabi.host_alloc(n); ht, ht_ptr = cabi.host_alloc(n)
    dp = C.POINTER(C.c_double)
    hx[:] = g["X_f"][:, 0]; ht[:] = g["X_f"][:, 1]
    p = make_inf(cabi, g)
    l_copy, g_copy, _ = p.loss_grad()
    p.set_collocation_mapped(C.cast(hx_ptr, dp), C.cast(ht_ptr, dp), n)
    l_map, g_map, _ = p.loss_grad()
    assert l_map == l_copy and np.array_equal(g_map, g_copy)
    assert rel(p.residual(n), g["residual"]) < 1e-10
    # new batch written in place
    rng = np.random.default_rng(3)
    Xn = g["lb"] + (g["ub"] - g["lb"]) * rng.random((n, 2))
    hx[:] = Xn[:, 0]; ht[:] = Xn[:, 1]
    p.set_collocation_mapped(C.cast(hx_ptr, dp), C.cast(ht_ptr, dp), n)
    l_new, g_new, _ = p.loss_grad()
    q = make_inf(cabi, g)
    q.set_collocation(Xn[:, 0], Xn[:, 1])
    l_ref, g_ref, _ = q.loss_grad()
    assert l_new == l_ref and np.array_equal(g_new, g_ref) and l_new != l_copy
    # switching back to the copied path drops the mapping
    p.set_collocation(g["X_f"][:, 0], g["X_f"][:, 1])
    assert p.loss_grad()[0] == l_copy
    p.close(); q.close()


def test_mapped_collocation_first_then_growing_data_block(cabi):
    """Regression (ADVICE r1): a fresh handle whose ONLY collocation set is a zero-copy mapping has no device collocation
    region (capacity 0); growing the data block afterwards must not copy n_c doubles out of it.  (Now one case of the seeded
    histories of tests/test_gpu_handle_state.py: "data region regrown under a mapped batch".)"""
    import ctypes as C
    rng = np.random.default_rng(21)
    lb, ub = np.array([-1.0, 0.0]), np.array([1.0, 0.99])
    n = 100000
    Xf = lb + (ub - lb) * rng.random((n, 2))
    Xu = lb + (ub - lb) * rng.random((2000, 2)); u = rng.uniform(-1, 1, (2000, 1))
    w = load_golden("burgers_inf")["w"]
    hx, hx_ptr = cabi.host_alloc(n); ht, ht_ptr = cabi.host_alloc(n)
    hx[:] = Xf[:, 0]; ht[:] = Xf[:, 1]
    dp = C.POINTER(C.c_double)
    p = cabi.Pinn(cabi.BURGERS_INF, LAYERS, lb, ub)
    p.set_pde_params([0.01 / np.pi])
    p.set_collocation_mapped(C.cast(hx_ptr, dp), C.cast(ht_ptr, dp), n)     # before any device-resident set exists
    p.set_data(Xu, u)                                                       # 2000 rows > the initial data capacity: regrow
    l_map, g_map, _ = p.loss_grad(w=w)
    q = cabi.Pinn(cabi.BURGERS_INF, LAYERS, lb, ub)
    q.set_pde_params([0.01 / np.pi]); q.set_data(Xu, u); q.set_collocation(Xf[:, 0], Xf[:, 1])
    l_ref, g_ref, _ = q.loss_grad(w=w)
    assert l_map == l_ref and np.array_equal(g_map, g_ref)
    # ... and the reverse order of growth: a larger copied set after the mapping was dropped
    p.set_collocation(Xf[:50000, 0], Xf[:50000, 1])
    q.set_collocation(Xf[:50000, 0], Xf[:50000, 1])
    assert p.loss_grad(w=w)[0] == q.loss_grad(w=w)[0]
    p.close(); q.close()


def test_residual_buffer_is_sized_by_the_library(cabi):
    """pinn_residual takes the row count of the caller's buffer and refuses a mismatch (ADVICE r1: it used to write n_c rows
    into whatever it was given).  (That a refused call leaves the handle as it was is tests/test_gpu_handle_state.py's.)"""
    import ctypes as C
    g = load_golden("burgers_inf")
    p = make_inf(cabi, g)
    n = g["X_f"].shape[0]
    assert p.residual().shape == (n, 1) and p.residual(n).shape == (n, 1)
    with pytest.raises(cabi.PinnError, match="residual points are stored"):
        p.residual(n - 1)
    small = np.empty(n - 1)
    rc = p.lib.pinn_residual(p.h, small.ctypes.data_as(C.POINTER(C.c_double)), n - 1)
    assert rc != 0 and b"rows" in p.lib.pinn_last_error()
    p.close()


def test_small_sets_use_fewer_chain_warps_per_cta(cabi):
    """N = 2000 identification (BASELINE configs[3] size): 250 tiles run as 125 CTAs x 2 chain warps; results are those of the
    Taylor oracle, and of the same points evaluated inside a large launch (different tile -> CTA mapping)."""
    from oracle import taylor as ty
    rng = np.random.default_rng(17)
    lb, ub = np.array([-1.0, 0.0]), np.array([1.0, 0.99])
    X = lb + (ub - lb) * rng.random((2000, 2)); u = rng.uniform(-1, 1, (2000, 1))
    w = np.concatenate([load_golden("burgers_inf")["w"], [0.3, -5.0]])
    p = cabi.Pinn(cabi.BURGERS_IDE, LAYERS, lb, ub)
    p.set_data(X, u)
    loss, grad, _ = p.loss_grad(w=w)
    f2, g2, _ = ty.burgers_loss_grad(w, LAYERS, lb, ub, None, X, u, identification=True)
    assert abs(loss - f2) <= 1e-10 * abs(f2) and rel(grad, g2) < 1e-10
    X3, u3 = np.vstack([X, 0.9 * X, 0.8 * X]), np.vstack([u, u, u])
    sms = p.kernel_info()["sms"]
    # around the chains-per-CTA switch points (one and four 8-point tiles per SM: 132 and 528 tiles on an H100)
    for n in (8, 9, 300, 8 * sms, 8 * sms + 1, 32 * sms - 1, 32 * sms + 1):
        p.set_data(X3[:n], u3[:n])
        l, gr, _ = p.loss_grad(w=w)
        f2, g2, _ = ty.burgers_loss_grad(w, LAYERS, lb, ub, None, X3[:n], u3[:n], identification=True)
        assert abs(l - f2) <= 1e-10 * abs(f2) and rel(gr, g2) < 1e-10, n
    p.close()


def test_quarter_million_point_shard(cabi):
    """BASELINE configs[4] per-GPU share (2 000 000 points over 8 GPUs = 250 000 per rank, MSE_f weighted by the GLOBAL count)
    against the numpy Taylor oracle."""
    from oracle import taylor as ty
    rng = np.random.default_rng(250)
    lb, ub = np.array([-1.0, 0.0]), np.array([1.0, 0.99])
    n = 250000
    X_f = lb + (ub - lb) * rng.random((n, 2))
    X_u = lb + (ub - lb) * rng.random((100, 2)); u = rng.uniform(-1, 1, (100, 1))
    w = load_golden("burgers_inf")["w"]
    p = cabi.Pinn(cabi.BURGERS_INF, LAYERS, lb, ub)
    p.set_pde_params([0.01 / np.pi]); p.set_data(X_u, u, weight=0.0)
    p.set_collocation(X_f[:, 0], X_f[:, 1], n_global=2000000)
    loss, grad, parts = p.loss_grad(w=w)
    f2, g2, _ = ty.burgers_loss_grad(w, LAYERS, lb, ub, X_f, X_u, u, nu=0.01 / np.pi, n_f_global=2000000, data_weight=0.0)
    assert abs(loss - f2) <= 1e-10 * abs(f2) and rel(grad, g2) < 1e-10 and parts[0] == 0.0
    p.close()


def test_gram_formulation_of_lbfgs_matches_the_literal_loop_on_short_runs():
    """PINN_LBFGS=gram (opt-in; see pinn_api.cu and DESIGN.md section 4.3): the golden
    6-iteration trace and a 60-iteration run with history overflow (n_corr = 7) against the default literal kernel."""
    import os
    import subprocess
    import sys
    from conftest import ROOT
    code = r'''
import os, sys, json, numpy as np
ROOT = %r
sys.path[:0] = [ROOT, os.path.join(ROOT, "pinns-tf2.0_b200", "utils")]
import pinn_cabi
g = np.load(os.path.join(ROOT, "tests", "golden", "burgers_inf.npz"))
out = {}
for n_corr, its in ((50, 6), (7, 60)):
    p = pinn_cabi.Pinn(pinn_cabi.BURGERS_INF, [2] + [20] * 8 + [1], g["lb"], g["ub"])
    p.set_pde_params([float(g["nu"])]); p.set_collocation(g["X_f"][:, 0], g["X_f"][:, 1]); p.set_data(g["X_u"], g["u"]); p.set_weights(g["w"])
    r = p.lbfgs(its, learning_rate=0.8, n_correction=n_corr, tol_fun=float(np.finfo(float).eps), sync_every=4, want_x_final=True)
    out[str(n_corr)] = {"f": r["f_hist"], "x": r["x_final"].tolist(), "n_iter": r["n_iter"], "n_eval": r["n_eval"]}
print(json.dumps(out))
''' % ROOT
    res = {}
    for mode in ("serial", "gram"):
        env = dict(os.environ, PINN_LBFGS=mode)
        r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, r.stderr[-2000:]
        import json
        res[mode] = json.loads(r.stdout.strip().splitlines()[-1])
    g = load_golden("burgers_inf")
    for key, tol in (("50", 1e-9), ("7", 1e-5)):
        a, b = res["serial"][key], res["gram"][key]
        assert a["n_iter"] == b["n_iter"] and a["n_eval"] == b["n_eval"]
        assert rel(b["f"], a["f"]) < tol and rel(b["x"], a["x"]) < tol
    assert rel(res["gram"]["50"]["f"], g["lbfgs_f"]) < 1e-7


def test_batched_adam_steps_and_the_in_kernel_tail_leave_the_trajectory_unchanged():
    """pinn_adam_steps(n) == n x pinn_adam_step, and the single-launch step (reduction + Adam done by the last CTAs of the fused
    kernel) == the two-launch step (PINN_FUSED_TAIL=0): same summation order, so weights and losses agree bit for bit."""
    import json
    import os
    import subprocess
    import sys
    from conftest import ROOT
    code = r'''
import os, sys, json, numpy as np
ROOT = %r
sys.path[:0] = [ROOT, os.path.join(ROOT, "pinns-tf2.0_b200", "utils")]
import pinn_cabi
g = np.load(os.path.join(ROOT, "tests", "golden", "burgers_inf.npz"))
out = {}
for mode in ("single", "batched"):
    p = pinn_cabi.Pinn(pinn_cabi.BURGERS_INF, [2] + [20] * 8 + [1], g["lb"], g["ub"])
    p.set_pde_params([float(g["nu"])]); p.set_collocation(g["X_f"][:, 0], g["X_f"][:, 1]); p.set_data(g["X_u"], g["u"]); p.set_weights(g["w"])
    if mode == "single":
        for _ in range(25):
            p.adam_step(0.01, sync=False)
    else:
        p.adam_steps(25, 0.01)
    out[mode] = {"w": p.get_weights().tolist(), "loss": p.last_loss(), "launches": p.kernel_info().get("launches")}
print(json.dumps(out))
''' % ROOT
    res = {}
    for tail in ("1", "0"):
        r = subprocess.run([sys.executable, "-c", code], env=dict(os.environ, PINN_FUSED_TAIL=tail), capture_output=True, text=True,
                           timeout=600)
        assert r.returncode == 0, r.stderr[-2000:]
        res[tail] = json.loads(r.stdout.strip().splitlines()[-1])
    ref = res["0"]["single"]
    for tail in ("1", "0"):
        for mode in ("single", "batched"):
            assert res[tail][mode]["w"] == ref["w"] and res[tail][mode]["loss"] == ref["loss"], (tail, mode)


def test_two_handles_stepping_concurrently_on_one_device():
    """Two handles enqueue asynchronous Adam steps alternately on their own streams.  Only one of two concurrent launches may keep
    its last CTAs spinning for the in-kernel tail (pinn_api.cu: tail_slot_free); the other falls back to the tail kernel.  The run
    must finish (a subprocess with a timeout guards the test session) and both trajectories must equal a handle stepped alone."""
    import json
    import os
    import subprocess
    import sys
    from conftest import ROOT
    code = r'''
import os, sys, json, numpy as np
ROOT = %r
sys.path[:0] = [ROOT, os.path.join(ROOT, "pinns-tf2.0_b200", "utils")]
import pinn_cabi
g = np.load(os.path.join(ROOT, "tests", "golden", "burgers_inf.npz"))
def make():
    p = pinn_cabi.Pinn(pinn_cabi.BURGERS_INF, [2] + [20] * 8 + [1], g["lb"], g["ub"])
    p.set_pde_params([float(g["nu"])]); p.set_collocation(g["X_f"][:, 0], g["X_f"][:, 1]); p.set_data(g["X_u"], g["u"]); p.set_weights(g["w"])
    return p
a, b = make(), make()
for _ in range(200):
    a.adam_step(0.01, sync=False)
    b.adam_step(0.01, sync=False)
a.sync(); b.sync()
wa, wb = a.get_weights().tolist(), b.get_weights().tolist()
a.close(); b.close()
c = make()
c.adam_steps(200, 0.01)
print(json.dumps({"a": wa, "b": wb, "c": c.get_weights().tolist()}))
''' % ROOT
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
    d = json.loads(r.stdout.strip().splitlines()[-1])
    assert d["a"] == d["c"] and d["b"] == d["c"]
