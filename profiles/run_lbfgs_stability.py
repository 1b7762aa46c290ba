"""Long fixed-step L-BFGS runs (the reference takes no line search, so a bad direction is never corrected): final loss of the
Gram-matrix formulation against the literal single-CTA kernel (PINN_LBFGS=serial) from several starting points.
    python profiles/run_lbfgs_stability.py           # spawns one subprocess per (mode, start)"""
import json, os, subprocess, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WORKER = r'''
import json, os, sys, numpy as np
ROOT = %r
for p in (ROOT, os.path.join(ROOT, "pinns-tf2.0_b200", "utils")):
    sys.path.insert(0, p)
import pinn_cabi
g = np.load(os.path.join(ROOT, "tests", "golden", "burgers_accuracy.npz"))
adam, its = int(sys.argv[1]), int(sys.argv[2])
p = pinn_cabi.Pinn(pinn_cabi.BURGERS_INF, [2] + [20] * 8 + [1], g["lb"], g["ub"])
p.set_pde_params([0.01 / np.pi]); p.set_collocation(g["X_f"][:, 0], g["X_f"][:, 1]); p.set_data(g["X_u"], g["u"]); p.set_weights(g["w0"])
for _ in range(adam):
    p.adam_step(0.03, sync=False)
l_adam = p.loss_grad()[0]
fs = []
r = p.lbfgs(its, learning_rate=0.8, n_correction=50, tol_fun=float(np.finfo(float).eps), sync_every=50, log_fn=lambda it, f: fs.append(f))
fs = np.array(fs)
print(json.dumps({"adam_epochs": adam, "loss_after_adam": l_adam, "n_iter": r["n_iter"], "reason": r["reason_str"], "final_loss": p.loss_grad()[0],
                  "min_loss": float(fs.min()), "max_loss": float(fs.max()), "first_above_1": int(np.argmax(fs > 1.0)) if (fs > 1.0).any() else -1}))
''' % ROOT
for mode in ("serial", "gram"):
    for adam in (100, 1900, 2000, 2100):
        env = dict(os.environ, PINN_LBFGS=mode)         # explicit for both: the serial kernel is the default
        r = subprocess.run([sys.executable, "-c", WORKER, str(adam), "3000"], env=env, capture_output=True, text=True, timeout=600)
        line = r.stdout.strip().splitlines()[-1] if r.stdout.strip() else json.dumps({"error": r.stderr[-300:]})
        print(json.dumps({"mode": mode, **json.loads(line)}), flush=True)
