"""Adam-step time of the small BASELINE configurations (cfg1: N_f=10000 inference; cfg4: N=2000 identification).  Run from the repo
root."""
import os, sys, json
import numpy as np
sys.path.insert(0, os.getcwd())
sys.path.insert(0, os.path.join(os.getcwd(), "pinns-tf2.0_b200", "utils"))
import pinn_cabi
from bench import synthetic_problem, init_weights, LB, UB, NU, ADAM_LR, LAYERS, timed_adam_steps
out = {}
X_f, X_u, u = synthetic_problem(7, 10000)
p = pinn_cabi.Pinn(pinn_cabi.BURGERS_INF, LAYERS, LB, UB)
p.set_pde_params([NU]); p.set_data(X_u, u); p.set_collocation(X_f[:, 0], X_f[:, 1]); p.set_weights(init_weights())
for _ in range(20):
    p.adam_step(ADAM_LR, sync=False)
p.sync()
out["cfg1_10k_step_ms"] = float(np.median(timed_adam_steps(p, 400, flush=False)))
out["cfg1_kernel_ms"] = p.time_kernel_ms(50) / 50
p.event_record(0); p.adam_steps(400, ADAM_LR); p.event_record(1); p.sync()
out["cfg1_10k_step_ms_batched"] = p.event_elapsed_ms(0, 1) / 400
p.close()
rng = np.random.default_rng(3)
X = LB + (UB - LB) * rng.random((2000, 2)); uu = rng.uniform(-1, 1, (2000, 1))
q = pinn_cabi.Pinn(pinn_cabi.BURGERS_IDE, LAYERS, LB, UB)
q.set_data(X, uu); q.set_weights(np.concatenate([init_weights(), [0.0, -6.0]]))
for _ in range(20):
    q.adam_step(ADAM_LR, sync=False)
q.sync()
out["cfg4_2k_step_ms"] = float(np.median(timed_adam_steps(q, 400, flush=False)))
out["cfg4_kernel_ms"] = q.time_kernel_ms(50) / 50
q.event_record(0); q.adam_steps(400, ADAM_LR); q.event_record(1); q.sync()
out["cfg4_2k_step_ms_batched"] = q.event_elapsed_ms(0, 1) / 400
q.close()
print(json.dumps(out))
