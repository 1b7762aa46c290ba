"""Continuous-time identification of the 2-D incompressible Navier-Stokes equations (PINNs/main/continuous_time_identification
(Navier-Stokes)/NavierStokes.py) on the fused sm_90a kernel: a net [3, 20 x 8, 2] maps (x, y, t) to the stream function and the
pressure, and lambda_1, lambda_2 of  u_t + l1 (u u_x + v u_y) = -p_x + l2 (u_xx + u_yy)  are trained with it.

    python 2d-navier-stokes/ide_cont_navier_stokes.py [path/to/cylinder_nektar_wake.mat]

Without a path the TG vortex of navierstokesutil.py (lambda_1 = 1, lambda_2 = nu) is used; PINN_NS_HP (JSON) overrides hp entries."""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [HERE, os.path.join(HERE, "..", "utils")]

from logger import Logger  # noqa: E402
from navierstokesutil import TG_NU, prep_data  # noqa: E402
from neuralnetwork import NeuralNetwork  # noqa: E402

hp = {"N_train": 5000, "layers": [3] + 8 * [20] + [2], "tf_epochs": 200, "tf_lr": 0.001, "tf_b1": 0.9, "tf_eps": None,
      "nt_epochs": 1000, "nt_lr": 0.8, "nt_ncorr": 50, "log_frequency": 100, "noise": 0.0}
hp.update(json.loads(os.environ.get("PINN_NS_HP", "{}")))


class NavierStokesInformedNN(NeuralNetwork):
    pde = "ns_ide"

    def __init__(self, hp, logger, ub, lb):
        super().__init__(hp, logger, ub, lb)
        self.lambda_1, self.lambda_2 = 0.0, 0.0


if __name__ == "__main__":
    path = sys.argv[1] if len(sys.argv) > 1 else None
    X_train, uv_train, lb, ub, (X_star, u_star, v_star, p_star) = prep_data(path, hp["N_train"], hp["noise"])
    logger = Logger(hp)
    pinn = NavierStokesInformedNN(hp, logger, ub, lb)

    def error():
        u, v, _ = pinn.predict(X_train)
        return np.linalg.norm(uv_train[:, 0:1] - u, 2) / np.linalg.norm(uv_train[:, 0:1], 2)

    logger.set_error_fn(error)
    pinn.fit(X_train, uv_train)
    l1, l2 = pinn.get_params(numpy=True)
    nu = 0.01 if path is not None else TG_NU                      # the cylinder wake is at Re = 100
    print(f"Error l1: {abs(l1 - 1.0) * 100:.5f}%")
    print(f"Error l2: {abs(l2 - nu) / nu * 100:.5f}%")
