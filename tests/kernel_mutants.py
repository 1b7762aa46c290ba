"""Value mutants of the CUDA kernels, and the tests expected to kill each one.

A mutant is one small edit of the kernel source that stands for a plausible real bug: a wrong coefficient, a dropped term, a
swapped operand, a flipped stop-test comparison.  tests/test_gpu_kernel_mutants.py builds every mutant into a library of its own
and runs the mutant's `kill` selection against it; a selection that still passes means the suite does not guard that line.

Every mutant changes a floating-point value only, never an integer, an index, a pointer, a loop bound, a predicate that guards a
memory access, a barrier, an mbarrier or ring phase, an atomic, a flag, a counter or a wait: a mutant must not be able to fault
or hang the GPU it runs on.  The one exception is the comparisons and the 1e-10 of the L-BFGS stop and curvature tests, which
only decide a stop status that max_iter and max_eval bound.  check_safe() enforces a conservative deny-list on the tokens that
differ between `before` and `after`.

Fields: name; file (relative to pinns-tf2.0_b200/csrc); before (occurs exactly once in the file) and after; models (the bug it
stands for); kill (pytest node ids, relative to the repository root); equivalent (None, or why no test can tell the mutant from
the product within the project's stated accuracy).
"""
import difflib
import os
import re
import shutil
import subprocess
import sys
from collections import namedtuple

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC_REL = os.path.join("pinns-tf2.0_b200", "csrc")

Mutant = namedtuple("Mutant", "name file before after models kill equivalent")

# node ids the selections below share
T_TANH = "tests/test_gpu_burgers.py::test_device_tanh_accuracy"
T_BURGERS = "tests/test_gpu_burgers.py::test_loss_grad_matches_golden"
T_BURGERS_IDE = "tests/test_gpu_burgers.py::test_identification_matches_golden"
T_V1 = "tests/test_gpu_precision.py::test_burgers_kernel_per_block[inf_shifted_nu1-v1]"
T_V2_IDE = "tests/test_gpu_precision.py::test_burgers_kernel_per_block[ide_std_neg_w025-v2]"
T_NLS = "tests/test_gpu_nls.py::test_loss_grad_parts_both_ic_modes"
T_NLS_RAGGED = "tests/test_gpu_nls.py::test_ragged_sizes_against_taylor_oracle[15-3-2]"
T_GEN_DMMA = "tests/test_gpu_precision.py::test_generic_kernel_shape_edges_per_block[w8k_pm1-dmma]"
T_GEN_DFMA = "tests/test_gpu_precision.py::test_generic_kernel_shape_edges_per_block[w8k_pm1-dfma]"
T_DISC_WIDE = "tests/test_gpu_precision.py::test_discrete_time_heads_per_block[disc_q511-dmma]"
T_GEN_NLS = "tests/test_gpu_generic.py::test_schrodinger_any_layers"
T_KDV = "tests/test_gpu_kdv_ac.py::test_golden_loss_grad_at_two_points[kdv_ide_disc]"
T_AC = "tests/test_gpu_kdv_ac.py::test_golden_loss_grad_at_two_points[ac_disc]"
T_POLY = "tests/test_gpu_poly.py::test_stress_spec_per_block_against_longdouble"
T_POLY_SRC = "tests/test_gpu_poly.py::test_source_is_reset_by_new_residual_points"
T_NS = "tests/test_gpu_ns.py::test_golden_loss_grad_at_two_points"
T_ADAM = "tests/test_gpu_burgers.py::test_adam_trajectory"
T_FOREIGN = "tests/test_gpu_lbfgs_foreign.py::test_foreign_closure_takes_every_exit_like_the_reference"
T_REPLAY = "tests/test_gpu_optimizer_replay.py::test_lbfgs_iteration_by_iteration_against_longdouble"
T_EXCHANGE = "tests/test_gpu_exchange_sim.py::test_exchange_is_bit_exact_and_both_forms_agree"
T_PROBES = "tests/test_gpu_precision.py::test_probes_per_stream[burgers_shifted]"
T_PROBES_Q1 = "tests/test_gpu_precision.py::test_probes_on_one_column_input"
T_KDV_PROBES = "tests/test_gpu_kdv_ac.py::test_derivatives_including_u_xxx"

M = Mutant
MUTANTS = [
    # ------------------------------------------------------------------------------------------------ pinn_common.cuh: tanh
    M("tanh_residual_correction_dropped", "pinn_common.cuh",
      "qd = fma(fma(-den, qd, num), rc, qd);", "qd = fma(0.0 * fma(-den, qd, num), rc, qd);",
      "the quotient's residual correction is lost, leaving the error of one Newton step on the reciprocal seed",
      [T_TANH], None),
    M("tanh_coef_5fact_is_4fact", "pinn_common.cuh",
      "q = fma(q, r, 0.008333333333333333);", "q = fma(q, r, 0.041666666666666664);",
      "the 1/5! Taylor coefficient copied from the 1/4! line", [T_TANH], None),
    M("tanh_coef_5fact_short", "pinn_common.cuh",
      "q = fma(q, r, 0.008333333333333333);", "q = fma(q, r, 0.0083333333333333);",
      "the 1/5! Taylor coefficient written with 14 significant digits", [T_TANH],
      "the coefficient's relative error is 4e-15 and its term is at most r^4/5! = 1.2e-4 of p(r) for |r| <= ln2/2, so p "
      "changes by < 5e-19 relative, far below the 2.5 ulp (5.6e-16) the tanh is documented to keep"),
    # ------------------------------------------------------------------------------------------------ burgers_fused_v2.cuh
    M("v2_zbar_x_coef", "burgers_fused_v2.cuh",
      "A[1][j] = fma(-4.0 * a * ax, Axx, s * Ax);", "A[1][j] = fma(-2.0 * a * ax, Axx, s * Ax);",
      "Z_x-bar coefficient -4 a a_x written as -2 a a_x", [T_BURGERS], None),
    M("v2_zbar_axx_term_dropped", "burgers_fused_v2.cuh",
      "z = fma(-2.0 * Axx, u2, z);", "z = fma(0.0 * (-2.0 * Axx), u2, z);",
      "the -2 A_xx (a a_xx + a_x^2) term of Z-bar is dropped", [T_BURGERS], None),
    M("v2_fwd_uxx_coef", "burgers_fused_v2.cuh",
      "V[3][j] = s * fma(-2.0 * a * zx, zx, V[3][j]);", "V[3][j] = s * fma(-1.0 * a * zx, zx, V[3][j]);",
      "the forward u_xx epilogue uses -a z_x^2 instead of -2 a z_x^2", [T_BURGERS], None),
    M("v2_l0_t_stream_scale", "burgers_fused_v2.cuh",
      "V[2][j] = sc1 * w1;", "V[2][j] = sc0 * w1;",
      "layer 0 seeds the t stream with the x scale 2/dx0", [T_BURGERS], None),
    M("v2_l0_wgrad_t_scale", "burgers_fused_v2.cuh",
      "g0t[j] = fma(th, A[0][j], fma(sc1, A[2][j], g0t[j]));", "g0t[j] = fma(th, A[0][j], fma(sc0, A[2][j], g0t[j]));",
      "the layer-0 weight gradient of the t input uses the x scale", [T_BURGERS], None),
    M("v2_u_seed_l1_dropped", "burgers_fused_v2.cuh",
      "seed[0] = fma(cc * l1, ux, 2.0 * wd * r);", "seed[0] = fma(cc, ux, 2.0 * wd * r);",
      "lambda_1 is missing from the u seed of the identification residual", [T_BURGERS_IDE, T_V2_IDE], None),
    M("v2_dlambda2_sign", "burgers_fused_v2.cuh",
      "gl2 = fma(-cc * kap, uxx, gl2);", "gl2 = fma(cc * kap, uxx, gl2);",
      "d/d lambda_2 with the wrong sign", [T_BURGERS_IDE], None),
    M("v2_uxx_seed_nu_for_kappa", "burgers_fused_v2.cuh",
      "seed[3] = -cc * kap;", "seed[3] = -cc * p.nu;",
      "the u_xx seed uses the inference nu instead of e^lambda_2", [T_BURGERS_IDE], None),
    M("v2_data_seed_weight", "burgers_fused_v2.cuh",
      "seed[0] = fma(cc * l1, ux, 2.0 * wd * r);", "seed[0] = fma(cc * l1, ux, 2.0 * wf * r);",
      "the data residual's seed weighted by the residual weight 1/n_f", [T_BURGERS], None),
    M("v2_chain_partials_reassociated", "burgers_fused_v2.cuh",
      "return red[i] + red[R + i] + red[2 * R + i] + red[3 * R + i];",
      "return (red[i] + red[R + i]) + (red[2 * R + i] + red[3 * R + i]);",
      "the per-CTA sum of the four chain warps' partials in another order", [T_BURGERS],
      "a reassociated sum of four doubles differs by a few ulp of the CTA partial; the kernel is held to the longdouble oracle "
      "at 1e-13 relative per parameter block plus 32x the float64 gap (test_gpu_precision.check), and every bit-for-bit test "
      "compares this kernel with itself or with the tail of the same partials"),
    # ------------------------------------------------------------------------------------------------ burgers_fused.cuh (v1)
    M("v1_zbar_x_coef", "burgers_fused.cuh",
      "A[1][nt][e] = s * fma(-2.0 * two_a * zx, Axx, Ax);", "A[1][nt][e] = s * fma(-1.0 * two_a * zx, Axx, Ax);",
      "Z_x-bar coefficient -4 a z_x written as -2 a z_x", [T_V1], None),
    M("v1_l0_t_stream_scale", "burgers_fused.cuh",
      "S[2][nt][e] = sc1 * w1;", "S[2][nt][e] = sc0 * w1;",
      "layer 0 seeds the t stream with the x scale 2/dx0", [T_V1], None),
    # ------------------------------------------------------------------------------------------------ nls_fused.cuh
    M("nls_fv_half_uxx_sign", "nls_fused.cuh",
      "const double fv = vt - 0.5 * uxx - h2 * u;", "const double fv = vt + 0.5 * uxx - h2 * u;",
      "f_v = v_t + u_xx/2 - |h|^2 u: the sign of the half u_xx flipped", [T_NLS], None),
    M("nls_v_seed_3vv", "nls_fused.cuh",
      "sd[1] = cu * (u * u + 3.0 * v * v) - cv * 2.0 * u * v;", "sd[1] = cu * (u * u + v * v) - cv * 2.0 * u * v;",
      "d f_u / dv = u^2 + 3 v^2 written as u^2 + v^2", [T_NLS], None),
    M("nls_boundary_seed_sign", "nls_fused.cuh",
      "sd[c] = sgn * 2.0 * p.wb * d;", "sd[c] = 2.0 * p.wb * d;",
      "the ub point of a periodic pair gets the lb point's seed", [T_NLS], None),
    M("nls_boundary_loss_weight", "nls_fused.cuh",
      "if (is_lb) lbd += p.wb * acc;", "if (is_lb) lbd += p.w0 * acc;",
      "the boundary loss weighted by 1/n0 instead of 1/nb (the same number when n0 == nb)", [T_NLS_RAGGED], None),
    # ------------------------------------------------------------------------------------------------ generic_fused.cuh
    M("gen_dmma_rows_k_remainder", "generic_fused.cuh",
      "b[j] = (bok[j] && kok) ? __ldg(bp[j] + (size_t)kc * ldk) : 0.0;",
      "b[j] = (bok[j] && kok) ? 0.0 * __ldg(bp[j] + (size_t)kc * ldk) : 0.0;",
      "the K % 4 remainder step of dmma_rows contributes nothing", [T_GEN_DMMA], None),
    M("gen_wgrad_npts_tail", "generic_fused.cuh",
      "b[j] = (ok && j < ntn) ? Aoth[st * so + ptc * fo + nc[j]] : 0.0;",
      "b[j] = (ok && j < ntn) ? 0.0 * Aoth[st * so + ptc * fo + nc[j]] : 0.0;",
      "the npts % 4 tail of the DMMA weight gradient contributes nothing",
      [T_GEN_DMMA, "tests/test_gpu_precision.py::test_generic_kernel_shape_edges_per_block[h128x128-dmma]"], None),
    M("gen_bias_row_all_streams", "generic_fused.cuh",
      "const double one = st == 0 ? 1.0 : 0.0;", "const double one = st == 0 ? 1.0 : 1.0;",
      "the bias row of the DMMA weight gradient takes 1 on the derivative streams too", [T_GEN_DMMA], None),
    M("gen_dfma_l0_t_scale", "generic_fused.cuh",
      "fma(th, z[0], sc1 * z[2 * so])", "fma(th, z[0], sc0 * z[2 * so])",
      "the layer-0 weight gradient of the t input uses the x scale", [T_GEN_DFMA], None),
    M("gen_wide_head_drops_uxx", "generic_fused.cuh",
      "if (lane == 0) Acur[s * sl + (size_t)pt * fl + i] = v;", "if (lane == 0) Acur[s * sl + (size_t)pt * fl + i] = v * fmin(1.0, 3.0 - s);",
      "the wide-head (out >= 64) input adjoint loses the u_xx stream", [T_DISC_WIDE], None),
    M("gen_nbar_drops_a3", "generic_fused.cuh",
      "acc = ((a0 + a1) + (a2 + a3)) * p.dt;", "acc = ((a0 + a1) + (a2 + 0.0 * a3)) * p.dt;",
      "one of the four N-bar accumulators is left out of the sum", [T_DISC_WIDE], None),
    M("gen_ac_slope_seed", "generic_fused.cuh",
      "if (gp >= p.n0p) sx = 2.0 *", "if (gp >= p.n0p) sx = 1.0 *",
      "the Allen-Cahn periodic slope seed is (U_x - U_x') instead of 2 (U_x - U_x')", [T_AC], None),
    M("gen_kdv_seed_sign", "generic_fused.cuh",
      "sdp[2 * out + k] = kap * nb_;", "sdp[2 * out + k] = -kap * nb_;",
      "the KdV u_xxx seed with the sign of the Burgers u_xx seed", [T_KDV], None),
    M("gen_pick_dpow_cubic", "generic_fused.cuh",
      "(e == 2 ? 2.0 * v : 3.0 * v2)", "(e == 2 ? 2.0 * v : 2.0 * v2)",
      "d(v^3)/dv = 2 v^2", [T_POLY], None),
    M("gen_poly_dlambda1_exp", "generic_fused.cuh",
      "f1 = fma(kind == 1 ? 1.0 : e1, m, f1);", "f1 = fma(kind == 1 ? 1.0 : 1.0, m, f1);",
      "the e^lambda_1 factor is missing from df/d lambda_1 of a kappa = e^lambda_1 term", [T_POLY], None),
    M("gen_poly_source_sign", "generic_fused.cuh",
      "if (res && p.src) f -= __ldg(p.src + (gp - p.c0));", "if (res && p.src) f -= -__ldg(p.src + (gp - p.c0));",
      "the source term added to the residual instead of subtracted", [T_POLY_SRC], None),
    M("gen_nls_half_coefs", "generic_fused.cuh",
      "sd[6] = -0.5 * cv; sd[7] = 0.5 * cu;", "sd[6] = -1.0 * cv; sd[7] = 1.0 * cu;",
      "the Schrodinger head seeds u_xx and v_xx without the 1/2", [T_GEN_NLS], None),
    # ------------------------------------------------------------------------------------------------ navier_stokes_fused.cuh
    M("ns_tanh_stream_xxy", "navier_stokes_fused.cuh",
      "fma(z[4], zy, 2.0 * z[5] * zx)", "fma(z[4], zy, 1.0 * z[5] * zx)",
      "the mixed third-order stream a_xxy counts z_xy z_x once instead of twice", [T_NS], None),
    M("ns_lambda2_drops_uyy", "navier_stokes_fused.cuh",
      "const double lap_u = pxxy + pyyy,", "const double lap_u = pxxy + 0.0 * pyyy,",
      "u_yy = psi_yyy is missing from the lambda_2 term of f_u", [T_NS], None),
    M("ns_fv_py_sign", "navier_stokes_fused.cuh",
      "fma(l1, adv_v, qy - pxt)", "fma(l1, adv_v, -qy - pxt)",
      "f_v with -p_y", [T_NS], None),
    # ------------------------------------------------------------------------------------------------ optim_kernels.cuh: Adam
    M("adam_eps_inside_sqrt", "optim_kernels.cuh",
      "w[i] -= (mi * alpha) / (sqrt(vi) + eps);", "w[i] -= (mi * alpha) / sqrt(vi + eps);",
      "Adam with eps under the square root", [T_ADAM], None),
    M("adam_bias_correction_t_plus_1", "optim_kernels.cuh",
      "(1.0 - pow(b1, (double)t));", "(1.0 - pow(b1, (double)t + 1.0));",
      "the first-moment bias correction one step ahead", [T_ADAM], None),
    M("adam_v_uses_b1", "optim_kernels.cuh",
      "(g * g - v[i]) * (1.0 - b2);", "(g * g - v[i]) * (1.0 - b1);",
      "the second moment decays with beta_1", [T_ADAM], None),
    M("combine8_reassociated", "optim_kernels.cuh",
      "return ((red[lane] + red[32 + lane]) + (red[64 + lane] + red[96 + lane])) +",
      "return (((red[lane] + red[32 + lane]) + red[64 + lane]) + red[96 + lane]) +",
      "the eight warp sums of the evaluation tail combined in another order (ranks would disagree bitwise)", [T_EXCHANGE], None),
    # ------------------------------------------------------------------------------------------------ optim_kernels.cuh: L-BFGS
    M("lbfgs_initial_optimality_strict", "optim_kernels.cuh",
      "if (n_iter == 0) return g1 <= st->tol_fun ? 7 : 0;", "if (n_iter == 0) return g1 < st->tol_fun ? 7 : 0;",
      "|g|_1 == tolFun at the start no longer counts as optimal", [T_FOREIGN], None),
    M("lbfgs_optimality_strict", "optim_kernels.cuh",
      "if (g1 <= st->tol_fun) return 3;", "if (g1 < st->tol_fun) return 3;",
      "|g|_1 == tolFun after a step no longer counts as optimal", [T_FOREIGN], None),
    M("lbfgs_step_tol_strict", "optim_kernels.cuh",
      "if (s1 <= st->tol_x) return 4;", "if (s1 < st->tol_x) return 4;",
      "a step of exactly tolX no longer stops the run", [T_FOREIGN], None),
    M("lbfgs_f_tol_non_strict", "optim_kernels.cuh",
      "if (fabs(f_new - st->f_old) < st->tol_x) return 5;", "if (fabs(f_new - st->f_old) <= st->tol_x) return 5;",
      "an f change of exactly tolX stops the run", [T_FOREIGN], None),
    M("lbfgs_no_progress_non_strict", "optim_kernels.cuh",
      "s.stop = gtd > -st->tol_x;", "s.stop = gtd >= -st->tol_x;",
      "g.d == -tolX counts as no progress", [T_FOREIGN], None),
    M("lbfgs_first_step_unclamped", "optim_kernels.cuh",
      "fmin(1.0, 1.0 / g1)", "1.0 / g1",
      "the first step is 1/|g|_1 without the min(1, .)", [T_FOREIGN], None),
    M("lbfgs_iterate_curvature_non_strict", "optim_kernels.cuh",
      "if (ys > 1e-10) {", "if (ys >= 1e-10) {",
      "the literal kernel keeps a pair with y.s == 1e-10", [T_FOREIGN], None),
    M("lbfgs_iterate_curvature_1e9", "optim_kernels.cuh",
      "if (ys > 1e-10) {", "if (ys > 1e-9) {",
      "the literal kernel's curvature threshold 1e-9", [T_FOREIGN], None),
    M("lbfgs_iterate_h_diag_inverted", "optim_kernels.cuh",
      "h_diag = ys / yy;", "h_diag = yy / ys;",
      "the literal kernel's initial Hessian scale y.y / y.s", [T_FOREIGN], None),
    M("lbfgs_solve_curvature_non_strict", "optim_kernels.cuh",
      "const bool accept = ys > 1e-10;", "const bool accept = ys >= 1e-10;",
      "the Gram kernel keeps a pair with y.s == 1e-10", [T_REPLAY], None),
    M("lbfgs_solve_curvature_1e9", "optim_kernels.cuh",
      "const bool accept = ys > 1e-10;", "const bool accept = ys > 1e-9;",
      "the Gram kernel's curvature threshold 1e-9", [T_REPLAY], None),
    M("lbfgs_solve_h_diag_inverted", "optim_kernels.cuh",
      "h_diag = ys / dots[4];", "h_diag = dots[4] / ys;",
      "the Gram kernel's initial Hessian scale y.y / y.s", [T_REPLAY], None),
    # ------------------------------------------------------------------------------------------------ optim_kernels.cuh: probes
    M("probe_xxx_bracket_coef", "optim_kernels.cuh",
      "return fma(-6.0 * a * zx, zxx,", "return fma(-4.0 * a * zx, zxx,",
      "the third-order probe's -6 a z_x z_xx written as -4 a z_x z_xx", [T_KDV_PROBES], None),
    M("probe_q1_t_zero", "optim_kernels.cuh",
      "(in_dim == 1 ? x : X[p * in_dim + 1])", "(in_dim == 1 ? 0.0 : X[p * in_dim + 1])",
      "an (n, 1) input on a 2-D net takes t := 0 instead of the broadcast t := x", [T_PROBES_Q1], None),
    M("probe_t_seed_dx0", "optim_kernels.cuh",
      "h[2][0] = 0.0;          h[2][1] = 2.0 / nd.dx1;", "h[2][0] = 0.0;          h[2][1] = 2.0 / nd.dx0;",
      "the probe seeds the t stream with the x scale", [T_PROBES], None),
    M("probe_uxx_epilogue_coef", "optim_kernels.cuh",
      "h[3][j] = sd * fma(-2.0 * a * zx, zx, z[3][j]);", "h[3][j] = sd * fma(-1.0 * a * zx, zx, z[3][j]);",
      "the probe's u_xx epilogue uses -a z_x^2 instead of -2 a z_x^2", [T_PROBES], None),
]
del M

# ------------------------------------------------------------------------------------------------------------- safety rule
# A token of the diff that is, or (for identifiers) contains, one of these rejects the mutant.
DENY_EXACT = {"while", "for", "[", "]", "++", "--", "+=", "-=", "*=", "/=", "&=", "|=", "^=", "<<=", ">>=", "goto", "return",
              "break", "continue", "if", "asm", "volatile"}
DENY_SUBSTR = ("sync", "mbar", "atomic", "nanosleep", "acquire", "release", "flag", "seq", "parity", "ticket", "n_total", "npts",
               "pts", "grid", "fence", "wait", "ring", "phase", "ctr", "slot", "head", "status", "n_iter", "n_eval", "max_iter")
# the comparisons a mutant may change: only those of the L-BFGS stop and curvature tests (optim_kernels.cuh)
COMPARISONS = {"<", "<=", ">", ">=", "==", "!="}
LBFGS_STOP_TEST_LINES = ("g1 <= st->tol_fun", "s1 <= st->tol_x", "fabs(f_new - st->f_old) < st->tol_x", "gtd > -st->tol_x",
                         "ys > 1e-10")

_TOKEN = re.compile(r"\d+\.\d*(?:[eE][-+]?\d+)?|\d+[eE][-+]?\d+|\.\d+(?:[eE][-+]?\d+)?|\d+|[A-Za-z_]\w*|->|<<=|>>=|\+\+|--"
                    r"|[-+*/%&|^<>=!]=|&&|\|\||<<|>>|\S")


def tokens(src):
    return _TOKEN.findall(src)


def changed_tokens(before, after):
    """The tokens that differ between before and after (both sides of every replaced, deleted or inserted run)."""
    a, b = tokens(before), tokens(after)
    out = []
    for op, i1, i2, j1, j2 in difflib.SequenceMatcher(None, a, b, autojunk=False).get_opcodes():
        if op != "equal":
            out += a[i1:i2] + b[j1:j2]
    return out


def check_safe(m):
    """Raise ValueError if the mutant's diff touches anything but a floating-point value."""
    diff = changed_tokens(m.before, m.after)
    if not diff:
        raise ValueError("%s: after does not differ from before" % m.name)
    for t in diff:
        low = t.lower()
        if t in DENY_EXACT or (re.match(r"[A-Za-z_]", t) and any(s in low for s in DENY_SUBSTR)):
            raise ValueError("%s: the diff touches %r" % (m.name, t))
        if re.fullmatch(r"\d+", t):
            raise ValueError("%s: the diff changes the integer literal %r" % (m.name, t))
        if t in COMPARISONS and not (m.file == "optim_kernels.cuh" and any(s in m.before for s in LBFGS_STOP_TEST_LINES)):
            raise ValueError("%s: the diff changes the comparison %r outside the L-BFGS stop and curvature tests" % (m.name, t))
    return diff


def source(m, src_root=ROOT):
    with open(os.path.join(src_root, CSRC_REL, m.file)) as f:
        return f.read()


def apply(src_root, mutant, dest):
    """Copy pinns-tf2.0_b200/csrc and include/ of src_root into dest, with their relative layout (pinn_api.cu includes
    ../../include/pinn_b200.h), and replace the mutant's `before` by its `after`.  Returns the mutated csrc directory."""
    check_safe(mutant)
    csrc = os.path.join(dest, CSRC_REL)
    shutil.copytree(os.path.join(src_root, CSRC_REL), csrc)
    shutil.copytree(os.path.join(src_root, "include"), os.path.join(dest, "include"))
    path = os.path.join(csrc, mutant.file)
    with open(path) as f:
        text = f.read()
    n = text.count(mutant.before)
    if n != 1:
        raise ValueError("%s: `before` occurs %d times in %s" % (mutant.name, n, mutant.file))
    with open(path, "w") as f:
        f.write(text.replace(mutant.before, mutant.after))
    return csrc


def build(src_root, mutant, dest, nvcc=None, flags=None):
    """apply() into dest, then compile the mutated pinn_api.cu with the library's own nvcc flags; returns the .so path."""
    pkg = os.path.join(src_root, "pinns-tf2.0_b200")
    if pkg not in sys.path:
        sys.path.insert(0, pkg)
    import build as pinn_build
    csrc = apply(src_root, mutant, dest)
    out = os.path.join(dest, "libpinn_b200.so")
    cmd = [nvcc or pinn_build._nvcc()] + list(flags or pinn_build.NVCC_FLAGS) + ["-o", out] + \
          [os.path.join(csrc, s) for s in pinn_build.SOURCES] + ["-lcudart", "-ldl"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("%s: nvcc failed:\n%s\n%s%s" % (mutant.name, " ".join(cmd), r.stdout, r.stderr))
    return out


def by_name(name):
    for m in MUTANTS:
        if m.name == name:
            return m
    raise KeyError(name)
