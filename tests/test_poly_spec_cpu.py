"""CPU: residual strings of user-defined PDEs (utils/poly_spec.py and NeuralNetwork with pde = "poly") -- expansion and
combining of like terms, every rejection, name resolution, and the inference / identification choice."""
import numpy as np
import pytest

import pinn_cabi
import poly_spec
from neuralnetwork import NeuralNetwork


def terms(text, **names):
    return poly_spec.parse(text, names.get).terms


def as_dict(ts):
    return {(k,) + e: c for c, k, e in ts}


def test_burgers_string():
    s = poly_spec.parse("u_t + u*u_x - nu*u_xx", {"nu": 0.01}.get)
    assert s.terms == [(1.0, 0, (0, 0, 1, 0)), (1.0, 0, (1, 1, 0, 0)), (-0.01, 0, (0, 0, 0, 1))]
    assert not s.identification
    s = poly_spec.parse("u_t + l1*u*u_x - exp(l2)*u_xx")
    assert s.terms == [(1.0, 0, (0, 0, 1, 0)), (1.0, 1, (1, 1, 0, 0)), (-1.0, 4, (0, 0, 0, 1))]
    assert s.identification


def test_expansion_and_like_terms():
    d = as_dict(terms("(u + u_x)**2 - 2*u*u_x + 3*(u_t - u_t) + u*(1 - u)"))
    assert d == {(0, 0, 2, 0, 0): 1.0, (0, 1, 0, 0, 0): 1.0}        # u^2 and u_t cancel and are dropped
    assert as_dict(terms("u_t - 1e-4*u_xx + 5*u**3 - 5*u")) == {(0, 0, 0, 1, 0): 1.0, (0, 0, 0, 0, 1): -1e-4, (0, 3, 0, 0, 0): 5.0,
                                                                 (0, 1, 0, 0, 0): -5.0}
    # Fisher-KPP with the lambdas distributed over a product of sums
    assert as_dict(terms("u_t - exp(l2)*u_xx - l1*u*(1 - u)")) == {(0, 0, 0, 1, 0): 1.0, (4, 0, 0, 0, 1): -1.0,
                                                                   (1, 1, 0, 0, 0): -1.0, (1, 2, 0, 0, 0): 1.0}
    # nonlinear diffusion in expanded form, unary minus, ** 0 and ** 1, float powers of numbers
    assert as_dict(terms("u_t - (u*u_xx + u_x**2)")) == {(0, 0, 0, 1, 0): 1.0, (0, 1, 0, 0, 1): -1.0, (0, 0, 2, 0, 0): -1.0}
    assert as_dict(terms("-(-u_x)**1 * u**0 + 2**3*u")) == {(0, 0, 1, 0, 0): 1.0, (0, 1, 0, 0, 0): 8.0}
    assert as_dict(terms("u_xx**3*u_t**3*u_x**3*u**3")) == {(0, 3, 3, 3, 3): 1.0}


def test_sixteen_terms_and_order_of_first_appearance():
    t = terms("(1 + u)**3 * (1 + u_x)**3 - 1")          # 4 x 4 = 16 products, the constant cancels -> 15 terms
    assert len(t) == 15
    t = terms("u_x + u")
    assert [e for _, _, e in t] == [(0, 1, 0, 0), (1, 0, 0, 0)]


@pytest.mark.parametrize("text,match", [
    ("u**4", "'u \\*\\* 4': u appears to the power 4"),
    ("u**2 * u_x * u**2", "u appears to the power 4"),
    ("(u + u_x + u_t + u_xx)**3", "expands to 20 terms; at most 16"),
    ("l1*l2*u", "product of two lambda factors"),
    ("exp(l1)*l1*u", "product of two lambda factors"),
    ("l1**2*u", "product of two lambda factors"),
    ("u_t / 2", "division"),
    ("u_t - u_xx / nu", "'u_xx / nu': division"),
    ("u**2.0", "literal non-negative integer"),
    ("u**-1", "literal non-negative integer"),
    ("u**n", "literal non-negative integer"),
    ("sin(u)", "'sin\\(u\\)': the only calls are exp\\(l1\\) and exp\\(l2\\)"),
    ("exp(u)", "the only calls"),
    ("u_t + foo*u", "name 'foo' is neither a stream"),
    ("u_t + x*u", "name 'x' is neither"),
    ("u_t + 1", "no stream factor"),
    ("u_t + l1", "no stream factor"),
    ("u - u", "identically zero"),
    ("u_t +", "cannot parse"),
    ("u_t if u else u", "is not supported"),
    ("u_t @ u", "is not supported"),
    ("u.x", "is not supported"),
    ("'u'", "only numbers"),
    ("True*u", "only numbers"),
])
def test_rejections_name_the_offending_piece(text, match):
    with pytest.raises(poly_spec.SpecError, match=match):
        poly_spec.parse(text, {"nu": 0.5}.get)


def test_rejects_non_string():
    with pytest.raises(poly_spec.SpecError, match="must be a string"):
        poly_spec.parse(None)


def test_evaluate_matches_the_terms():
    rng = np.random.default_rng(1)
    V = [rng.standard_normal((5, 1)) for _ in range(4)]
    t = terms("u_t - exp(l2)*u_xx - l1*u*(1 - u) + 0.5*u_x**2*u_xx")
    f = poly_spec.evaluate(t, V, 0.3, -0.7)
    u, ux, ut, uxx = V
    assert np.allclose(f, ut - np.exp(-0.7) * uxx - 0.3 * u * (1 - u) + 0.5 * ux ** 2 * uxx, rtol=1e-14, atol=1e-14)
    assert poly_spec.format_terms(terms("u_t - 2*u*u_x**2")) == "1.0*u_t + -2.0*u*u_x**2"


def _net(cls):
    hp = {"layers": [2, 5, 1], "tf_epochs": 0, "tf_lr": 1e-3, "tf_b1": 0.9, "tf_eps": None, "nt_epochs": 0, "nt_lr": 1.0,
          "nt_ncorr": 10}
    return cls(hp, None, [1.0, 1.0], [-1.0, 0.0])


def test_name_resolution_and_the_inf_ide_choice():
    class Heat(NeuralNetwork):
        pde = "poly"
        residual = "u_t - k*u_xx - c2*u"
        k = 0.25

        def __init__(self, *a):
            super().__init__(*a)
            self.c2 = np.array([[2.0]])                   # a one-element array resolves like a number

    h = _net(Heat)
    assert h._pde_id() == pinn_cabi.POLY_INF
    assert h._poly_spec().terms == [(1.0, 0, (0, 0, 1, 0)), (-0.25, 0, (0, 0, 0, 1)), (-2.0, 0, (1, 0, 0, 0))]

    class Fisher(NeuralNetwork):
        pde = "poly"
        residual = "u_t - exp(l2)*u_xx - l1*u + l1*u**2"

    assert _net(Fisher)._pde_id() == pinn_cabi.POLY_IDE

    class Bad(NeuralNetwork):
        pde = "poly"
        residual = "u_t - D*u_xx"
        D = "0.1"                                          # not numeric

    with pytest.raises(pinn_cabi.PinnError, match="Bad.residual: name 'D' is neither"):
        _net(Bad)._pde_id()

    class Method(NeuralNetwork):
        pde = "poly"
        residual = "u_t - source*u_xx"                     # a method is not a number

        def source(self, x, t):
            return 0 * x

    with pytest.raises(pinn_cabi.PinnError, match="name 'source' is neither"):
        _net(Method)._pde_id()

    class NoString(NeuralNetwork):
        pde = "poly"

    with pytest.raises(pinn_cabi.PinnError, match="must be a string"):
        _net(NoString)._pde_id()
