"""CPU: source tables of the polynomial residual models (pinn_set_source_terms, DESIGN §4.8).

The longdouble restatement (oracle/source_terms.py) against mpmath evaluations of the original strings; the string parser's tables
and its refusals; the binding's argument checks, which restate the header's validation; the mirror's schedule with string,
callable and absent sources on a stand-in handle; and the new kernels' spill-free resource use."""
import math
import re
import subprocess

import numpy as np
import pytest

from oracle import source_terms as st

import pinn_cabi
import poly_spec as ps

K, NU = 0.5, 0.01 / math.pi
NAMES = {"k": K, "nu": NU}
HEAT = "(k*pi**2 - 1)*sin(pi*x)*exp(-t)"                                           # u_t - k u_xx, u = sin(pi x) e^-t
BURGERS = "-sin(pi*x)*exp(-t) + 0.5*pi*sin(2*pi*x)*exp(-2*t) + nu*pi**2*sin(pi*x)*exp(-t)"   # u_t + u u_x - nu u_xx
PULSE = "3*exp(-100*(x - 0.3)**2 - 4*(t - 0.5)**2)"
MIXED = "x**3*t**2*cos(2*x + 0.5)*sin(3*t - 1)*exp(0.1*x - 0.02*x**2 + 0.3*t - 0.05*t**2) - 2*x*t + 0.7 + t**3*cos(5*t)"
STRINGS = [HEAT, BURGERS, PULSE, MIXED]


def table(text):
    return pinn_cabi.pack_source_terms(ps.parse_source(text, NAMES.get))


def mp_eval(text, x, t):
    """The original string at one point in 50-digit arithmetic."""
    import mpmath
    mpmath.mp.dps = 50
    env = {"x": mpmath.mpf(float(x)), "t": mpmath.mpf(float(t)), "pi": mpmath.pi, "sin": mpmath.sin, "cos": mpmath.cos,
           "exp": mpmath.exp, "k": mpmath.mpf(K), "nu": mpmath.mpf(NU)}
    return eval(compile(text, "<source>", "eval"), {"__builtins__": {}}, env)


# ---------------------------------------------------------------------------------------------------------------- oracle
def mp_table(form, par, x, t):
    """The table at one point as the header defines it: the trig and exp arguments formed in fp64 (Python floats, each operation
    rounded), everything else in 50-digit arithmetic."""
    import mpmath
    mpmath.mp.dps = 50
    x, t = float(x), float(t)
    s = mpmath.mpf(0)
    for f, c in zip(form, par):
        a, om, ph, nu, ps_, al, ga, be, de = (float(v) for v in c)
        m = mpmath.mpf(a) * mpmath.mpf(x) ** (int(f) & 3) * mpmath.mpf(t) ** ((int(f) >> 2) & 3)
        for kind, arg in (((int(f) >> 4) & 3, om * x + ph), ((int(f) >> 6) & 3, nu * t + ps_)):
            if kind:
                m *= (mpmath.sin if kind == 1 else mpmath.cos)(mpmath.mpf(arg))
        if (al, ga, be, de) != (0.0, 0.0, 0.0, 0.0):
            m *= mpmath.exp(mpmath.mpf(((al * x + ga * (x * x)) + be * t) + de * (t * t)))
        s += m
    return s


def term_scale(form, par, x, t):
    """sum_k |m_k| (1 + the magnitudes of the pieces of its trig and exp arguments): what fp64 rounding of the table's constants
    and arguments can move the value by, in units of u."""
    out = 0.0
    for f, c in zip(form, par):
        a, om, ph, nu, ps_, al, ga, be, de = (float(v) for v in c)
        m = abs(a * x ** (int(f) & 3) * t ** ((int(f) >> 2) & 3))
        pieces = 1.0
        if (int(f) >> 4) & 3:
            pieces += abs(om * x) + abs(ph)
        if (int(f) >> 6) & 3:
            pieces += abs(nu * t) + abs(ps_)
        z = ((al * x + ga * (x * x)) + be * t) + de * (t * t)
        pieces += abs(al * x) + abs(ga * x * x) + abs(be * t) + abs(de * t * t) + abs(z)    # |z| also covers the folded e^c0
        out += m * math.exp(z) * pieces
    return out


@pytest.mark.parametrize("text", STRINGS)
def test_oracle_equals_mpmath_on_the_table(text):
    """The longdouble evaluation and its fp64 arguments against 50-digit arithmetic on the same arguments: within longdouble
    rounding, far inside the device bound."""
    pytest.importorskip("mpmath")
    rng = np.random.default_rng(7)
    x, t = rng.uniform(-1, 1, 200), rng.uniform(0, 1, 200)
    form, par = table(text)
    s = st.source(form, par, x, t)
    b = st.error_bound(form, par, x, t)
    for i in range(x.size):
        want = mp_table(form, par, x[i], t[i])
        assert abs(float(s[i] - np.longdouble(str(want)))) <= float(b[i]) / 256, (text, x[i], t[i])


@pytest.mark.parametrize("text", STRINGS)
def test_table_equals_mpmath_on_the_original_strings(text):
    """The parser's table against the string itself: they differ only by the fp64 rounding of folded constants and arguments."""
    pytest.importorskip("mpmath")
    rng = np.random.default_rng(7)
    x, t = rng.uniform(-1, 1, 200), rng.uniform(0, 1, 200)
    form, par = table(text)
    s = st.source(form, par, x, t)
    for i in range(x.size):
        want = mp_eval(text, x[i], t[i])
        tol = 4 * 2.0 ** -53 * (len(form) + 2) * term_scale(form, par, x[i], t[i])
        assert abs(float(s[i] - np.longdouble(str(want)))) <= tol, (text, x[i], t[i])


def test_oracle_bound_covers_a_perturbed_evaluation():
    """The bound is not loose by orders of magnitude: a relative perturbation of 64 u (u = 2^-53) breaks it somewhere."""
    form, par = table(MIXED)
    rng = np.random.default_rng(3)
    x, t = rng.uniform(-1, 1, 2000), rng.uniform(0, 1, 2000)
    s = st.source(form, par, x, t).astype(np.float64)
    assert st.check(s, form, par, x, t)[0] <= 1.0
    worst, _ = st.check(s * (1 + 64 * 2.0 ** -53), form, par, x, t)
    assert worst > 1.0


def test_oracle_trig_is_nan_from_2_pow_31():
    form, par = pinn_cabi.pack_source_terms([(1.0, 0, 0, 1, 1.0, 0.0, 0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0)])
    x = np.array([2.0 ** 31 - 1, 2.0 ** 31, -2.0 ** 31, np.inf, np.nan])
    s = st.source(form, par, x, np.zeros(5))
    assert np.isfinite(s[0]) and np.isnan(s[1:]).all()


# ---------------------------------------------------------------------------------------------------------------- parser
def T(a, p=0, q=0, xk=0, om=0.0, ph=0.0, tk=0, nu=0.0, psi=0.0, al=0.0, ga=0.0, be=0.0, de=0.0):
    return ps.SourceTerm(a, p, q, xk, om, ph, tk, nu, psi, al, ga, be, de)


def test_parser_tables_of_manufactured_solutions():
    assert ps.parse_source(HEAT, NAMES.get) == [T(K * math.pi ** 2 - 1, xk=1, om=math.pi, be=-1.0)]
    got = ps.parse_source(BURGERS, NAMES.get)
    assert got == [T(-1.0 + NU * math.pi ** 2, xk=1, om=math.pi, be=-1.0), T(0.5 * math.pi, xk=1, om=2 * math.pi, be=-2.0)]
    (g,) = ps.parse_source(PULSE)
    assert g._replace(a=0.0) == T(0.0, al=60.0, ga=-100.0, be=4.0, de=-4.0)
    assert g.a == pytest.approx(3 * math.exp(-9.0 - 1.0), rel=1e-15)
    assert ps.parse_source("0") == [] and ps.parse_source("x - x") == []
    assert ps.parse_source("2.5") == [T(2.5)]
    assert ps.parse_source("cos(2*t + 1)*exp(x)**2*3*x**2*t") == [T(3.0, p=2, q=1, tk=2, nu=2.0, psi=1.0, al=2.0)]
    assert ps.parse_source("sin(pi*(x + 1))") == [T(1.0, xk=1, om=math.pi, ph=math.pi)]
    assert ps.parse_source("sin(0.5)*x") == [T(math.sin(0.5), p=1)]
    # a table from the parser passes the binding's checks and the oracle evaluates it
    for text in STRINGS:
        form, par = table(text)
        assert np.all(np.isfinite(st.source(form, par, np.linspace(-1, 1, 5), np.linspace(0, 1, 5))))


@pytest.mark.parametrize("text, msg", [
    ("sin(pi*x)*cos(pi*x)", "two trig factors in x"),
    ("sin(t)**2", "two trig factors in t"),
    ("x**4", "x appears to the power 4"),
    ("x**2*t*(x + 1)*t**3", "power"),
    ("x/2", "division"),
    ("tanh(x)", "unknown function"),
    ("sin(x + t)", "affine function of one variable"),
    ("sin(x**2)", "affine function of one variable"),
    ("sin(exp(x))", "sin takes an affine function"),
    ("exp(x*t)", "without an x\\*t term"),
    ("exp(x**3)", "degree <= 2"),
    ("exp(sin(x))", "exp takes a polynomial"),
    ("y*x", "name 'y'"),
    ("x**t", "literal non-negative integer"),
    (" + ".join("%d*x**%d*t**%d" % (i + 1, i // 4, i % 4) for i in range(16)) + " + sin(x)", "17 terms"),
    ("x +", "cannot parse"),
])
def test_parser_rejections_name_the_piece(text, msg):
    with pytest.raises(ps.SpecError, match=msg):
        ps.parse_source(text, NAMES.get)


@pytest.mark.parametrize("text, msg", [
    ("3*exp(-100*(x - 3)**2)", r"'exp\(-100 \* \(x - 3\) \*\* 2\)': the constant part of its exponent, exp\(-900.0\) is 0.0, below "
                               r"the normal fp64 range.*w\*x0\*\*2 below about 708"),
    ("exp(-(x - 30)**2)", r"exp\(-900.0\) is 0.0, below the normal fp64 range"),
    ("exp(-100*(t - 5)**2)", r"exp\(-2500.0\) is 0.0"),
    ("3*exp(-100*(x - 2.7)**2)", r"exp\(-729.0000000000001\) is 2.5\d*e-317, below the normal fp64 range"),
    ("exp(800)*exp(-x)", r"'exp\(800\)': the constant part of its exponent, exp\(800.0\) overflows fp64"),
    ("exp(-700)*exp(-700)*x", r"'exp\(-700\) \* exp\(-700\)': the product of the coefficients is 0.0, below"),
    ("1e-310*x", r"'1e-310 \* x': the product of the coefficients is 1e-310, below the normal fp64 range"),
    ("1e200*1e200*x", r"'1e\+?200 \* 1e\+?200': the product of the coefficients overflows fp64"),
])
def test_parser_refuses_coefficients_that_folding_loses(text, msg):
    """A term whose folded coefficient overflows, underflows to 0 or drops below the normal range is refused, never silently
    turned into 0 or inf."""
    with pytest.raises(ps.SpecError, match=msg):
        ps.parse_source(text, NAMES.get)


def test_parser_keeps_pulses_inside_the_range():
    (g,) = ps.parse_source("3*exp(-100*(x - 2.6)**2)")
    assert g.a == pytest.approx(3 * math.exp(-676.0), rel=1e-12) and g.a >= np.finfo(np.float64).tiny
    assert (g.alpha, g.gamma) == (pytest.approx(520.0), -100.0)
    ps.check_source_range([g], [-50.0, 0.0], [50.0, 10.0])                  # the exponent peaks at 676 (x = 2.6)
    s = ps.evaluate_source([g], np.array([2.5, 2.6, 2.7]), np.zeros(3))
    assert np.allclose(s, 3 * np.exp(-100 * (np.array([2.5, 2.6, 2.7]) - 2.6) ** 2), rtol=1e-12)


def test_range_check_refuses_exponents_that_overflow_on_the_box():
    (g,) = ps.parse_source("exp(-10*(x - 8.4)**2)")                         # e^-705.6 exp(168 x - 10 x^2): peak 705.6 at 8.4
    ps.check_source_range([g], [-50.0, 0.0], [50.0, 10.0])
    (h,) = ps.parse_source("exp(0.5*x**2)")
    ps.check_source_range([h], [-1.0, 0.0], [1.0, 1.0])
    with pytest.raises(ps.SpecError, match=r"term 0 of the source: .* reaches 1250 on the box \[-50.0, 50.0\]"):
        ps.check_source_range([h], [-50.0, 0.0], [50.0, 10.0])
    (k,) = ps.parse_source("x*exp(t**2 + 100*t)")
    with pytest.raises(ps.SpecError, match="reaches 1100"):
        ps.check_source_range([k], [-1.0, 0.0], [1.0, 10.0])
    ps.check_source_range([k], [-1.0, 0.0], [1.0, 6.0])


def test_evaluate_source_follows_the_device_order():
    """The host evaluation of f_model(X) differs from the device only by numpy's sin, cos and exp: the products and sums are
    the table's, and trig arguments from 2^31 on give NaN."""
    rng = np.random.default_rng(5)
    x, t = rng.uniform(-1, 1, 500), rng.uniform(0, 1, 500)
    terms = ps.parse_source(MIXED, NAMES.get)
    s = ps.evaluate_source(terms, x, t)
    form, par = pinn_cabi.pack_source_terms(terms)
    worst, ok = st.check(s, form, par, x, t)
    assert ok and worst <= 1.0
    # the powers are repeated rounded products, a x^3 t^2 = ((((a x) x) x) t) t, not a * x**3 * t**2
    (cube,) = ps.parse_source("x**3*t**2")
    xs, ts = np.array([1.1, 0.7, -1.3]), np.array([0.3, 1.7, 2.9])
    assert np.array_equal(ps.evaluate_source([cube], xs, ts), (((1.0 * xs * xs) * xs) * ts) * ts)
    big = ps.evaluate_source(ps.parse_source("sin(x)"), np.array([2.0 ** 31 - 1, 2.0 ** 31]), np.zeros(2))
    assert np.isfinite(big[0]) and np.isnan(big[1])


def test_parser_refuses_non_strings():
    with pytest.raises(ps.SpecError, match="must be a string"):
        ps.parse_source(lambda x, t: x)


# ------------------------------------------------------------------------------------------------- binding validation
GOOD = (1.0, 1, 2, 1, 2.0, 0.5, 2, 3.0, -1.0, 0.1, -0.2, 0.3, -0.4)


def test_binding_packs_form_and_parameters():
    form, par = pinn_cabi.pack_source_terms([GOOD, T(2.0)])
    assert form.tolist() == [1 | 2 << 2 | 1 << 4 | 2 << 6, 0]
    assert par.tolist() == [[1.0, 2.0, 0.5, 3.0, -1.0, 0.1, -0.2, 0.3, -0.4], [2.0] + [0.0] * 8]
    assert st.unpack(form)[0].tolist() == [1, 0]
    form, par = pinn_cabi.pack_source_terms([])
    assert form.size == 0 and par.shape == (0, 9)


@pytest.mark.parametrize("i, v, msg", [(1, 4, "p = 4"), (2, -1, "q = -1"), (3, 3, "xkind = 3"), (6, 3, "tkind = 3"),
                                       (1, 1.0, "p = 1.0"), (3, True, "xkind = True")] +
                         [(j, bad, "parameter %s is not finite" % name)
                          for j, name in zip((0, 4, 5, 7, 8, 9, 10, 11, 12),
                                             ("a", "omega", "phi", "nu", "psi", "alpha", "gamma", "beta", "delta"))
                          for bad in (float("nan"), float("inf"), -float("inf"))])
def test_binding_refuses_what_the_header_refuses(i, v, msg):
    term = list(GOOD)
    term[i] = v
    with pytest.raises(pinn_cabi.PinnError, match="term 1: " + re.escape(msg)):
        pinn_cabi.pack_source_terms([GOOD, term])


def test_binding_refuses_too_many_terms_and_short_terms():
    with pytest.raises(pinn_cabi.PinnError, match="17 terms"):
        pinn_cabi.pack_source_terms([GOOD] * 17)
    pinn_cabi.pack_source_terms([GOOD] * 16)
    with pytest.raises(pinn_cabi.PinnError, match="12 entries"):
        pinn_cabi.pack_source_terms([GOOD[:12]])


# ------------------------------------------------------------------------------------------------------- mirror schedule
class StandIn(object):
    """Records every call the mirror makes on its handle (pinn_cabi.Pinn's method names)."""
    log = []

    def __init__(self, pde, layers, lb, ub, device=0, rank=0, world=1, nccl_uid=None):
        self.pde = pde

    def __getattr__(self, name):
        def call(*args, **kw):
            StandIn.log.append((name, args, kw))
            if name == "get_collocation":
                return np.zeros(40), np.zeros(40)
            return 0.5 if name == "last_loss" else None
        return call


class QuietLogger(object):
    def log_train_opt(self, name):
        pass

    def log_train_epoch(self, epoch, loss, custom="", is_iter=False):
        float(loss)


@pytest.fixture()
def mirror(monkeypatch):
    import neuralnetwork
    monkeypatch.setattr(pinn_cabi, "Pinn", StandIn)
    StandIn.log = []
    return neuralnetwork


def heat(nn, source, epochs=7, **hp_extra):
    hp = {"layers": [2, 8, 1], "tf_epochs": epochs, "tf_lr": 1e-3, "tf_b1": 0.9, "tf_eps": None, "nt_epochs": 0, "nt_lr": 0.8,
          "nt_ncorr": 50}
    hp.update(hp_extra)
    attrs = {"pde": "poly", "residual": "u_t - k*u_xx", "k": K}
    if source is not None:
        attrs["source"] = source

    def __init__(self):
        nn.NeuralNetwork.__init__(self, hp, QuietLogger(), np.array([1.0, 1.0]), np.array([-1.0, 0.0]))
        self.x_f, self.t_f = np.zeros((40, 1)), np.zeros((40, 1))
    attrs["__init__"] = __init__
    return type("Heat", (nn.NeuralNetwork,), attrs)()


def names(*which):
    return [n for n, _, _ in StandIn.log if n in which]


def callable_source(self, x, t):
    return np.sin(np.pi * x) * np.exp(-t)


def test_mirror_string_source_sets_a_table_and_never_reads_back(mirror):
    net = heat(mirror, HEAT, resample_every=2)
    net.tf_optimization(np.zeros((5, 2)), np.zeros((5, 1)))
    tables = [a for n, a, _ in StandIn.log if n == "set_source_terms"]
    assert tables == [(ps.parse_source(HEAT, NAMES.get),)]
    assert names("get_collocation", "set_source") == []
    want = []
    for e in range(7):
        want += (["draw_collocation"] if e > 0 and e % 2 == 0 else []) + ["adam_step"]
    assert names("draw_collocation", "adam_step") == want


def test_mirror_callable_source_keeps_one_read_back_per_draw(mirror):
    net = heat(mirror, callable_source, resample_every=2)
    net.tf_optimization(np.zeros((5, 2)), np.zeros((5, 1)))
    assert names("set_source_terms") == []
    assert names("draw_collocation", "get_collocation", "set_source") == ["set_source"] + \
        ["draw_collocation", "get_collocation", "set_source"] * 3


def test_mirror_absent_source_sets_nothing(mirror):
    heat(mirror, None, resample_every=2).tf_optimization(np.zeros((5, 2)), np.zeros((5, 1)))
    assert names("set_source_terms", "set_source", "get_collocation") == []


def test_mirror_rad_gate_takes_string_sources_only(mirror):
    for source in (HEAT, "0"):
        StandIn.log = []
        heat(mirror, source, rad_every=3, resample_seed=5).tf_optimization(np.zeros((5, 2)), np.zeros((5, 1)))
        assert [a for n, a, _ in StandIn.log if n == "draw_collocation_rad"] == [(5, d, 40, 400, 1, 1.0) for d in (1, 2)]
        assert names("get_collocation", "set_source") == []
    for source in (None, callable_source):
        StandIn.log = []
        with pytest.raises(pinn_cabi.PinnError, match="rad_every.*string source"):
            heat(mirror, source, rad_every=3).tf_optimization(np.zeros((5, 2)), np.zeros((5, 1)))
        assert names("draw_collocation_rad") == []


def test_mirror_reports_bad_source_strings(mirror):
    with pytest.raises(pinn_cabi.PinnError, match="Heat.source: .*two trig factors in x"):
        heat(mirror, "sin(x)*cos(x)").tf_optimization(np.zeros((5, 2)), np.zeros((5, 1)))
    with pytest.raises(pinn_cabi.PinnError, match="Heat.source: .*exp\\(-900.0\\) is 0.0"):
        heat(mirror, "exp(-100*(x - 3)**2)").tf_optimization(np.zeros((5, 2)), np.zeros((5, 1)))
    with pytest.raises(pinn_cabi.PinnError, match=r"Heat.source: term 0 of the source: .* reaches 800 on the box \[-1.0, 1.0\]"):
        heat(mirror, "exp(800*x**2)").tf_optimization(np.zeros((5, 2)), np.zeros((5, 1)))
    assert names("set_source_terms") == []


# ------------------------------------------------------------------------------------------------------------- library
def test_library_exports_and_binds_the_source_calls(lib_built):
    import ctypes
    lib = ctypes.CDLL(lib_built)
    for name in ("pinn_set_source_terms", "pinn_get_source"):
        assert hasattr(lib, name) and name in pinn_cabi.SIGNATURES


def test_source_kernels_have_no_stack_and_no_local_memory(lib_built):
    out = subprocess.run(["cuobjdump", "-res-usage", lib_built], capture_output=True, text=True).stdout
    m = re.findall(r"Function (\S*4pinn6source\S*?):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:\d+ LOCAL:(\d+)", out)
    assert sorted(re.search(r"source\d+(\w+?)_kernel", name).group(1) for name, *_ in m) == ["eval", "pool_head"], m
    for name, regs, stack, local in m:
        assert int(stack) == 0 and int(local) == 0, name
    elf = subprocess.run(["cuobjdump", "-lelf", lib_built], capture_output=True, text=True).stdout
    assert "sm_90a" in elf
