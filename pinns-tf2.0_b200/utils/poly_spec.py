"""Residual strings of user-defined PDEs -> the term table of ``pinn_set_residual`` (include/pinn_b200.h).

    parse("u_t + u*u_x - nu*u_xx", resolve) -> Spec(terms=[(coef, kind, (e_u, e_ux, e_ut, e_uxx)), ...], identification)

The string is read with ``ast`` (never ``eval``).  It may use numbers; the streams ``u``, ``u_x``, ``u_t``, ``u_xx``; the raw
trainable scalars ``l1``, ``l2`` and ``exp(l1)``, ``exp(l2)``; any other name that ``resolve`` maps to a number (the
subclass's numeric attributes); ``+``, ``-``, ``*``, parentheses, and ``**`` with a literal non-negative integer exponent.
Products of sums are expanded and like terms combined.  Anything outside the class the kernel evaluates -- a stream exponent
above 3, more than 16 terms, a product of two lambda factors, division, a term without a stream factor -- is rejected with a
message that names the offending piece.
"""
import ast
from collections import namedtuple

import numpy as np

STREAMS = ("u", "u_x", "u_t", "u_xx")
LAMBDAS = {"l1": 1, "l2": 2}
EXP_LAMBDAS = {"l1": 3, "l2": 4}
KIND_NAMES = ("1", "l1", "l2", "exp(l1)", "exp(l2)")
MAX_TERMS = 16
MAX_EXP = 3

Spec = namedtuple("Spec", "terms identification")


class SpecError(ValueError):
    pass


def _piece(node):
    return "'%s'" % ast.unparse(node)


def _mul(a, b, node):
    """Product of two polynomials {(kind, e_u, e_ux, e_ut, e_uxx): coef}."""
    out = {}
    for ka, ca in a.items():
        for kb, cb in b.items():
            if ka[0] and kb[0]:
                raise SpecError("%s: product of two lambda factors (%s * %s); each term takes at most one of l1, l2, exp(l1), "
                                "exp(l2)" % (_piece(node), KIND_NAMES[ka[0]], KIND_NAMES[kb[0]]))
            e = tuple(x + y for x, y in zip(ka[1:], kb[1:]))
            for j, v in enumerate(e):
                if v > MAX_EXP:
                    raise SpecError("%s: %s appears to the power %d; stream exponents go up to %d" % (_piece(node), STREAMS[j], v,
                                                                                                 MAX_EXP))
            key = (ka[0] or kb[0],) + e
            out[key] = out.get(key, 0.0) + ca * cb
    return out


def _add(a, b, sign=1.0):
    out = dict(a)
    for k, c in b.items():
        out[k] = out.get(k, 0.0) + sign * c
    return out


def _const(c):
    return {(0, 0, 0, 0, 0): float(c)}


def _expand(node, resolve):
    if isinstance(node, ast.Expression):
        return _expand(node.body, resolve)
    if isinstance(node, ast.Constant):
        if isinstance(node.value, bool) or not isinstance(node.value, (int, float)):
            raise SpecError("%s: only numbers may appear as constants" % _piece(node))
        return _const(node.value)
    if isinstance(node, ast.Name):
        if node.id in STREAMS:
            e = [0, 0, 0, 0]
            e[STREAMS.index(node.id)] = 1
            return {(0,) + tuple(e): 1.0}
        if node.id in LAMBDAS:
            return {(LAMBDAS[node.id], 0, 0, 0, 0): 1.0}
        v = resolve(node.id) if resolve is not None else None
        if v is None:
            raise SpecError("name %s is neither a stream (u, u_x, u_t, u_xx), a lambda (l1, l2) nor a numeric attribute" %
                            _piece(node))
        return _const(v)
    if isinstance(node, ast.Call):
        if (isinstance(node.func, ast.Name) and node.func.id == "exp" and len(node.args) == 1 and not node.keywords
                and isinstance(node.args[0], ast.Name) and node.args[0].id in EXP_LAMBDAS):
            return {(EXP_LAMBDAS[node.args[0].id], 0, 0, 0, 0): 1.0}
        raise SpecError("%s: the only calls are exp(l1) and exp(l2)" % _piece(node))
    if isinstance(node, ast.UnaryOp) and isinstance(node.op, (ast.UAdd, ast.USub)):
        p = _expand(node.operand, resolve)
        return p if isinstance(node.op, ast.UAdd) else {k: -c for k, c in p.items()}
    if isinstance(node, ast.BinOp):
        if isinstance(node.op, (ast.Div, ast.FloorDiv, ast.Mod)):
            raise SpecError("%s: division is not supported; write the reciprocal as a number or a numeric attribute" %
                            _piece(node))
        if isinstance(node.op, ast.Pow):
            n = node.right
            if not (isinstance(n, ast.Constant) and isinstance(n.value, int) and not isinstance(n.value, bool) and n.value >= 0):
                raise SpecError("%s: the exponent of ** must be a literal non-negative integer" % _piece(node))
            base = _expand(node.left, resolve)
            out = _const(1.0)
            for _ in range(n.value):
                out = _mul(out, base, node)
            return out
        a, b = _expand(node.left, resolve), _expand(node.right, resolve)
        if isinstance(node.op, ast.Add):
            return _add(a, b)
        if isinstance(node.op, ast.Sub):
            return _add(a, b, -1.0)
        if isinstance(node.op, ast.Mult):
            return _mul(a, b, node)
    raise SpecError("%s is not supported (numbers, u, u_x, u_t, u_xx, l1, l2, exp(l1), exp(l2), numeric attributes, "
                    "+, -, *, ** with an integer literal, parentheses)" % _piece(node))


def parse(text, resolve=None):
    """The residual string -> Spec.  resolve(name) returns the number a free name stands for, or None."""
    if not isinstance(text, str):
        raise SpecError("the residual must be a string such as 'u_t + u*u_x - nu*u_xx'")
    try:
        tree = ast.parse(text.strip(), mode="eval")
    except SyntaxError as e:
        raise SpecError("cannot parse the residual %r: %s" % (text, e.msg))
    poly = _expand(tree, resolve)
    terms = []
    for key, c in poly.items():
        if c == 0.0:
            continue
        if not np.isfinite(c):
            raise SpecError("the coefficient of a term is not finite (%r)" % c)
        kind, e = key[0], key[1:]
        if not any(e):
            raise SpecError("the term %s has no stream factor; a term without u, u_x, u_t or u_xx belongs in source(x, t)" %
                            _format_term(c, kind, e))
        terms.append((float(c), int(kind), tuple(int(v) for v in e)))
    if not terms:
        raise SpecError("the residual %r is identically zero" % text)
    if len(terms) > MAX_TERMS:
        raise SpecError("the residual expands to %d terms; at most %d are supported" % (len(terms), MAX_TERMS))
    return Spec(terms, any(k != 0 for _, k, _ in terms))


def _format_term(c, kind, e):
    f = [repr(c)] + ([KIND_NAMES[kind]] if kind else [])
    f += [s if v == 1 else "%s**%d" % (s, v) for s, v in zip(STREAMS, e) if v]
    return "*".join(f)


def format_terms(terms):
    return " + ".join(_format_term(c, k, e) for c, k, e in terms)


def evaluate(terms, streams, l1=0.0, l2=0.0):
    """f without the source: sum_k c_k kappa_k u^a u_x^b u_t^c u_xx^d on arrays streams = (u, u_x, u_t, u_xx)."""
    kv = (1.0, l1, l2, np.exp(l1), np.exp(l2))
    f = 0.0
    for c, k, e in terms:
        m = c * kv[k]
        for v, p in zip(streams, e):
            if p:
                m = m * np.asarray(v) ** p
        f = f + m
    return f


# ------------------------------------------------------------------------------------------------- source s(x, t)
# A source string -> the term table of pinn_set_source_terms: a sum of up to 16 terms
#   a x^p t^q X(x) T(t) exp(alpha x + gamma x^2 + beta t + delta t^2),  X, T in {1, sin(affine), cos(affine)}.
SourceTerm = namedtuple("SourceTerm", "a p q xkind omega phi tkind nu psi alpha gamma beta delta")
SOURCE_VARS = ("x", "t")
TRIG = {"sin": 1, "cos": 2}
_NO_EXP = (0.0, 0.0, 0.0, 0.0)          # (alpha, gamma, beta, delta)
TINY = float(np.finfo(np.float64).tiny)  # the least normal fp64 number
EXP_MAX = float(np.log(np.finfo(np.float64).max))   # 709.78...: exp overflows above it


def _folded(c, node, what, hint=""):
    """A coefficient that folding constants made: refused when it overflowed, or when a nonzero value fell to 0 or below the
    normal range (it would silently drop the term, or keep only a few significant bits of it)."""
    if not np.isfinite(c):
        raise SpecError("%s: %s overflows fp64" % (_piece(node), what))
    if abs(c) < TINY:
        raise SpecError("%s: %s is %r, below the normal fp64 range, so the term's coefficient a would lose it%s" %
                        (_piece(node), what, c, hint))
    return c


def _skey(p=0, q=0, xf=None, tf=None, ex=_NO_EXP):
    """Key of a source monomial: powers of x and t, the trig factor in x and in t ((kind, omega, phi) or None), the exponent."""
    return (p, q, xf, tf, ex)


def _smul(a, b, node):
    out = {}
    for ka, ca in a.items():
        for kb, cb in b.items():
            p, q = ka[0] + kb[0], ka[1] + kb[1]
            for var, v in (("x", p), ("t", q)):
                if v > MAX_EXP:
                    raise SpecError("%s: %s appears to the power %d; powers of x and t go up to %d" % (_piece(node), var, v, MAX_EXP))
            for i, var in ((2, "x"), (3, "t")):
                if ka[i] is not None and kb[i] is not None:
                    raise SpecError("%s: two trig factors in %s; a term takes at most one sin or cos of each variable" %
                                    (_piece(node), var))
            ex = tuple(u + v for u, v in zip(ka[4], kb[4]))
            key = _skey(p, q, ka[2] if ka[2] is not None else kb[2], ka[3] if ka[3] is not None else kb[3], ex)
            c = ca * cb
            if ca != 0.0 and cb != 0.0:
                c = _folded(c, node, "the product of the coefficients")
            out[key] = out.get(key, 0.0) + c
    return out


def _sconst(c):
    return {_skey(): float(c)}


def _plain(poly, node, what):
    """A source polynomial without trig or exp factors -> {(p, q): coef}."""
    out = {}
    for k, c in poly.items():
        if k[2] is not None or k[3] is not None or k[4] != _NO_EXP:
            raise SpecError("%s: %s" % (_piece(node), what))
        if c != 0.0:
            out[(k[0], k[1])] = out.get((k[0], k[1]), 0.0) + c
    return out


def _sexpand(node, resolve):
    import math
    if isinstance(node, ast.Expression):
        return _sexpand(node.body, resolve)
    if isinstance(node, ast.Constant):
        if isinstance(node.value, bool) or not isinstance(node.value, (int, float)):
            raise SpecError("%s: only numbers may appear as constants" % _piece(node))
        return _sconst(node.value)
    if isinstance(node, ast.Name):
        if node.id == "x":
            return {_skey(p=1): 1.0}
        if node.id == "t":
            return {_skey(q=1): 1.0}
        if node.id == "pi":
            return _sconst(math.pi)
        v = resolve(node.id) if resolve is not None else None
        if v is None:
            raise SpecError("name %s is neither x, t, pi nor a numeric attribute" % _piece(node))
        return _sconst(v)
    if isinstance(node, ast.Call):
        fn = node.func.id if isinstance(node.func, ast.Name) else None
        if fn not in ("sin", "cos", "exp"):
            raise SpecError("%s: unknown function; the source may call sin, cos and exp" % _piece(node))
        if len(node.args) != 1 or node.keywords:
            raise SpecError("%s: %s takes one argument" % (_piece(node), fn))
        arg = _sexpand(node.args[0], resolve)
        if fn == "exp":
            poly = _plain(arg, node, "exp takes a polynomial of degree <= 2 in x and t without an x*t term")
            ex, c0 = [0.0, 0.0, 0.0, 0.0], 0.0
            slots = {(1, 0): 0, (2, 0): 1, (0, 1): 2, (0, 2): 3}
            for (p, q), c in poly.items():
                if (p, q) == (0, 0):
                    c0 = c
                elif (p, q) in slots:
                    ex[slots[(p, q)]] = c
                else:
                    raise SpecError("%s: exp takes a polynomial of degree <= 2 in x and t without an x*t term (it has x^%d t^%d)" %
                                    (_piece(node), p, q))
            # the constant part moves into a: a Gaussian exp(-w (x - x0)^2) becomes e^(-w x0^2) exp(2 w x0 x - w x^2), and
            # e^(-w x0^2) must be a normal fp64 number (w x0^2 below about 708)
            try:
                a = math.exp(c0)
            except OverflowError:
                a = math.inf
            return {_skey(ex=tuple(ex)): _folded(a, node, "the constant part of its exponent, exp(%r)" % c0,
                                                 "; a Gaussian exp(-w*(x - x0)**2) needs w*x0**2 below about 708")}
        poly = _plain(arg, node, "%s takes an affine function of x or of t" % fn)
        c0 = poly.pop((0, 0), 0.0)
        if not poly:
            return _sconst(math.sin(c0) if fn == "sin" else math.cos(c0))
        if len(poly) != 1 or list(poly)[0] not in ((1, 0), (0, 1)):
            raise SpecError("%s: %s takes an affine function of one variable, omega*x + phi or nu*t + psi" % (_piece(node), fn))
        (p, q), w = list(poly.items())[0]
        f = (TRIG[fn], w, c0)
        return {_skey(xf=f) if p else _skey(tf=f): 1.0}
    if isinstance(node, ast.UnaryOp) and isinstance(node.op, (ast.UAdd, ast.USub)):
        p = _sexpand(node.operand, resolve)
        return p if isinstance(node.op, ast.UAdd) else {k: -c for k, c in p.items()}
    if isinstance(node, ast.BinOp):
        if isinstance(node.op, (ast.Div, ast.FloorDiv, ast.Mod)):
            raise SpecError("%s: division is not supported; write the reciprocal as a number or a numeric attribute" %
                            _piece(node))
        if isinstance(node.op, ast.Pow):
            n = node.right
            if not (isinstance(n, ast.Constant) and isinstance(n.value, int) and not isinstance(n.value, bool) and n.value >= 0):
                raise SpecError("%s: the exponent of ** must be a literal non-negative integer" % _piece(node))
            base = _sexpand(node.left, resolve)
            out = _sconst(1.0)
            for _ in range(n.value):
                out = _smul(out, base, node)
            return out
        a, b = _sexpand(node.left, resolve), _sexpand(node.right, resolve)
        if isinstance(node.op, (ast.Add, ast.Sub)):
            out = dict(a)
            for k, c in b.items():
                out[k] = out.get(k, 0.0) + (c if isinstance(node.op, ast.Add) else -c)
            return out
        if isinstance(node.op, ast.Mult):
            return _smul(a, b, node)
    raise SpecError("%s is not supported (numbers, x, t, pi, numeric attributes, +, -, *, ** with an integer literal, "
                    "sin and cos of an affine function of x or t, exp of a quadratic in x and t, parentheses)" % _piece(node))


def parse_source(text, resolve=None):
    """The source string -> [SourceTerm, ...] for pinn_set_source_terms (an empty list for a zero source, e.g. "0").  Products of
    sums are expanded, products of exp factors add their exponents, a constant in an exponent moves into a, and like terms are
    combined.  resolve(name) returns the number a free name stands for, or None."""
    if not isinstance(text, str):
        raise SpecError("the source must be a string such as '(k*pi**2 - 1)*sin(pi*x)*exp(-t)'")
    try:
        tree = ast.parse(text.strip(), mode="eval")
    except SyntaxError as e:
        raise SpecError("cannot parse the source %r: %s" % (text, e.msg))
    terms = []
    for (p, q, xf, tf, ex), c in _sexpand(tree, resolve).items():
        if c == 0.0:
            continue
        if not all(np.isfinite(v) for v in (c,) + (xf or (0, 0, 0))[1:] + (tf or (0, 0, 0))[1:] + ex):
            raise SpecError("a term of the source has a parameter that is not finite (coefficient %r)" % c)
        if abs(c) < TINY:
            raise SpecError("the coefficient of a term of the source is below the normal fp64 range (%r)" % c)
        xk, om, ph = xf or (0, 0.0, 0.0)
        tk, nu, ps = tf or (0, 0.0, 0.0)
        terms.append(SourceTerm(float(c), p, q, xk, float(om), float(ph), tk, float(nu), float(ps), *(float(v) for v in ex)))
    if len(terms) > MAX_TERMS:
        raise SpecError("the source expands to %d terms; at most %d are supported" % (len(terms), MAX_TERMS))
    return terms


def check_source_range(terms, lb, ub):
    """Refuse a table whose exp factor overflows somewhere on the box [lb, ub] of (x, t): the largest exponent
    alpha x + gamma x^2 + beta t + delta t^2 there must stay below log(DBL_MAX) = 709.78."""
    def top(c1, c2, lo, hi):
        cand = [lo, hi] + ([-c1 / (2 * c2)] if c2 < 0 and lo < -c1 / (2 * c2) < hi else [])
        return max(c1 * v + c2 * v * v for v in cand)
    for k, tm in enumerate(terms):
        z = top(tm.alpha, tm.gamma, float(lb[0]), float(ub[0])) + top(tm.beta, tm.delta, float(lb[1]), float(ub[1]))
        if z > EXP_MAX:
            raise SpecError("term %d of the source: its exponent %r x + %r x^2 + %r t + %r t^2 reaches %.6g on the box [%r, %r] x "
                            "[%r, %r], where exp overflows (above %.6g); centre the exponent or shrink it" %
                            (k, tm.alpha, tm.gamma, tm.beta, tm.delta, z, float(lb[0]), float(ub[0]), float(lb[1]), float(ub[1]),
                             EXP_MAX))


def evaluate_source(terms, x, t):
    """s(x, t) of a source table on arrays in fp64, in the device's order with every product and sum rounded (numpy does not
    contract), NaN trig factors from |argument| >= 2^31, and numpy's sin, cos and exp in place of CUDA's: the two differ only by
    those functions' last bits (definition: include/pinn_b200.h, pinn_set_source_terms)."""
    x, t = np.asarray(x, dtype=np.float64), np.asarray(t, dtype=np.float64)
    s = np.zeros(np.broadcast(x, t).shape)

    def trig(kind, arg):
        with np.errstate(invalid="ignore"):
            v = (np.sin if kind == 1 else np.cos)(arg)
        return np.where(np.abs(arg) < 2.0 ** 31, v, np.nan)

    with np.errstate(all="ignore"):
        for a, p, q, xk, om, ph, tk, nu, ps, al, ga, be, de in terms:
            m = np.full(s.shape, float(a))
            for _ in range(p):
                m = m * x
            for _ in range(q):
                m = m * t
            if xk:
                m = m * trig(xk, om * x + ph)
            if tk:
                m = m * trig(tk, nu * t + ps)
            if al != 0.0 or ga != 0.0 or be != 0.0 or de != 0.0:
                m = m * np.exp(((al * x + ga * (x * x)) + be * t) + de * (t * t))
            s = s + m
    return s
