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
