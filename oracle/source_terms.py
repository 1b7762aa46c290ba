"""Extended-precision restatement of the source tables of pinn_set_source_terms (include/pinn_b200.h, DESIGN §4.8).

    s_ld = source(form, par, x, t)          longdouble s(x, t): the table's value at the fp64 trig and exp arguments
    b = error_bound(form, par, x, t)        the bound the device's fp64 s keeps to s_ld: |s - s_ld| <= b

CUDA's sin, cos and exp are not correctly rounded, so numpy cannot restate the device's bits.  Instead the arguments of sin, cos
and exp are formed exactly as the device forms them (fp64, each product and sum rounded; numpy's fp64 operations round the same
way), the functions are evaluated in longdouble on those arguments, and the products and the sum are taken in longdouble.  The
device's result then differs from s_ld only by the errors of its own operations (u = 2^-53):
  - each fp64 product and sum: at most u relative;
  - sin, cos: at most 2 ulp (4u relative), exp: at most 1 ulp (2u relative), CUDA Math API error table (double precision);
so a term with c multiplications, n_x + n_t trig factors and n_e exp factors is within
((c + 4 (n_x + n_t) + 2 n_e) u)(1 + 0.01) of its value, and the left-to-right sum of n terms adds (n - 1) u times the sum of |terms|.
The bound is sum_k |m_k| ((c_k + 4 (n_x + n_t)_k + 2 n_e,k + n) u)(1.01) + sum_k (|m_k without exp| + 1) 2^-1070: the last part
covers an exp result in the subnormal range, where the relative bounds do not hold.  sin and cos of an argument of magnitude
2^31 or more are NaN, as on the device.
"""
import numpy as np

LD = np.longdouble
U = 2.0 ** -53
TRIG_MAX = 2.0 ** 31


def unpack(form):
    f = np.asarray(form, dtype=np.int64)
    return f & 3, (f >> 2) & 3, (f >> 4) & 3, (f >> 6) & 3


def _trig(kind, arg64):
    a = np.asarray(arg64, dtype=np.float64)
    v = (np.sin if kind == 1 else np.cos)(a.astype(LD))
    return np.where(np.abs(a) < TRIG_MAX, v, LD(np.nan))


def _terms(form, par, x, t):
    """Per term: (|m| of the longdouble term, |m| without its exp factor, operation count c + 4 n_trig + 2 n_exp, the term)."""
    x = np.asarray(x, dtype=np.float64)
    t = np.asarray(t, dtype=np.float64)
    P, Q, XK, TK = unpack(form)
    par = np.asarray(par, dtype=np.float64).reshape(-1, 9)
    out = []
    with np.errstate(all="ignore"):
        for k in range(par.shape[0]):
            a, om, ph, nu, ps, al, ga, be, de = par[k]
            m = np.full(x.shape, LD(a))
            ops = int(P[k] + Q[k])
            m = m * x.astype(LD) ** int(P[k]) * t.astype(LD) ** int(Q[k])
            if XK[k]:
                m = m * _trig(XK[k], om * x + ph)          # fp64 argument, as on the device
                ops += 5
            if TK[k]:
                m = m * _trig(TK[k], nu * t + ps)
                ops += 5
            pre = np.abs(m)
            if al != 0.0 or ga != 0.0 or be != 0.0 or de != 0.0:
                z = ((al * x + ga * (x * x)) + be * t) + de * (t * t)
                m = m * np.exp(z.astype(LD))
                ops += 3
            out.append((np.abs(m), pre, ops, m))
    return out


def source(form, par, x, t):
    """s(x, t) in longdouble; NaN wherever the device's s is NaN (non-finite points, trig arguments from 2^31 on)."""
    x = np.asarray(x, dtype=np.float64)
    s = np.zeros(x.shape, dtype=LD)
    for _, _, _, m in _terms(form, par, x, t):
        s = s + m
    return s


def error_bound(form, par, x, t):
    terms = _terms(form, par, x, t)
    n = len(terms)
    b = np.zeros(np.asarray(x).shape, dtype=LD)
    for am, pre, ops, _ in terms:
        b = b + am * LD((ops + n) * U * 1.01) + (pre + 1) * LD(2.0 ** -1070)
    return b


def check(s_dev, form, par, x, t):
    """(worst |s_dev - s_ld| / bound over the finite entries, whether s_dev is non-finite exactly where s_ld is)."""
    s_ld = source(form, par, x, t)
    b = error_bound(form, par, x, t)
    s_dev = np.asarray(s_dev, dtype=np.float64)
    fin = np.isfinite(s_ld)
    same_nonfinite = bool(np.array_equal(fin, np.isfinite(s_dev)))
    with np.errstate(all="ignore"):
        r = np.abs(s_dev[fin].astype(LD) - s_ld[fin]) / b[fin]
    return (float(r.max()) if r.size else 0.0), same_nonfinite
