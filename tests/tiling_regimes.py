"""The tiling regimes of the generic and Navier-Stokes fused kernels, restated from their launch and item formulas, and a
deterministic sweep of shapes that reaches every one of them.

Both kernels split their work with integer formulas: points over CTAs (pinn_api.cu: generic_launch_eval, ns_launch_eval), and,
inside a CTA, GEMM work items over point groups, column groups, row tiles and k steps (generic_fused.cuh: fused_loss_grad and
dmma_rows; navier_stokes_fused.cuh: fused_loss_grad and gemm13).  A wrong split (a group dropped, a tail skipped, a bias row
lost) is only visible at the shapes whose split takes that branch.  This module

* declares the regime cells one evaluation can touch (universe(), one place) and computes the cells of one evaluation
  (generic_cells, ns_cells);
* builds sweep(sms): layer lists, point counts and heads, chosen greedily from a fixed seed until every cell is reached;
* walks the item decomposition of every GEMM phase in numpy (walk_generic_layer, walk_ns_layer, walk_cta_split): how often each
  output element is written and how often each k term is added to it.  `bugs` names broken decompositions (BUGS) that the walk
  can apply; they exist only here, in numpy, and are never compiled.

Every item list of the kernels is a product: (point groups x column groups) or (row tiles x column groups), and inside an item
the same k steps.  The walk builds each phase from those factors (point_groups, col_groups, row_tiles, ksteps), so a phase is
exact-once exactly when each factor is; tests/test_tiling_regimes_cpu.py checks the factors over their whole ranges and the
composed walk on every sweep shape.
"""
import numpy as np

NTW = 4                 # generic_fused.cuh: N tiles (of 8 columns) per DMMA work item
WARPS = 8               # 256-thread CTAs
MAXW = 128              # optim_kernels.cuh: mlp_forward_generic's narrow instantiation; MAXW_WIDE = 256 above it
MAX_HIDDEN = 14         # 15 Dense layers at most
HEADS = ("inf", "ide", "nls", "disc", "kdv")   # Burgers inference / identification, Schrodinger, Burgers disc (pde 3), KdV

# Broken decompositions the walk can apply (name: what it stands for)
BUGS = {
    "tpg_floor": "tiles per column group rounded down: tpg = nt // ngrp",
    "ntn_no_min": "tiles of a column group without the min: ntn = nt - grp * tpg",
    "k_tail_dropped": "the K & 3 tail of dmma_rows / gemm13 skipped",
    "bias_row_pos7": "the bias row lost when it is the last row of its 8-row tile (fi % 8 == 7)",
    "last_point_group_dropped": "point groups counted as npts >> 3 (16-point tiles: npts >> 4)",
    "wgrad_npts_tail_dropped": "the npts & 3 tail of the weight-gradient K loop skipped",
    "ns_bias_tile_off_by_one": "Navier-Stokes weight-gradient row tiles (fi + 15) >> 4: no tile for a bias row at 16 m",
    "cta_base_per": "each CTA's first point taken as blockIdx * per instead of blockIdx * pts",
}


def cdiv(a, b):
    return -(-a // b)


# --------------------------------------------------------------------------------------------------------- factor walks
def col_groups(N, bugs=()):
    """generic_fused.cuh: the columns of each column group of a DMMA phase over N columns (forward: N = fo, input adjoint and
    weight-gradient columns as stated there):  nt = ceil(N/8), ngrp = ceil(nt/NTW), tpg = ceil(nt/ngrp),
    n0 = 8 grp tpg, ntn = min(tpg, nt - grp tpg); tile j < ntn, column n0 + 8j + c stored while < N."""
    nt = cdiv(N, 8)
    ngrp = cdiv(nt, NTW)
    tpg = nt // ngrp if "tpg_floor" in bugs else cdiv(nt, ngrp)
    out = []
    for grp in range(ngrp):
        n0 = 8 * grp * tpg
        ntn = nt - grp * tpg if "ntn_no_min" in bugs else min(tpg, nt - grp * tpg)
        out.append([n0 + 8 * j + c for j in range(NTW) if j < ntn for c in range(8) if n0 + 8 * j + c < N])
    return out


def group_signature(N):
    """The tiles of each column group: the regime of the forward / adjoint column split over N columns."""
    nt = cdiv(N, 8)
    ngrp = cdiv(nt, NTW)
    tpg = cdiv(nt, ngrp)
    return tuple(min(tpg, nt - g * tpg) for g in range(ngrp))


def point_groups(npts, rows, bugs=()):
    """Point groups of `rows` points (generic 8, Navier-Stokes 16): ceil(npts / rows) groups, row r stored while < npts."""
    n = npts // rows if "last_point_group_dropped" in bugs else cdiv(npts, rows)
    return [[rows * p + r for r in range(rows) if rows * p + r < npts] for p in range(n)]


def ksteps(K, tail_bug=None, bugs=()):
    """The k terms a DMMA k loop adds: K >> 2 full steps of 4, then (K & 3) the tail with k >= K masked to zero."""
    ks = list(range(4 * (K >> 2)))
    if K & 3 and tail_bug not in bugs:
        ks += [k for k in range(4 * (K >> 2), 4 * (K >> 2) + 4) if k < K]
    return ks


def row_tiles(fi, rows, bugs=()):
    """Row tiles of [W_l ; b_l] in the weight gradient: generic ceil((fi + 1) / 8) tiles of 8 (generic_fused.cuh: mt_w),
    Navier-Stokes (fi + 1 + 15) >> 4 tiles of 16; row fi is the bias, rows above fi are not stored."""
    if rows == 16 and "ns_bias_tile_off_by_one" in bugs:
        mt = (fi + 15) >> 4
    else:
        mt = cdiv(fi + 1, rows)
    out = []
    for t in range(mt):
        rs = [rows * t + r for r in range(rows) if rows * t + r <= fi]
        if rows == 8 and "bias_row_pos7" in bugs and fi % 8 == 7:
            rs = [i for i in rs if i != fi]
        out.append(rs)
    return out


def ns_col_tiles(N):
    """navier_stokes_fused.cuh: column tiles of 8, one per item: nt = (N + 7) >> 3, column n0 + 2q + e stored while < N."""
    return [[8 * t + c for c in range(8) if 8 * t + c < N] for t in range(cdiv(N, 8))]


def compose(row_items, col_items, kidx, R, Cn, K):
    """Counts of an item list row_items x col_items (item it -> row item it // len(col_items), column item the rest, as the
    kernels decode it), every item adding the k terms kidx.  Returns (writes [R, Cn], adds [R, Cn, K]); entries past R, Cn or K
    would be a write out of range and raise."""
    writes = np.zeros((R, Cn), np.int64)
    adds = np.zeros((R, Cn, K), np.int64)
    kc = np.bincount(np.asarray(kidx, np.int64), minlength=K) if len(kidx) else np.zeros(K, np.int64)
    if len(kc) > K:
        raise IndexError("k term out of range")
    ncol = len(col_items)
    for it in range(len(row_items) * ncol):
        rows, cols = row_items[it // ncol], col_items[it % ncol]
        if not rows or not cols:
            continue
        ix = np.ix_(rows, cols)
        writes[ix] += 1
        adds[ix] += kc
    return writes, adds


def walk_generic_layer(fi, fo, npts, bugs=()):
    """The three DMMA phases of a hidden-to-hidden layer (fi -> fo) of generic_fused.cuh over one CTA's npts points:
    forward  [npts x fo] over K = fi;  weight gradient [(fi + 1) x fo] over K = the CTA's points;  input adjoint [npts x fi]
    over K = fo."""
    pg = point_groups(npts, 8, bugs)
    return {
        "forward": compose(pg, col_groups(fo, bugs), ksteps(fi, "k_tail_dropped", bugs), npts, fo, fi),
        "weight gradient": compose(row_tiles(fi, 8, bugs), col_groups(fo, bugs), ksteps(npts, "wgrad_npts_tail_dropped", bugs),
                                   fi + 1, fo, npts),
        "input adjoint": compose(pg, col_groups(fi, bugs), ksteps(fo, "k_tail_dropped", bugs), npts, fi, fo),
    }


def walk_ns_layer(fi, fo, npts, bugs=()):
    """The three DMMA.16x8x4 phases of a hidden-to-hidden layer of navier_stokes_fused.cuh (items of 16 points x 8 columns,
    weight-gradient row tiles of 16)."""
    pt = point_groups(npts, 16, bugs)
    return {
        "forward": compose(pt, ns_col_tiles(fo), ksteps(fi, "k_tail_dropped", bugs), npts, fo, fi),
        "weight gradient": compose(row_tiles(fi, 16, bugs), ns_col_tiles(fo), ksteps(npts, "wgrad_npts_tail_dropped", bugs),
                                   fi + 1, fo, npts),
        "input adjoint": compose(pt, ns_col_tiles(fi), ksteps(fo, "k_tail_dropped", bugs), npts, fi, fo),
    }


def exact_once(phases):
    """The phases (name: (writes, adds)) whose counts are not all 1."""
    return [name for name, (w, a) in phases.items() if not (np.all(w == 1) and np.all(a == 1))]


# ------------------------------------------------------------------------------------------------------------ point splits
def generic_split(n_total, sms):
    """pinn_api.cu: generic_launch_eval with C = 2 x SM count CTAs (pinn_create): per = ceil(n / C), pts rounded up to a multiple
    of 16 from 16 on and to an even count below; grid = ceil(n / pts), only CTAs that own points."""
    C = 2 * sms
    per = cdiv(n_total, C)
    pts = cdiv(per, 16) * 16 if per >= 16 else cdiv(per, 2) * 2
    return dict(n_cta=C, per=per, pts=pts, grid=cdiv(n_total, pts))


def ns_split(n_total, sms):
    """pinn_api.cu: ns_launch_eval, one CTA per SM: pts = ceil(n / SMs), grid = ceil(n / pts)."""
    pts = cdiv(n_total, sms)
    return dict(n_cta=sms, per=pts, pts=pts, grid=cdiv(n_total, pts))


def walk_cta_split(n_total, split, bugs=()):
    """(first point, point count) of every CTA, as fused_loss_grad derives them: base = blockIdx * pts,
    npts = clamp(n - base, 0, pts); and how often each of the n points is owned."""
    step = split["per"] if "cta_base_per" in bugs else split["pts"]
    ctas, owned = [], np.zeros(n_total, np.int64)
    for b in range(split["grid"]):
        base = b * step
        npts = max(0, min(split["pts"], n_total - base))
        ctas.append((base, npts))
        owned[base:base + npts] += 1
    return ctas, owned


def cta_counts(n_total, split):
    """The distinct point counts of the CTAs (full CTAs, then the last one)."""
    return sorted({npts for _, npts in walk_cta_split(n_total, split)[0]})


# ------------------------------------------------------------------------------------------------------------------- cells
def layer_cells(fi, fo, o3=False):
    """Cells of one hidden-to-hidden layer in the generic kernel's DMMA form."""
    cs = {("fwd k tail fi%4", fi % 4), ("fwd groups over fo", group_signature(fo)), ("fwd fo%8", fo % 8),
          ("adj k tail fo%4", fo % 4), ("adj groups over fi", group_signature(fi)), ("adj fi%8", fi % 8),
          ("bias row fi%8", fi % 8), ("bias row opens a tile", fi % 8 == 0),
          ("(fi%4, fo%4)", (fi % 4, fo % 4)), ("(fi%8, fo%8)", (fi % 8, fo % 8))}
    if o3:
        cs |= {("o3 " + k, v) for k, v in cs if k.startswith(("fwd", "bias"))}
    return cs


def ns_layer_cells(fi, fo):
    return {("ns fwd k tail fi%4", fi % 4), ("ns fo%8", fo % 8), ("ns adj k tail fo%4", fo % 4), ("ns adj fi%8", fi % 8),
            ("ns bias row (fi+1)%16", (fi + 1) % 16)}


def probe_cells(layers):
    """pinn_api.cu: forward_generic picks mlp_forward_generic<.., MAXW> when the widest of layers[1:] is <= 128."""
    w = max(layers[1:])
    return {("probe max width", (w, layers[0]))} if w in (MAXW, MAXW + 1) else set()


def generic_cells(layers, n_total, sms, form, pde):
    """The cells one evaluation of the generic kernel touches: `form` "dmma" or "dfma" (PINN_GENERIC_DFMA=1), `pde` one of
    HEADS.  Point cells carry the form; the DFMA form's loops are thread-per-entry, so only the DMMA form has shape cells."""
    sp = generic_split(n_total, sms)
    regime = "per<16" if sp["per"] < 16 else "per>=16"
    cs = {(form + " regime", regime), (form + " grid<n_cta", sp["grid"] < sp["n_cta"])}
    counts = cta_counts(n_total, sp)
    for npts in counts:
        cs |= {(form + " CTA npts%8", (regime, npts % 8)), (form + " CTA npts%4", npts % 4)}
    hidden = layers[1:-1]
    if form == "dmma":
        for fi, fo in zip(hidden, hidden[1:]):
            cs |= layer_cells(fi, fo, o3=pde == "kdv")
            for npts in counts:
                if cdiv(npts, 8) * len(group_signature(fo)) < WARPS:
                    cs.add(("dmma phase with < 8 items", "forward"))
                if cdiv(fi + 1, 8) * len(group_signature(fo)) + cdiv(npts, 8) * len(group_signature(fi)) < WARPS:
                    cs.add(("dmma phase with < 8 items", "backward"))
    out = layers[-1]
    if pde in ("disc", "kdv"):
        cs.add(("disc head out%16", (out % 16, out >= 16)))
        if out in (63, 64, 65):                   # both heads: the KdV seeds leave the u_xx slot at 0, Burgers' the t slot
            cs.add(("wide-head switch (out, head)", (out, pde)))
    else:
        cs.add(("continuous head out", out))
    return cs | probe_cells(layers)


def ns_cells(layers, n_total, sms):
    sp = ns_split(n_total, sms)
    cs = {("ns pts<16", sp["pts"] < 16)}
    for npts in cta_counts(n_total, sp):
        cs |= {("ns CTA npts%16", npts % 16), ("ns CTA npts%4", npts % 4)}
    hidden = layers[1:-1]
    for fi, fo in zip(hidden, hidden[1:]):
        cs |= ns_layer_cells(fi, fo)
    return cs


def universe():
    """Every cell: {"generic": set, "ns": set}."""
    g = set()
    for form in ("dmma", "dfma"):
        g |= {(form + " regime", r) for r in ("per<16", "per>=16")}
        g |= {(form + " grid<n_cta", b) for b in (True, False)}
        g |= {(form + " CTA npts%8", (r, m)) for r in ("per<16", "per>=16") for m in range(8)}
        g |= {(form + " CTA npts%4", m) for m in range(4)}
    for fi in range(1, 257):
        for fo in range(1, 257):
            if fi <= 8 or fo <= 8 or fi % 8 == 0 or fo % 8 == 0 or fi > 248 or fo > 248:   # every residue and signature
                g |= layer_cells(fi, fo, o3=True)
    g |= {("dmma phase with < 8 items", p) for p in ("forward", "backward")}
    g |= {("disc head out%16", (m, big)) for m in range(16) for big in (False, True) if big or m > 0}
    g |= {("wide-head switch (out, head)", (o, h)) for o in (63, 64, 65) for h in ("disc", "kdv")}
    g |= {("continuous head out", o) for o in (1, 2)}
    g |= {("probe max width", (w, d)) for w in (MAXW, MAXW + 1) for d in (1, 2)}
    ns = {("ns pts<16", b) for b in (True, False)}
    ns |= {("ns CTA npts%16", m) for m in range(16)} | {("ns CTA npts%4", m) for m in range(4)}
    for fi in range(1, 33):
        for fo in range(1, 33):
            ns |= ns_layer_cells(fi, fo)
    return {"generic": g, "ns": ns}


# ------------------------------------------------------------------------------------------------------------------- shapes
def n_total(shape):
    """The kernel's point count of a shape (pinn_api.cu: upload_points / assemble_points): Burgers inference data + collocation,
    identification data, Schrodinger [n_0 | pad to even | 2 n_b | collocation], disc [x_0 | 2 boundary points], KdV n_0 + n_1,
    Navier-Stokes data."""
    c, h = shape["counts"], shape["head"]
    if h == "inf":
        return c["n_u"] + c["n_f"]
    if h == "ide":
        return c["n_u"]
    if h == "nls":
        return (c["n_0"] + 1) // 2 * 2 + 2 * c["n_b"] + c["n_f"]
    if h == "disc":
        return c["n_0"] + 2
    if h == "kdv":
        return c["n_0"] + c["n_1"]
    return c["n"]


def shape_cells(shape, sms):
    if shape["head"] == "ns":
        return ns_cells(shape["layers"], n_total(shape), sms)
    return set().union(*(generic_cells(shape["layers"], n_total(shape), sms, f, shape["head"]) for f in ("dmma", "dfma")))


def shape_cost(shape):
    L = shape["layers"]
    return n_total(shape) * sum(a * b for a, b in zip(L, L[1:])) * (13 if shape["head"] == "ns" else 4)


def _counts(head, n, rng):
    """Split a kernel point count n over the head's sets (None when the head cannot take n points)."""
    if head == "inf":
        if n < 2:
            return None
        n_u = int(rng.integers(1, min(n - 1, 40) + 1))
        return {"n_u": n_u, "n_f": n - n_u}
    if head == "ide":
        return {"n_u": n}
    if head == "nls":                                   # at least one point in each of the three sets
        if n < 5:
            return None
        n_0 = int(rng.integers(1, min(n - 4, 30) + 1))
        n_b = min(int(rng.integers(1, (n - (n_0 + 1) // 2 * 2 - 1) // 2 + 1)), 20)
        return {"n_0": n_0, "n_b": n_b, "n_f": n - (n_0 + 1) // 2 * 2 - 2 * n_b}
    if head == "disc":
        return {"n_0": n - 2} if n >= 3 else None
    if head == "kdv":
        if n < 2:
            return None
        n_0 = int(rng.integers(1, n))
        return {"n_0": n_0, "n_1": n - n_0}
    return {"n": n}


class _Builder:
    def __init__(self, sms, seed):
        self.sms, self.rng = sms, np.random.default_rng(seed)
        self.C = 2 * sms

    def r(self, lo, hi):                                  # integer in [lo, hi]
        return int(self.rng.integers(lo, hi + 1))

    def chain(self, first, want, o3, ns, length, maxw):
        """Hidden widths from `first` on, each next width the one whose layer covers the most cells of `want` (ties: the
        narrower), until nothing more is gained or the chain is `length` long."""
        ws = list(first)
        cells = ns_layer_cells if ns else (lambda a, b: layer_cells(a, b, o3))
        while len(ws) < length:
            prev = ws[-1]
            best, gain = None, 0
            for w in range(1, maxw + 1):
                g = len(cells(prev, w) & want)
                if g > gain:
                    best, gain = w, g
            if best is None:
                break
            want = want - cells(prev, best)
            ws.append(best)
        return ws

    def head_out(self, head, want):
        """An output width for the head: continuous heads 1 (Burgers) / 2 (Schrodinger); discrete-time heads an uncovered
        out%16 cell if any."""
        if head in ("inf", "ide"):
            return 1
        if head == "nls":
            return 2
        lo = 2 if head == "disc" else 1
        for o in list(range(lo, 16)) + [16 * self.r(1, 3) + m for m in range(16)] + [63, 64, 65]:
            if o >= lo and {("disc head out%16", (o % 16, o >= 16)), ("wide-head switch (out, head)", (o, head))} & want:
                return o
        return self.r(lo, 40)

    def shape(self, head, hidden, n, dom=None, out=None, want=frozenset()):
        counts = _counts(head, n, self.rng)
        if counts is None:
            return None
        if head == "ns":
            layers = [3] + hidden + [2]
            dom = dom or ("upstream", "small box")[self.r(0, 1)]
        else:
            out = self.head_out(head, want) if head in ("inf", "ide", "nls") or out is None else out
            layers = [1 if head in ("disc", "kdv") else 2] + hidden + [out]
            dom = dom or ("shifted", "small")[self.r(0, 1)]
        return {"head": head, "layers": layers, "counts": counts, "dom": dom, "seed": self.r(0, 10 ** 6)}

    # targeted candidates: a shape built to reach one cell, the rest of it drawn from the seed
    def generic_candidate(self, cell, want):
        key, val = cell
        C = self.C
        small = lambda: self.r(1, 48)                      # few points for nets built around their layers
        heads = HEADS
        if key.endswith("regime") or "CTA npts" in key or key.endswith("grid<n_cta"):
            if key.endswith("grid<n_cta"):
                n = 2 * C if not val else self.r(3, 2 * C - 3)
            elif key.endswith("regime"):
                n = self.r(3, 14 * C) if val == "per<16" else 16 * C + self.r(1, 32)
            else:
                regime, m = val if "npts%8" in key else (("per<16", "per>=16")[self.r(0, 1)], val + 4 * self.r(0, 1))
                last = m if m else 8
                if regime == "per<16":                       # C CTAs of pts (even, < 16) points, the last one `last`
                    n = (C - 1) * 2 * self.r(cdiv(last, 2), 7) + last
                else:                                        # pts = 32 over SMs + 1 CTAs, the last one the rest
                    n = 16 * C + (m if m else 8 * self.r(1, 4))
            hidden = [self.r(2, 12) for _ in range(self.r(2, 3))]
            head = heads[self.r(0, len(heads) - 1)]
            return self.shape(head, hidden, n, want=want)
        if key == "dmma phase with < 8 items":
            return self.shape(heads[self.r(0, 4)], [self.r(1, 8), self.r(1, 8)], self.r(3, 2 * C), want=want)
        if key in ("disc head out%16", "wide-head switch (out, head)"):
            if key == "disc head out%16":
                out = val[0] if not val[1] else 16 * self.r(1, 3) + val[0]
                head = "kdv" if out == 1 or self.r(0, 1) else "disc"
            else:
                out, head = val
            hidden = self.chain([self.r(1, 40)], want, head == "kdv", False, self.r(2, 5), 64)
            return self.shape(head, hidden, self.r(3, 60), out=out, want=want)
        if key == "continuous head out":
            return self.shape(("inf", "ide")[self.r(0, 1)] if val == 1 else "nls", [self.r(1, 30), self.r(1, 30)], small() + 3,
                              want=want)
        if key == "probe max width":
            w, d = val
            head = ("disc", "kdv")[self.r(0, 1)] if d == 1 else ("inf", "ide", "nls")[self.r(0, 2)]
            return self.shape(head, [self.r(1, 40), w, self.r(1, 40)], self.r(3, 40), out=self.r(2, min(w, 40)), want=want)
        # a layer cell: a first layer that has it, then the chain
        o3 = key.startswith("o3 ")
        fits = _layer_index()[cell]
        narrow = [f for f in fits if max(f) <= 48]
        fits = narrow or fits
        a, b = fits[self.r(0, len(fits) - 1)]
        head = "kdv" if o3 else heads[self.r(0, len(heads) - 1)]
        hidden = self.chain([a, b], want, head == "kdv", False, self.r(4, 8), 256)
        return self.shape(head, hidden, small() + 3, want=want)

    def ns_candidate(self, cell, want):
        key, val = cell
        sms = self.sms
        if key == "ns pts<16" or "npts" in key:
            if key == "ns pts<16":
                pts = self.r(2, 15) if val else self.r(16, 24)
            else:
                m = val if "%16" in key else val + 4 * self.r(0, 3)
                pts = m if m else 16
            last = self.r(1, pts)
            n = (sms - 1) * pts + last                      # SMs CTAs of pts points, the last one `last`
            hidden = self.chain([self.r(1, 32)], want, False, True, self.r(2, 4), 24)
            return self.shape("ns", hidden, n)
        fits = [(a, b) for a in range(1, 33) for b in range(1, 33) if cell in ns_layer_cells(a, b)]
        a, b = fits[self.r(0, len(fits) - 1)]
        hidden = self.chain([a, b], want, False, True, self.r(4, 7), 32)
        return self.shape("ns", hidden, self.r(1, 3 * sms))


_INDEX = {}


def _layer_index():
    """cell -> the (fi, fo) layers of width <= 256 that have it (o3 cells included)."""
    if not _INDEX:
        for a in range(1, 257):
            for b in range(1, 257):
                for c in layer_cells(a, b, True):
                    _INDEX.setdefault(c, []).append((a, b))
    return _INDEX


def _greedy(kind, U, builder, candidate, per_step=6):
    shapes, covered = [], set()
    order = sorted(U, key=repr)
    while True:
        todo = [c for c in order if c not in covered]
        if not todo:
            return shapes
        want = frozenset(todo)
        cands = []
        for cell in todo[:per_step]:
            for _ in range(2):
                s = candidate(cell, want)
                if s is not None:
                    cands.append((len(shape_cells(s, builder.sms) & want), -shape_cost(s), s))
        gain, _, best = max(cands, key=lambda t: (t[0], t[1]))
        assert gain > 0, (kind, todo[:5])
        best["name"] = "%s%02d_%s_%s" % (kind, len(shapes), best["head"], "x".join(map(str, best["layers"][1:-1])))
        shapes.append(best)
        covered |= shape_cells(best, builder.sms)


def sweep(sms, seed=2026):
    """{"generic": [shape], "ns": [shape]}: deterministic for (sms, seed); together the shapes reach every cell of universe()."""
    U = universe()
    b = _Builder(sms, seed)
    return {"generic": _greedy("g", U["generic"], b, b.generic_candidate),
            "ns": _greedy("ns", U["ns"], b, b.ns_candidate)}
