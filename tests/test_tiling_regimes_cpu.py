"""CPU: the regime cells of tests/tiling_regimes.py, the sweep that reaches them, and the numpy walk of the kernels' item lists.

* sweep(sms) reaches every declared cell at 132, 114 and 78 SMs (H100 SXM, H100 PCIe and an odd count); the cell counts are
  printed, and so is the fraction the layer lists of the existing GPU tests reach (run with -s).
* The item walk is exact-once: every factor of every item list over its whole range (columns and k up to 256, rows of [W ; b]
  up to fi = 256, points up to 33), the composed phases on every sweep shape at every CTA point count, and the split of the
  points over the CTAs.
* The sweep discriminates: each broken decomposition of tiling_regimes.BUGS breaks exact-once coverage on some sweep shape.
  Which of them the existing tests' shapes would miss is printed.  The broken forms exist only in the numpy walk."""
import ast
import glob
import os
import re

import numpy as np
import pytest

import tiling_regimes as tr

TESTS = os.path.dirname(os.path.abspath(__file__))
SMS = (132, 114, 78)


@pytest.fixture(scope="module")
def sweeps():
    return {s: tr.sweep(s) for s in SMS}


@pytest.mark.parametrize("sms", SMS)
def test_sweep_reaches_every_cell(sweeps, sms):
    S, U = sweeps[sms], tr.universe()
    for kind in ("generic", "ns"):
        reached = set().union(*(tr.shape_cells(s, sms) for s in S[kind]))
        assert reached <= U[kind], sorted(reached - U[kind], key=repr)[:5]       # no cell outside the declared universe
        missing = sorted(U[kind] - reached, key=repr)
        print("[cells] %d SMs, %-7s: %d shapes reach %d of %d cells" % (sms, kind, len(S[kind]), len(reached), len(U[kind])))
        assert not missing, missing[:10]
    assert sweeps[sms] == tr.sweep(sms)                                               # deterministic
    assert 20 <= len(S["generic"]) <= 60 and 6 <= len(S["ns"]) <= 16
    sig32 = tr.group_signature(256)
    for s in S["generic"] + S["ns"]:
        assert len(s["layers"]) <= tr.MAX_HIDDEN + 2 and max(s["layers"][1:-1]) <= 256
        if max(s["layers"][1:-1]) > 248:              # the widest layers only where the 32-tile column split needs them
            assert any("groups" in c[0] and c[1] == sig32 for c in tr.shape_cells(s, sms)), s["name"]


# ------------------------------------------------------------------------------------------------------- exact-once walks
def _once(counts, n):
    c = np.bincount(np.asarray(counts, np.int64), minlength=n) if len(counts) else np.zeros(n, np.int64)
    return len(c) == n and np.all(c == 1)


def test_every_factor_is_exact_once_over_its_whole_range():
    for N in range(1, 257):
        assert _once(sum(tr.col_groups(N), []), N), N
        assert _once(sum(tr.ns_col_tiles(N), []), N), N
        assert _once(tr.ksteps(N, "k_tail_dropped"), N), N
        assert _once(sum(tr.row_tiles(N, 8), []), N + 1), N                 # rows 0..fi, the bias at fi
        assert _once(sum(tr.row_tiles(N, 16), []), N + 1), N
        assert len(tr.col_groups(N)) == len(tr.group_signature(N)) and all(map(len, tr.col_groups(N)))
    for npts in range(1, 34):
        assert _once(sum(tr.point_groups(npts, 8), []), npts) and _once(sum(tr.point_groups(npts, 16), []), npts)
        assert _once(tr.ksteps(npts, "wgrad_npts_tail_dropped"), npts)
    assert {tr.group_signature(N) for N in range(1, 257)} == {tr.group_signature(8 * k) for k in range(1, 33)}


def test_composed_phases_are_exact_once_across_widths_and_point_counts():
    """Every fi <= 256 with fo = 257 - fi, npts cycling through 1..33 (generic) and 1..40 (Navier-Stokes)."""
    for fi in range(1, 257):
        assert not tr.exact_once(tr.walk_generic_layer(fi, 257 - fi, fi % 33 + 1)), fi
    for fi in range(1, 65):
        assert not tr.exact_once(tr.walk_ns_layer(fi, 65 - fi, fi % 40 + 1)), fi


def _walk_shape(shape, sms, bugs=()):
    """The phases and the CTA split of one sweep shape that are not exact-once under `bugs`."""
    n = tr.n_total(shape)
    ns = shape["head"] == "ns"
    split = (tr.ns_split if ns else tr.generic_split)(n, sms)
    ctas, owned = tr.walk_cta_split(n, split, bugs)
    bad = [] if np.all(owned == 1) else ["CTA split"]
    hidden = shape["layers"][1:-1]
    walk = tr.walk_ns_layer if ns else tr.walk_generic_layer
    for npts in sorted({c for _, c in ctas if c > 0}):
        for fi, fo in zip(hidden, hidden[1:]):
            bad += ["%s %dx%d at %d points" % (p, fi, fo, npts) for p in tr.exact_once(walk(fi, fo, npts, bugs))]
    return bad


def test_the_walk_is_exact_once_on_every_sweep_shape(sweeps):
    for sms in SMS:
        for s in sweeps[sms]["generic"] + sweeps[sms]["ns"]:
            assert not _walk_shape(s, sms), (sms, s["name"])


# ------------------------------------------------------------------------------------------- the existing tests' shapes
def _layer_lists(path):
    """Layer-list literals of a test module: [a, b, ...] and [a] + [b] * k + [c] forms that start with 1, 2 or 3."""
    src = open(path).read()
    found = []
    for m in re.finditer(r"\[\d+\](?:\s*\+\s*\[\d+(?:\s*,\s*\d+)*\](?:\s*\*\s*\d+)?)+|\[\d+(?:\s*,\s*\d+){2,}\]", src):
        try:
            v = eval(compile(ast.parse(m.group(0), mode="eval"), "<layers>", "eval"), {"__builtins__": {}})
        except Exception:
            continue
        if len(v) >= 3 and v[0] in (1, 2, 3) and all(1 <= x <= 512 for x in v) and max(v[1:-1]) <= 256:
            found.append(list(v))
    return found


def existing_shapes(sms):
    """(head, layers, n_total or None) of the generic and Navier-Stokes nets in the GPU tests: the structured case lists of the
    precision modules with their point counts, and the layer-list literals of the other modules without."""
    import test_gpu_ns as tns
    import test_gpu_precision as tp
    import test_gpu_precision_heads as th
    import test_gpu_precision_load as tl
    out = []
    for c in tp.GENERIC_CASES:
        out.append((c[1], c[2], c[5] + c[4] if c[1] == "inf" else c[5]))
    for c in tp.DISC_CASES:
        d = tp.disc_inputs(c)
        out.append(("ide_disc" if d["ide"] else "disc", d["layers"], len(d["x_0"]) + len(d["x_1"])))
    for c in tl.GENERIC_LOAD:
        if c[1] == "nls" and c[2] == tp.NLS:
            continue                                   # the specialised Schrodinger kernel's net, forced generic in its file
        out.append((c[1], c[2], tl.generic_set(c, sms)["n_total"]))
    for c in th.KDV_CASES:
        d = th.kdv_inputs(c, sms)
        out.append(("kdv", d["layers"], len(d["x_0"]) + len(d["x_1"])))
    for c in th.AC_CASES:
        n = th.n_points(c[7], sms)
        out.append(("ac", [1] + list(c[6]) + [c[5]], (n + 1) // 2 * 2 + 2))
    out += [("poly", th.POLY_NET, c[6] + (0 if c[1] else c[7])) for c in th.POLY_CASES]
    out += [("ns", [3] + list(h) + [2], n) for h, n in tns.CASES]
    out += [("ns", [3] + list(h) + [2], n) for _, h, n, _, _, _ in tns.PREC]
    out += [("ns", [3] + tl.NS_NET + [2], B * R) for _, _, _, _, B, R, _ in tl.NS_LOAD]
    structured = {os.path.basename(m.__file__) for m in (tns, tp, th, tl)}
    seen = {tuple(l) for _, l, _ in out}
    for path in sorted(glob.glob(os.path.join(TESTS, "test_gpu_*.py"))):
        if os.path.basename(path) in structured or "tiling" in path:
            continue
        for layers in _layer_lists(path):
            if tuple(layers) not in seen and layers not in ([2] + [20] * 8 + [1], [2, 100, 100, 100, 100, 2]):
                seen.add(tuple(layers))
                out.append(("ns" if layers[0] == 3 else "disc" if layers[0] == 1 else "inf", layers, None))
    return out


def _existing_cells(shapes, sms):
    g, ns = set(), set()
    for head, layers, n in shapes:
        hidden = layers[1:-1]
        if head == "ns":
            ns |= set().union(*[tr.ns_layer_cells(a, b) for a, b in zip(hidden, hidden[1:])]) if len(hidden) > 1 else set()
            if n:
                ns |= tr.ns_cells(layers, n, sms)
            continue
        h = {"ide_disc": "disc", "ac": "disc", "poly": "inf"}.get(head, head)
        if n:
            for form in ("dmma", "dfma"):
                g |= tr.generic_cells(layers, n, sms, form, h)
        else:
            for a, b in zip(hidden, hidden[1:]):
                g |= tr.layer_cells(a, b, h == "kdv")
            g |= tr.probe_cells(layers)
    return g, ns


def test_report_what_the_existing_tests_reach():
    """Prints the fraction of the cells the existing GPU tests' shapes reach, per kind of cell (no assertion on it)."""
    sms = 132
    shapes = existing_shapes(sms)
    g, ns = _existing_cells(shapes, sms)
    U = tr.universe()
    print("\n[existing] %d nets from the GPU tests" % len(shapes))
    for kind, reached in (("generic", g), ("ns", ns)):
        groups = {}
        for c in U[kind]:
            groups.setdefault(c[0], [0, 0])[1] += 1
            groups[c[0]][0] += c in reached
        print("[existing] %-7s %d of %d cells (%.0f %%)" % (kind, len(reached & U[kind]), len(U[kind]),
                                                           100.0 * len(reached & U[kind]) / len(U[kind])))
        for k, (a, b) in sorted(groups.items()):
            print("[existing]   %-32s %3d / %3d" % (k, a, b))
    assert len(shapes) >= 40


# ------------------------------------------------------------------------------------------------------ the sweep discriminates
@pytest.mark.parametrize("bug", sorted(tr.BUGS))
def test_the_sweep_catches_every_broken_decomposition(sweeps, bug):
    sms = 132
    S = sweeps[sms]
    caught = [(s["name"], b[0]) for s in S["generic"] + S["ns"] for b in [_walk_shape(s, sms, (bug,))] if b]
    ex = [(head, layers, n) for head, layers, n in existing_shapes(sms) if n]
    ex_caught = []
    for head, layers, n in ex:
        shape = {"head": "ns" if head == "ns" else "ide", "layers": layers, "counts": {"n_u": n, "n": n}}
        if _walk_shape(shape, sms, (bug,)):
            ex_caught.append(layers)
    print("\n[bugs] %-26s sweep: broken on %d of %d shapes (first: %s, %s); existing shapes with point counts: %s"
          % (bug, len(caught), len(S["generic"]) + len(S["ns"]), caught[0][0] if caught else "-", caught[0][1] if caught else "-",
             "caught on %d" % len(ex_caught) if ex_caught else "MISSED"))
    assert caught, (bug, tr.BUGS[bug])
