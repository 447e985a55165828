"""Exact reference of the Triangulation lookup (``tri_lookup``, csrc/common.cuh) and of the value operator's
rows (``operator_row``, csrc/value_opt.cu), in numpy and ``fractions.Fraction``; no torch, no CUDA.

Lookup semantics (the reference's ``_Triangulation``, ``functions.py:1103-1158, 1473-1499``):

* cell: per dimension ``np.digitize(x, discrete_points) - 1`` clipped to ``[0, n - 2]``;
* unit coordinates: ``clip(x - offset, 2 eps, range - 2 eps) % unit_maxes`` -- one subtraction, a clip
  and an exact ``fmod``, each reproduced bit for bit here.  So a point on a grid line can be looked up
  in a simplex of the wrong side of its cell (DESIGN.md §3.2 Q6), as upstream;
* simplex: the first unit-cell simplex whose barycentric weights at the unit coordinates are all
  >= -W_TOL, else the one with the largest smallest weight; a point clipped in every dimension
  (d > 1) takes Qhull's simplex of its corner pattern (``corner_simplex``, functions.py restates it);
* value: the barycentric weights of the point (clipped to the limits when ``project``) in that
  simplex of that cell, ``sum_k w_k value[vertex_k]``; gradient ``G (V_1..d - V_0)``, G the inverse edge
  matrix; row ``(vertices, weights)``.

Rounding model: every fp64 operation rounds with relative error at most u = 2^-53, fused or not;
gamma_n = n u / (1 - n u).  A sum of products in any order along which a term passes at most n
roundings is off by at most gamma_n sum |terms|.

Admissible simplices.  The kernel screens with w_c = sum_k (unit_k - o_k) H_kc (o the simplex's first
vertex in the unit cell, H the fp64 ``hyperplanes``: ``np.linalg.inv`` of the cell-0 edge matrix),
w_0 = 1 - sum_c w_c, possibly contracted.  Against the exact weights (unit - o) E^-1 of the unit-cell
simplex (E its exact edge matrix), with D = |H - E^-1| computed exactly once per simplex:

    delta_c = sum_k |unit_k - o_k| (D_kc + gamma_{d+1} |H_kc|)          (d products, d - 1 adds, the
                                                                          subtraction: d + 1 roundings)
    delta_0 = sum_c delta_c + gamma_d (1 + sum_c (|w_c| + delta_c))     (d - 1 adds and 1 - sum)
    delta   = max(delta_0, ..., delta_d)                                  (|min w^ - min w| <= delta)

With exact smallest weight m_s, first-fit surely takes s when m_s >= -W_TOL + delta and surely skips it
when m_s < -W_TOL - delta.  ``admissible`` returns the simplices first-fit can pick: in order, every s
not surely skipped, up to the first surely taken.  m_s is screened in fp64 (itself within delta of m_s)
and decided in Fractions only inside the margin.

Rounding bound of one evaluation in simplex s of a cell.  G = E_cell^-1 exactly, from the vertex
coordinates ``index_to_state`` returns (H is reused for every cell, so D_cell = |H - G| carries the
coordinates' rounding as well as the inverse's), r = x - vertex_0 (x projected under ``project``),
lambda the exact weights:

    e_c = sum_k |r_k| (D_kc + gamma_{d+1} |H_kc|)                         c = 1..d
    e_0 = sum_c e_c + gamma_d (1 + sum_c (|lambda_c| + e_c))
    value:    E_o = sum_k e_k |V_ko| + gamma_{d+1} sum_k (|lambda_k| + e_k) |V_ko|   (d + 1 term gather)
    gradient: E_k = sum_c D_kc (|V_c| + |V_0|) + gamma_{2d} sum_c |H_kc| (|V_c| + |V_0|)
              (hs = sum_c H_kc by d - 1 adds, times V_0, then d adds: 2d roundings on the longest path)
    row:      weight k within e_k of lambda_k.

Bounds are evaluated in fp64 from exact inputs and multiplied by (1 + 8 (d + 2) u), which covers the
rounding of evaluating them.
"""
from fractions import Fraction

import numpy as np

W_TOL = 1e-12
EPS = np.finfo(np.float64).eps
U = EPS / 2
QHULL_EPS = 100 * EPS        # scipy's find_simplex tolerance on its barycentric coordinates


def gamma(n):
    return n * U / (1 - n * U)


def _fr(a):
    return [Fraction(float(v)) for v in np.ravel(a)]


def _inverse(E):
    """Exact inverse of a d x d matrix of Fractions (Gauss-Jordan)."""
    d = len(E)
    A = [list(row) + [Fraction(int(i == j)) for j in range(d)] for i, row in enumerate(E)]
    for c in range(d):
        p = next(r for r in range(c, d) if A[r][c] != 0)
        A[c], A[p] = A[p], A[c]
        piv = A[c][c]
        A[c] = [v / piv for v in A[c]]
        for r in range(d):
            if r != c and A[r][c] != 0:
                f = A[r][c]
                A[r] = [a - f * b for a, b in zip(A[r], A[c])]
    return [row[d:] for row in A]


def _tofloat(q):
    """A Fraction as the nearest double, +-inf beyond the double range."""
    try:
        return float(q)
    except OverflowError:
        return float("inf") if q > 0 else float("-inf")


def _up(a, d):
    return np.asarray(a, dtype=np.float64) * (1 + 8 * (d + 2) * U)


def corner_simplex(grid, triangulation):
    """Qhull's simplex for each corner pattern (bit c set: clipped at the upper limit of dimension c),
    one isolated query per pattern (functions.py builds the library's table the same way)."""
    d = grid.ndim
    table = np.zeros(2 ** d, dtype=np.int64)
    if d > 1:
        lo = grid.offset_limits[:, 0] + 2 * EPS
        hi = grid.offset_limits[:, 1] - 2 * EPS
        for pattern in range(2 ** d):
            bits = np.array([(pattern >> c) & 1 for c in range(d)], dtype=bool)
            unit = np.where(bits, hi, lo) % grid.unit_maxes
            table[pattern] = int(triangulation.find_simplex(unit[None, :])[0])
    return table


class Lookup(object):
    """The lookup of one Triangulation: ``grid`` an ``oracle.GridWorld``; ``unit_simplices`` [S, d + 1]
    grid indices of the unit cell's simplices and ``hyperplanes`` [S, d, d] (``oracle.Triangulation``'s,
    which the fixtures pin to the reference's); ``corner`` the corner-pattern table; ``qhull_transform``
    [S, d + 1, d] scipy's barycentric transforms of the unit cell's Delaunay triangulation (d > 1), used only
    to list the simplices the reference's own lookup may take (``containing``)."""

    def __init__(self, grid, unit_simplices, hyperplanes, corner, project, qhull_transform=None):
        self.grid = grid
        self.T = None if qhull_transform is None else np.asarray(qhull_transform, dtype=np.float64)
        self.d = d = grid.ndim
        self.simp = np.asarray(unit_simplices, dtype=np.int64)
        self.H = np.asarray(hyperplanes, dtype=np.float64)
        self.corner_table = np.asarray(corner)
        self.project = bool(project)
        self.S = len(self.simp)
        ijk = np.array(np.unravel_index(self.simp[:, 0], grid.num_points), dtype=np.float64).T
        self.o = ijk * grid.unit_maxes                                   # [S, d], exact (ijk in {0, 1})
        self._unit_inv = {}
        self._cell_inv = {}
        self.D_unit = np.empty_like(self.H)
        for s in range(self.S):
            G = self.unit_inverse(s)
            self.D_unit[s] = _up([[abs(Fraction(float(self.H[s, i, j])) - G[i][j]) for j in range(d)]
                                  for i in range(d)], d)

    @classmethod
    def of(cls, otri):
        """From an ``oracle.Triangulation``."""
        return cls(otri.discretization, otri.unit_simplices, otri.hyperplanes,
                   corner_simplex(otri.discretization, otri.triangulation), otri.project,
                   getattr(otri.triangulation, "transform", None))

    # ---------------------------------------------------------------- exact inverse edge matrices
    def unit_inverse(self, s):
        if s not in self._unit_inv:
            ijk = np.array(np.unravel_index(self.simp[s], self.grid.num_points), dtype=np.float64).T
            P = [_fr(row * self.grid.unit_maxes) for row in ijk]
            self._unit_inv[s] = _inverse([[a - b for a, b in zip(P[k], P[0])] for k in range(1, self.d + 1)])
        return self._unit_inv[s]

    def vertices(self, s, corner):
        return self.grid.index_to_state(self.simp[s] + corner)          # [d + 1, d], fp64

    def cell_inverse(self, s, corner):
        key = (s, corner)
        if key not in self._cell_inv:
            P = [_fr(row) for row in self.vertices(s, corner)]
            self._cell_inv[key] = _inverse([[a - b for a, b in zip(P[k], P[0])] for k in range(1, self.d + 1)])
        return self._cell_inv[key]

    # ---------------------------------------------------------------- cell and unit coordinates
    def cell(self, x):
        """(corner index, unit coordinates, all_clipped, pattern) of one point, as tri_lookup forms them."""
        g = self.grid
        x = np.asarray(x, dtype=np.float64)
        ks = []
        for c, (pts, n) in enumerate(zip(g.discrete_points, g.num_points)):
            ks.append(int(np.clip(np.digitize(x[c], pts) - 1, 0, n - 2)))
        corner = int(np.ravel_multi_index(ks, g.num_points))
        cen = x - g.offset
        lo = g.offset_limits[:, 0] + 2 * EPS
        hi = g.offset_limits[:, 1] - 2 * EPS
        pattern = int(np.sum((cen > hi) << np.arange(self.d)))
        all_clipped = bool(np.all((cen < lo) | (cen > hi)))
        unit = np.fmod(np.clip(cen, lo, hi), g.unit_maxes)
        return corner, unit, all_clipped, pattern

    def cell_unit(self, x, corner):
        """The repair's unit coordinates (TRI_CELL): clip(x, limits) - the cell's lowest vertex."""
        g = self.grid
        return np.minimum(np.maximum(x, g.limits[:, 0]), g.limits[:, 1]) - g.index_to_state(corner)[0]

    # ---------------------------------------------------------------- admissible simplices
    def screen(self, unit):
        """(fp64 smallest weights [S], delta [S]) at unit coordinates."""
        d = self.d
        A = np.abs(unit[None, :] - self.o)                               # [S, d]
        w = np.einsum("sk,skc->sc", unit[None, :] - self.o, self.H)
        m = np.minimum(w.min(axis=1), 1.0 - w.sum(axis=1))
        dc = np.einsum("sk,skc->sc", A, self.D_unit + gamma(d + 1) * np.abs(self.H))
        wabs = np.einsum("sk,skc->sc", A, np.abs(self.H)) * (1 + gamma(d + 1))
        d0 = dc.sum(axis=1) + gamma(d) * (1 + (wabs + dc).sum(axis=1))
        return m, _up(np.maximum(d0, dc.max(axis=1)), d)

    def exact_min_weight(self, s, unit):
        G = self.unit_inverse(s)
        r = [Fraction(float(a)) - Fraction(float(b)) for a, b in zip(unit, self.o[s])]
        lam = [sum(r[k] * G[k][c] for k in range(self.d)) for c in range(self.d)]
        return min(min(lam), 1 - sum(lam))

    def admissible(self, unit):
        """The simplices first-fit can pick at these unit coordinates (see the module docstring)."""
        m, delta = self.screen(unit)
        tol = Fraction(W_TOL)
        out = []
        for s in range(self.S):
            lo, hi = m[s] - delta[s], m[s] + delta[s]                   # exact m_s lies in [lo, hi]
            if hi < -W_TOL - delta[s]:
                continue                                                  # surely skipped
            if lo >= -W_TOL + delta[s]:
                out.append(s)
                return out                                                # surely taken
            ms = self.exact_min_weight(s, unit)
            if ms < -tol - Fraction(float(delta[s])):
                continue
            out.append(s)
            if ms >= -tol + Fraction(float(delta[s])):
                return out
        raise AssertionError("no simplex surely contains the unit point %r: the largest-smallest-weight "
                             "fallback could apply" % (unit,))

    def containing(self, unit):
        """Every simplex scipy's find_simplex may return at these unit coordinates.  scipy accepts simplex s
        when every barycentric coordinate it computes from its own fp64 transform T_s (``Delaunay.transform``)
        lies in [-QHULL_EPS, 1 + QHULL_EPS]:  c_i = sum_j T_s[i, j] (x_j - T_s[d, j]) for i < d and
        c_d = 1 - sum_i c_i.  Against the exact c_i of the same T_s, a computed c_i is off by at most
        err_i = gamma_{d+1} sum_j |T_s[i, j]| |x_j - T_s[d, j]| (d products, d - 1 adds, the subtraction),
        and c_d by err_d = sum_i err_i + gamma_d (1 + sum_i |c_i|).  So s may be returned only if every
        exact c_i lies in [-QHULL_EPS - err_i, 1 + QHULL_EPS + err_i]; those are the simplices listed.
        (scipy's brute-force fallback with a wider tolerance for points next to degenerate simplices is not
        modelled: the unit cell has none, and a fixture row that needed it would fail its check.)"""
        if self.T is None:                                             # d = 1: one simplex
            return list(range(self.S))
        d = self.d
        r = unit[None, :] - self.T[:, d, :]                             # [S, d]
        c = np.einsum("sij,sj->si", self.T[:, :d, :], r)
        cabs = np.einsum("sij,sj->si", np.abs(self.T[:, :d, :]), np.abs(r)) * (1 + gamma(d + 1))
        err = gamma(d + 1) * cabs
        err_d = err.sum(axis=1) + gamma(d) * (1 + cabs.sum(axis=1))
        c = np.concatenate([c, 1 - c.sum(axis=1, keepdims=True)], axis=1)
        err = _up(np.concatenate([err, err_d[:, None]], axis=1), d)
        # screen: the numpy c is itself within err of the exact c, so 2 err covers both
        maybe = np.all((c >= -QHULL_EPS - 2 * err) & (c <= 1 + QHULL_EPS + 2 * err), axis=1)
        out = []
        for s in np.flatnonzero(maybe):
            T = [_fr(row) for row in self.T[s]]
            rf = [Fraction(float(a)) - b for a, b in zip(unit, T[d])]
            ce = [sum(T[i][j] * rf[j] for j in range(d)) for i in range(d)]
            ce.append(1 - sum(ce))
            if all(-Fraction(QHULL_EPS) - Fraction(float(e)) <= v <= 1 + Fraction(QHULL_EPS) + Fraction(float(e))
                   for v, e in zip(ce, err[s])):
                out.append(int(s))
        return out

    def fixture_set(self, x):
        """(corner, simplices) the reference's own lookup may take for an isolated query: first-fit's
        admissible set (the library's choice) and every simplex Qhull's walk may return."""
        corner, sims = self.lookup_set(x)
        _, unit, all_clipped, _ = self.cell(x)
        if not (all_clipped and self.d > 1):
            sims = sorted(set(sims) | set(self.containing(unit)))
        return corner, sims

    def lookup_set(self, x):
        """(corner, admissible simplices) of tri_lookup's first search (TRI_EVAL / TRI_WEIGHTS)."""
        corner, unit, all_clipped, pattern = self.cell(x)
        if all_clipped and self.d > 1:
            return corner, [int(self.corner_table[pattern])]
        return corner, self.admissible(unit)

    # ---------------------------------------------------------------- exact results of one simplex
    def query_point(self, x):
        g = self.grid
        return np.minimum(np.maximum(x, g.limits[:, 0]), g.limits[:, 1]) if self.project else np.asarray(x)

    def exact(self, x, corner, s, V=None):
        """Exact weights (Fractions, d + 1), their bounds e [d + 1], and, given vertex values V [nindex, m],
        the exact values [m] with bounds [m] and, for m = 1, the exact gradient [d] with bounds [d]."""
        d = self.d
        xq = self.query_point(x)
        P = self.vertices(s, corner)
        G = self.cell_inverse(s, corner)
        H = self.H[s]
        r = [Fraction(float(a)) - Fraction(float(b)) for a, b in zip(xq, P[0])]
        lam = [sum(r[k] * G[k][c] for k in range(d)) for c in range(d)]
        lam = [1 - sum(lam)] + lam
        D = _up([[abs(Fraction(float(H[i, j])) - G[i][j]) for j in range(d)] for i in range(d)], d)
        ra = np.array([abs(float(v)) for v in r]) * (1 + U)
        ec = ra @ (D + gamma(d + 1) * np.abs(H))
        lamabs = np.array([abs(_tofloat(v)) for v in lam]) * (1 + U)
        e0 = ec.sum() + gamma(d) * (1 + (lamabs[1:] + ec).sum())
        e = _up(np.concatenate([[e0], ec]), d)
        res = {"weights": lam, "weight_bound": e, "vertices": self.simp[s] + corner, "corner": corner,
               "simplex": s, "point": xq, "vertex_states": P}
        if V is not None:
            V = np.asarray(V, dtype=np.float64).reshape(self.grid.nindex, -1)
            Vs = V[self.simp[s] + corner]                                # [d + 1, m]
            vals, vb = [], []
            for o in range(Vs.shape[1]):
                vf = _fr(Vs[:, o])
                vals.append(_tofloat(sum(l * v for l, v in zip(lam, vf))))
                va = np.abs(Vs[:, o])
                vb.append(e @ va + gamma(d + 1) * (lamabs + e) @ va)
            res["value"], res["value_bound"] = np.array(vals), _up(vb, d)
            if Vs.shape[1] == 1:
                vf = _fr(Vs[:, 0])
                res["gradient"] = np.array([float(sum(G[k][c] * (vf[c + 1] - vf[0]) for c in range(d)))
                                            for k in range(d)])
                va = np.abs(Vs[:, 0])
                res["gradient_bound"] = _up((D + gamma(2 * d) * np.abs(H)) @ (va[1:] + va[0]), d)
        return res

    def candidates(self, x, V=None, fixture=False):
        """Exact results of every admissible simplex of tri_lookup at x (``fixture``: of every simplex
        the reference's lookup may take, ``fixture_set``)."""
        corner, sims = self.fixture_set(x) if fixture else self.lookup_set(x)
        with np.errstate(over="ignore", invalid="ignore"):      # value bounds of |x| ~ 1e308 are inf
            return [self.exact(x, corner, s, V) for s in sims]

    # ---------------------------------------------------------------- the value operator's row
    def row_candidates(self, x):
        """operator_row: (results, repaired) for every choice the kernel can make at next state x.  The
        first lookup's row is repaired -- re-searched from TRI_CELL's unit coordinates -- when its
        computed smallest weight is < -W_TOL and x is inside the grid or projected onto it."""
        g = self.grid
        inside = bool(np.all((x >= g.limits[:, 0]) & (x <= g.limits[:, 1])))
        out = []
        need_repair = False
        corner = None
        for res in self.candidates(x):
            corner = res["corner"]
            m = min(res["weights"])
            e = float(res["weight_bound"].max())
            if not (self.project or inside) or m >= -Fraction(W_TOL) + Fraction(e):
                out.append((res, False))
            elif m < -Fraction(W_TOL) - Fraction(e):
                need_repair = True
            else:
                out.append((res, False))
                need_repair = True
        if need_repair:
            for s in self.admissible(self.cell_unit(x, corner)):
                out.append((self.exact(x, corner, s), True))
        return out


# ------------------------------------------------------------------ checks used by the GPU tests
def _fail(what, i, detail):
    raise AssertionError("%s at point %d: %s" % (what, i, detail))


def check_values(lk, x, got, V, fixture=False):
    """Each row of got [n, m] within the bound of the exact value of some admissible simplex; NaN in
    x gives NaN."""
    for i, p in enumerate(x):
        if np.isnan(p).any():
            if not np.isnan(got[i]).all():
                _fail("value of a NaN point", i, got[i])
            continue
        cands = lk.candidates(p, V, fixture)
        if not any(np.all(np.abs(got[i] - c["value"]) <= c["value_bound"]) for c in cands):
            _fail("value", i, "got %r, admissible %r" % (got[i], [(c["simplex"], c["value"], c["value_bound"])
                                                               for c in cands]))


def check_gradients(lk, x, got, V, maxabs=False, fixture=False):
    """Gradient rows [n, d] (or their max-abs [n, 1]) within the bound of an admissible simplex's."""
    for i, p in enumerate(x):
        if np.isnan(p).any():
            if not np.isnan(got[i]).all():
                _fail("gradient of a NaN point", i, got[i])
            continue
        ok = False
        for c in lk.candidates(p, V, fixture):
            if maxabs:
                ok |= abs(got[i][0] - np.max(np.abs(c["gradient"]))) <= np.max(c["gradient_bound"])
            else:
                ok |= bool(np.all(np.abs(got[i] - c["gradient"]) <= c["gradient_bound"]))
        if not ok:
            _fail("gradient", i, "got %r" % (got[i],))


def check_affine(lk, x, got_value, got_grad, a, b, V):
    """Vertex values V = x_vertex a + b: every simplex interpolates the same affine function, so the value
    is xq a + b (xq projected under ``project``) within the evaluation bound plus the vertex values'
    own rounding (sum_k |lambda_k| |V_k - (a x_k + b)|, exact), and the gradient is a within the gradient
    bound plus its share of that rounding (sum_c |G_kc| |rounding_c - rounding_0|)."""
    d = lk.d
    af = [_fr(a[:, o]) for o in range(a.shape[1])]
    bf = _fr(b)
    for i, p in enumerate(x):
        if np.isnan(p).any():
            if not (np.isnan(got_value[i]).all() and (got_grad is None or np.isnan(got_grad[i]).all())):
                _fail("affine value of a NaN point", i, got_value[i])
            continue
        ok = False
        for c in lk.candidates(p, V):
            xq = _fr(c["point"])
            P = c["vertex_states"]
            Vs = V[c["vertices"]]
            lamabs = np.array([abs(float(v)) for v in c["weights"]])
            good = True
            for o in range(a.shape[1]):
                want = float(sum(xc * ac for xc, ac in zip(xq, af[o])) + bf[o])
                rnd = [float(Fraction(float(Vs[k, o])) - sum(pc * ac for pc, ac in zip(_fr(P[k]), af[o])) - bf[o])
                       for k in range(d + 1)]
                lim = c["value_bound"][o] + _up(lamabs @ np.abs(rnd), d)
                good &= abs(got_value[i][o] - want) <= lim
                if got_grad is not None and o == 0:
                    G = lk.cell_inverse(c["simplex"], c["corner"])
                    Ga = np.array([[abs(float(G[k][j])) for j in range(d)] for k in range(d)])
                    glim = c["gradient_bound"] + _up(Ga @ (np.abs(rnd[1:]) + abs(rnd[0])), d)
                    good &= bool(np.all(np.abs(got_grad[i] - a[:, 0]) <= glim))
            ok |= good
        if not ok:
            _fail("affine value", i, "got %r" % (got_value[i],))


def check_rows(lk, x, cols, weights):
    """Value-operator rows [n, d + 1]: columns in range; the row's simplex, read from cols - corner, one
    the kernel can pick under the repair rule; weights within e_k of the exact barycentrics and, summed
    exactly, within sum e_k of 1; sum_k w_k vertex_k, formed exactly, reconstructing the (projected) point
    within sum_k e_k |vertex_k|; weights >= -W_TOL for points inside the
    grid or projected onto it.  Returns the number of rows that can only come from the repair."""
    g = lk.grid
    d = lk.d
    repaired = 0
    for i, p in enumerate(x):
        c, w = cols[i].astype(np.int64), weights[i]
        if c.min() < 0 or c.max() >= g.nindex:
            _fail("row column out of range", i, c)
        match = [(res, rep) for res, rep in lk.row_candidates(p) if np.array_equal(res["vertices"], c)]
        if not match:
            _fail("row simplex", i, "cols %r not admissible" % (c,))
        res, rep = match[0]
        repaired += all(r for _, r in match)
        lam = np.array([float(v) for v in res["weights"]])
        e = res["weight_bound"]
        if np.any(np.abs(w - lam) > e):
            _fail("row weights", i, "got %r want %r +- %r" % (w, lam, e))
        s = sum(Fraction(float(v)) for v in w)
        if abs(float(s - 1)) > _up(e.sum(), d):         # sum lambda = 1: |sum w - 1| <= sum |w - lambda|
            _fail("row weight sum", i, float(s))
        P = res["vertex_states"]
        rec = [sum(Fraction(float(w[k])) * Fraction(float(P[k, j])) for k in range(d + 1)) for j in range(d)]
        lim = _up(e @ np.abs(P), d)                     # sum lambda_k P_k = x: sum (w_k - lambda_k) P_k
        dev = np.array([abs(float(rec[j] - Fraction(float(res["point"][j])))) for j in range(d)])
        if np.any(dev > lim):
            _fail("row reconstruction", i, dev)
        inside = np.all((p >= g.limits[:, 0]) & (p <= g.limits[:, 1]))
        if (lk.project or inside) and w.min() < -W_TOL:
            _fail("negative weight", i, w)
    return repaired


def check_fixture_rows(lk, x, cols, weights):
    """The reference's own rows (``parameter_derivative``): vertices of a simplex its lookup may take,
    weights within that simplex's e_k of the exact barycentrics."""
    for i, p in enumerate(x):
        match = [c for c in lk.candidates(p, fixture=True) if np.array_equal(c["vertices"], cols[i])]
        if not match:
            _fail("fixture row simplex", i, cols[i])
        lam = np.array([float(v) for v in match[0]["weights"]])
        if np.any(np.abs(weights[i] - lam) > match[0]["weight_bound"]):
            _fail("fixture row weights", i, weights[i] - lam)


# ------------------------------------------------------------------ the certified solve
def rho_exact(weights):
    """max_i sum_k |w_ik| exactly (as the next fp64 number up)."""
    s = max(sum(Fraction(float(abs(v))) for v in row) for row in weights)
    return float(s) * (1 + 2 * U)


def fixed_point(cols, weights, rewards, gamma_, target):
    """A fixed point of v = r + gamma T v (T: rows cols/weights) whose own error is certified below
    `target`: spsolve in fp64, then iterative refinement with residuals r - (I - gamma T) v computed in
    Fractions; ||v - v*||_inf <= ||residual||_inf / (1 - gamma rho).  Returns (v, certified error)."""
    import scipy.sparse as sp
    import scipy.sparse.linalg as spla
    n, k = cols.shape
    T = sp.csr_matrix((weights.ravel(), (np.repeat(np.arange(n), k), cols.ravel())), shape=(n, n))
    lu = spla.splu((sp.identity(n) - gamma_ * T).tocsc())
    v = lu.solve(np.asarray(rewards, dtype=np.float64))
    g = Fraction(float(gamma_))
    contraction = 1 - float(g) * rho_exact(weights)
    wf = [[Fraction(float(a)) for a in row] for row in weights]
    rf = [Fraction(float(a)) for a in rewards]
    for _ in range(6):
        vf = [Fraction(float(a)) for a in v]
        res = [rf[i] - vf[i] + g * sum(wf[i][j] * vf[cols[i, j]] for j in range(k)) for i in range(n)]
        err = float(max(abs(a) for a in res)) * (1 + 2 * U) / contraction
        if err <= target:
            return v, err
        v = v + lu.solve(np.array([float(a) for a in res]))
    raise AssertionError("refinement did not reach %g (at %g)" % (target, err))


def solve_slack(weights, rewards, gamma_, values, d, bound):
    """How far the kernel's values may sit from the exact fixed point v* beyond the certificate ``bound``
    it reports (``last_solve["bound"]``, q^ delta^ with q^ = gamma rho^ / (1 - gamma rho^) in fp64).

    The kernel computes v_k = F(v_{k-1}) + eps_k with |eps_k| <= eta = gamma_{d+3} (max |r| + gamma rho
    max |v|) (d + 1 products and d adds, times gamma, plus r: d + 3 roundings on the longest path).  With
    v* = F(v*): ||v_k - v*|| <= gamma rho ||v_{k-1} - v*|| + eta <= gamma rho (||v_k - v_{k-1}|| +
    ||v_k - v*||) + eta, so ||v_k - v*|| <= q ||v_k - v_{k-1}|| + eta / (1 - gamma rho), q and rho exact.
    The certificate is that first term rounded: rho^ (d adds of |w|) is within gamma_d rho of rho, so
    gamma rho^ is within (gamma_d + u) gamma rho and q^ within ((gamma_d + u) / (1 - gamma rho) + 2u) q
    (the subtraction and the division); delta^ = |v_k - v_{k-1}| is within u, and the product within u.
    So q delta <= bound (1 + c) with c = (gamma_d + u) / (1 - gamma rho) + 4u, and
        ||v_k - v*|| <= bound + slack,   slack = c bound + eta / (1 - gamma rho),
    with rho rounded up."""
    rho = rho_exact(weights)
    gr = gamma_ * rho * (1 + 2 * U)
    eta = gamma(d + 3) * (np.max(np.abs(rewards)) + gr * np.max(np.abs(values)) * (1 + 2 * U))
    c = (gamma(d) + U) / (1 - gr) + 4 * U
    return _up(c * bound + eta / (1 - gr), d)


def check_fixed_point(got, vstar, vstar_err, bound, slack):
    """||got - v*||_inf <= bound + slack, v* known to within vstar_err (fixed_point)."""
    dev = float(np.max(np.abs(np.asarray(got) - vstar)))
    lim = bound + slack + vstar_err
    if not dev <= lim:
        raise AssertionError("fixed point off by %.3g, certified %.3g" % (dev, lim))
    return dev, lim


# ------------------------------------------------------------------ the point classes of the tests
SHAPE_NUM = {1: [7], 2: [6, 5], 3: [4, 3, 5], 4: [3, 4, 3, 3], 5: [3] * 5, 6: [3, 2, 3, 2, 3, 2]}


def shape_grid(ns, d):
    """The d-dimensional test grid on [-1 - 0.1 c, 1 + 0.2 c] (``ns``: the oracle or the library)."""
    return ns.GridWorld([[-1.0 - 0.1 * c, 1.0 + 0.2 * c] for c in range(d)], SHAPE_NUM[d])


def _lines(grid, rng, per_line, with_ulps=True):
    """Points with one coordinate exactly on an interior grid line (and one ulp either side)."""
    lo, hi = grid.limits[:, 0], grid.limits[:, 1]
    out = []
    for c, pts in enumerate(grid.discrete_points):
        for j in range(1, len(pts) - 1):
            p = rng.uniform(lo, hi, (per_line, grid.ndim))
            p[:, c] = pts[j]
            out.append(p)
            if with_ulps:
                for to in (np.inf, -np.inf):
                    q = p.copy()
                    q[:, c] = np.nextafter(pts[j], to)
                    out.append(q)
    return out


def _outside(grid, rng):
    """Each single face outside (2 d points) and a point beyond each of the 2^d corner patterns."""
    d = grid.ndim
    lo, hi = grid.limits[:, 0], grid.limits[:, 1]
    span = hi - lo
    faces = []
    for c in range(d):
        for side in (0, 1):
            p = rng.uniform(lo, hi, (1, d))
            p[0, c] = hi[c] + rng.uniform(0.05, 0.5) * span[c] if side else lo[c] - rng.uniform(0.05, 0.5) * span[c]
            faces.append(p)
    bits = (np.arange(2 ** d)[:, None] >> np.arange(d)[None, :]) & 1
    corners = np.where(bits == 1, hi + rng.uniform(0.05, 0.5, (2 ** d, d)) * span,
                       lo - rng.uniform(0.05, 0.5, (2 ** d, d)) * span)
    return faces + [corners]


def _edges(grid, rng):
    """The boundary grid lines, and the clip edges offset + 2 eps, upper - 2 eps and upper exactly."""
    d = grid.ndim
    lo, hi = grid.limits[:, 0], grid.limits[:, 1]
    out = []
    for c in range(d):
        for val in (lo[c], hi[c], lo[c] + 2 * EPS, hi[c] - 2 * EPS):
            p = rng.uniform(lo, hi, (1, d))
            p[0, c] = val
            out.append(p)
    return out


def point_classes(grid, rng):
    """Inside, vertices, interior grid lines (on and +-1 ulp), boundary lines and clip edges, each single
    face outside, all 2^d corner patterns outside, coordinates of +-1e300, and a NaN."""
    d = grid.ndim
    lo, hi = grid.limits[:, 0], grid.limits[:, 1]
    verts = grid.all_points[rng.choice(grid.nindex, min(24, grid.nindex), replace=False)]
    big = []
    for c in range(d):
        p = rng.uniform(lo, hi, (2, d))
        p[0, c], p[1, c] = 1e300, -1e300
        big.append(p)
    big.append(np.array([[1e300] * d, [-1e300] * d]))
    nan = rng.uniform(lo, hi, (1, d))
    nan[0, rng.integers(d)] = np.nan
    return np.vstack([rng.uniform(lo, hi, (24, d)), verts] + _lines(grid, rng, 3) + _edges(grid, rng)
                     + _outside(grid, rng) + big + [nan])


def operator_points(grid, rng):
    """Next states for the value operator: inside, exact grid-line points (one coordinate, and two at
    once) with +-1 ulp, vertices, boundary lines and clip edges, and points outside that projection puts
    on the boundary."""
    d = grid.ndim
    lo, hi = grid.limits[:, 0], grid.limits[:, 1]
    two = []
    for p in _lines(grid, rng, 4, with_ulps=False):
        q = p.copy()
        c = rng.integers(d)
        q[:, c] = grid.discrete_points[c][rng.integers(len(grid.discrete_points[c]), size=len(q))]
        two.append(q)
    verts = grid.all_points[rng.choice(grid.nindex, min(16, grid.nindex), replace=False)]
    return np.vstack([rng.uniform(lo, hi, (16, d)), verts] + _lines(grid, rng, 8) + two
                     + _edges(grid, rng) + _outside(grid, rng))
