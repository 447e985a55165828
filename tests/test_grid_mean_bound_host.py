"""CPU check of the factored grid mean's arithmetic and its certified bound (csrc/filter.cu,
filter_grid_mean_kernel): the fp64 steps of one tile, factor and policy regime restated in numpy -- centred
differences, weights, the per-axis recurrence of the tables, the contraction and Q -- against the kernel
sum evaluated directly in extended precision at the grid's own points and the policy's rounded u.  The
error must stay within the bound the kernel computes, on ordinary and on adversarial tiles (wide tiles
in lengthscale units, far and near-dropped training rows, steep policies, tiles far from the origin)."""
import numpy as np
import pytest

U = 2.0 ** -53
EPS_K = 1.0e-13
RHO_MAX, K_DROP = 12.0, 600.0
GR = GC = 16


def _tile(rng, lo, unit, ls, row0, col0, gain, lim, regime, M, spread, centre_pull):
    l0, l1, l2 = ls
    # training inputs: around the tile (centre_pull) and far away (spread), plus rows near the drop line
    c = np.array([lo[0] + (row0 + 8) * unit[0], lo[1] + (col0 + 8) * unit[1], 0.0])
    X = c + rng.normal(scale=spread, size=(M, 3)) * np.array(ls)
    X[: M // 4] = c + rng.normal(scale=centre_pull, size=(M // 4, 3)) * np.array(ls)
    X[-2:, 0] = c[0] + np.array([24.4, 24.6]) * l0                      # |D|^2 around K_DROP
    gamma = rng.normal(size=M) * np.exp(rng.normal(scale=3.0, size=M))
    xs = X / np.array(ls)
    # the grid's own points (grid_index_to_state) and the policy's u, fp64 as the kernel computes them
    x0 = (np.arange(row0, row0 + GR) * unit[0]) + lo[0]
    x1 = (np.arange(col0, col0 + GC) * unit[1]) + lo[1]
    a, b = gain
    raw = (x0[:, None] * a) + (x1[None, :] * b)
    # the kernel's fp64 steps for this regime
    cw0 = (lo[0] + (row0 + 8) * unit[0]) / l0
    cw1 = (lo[1] + (col0 + 8) * unit[1]) / l1
    h0, h1 = unit[0] / l0, unit[1] / l1
    if regime == 2:
        alpha, beta = (a * l0) / l2, (b * l1) / l2
        cw2 = alpha * cw0 + beta * cw1
    else:
        alpha = beta = 0.0
        cw2 = lim[regime] / l2
    off = np.arange(-8, 8).astype(float)
    xi, eta = off * h0, off * h1
    dev = max(np.abs((x0 / l0 - cw0) - xi).max(), np.abs((x1 / l1 - cw1) - eta).max())
    mxi, meta = np.abs(xi).max(), np.abs(eta).max()
    rho = mxi * np.sqrt(alpha * alpha + 1) + meta * np.sqrt(beta * beta + 1)
    D = np.array([cw0, cw1, cw2]) - xs
    K = (D ** 2).sum(axis=1)
    keep = K <= K_DROP
    w = np.where(keep, np.exp(-0.5 * K), 0.0)
    p = np.where(keep, alpha * D[:, 2] + D[:, 0], 0.0)
    q = np.where(keep, beta * D[:, 2] + D[:, 1], 0.0)

    def table(h, v):                                  # g^o, o = -8 .. 7, by products outwards from o = 0
        gd, gu = np.exp(-h * v), np.exp(h * v)
        T = np.empty((16, v.size))
        T[8] = 1.0
        for o in range(1, 8):
            T[8 + o] = T[7 + o] * gd
        for o in range(1, 9):
            T[8 - o] = T[9 - o] * gu
        return T

    E0, E1 = table(h0, p), table(h1, q)
    S = (E0 * (gamma * w)) @ E1.T
    vv = alpha * xi[:, None] + beta * eta[None, :]
    Q = np.exp(-0.5 * (xi[:, None] ** 2 + eta[None, :] ** 2 + vv ** 2))
    mean = S * Q
    # the bound (filter_grid_mean_kernel)
    Mp = (M + 7) // 8 * 8
    W0, W1 = abs(cw0) + mxi, abs(cw1) + meta
    W2 = abs(alpha) * W0 + abs(beta) * W1 if regime == 2 else abs(cw2)
    sq = np.sqrt(rho * rho + 2.0) + rho
    kd = np.sqrt(K_DROP) - rho
    eps = 1.05 * (18.2 * EPS_K + U * (1.01 * (3.5 * sq * sq + 43.0) + 1.02 * (Mp + 4))
                  + 1.01 * dev * ((2.0 + abs(alpha) + abs(beta)) if regime == 2 else 2.0)
                  + U * (2.0 * (mxi + meta) + (10.0 * W2 if regime == 2 else 2.0 * W2))
                  + 4.5e-16 * (0.5 * (W0 * W0 + W1 * W1 + W2 * W2) + 0.5 * (xs ** 2).sum(1).max())
                  + 7e-16 * (M + 8) + np.exp(-0.5 * kd * kd))
    bound = eps * np.abs(gamma).sum() + 1e-150 * (Mp + 1)
    # extended-precision reference at the grid's points: zs = fl(x / l) and the u of the regime -- the
    # policy's rounded fl(x0 a) + fl(x1 b) on the affine one, the saturation constant otherwise (every
    # point of the tile is checked against the regime's arithmetic)
    L = np.longdouble
    ur = raw if regime == 2 else np.full_like(raw, lim[regime])
    zs = np.stack(np.broadcast_arrays((x0 / l0)[:, None], (x1 / l1)[None, :], ur / l2), axis=-1).astype(L)
    d2 = ((zs[:, :, None, :] - xs.astype(L)[None, None, :, :]) ** 2).sum(-1)
    ref = (np.exp(-d2 / 2) * gamma.astype(L)).sum(-1)
    return mean, ref, bound, rho, np.abs(gamma).sum()


@pytest.mark.parametrize("case", ["pendulum", "wide tile", "steep policy", "far tile", "tight cluster",
                                  "short lengthscales"])
@pytest.mark.parametrize("regime", [0, 1, 2])
def test_factored_tile_mean_within_bound(case, regime):
    rng = np.random.default_rng(7 + regime)
    kw = dict(lo=(-1.0, -1.0), unit=(2 / 255, 2 / 255), ls=(1.5, 1.5, 2.0), row0=96, col0=112,
              gain=(-0.9, -1.7), lim=(-1.0, 1.0), M=500, spread=1.0, centre_pull=0.3)
    if case == "wide tile":
        kw.update(ls=(0.12, 0.1, 0.3))
    if case == "steep policy":
        kw.update(gain=(-40.0, 25.0), ls=(0.8, 0.9, 0.5))
    if case == "far tile":
        kw.update(lo=(-3000.0, 2000.0), unit=(0.01, 0.013))
    if case == "tight cluster":
        kw.update(spread=0.05, centre_pull=0.01)
    if case == "short lengthscales":
        kw.update(ls=(0.07, 0.07, 0.5))
    mean, ref, bound, rho, g1 = _tile(rng, regime=regime, **kw)
    if not rho <= RHO_MAX:
        pytest.skip("tile outside the admissible range (its points take the fp64 route)")
    err = np.abs(mean.astype(np.longdouble) - ref).astype(float)
    assert (err <= bound).all(), "max err / bound = %g" % (err.max() / bound)
    # fp64-class; far from the origin the expanded distance of the full posterior itself rounds at
    # |w|^2 u (4.5e-16 (|w|^2 / 2 + hmax) of the bound)
    assert bound <= (1e-7 if case == "far tile" else 1e-9) * g1, "bound is not fp64-class: %g of sum |gamma|" % (
        bound / g1)
