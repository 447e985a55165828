"""Host-side rules of the policy-iteration kernels (no GPU): when ``slb_bellman_argmax`` takes the
factored tensor-core path of ``csrc/bellman_tile.cu`` and how much workspace it asks for, and the
slice size of the staged GP mean the Bellman kernels run (``mean_chunk_rows`` in
``csrc/gp_mean_staged.cuh``), restated here so that ``tests/test_gpu_bellman_shapes.py`` can place M
on its boundaries."""
import ctypes

import pytest


def mean_chunk_rows(din, nomax):
    """Rows per staged slice of the Bellman kernels' GP mean: a 24 KB budget for two buffers of
    [x / l, h] rows (din + 1 doubles) and the gammas of the factor's outputs (nomax doubles), at most
    256 rows, a multiple of 8."""
    return min(256, (24576 // (16 * (din + 1 + nomax))) & ~7)


def test_mean_chunk_rows_restatement():
    assert [mean_chunk_rows(din, 1) for din in range(1, 7)] == [256, 256, 256, 256, 216, 192]
    assert mean_chunk_rows(5, 4) == 152          # four outputs on one factor at d_in = 5
    assert mean_chunk_rows(6, 5) == 128
    assert mean_chunk_rows(4, 2) == 216


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__
    __graft_entry__.build()
    from safe_learning_b200 import _native
    return _native.load()


_DUMMY = (ctypes.c_double * 16)()                # any non-NULL address: the rule never reads it


def _bellman(d, m, M=(100,), outputs_factor=None, prims=0, gamma_f=True):
    """A Bellman descriptor with a d-dimensional grid, m actions and a GP stack of d outputs on
    len(M) factors (factor f with M[f] rows); output o sits on factor outputs_factor[o]."""
    from safe_learning_b200 import _native as nat
    cfg = nat.SlbBellman()
    cfg.grid.ndim = d
    cfg.fixed_action = 1
    cfg.policy.out_dim = m
    cfg.gp.num_outputs, cfg.gp.num_factors, cfg.gp.input_dim = d, len(M), d + m
    for f, rows in enumerate(M):
        cfg.gp.factors[f].M = rows
        cfg.gp.factors[f].kernel.num_prims = prims
    if outputs_factor is None:
        outputs_factor = [min(o, len(M) - 1) for o in range(d)]
    for o in range(d):
        cfg.gp.outputs[o].factor = outputs_factor[o]
        cfg.gp.outputs[o].gamma_f = ctypes.addressof(_DUMMY) if gamma_f else None
    return cfg


def _expected_bytes(cfg, n_actions):
    nrb = -(-n_actions // 8)
    return sum(nrb * -(-cfg.gp.factors[cfg.gp.outputs[o].factor].M // 8) * 64 * 8
               for o in range(cfg.gp.num_outputs))


@pytest.mark.parametrize("d", [1, 2])
@pytest.mark.parametrize("m", [1, 2])
def test_factored_argmax_workspace_plain_rbf(lib, d, m):
    """Plain RBF factors at d <= 2: the factored path applies for every n_actions >= 2, and the
    workspace holds one packed [ceil(n/8) x ceil(M/8)] block table of 64 doubles per output."""
    layouts = [dict(M=[127] * d), dict(M=[129, 40][:d]), dict(M=[500], outputs_factor=[0] * d)]
    for layout in layouts:
        cfg = _bellman(d, m, **layout)
        for n_actions in (2, 7, 8, 9, 101, 128, 129, 202):
            got = lib.slb_bellman_argmax_workspace(cfg, n_actions)
            assert got > 0
            assert got == _expected_bytes(cfg, n_actions), (layout, n_actions)
    # C3: 101 actions, two factors of 500 rows
    assert lib.slb_bellman_argmax_workspace(_bellman(2, 1, M=[500, 500]), 101) == 2 * 13 * 63 * 512


@pytest.mark.parametrize("m", [1, 2])
def test_factored_argmax_does_not_apply(lib, m):
    """Workspace 0 (the per-action kernel runs) for one action, a covariance expression, a factor
    without data, a missing gamma_f table, and every state dimension from 3 on: the tile's means
    take d * 128 * 64 doubles of shared memory, above the CTA's 227 KB at d = 3."""
    for d in (1, 2):
        assert lib.slb_bellman_argmax_workspace(_bellman(d, m), 1) == 0
        assert lib.slb_bellman_argmax_workspace(_bellman(d, m, prims=2), 9) == 0
        assert lib.slb_bellman_argmax_workspace(_bellman(d, m, gamma_f=False), 9) == 0
        assert lib.slb_bellman_argmax_workspace(_bellman(d, m), 0) == 0
    assert lib.slb_bellman_argmax_workspace(_bellman(1, m, M=[0]), 9) == 0
    assert lib.slb_bellman_argmax_workspace(_bellman(2, m, M=[0, 100]), 9) == 0
    assert lib.slb_bellman_argmax_workspace(_bellman(2, m, M=[100, 0]), 9) == 0
    for d in (3, 4, 5, 6):
        for layout in (dict(M=[100] * d), dict(M=[8], outputs_factor=[0] * d)):
            for n_actions in (2, 9, 101):
                assert lib.slb_bellman_argmax_workspace(_bellman(d, m, **layout), n_actions) == 0
    assert lib.slb_bellman_argmax_workspace(None, 9) == 0
