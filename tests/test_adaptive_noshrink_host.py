"""Host tests of ``update_safe_set(can_shrink=False)`` with adaptive refinement: the oracle's as-written
reading against the reference-generated fixture, the host replay ``adaptive_as_written`` (with a previous
safe set and refinement) against the oracle on random cases, and the argument checks of
``slb_no_shrink_scan`` / ``slb_no_shrink_resolve``, which fail before any launch."""
import os
import sys

import numpy as np
import pytest
from numpy.testing import assert_array_equal

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import oracle as O  # noqa: E402
from adaptive_noshrink_cases import fixture_cases, load_fixture, replay_fixture  # noqa: E402
from safe_learning_b200.lyapunov import adaptive_as_written  # noqa: E402

FIX, PAR = load_fixture()


def _oracle_reference(lyap, can_shrink, R, s):
    lyap.update_safe_set(can_shrink, R, s, refinement_mode="reference")


@pytest.mark.parametrize("case", fixture_cases(FIX), ids=lambda c: c[0])
def test_oracle_reference_mode_reproduces_fixture(case):
    replay_fixture(O, "oracle", FIX, PAR, case, _oracle_reference)


def test_fixture_is_not_trivial():
    """The recorded sequences grow the safe set past the initial set, refine cells, and change under
    can_shrink=False."""
    keys = [c[0] for c in fixture_cases(FIX)]
    assert any((FIX[k + "_3_refinement"] > 1).sum() > 50 for k in keys)
    assert any(not np.array_equal(FIX[k + "_1_safe_set"], FIX[k + "_3_safe_set"]) for k in keys)
    assert any(not np.array_equal(FIX[k + "_2_safe_set"], FIX[k + "_3_safe_set"]) for k in keys)


def _random_case(rng, num):
    """A deterministic pendulum whose V has up to 8-fold ties (P = I on a square symmetric grid)."""
    import bench_workloads as W
    par = W.make_pendulum(num_points=num, M=8, tau_scale=1.0)
    par["P"] = np.eye(2)
    par["tau"] = float(rng.choice([0.004, 0.01, 0.03]))
    grid = O.GridWorld(par["limits"], par["num_points"])
    policy = O.Saturation(O.LinearSystem(-par["K"]), -1., 1.)
    dyn = O.LinearSystem((par["A_true"], par["B_true"]))
    lyap = O.Lyapunov(grid, O.QuadraticFunction(par["P"]), dyn, par["L_dyn"],
                      O.AbsFunction(O.LinearSystem((2 * par["P"],))), par["tau"], policy,
                      initial_set=par["initial"], adaptive=True)
    return lyap


@pytest.mark.parametrize("seed", range(4))
def test_adaptive_as_written_matches_oracle(seed):
    """adaptive_as_written(safe_set=, refinement=) is the oracle's can_shrink=False reference reading, for
    batch sizes 1, 7, 64, N and N + 5, tied V and random previous safe sets and refinements."""
    rng = np.random.default_rng(seed)
    lyap = _random_case(rng, int(rng.integers(9, 16)))
    n = lyap.discretization.nindex
    states = lyap.discretization.all_points
    assert len(np.unique(lyap.values)) < n // 2            # heavily tied
    negative = lyap.negative(states)
    decrease, threshold = lyap.decrease_and_threshold(states)
    coef = np.broadcast_to(lyap.threshold(states, 1.0), decrease.shape)[:, 0]
    initial = lyap.initial_safe_set
    for batch in (1, 7, 64, n, n + 5):
        for R, s in ((4, 1.0), (16, 2.0), (2, 1.0)):
            prev = initial | (rng.random(n) < rng.choice([0.1, 0.5, 0.9]))
            refine = np.where(prev, rng.integers(0, R + 3, n), rng.integers(0, 2, n))
            old = O.config.gp_batch_size
            try:
                O.config.gp_batch_size = batch
                lyap.safe_set, lyap._refinement = prev.copy(), refine.copy()
                lyap.update_safe_set(False, R, s, refinement_mode="reference")
            finally:
                O.config.gp_batch_size = old
            safe, refinement, position = adaptive_as_written(
                lyap.values, negative, decrease[:, 0], threshold[:, 0], coef, initial, lyap.tau,
                batch, R, max(s, 1.0), safe_set=prev, refinement=refine)
            assert_array_equal(safe, lyap.safe_set)
            assert_array_equal(refinement, lyap._refinement)
            assert lyap.values[np.argsort(lyap.values, kind="stable")[position]] == lyap.c_max


# ------------------------------------------------------------------ host checks of the entry points
@pytest.fixture(scope="module")
def lib():
    import __graft_entry__
    __graft_entry__.build()
    from safe_learning_b200 import _native
    return _native.load()


FAKE = 64           # a non-null address: every call below fails its checks before touching memory


def _scan(lib, **kw):
    a = dict(order=FAKE, negative=FAKE, prev_safe=FAKE, initial=None, n_req=FAKE, n=100, batch=7, R=4,
             ws=FAKE, cand=FAKE)
    a.update(kw)
    return lib.slb_no_shrink_scan(None, a["order"], a["negative"], a["prev_safe"], a["initial"], a["n_req"],
                                  a["n"], a["batch"], a["R"], a["ws"], a["cand"])


def _resolve(lib, **kw):
    a = dict(order=FAKE, values=FAKE, negative=FAKE, prev_safe=FAKE, prev_ref=FAKE, initial=None,
             n_req=FAKE, refined=FAKE, n=100, batch=7, R=4, ws=FAKE, safe=FAKE, ref=FAKE, pos=FAKE,
             cmax=FAKE)
    a.update(kw)
    return lib.slb_no_shrink_resolve(None, a["order"], a["values"], a["negative"], a["prev_safe"], a["prev_ref"],
                                     a["initial"], a["n_req"], a["refined"], a["n"], a["batch"], a["R"],
                                     a["ws"], a["safe"], a["ref"], a["pos"], a["cmax"])


BAD = [(dict(n=-1), "negative n"), (dict(batch=0), "batch size"), (dict(R=0), "max_refinement"),
       (dict(ws=None), "null workspace"), (dict(order=None), "null order"),
       (dict(negative=None), "null order/negative"), (dict(prev_safe=None), "prev_safe"),
       (dict(n_req=None), "null n_req")]


@pytest.mark.parametrize("bad,message", BAD + [(dict(cand=None), "null candidates")])
def test_scan_rejects_bad_arguments(lib, bad, message):
    from safe_learning_b200 import _native as nat
    before = nat.launch_count()
    assert _scan(lib, **bad) != 0
    assert message in nat.last_error() and "slb_no_shrink_scan" in nat.last_error()
    assert nat.launch_count() == before


@pytest.mark.parametrize("bad,message", BAD + [
    (dict(values=None), "null values"), (dict(prev_ref=None), "prev_refinement"),
    (dict(refined=None), "refined"), (dict(safe=None), "null safe"), (dict(ref=None), "refinement output"),
    (dict(pos=None), "null c_max"), (dict(cmax=None), "null c_max")])
def test_resolve_rejects_bad_arguments(lib, bad, message):
    from safe_learning_b200 import _native as nat
    before = nat.launch_count()
    assert _resolve(lib, **bad) != 0
    assert message in nat.last_error() and "slb_no_shrink_resolve" in nat.last_error()
    assert nat.launch_count() == before


def test_workspace_size(lib):
    assert lib.slb_no_shrink_workspace(0, 1) == 16
    assert lib.slb_no_shrink_workspace(100, 7) == 8 * (2 + 3 * 15)
    assert lib.slb_no_shrink_workspace(100, 1000) == 8 * 5
    assert lib.slb_no_shrink_workspace(-1, 4) < 0 and lib.slb_no_shrink_workspace(10, 0) < 0
