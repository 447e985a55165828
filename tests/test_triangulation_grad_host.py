"""CPU tests of the Triangulation vertex gradient (``csrc/triangulation_grad.cu``): the exported symbols,
the host-side rejections of ``slb_function_vjp`` / ``slb_triangulation_rows`` for SLB_FN_TRIANGULATION
(every case fails before a launch), and the numpy oracle's restatement of
``_Triangulation.parameter_derivative`` against the reference's fixture."""
import os

import numpy as np
import pytest
import scipy.sparse

import oracle as O
from safe_learning_b200 import _native as nat
from safe_learning_b200.functions import GridWorld

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden",
                      "triangulation_param_derivative.npz")


def _lib():
    return nat.load()


def test_symbols_and_abi():
    lib = _lib()
    assert lib.slb_abi_version() == nat.ABI_VERSION
    for name in ("slb_function_vjp", "slb_function_vjp_workspace", "slb_triangulation_rows"):
        assert name in nat.SIGNATURES
        assert getattr(lib, name) is not None
    assert len(nat.SIGNATURES["slb_triangulation_rows"][1]) == 6


def _tri_desc(num_points=(5, 4), out_dim=1, flags=0):
    grid = GridWorld([[-1.0, 1.0]] * len(num_points), list(num_points))
    d = nat.SlbFunction()
    d.kind, d.in_dim, d.out_dim, d.flags = nat.FN_TRIANGULATION, grid.ndim, out_dim, flags
    d.matrix, d.hyperplanes, d.unit_simplices = 0x1000, 0x1100, 0x1200   # never dereferenced
    d.nsimplex = 2
    d.grid = grid.descriptor()
    d.grid.discrete_points = 0x1300
    return d


def _vjp(desc, n=10, points=0x2000, gout=0x3000, gin=None, gpar=0x5000, ws=None):
    return _lib().slb_function_vjp(None, desc, points, n, gout, gin, gpar, None, ws)


def test_vjp_rejects_point_gradient():
    assert _vjp(_tri_desc(), gin=0x4000, ws=0x6000) != 0
    assert "grad_in must be NULL" in nat.last_error()


@pytest.mark.parametrize("flag", [nat.FLAG_SATURATE, nat.FLAG_ABS, nat.FLAG_SCALE, nat.FLAG_GRADIENT])
def test_vjp_rejects_post_op_flags(flag):
    assert _vjp(_tri_desc(flags=flag), ws=0x6000) != 0
    assert "flags" in nat.last_error()


def test_vjp_rejects_null_buffers():
    assert _vjp(_tri_desc(), points=None, ws=0x6000) != 0
    assert "null points or cotangent" in nat.last_error()
    assert _vjp(_tri_desc(), gout=None, ws=0x6000) != 0
    assert "null points or cotangent" in nat.last_error()
    assert _vjp(_tri_desc(), ws=None) != 0
    assert "workspace" in nat.last_error()
    desc = _tri_desc()
    desc.matrix = None
    assert _vjp(desc, ws=0x6000) != 0
    assert "tables missing" in nat.last_error()


def test_vjp_rejects_negative_n():
    assert _vjp(_tri_desc(), n=-1, ws=0x6000) != 0
    assert "negative n" in nat.last_error()
    assert _lib().slb_function_vjp_workspace(_tri_desc(), -1) == -1


def test_vjp_rejects_key_overflow():
    # 2^60 vertices need 60 key bits; 100 points x 4 rows need 9 more
    desc = _tri_desc(num_points=(1 << 20,) * 3)
    assert _vjp(desc, n=100, ws=0x6000) != 0
    assert "64 bits" in nat.last_error()
    assert _lib().slb_function_vjp_workspace(desc, 100) == -1
    assert "64 bits" in nat.last_error()


def test_vjp_workspace_of_an_empty_batch_is_zero():
    assert _lib().slb_function_vjp_workspace(_tri_desc(), 0) == 0


def _rows(desc, n=10, points=0x2000, cols=0x3000, w=0x4000):
    return _lib().slb_triangulation_rows(None, desc, points, n, cols, w)


def test_rows_rejections():
    net = nat.SlbFunction()
    net.kind, net.in_dim, net.out_dim = nat.FN_LINEAR, 2, 1
    net.matrix = 0x1000
    assert _rows(net) != 0 and "not a Triangulation" in nat.last_error()
    assert _rows(_tri_desc(flags=nat.FLAG_SATURATE)) != 0 and "flags" in nat.last_error()
    assert _rows(_tri_desc(), n=-1) != 0 and "negative n" in nat.last_error()
    assert _rows(_tri_desc(), cols=None) != 0 and "null buffer" in nat.last_error()
    assert _rows(_tri_desc(), points=None) != 0 and "null buffer" in nat.last_error()
    assert _rows(_tri_desc(), n=0, points=None, cols=None, w=None) == 0


# ---------------------------------------------------------------- oracle against the reference fixture
def oracle_parameter_derivative(tri, points):
    """``_Triangulation.parameter_derivative`` restated on the numpy oracle, one query at a time as the
    fixture was made."""
    cols, weights = [], []
    for p in np.atleast_2d(points):
        w, c = tri.weights(p[None, :])
        cols.append(c[0])
        weights.append(w[0])
    cols, weights = np.array(cols, dtype=np.int64), np.array(weights)
    n, nsimp = cols.shape
    return scipy.sparse.coo_matrix((weights.ravel(), (np.repeat(np.arange(n), nsimp), cols.ravel())),
                                   shape=(n, tri.nindex))


def fixture_cases():
    fix = np.load(GOLDEN)
    for key in sorted(k[:-len("_points")] for k in fix.files if k.endswith("_points")):
        tag, proj, group = key.split("_", 2)
        yield key, tag, proj == "proj", group


@pytest.mark.parametrize("key,tag,project,group", list(fixture_cases()))
def test_oracle_parameter_derivative_matches_reference(key, tag, project, group):
    fix = np.load(GOLDEN)
    grid = O.GridWorld(fix[tag + "_limits"], fix[tag + "_num"])
    tri = O.Triangulation(grid, np.zeros((grid.nindex, 1)), project=project)
    got = oracle_parameter_derivative(tri, fix[key + "_points"])
    n, nsimp = fix[key + "_cols"].shape
    np.testing.assert_array_equal(got.row, np.repeat(np.arange(n), nsimp))
    np.testing.assert_array_equal(got.col.reshape(n, nsimp), fix[key + "_cols"])
    np.testing.assert_array_equal(got.data.reshape(n, nsimp), fix[key + "_weights"])
