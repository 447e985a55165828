"""Import the UNMODIFIED reference package (a befelix/safe_learning @ f1aad5a checkout whose
directory $SAFE_LEARNING_REFERENCE names) on top of the API shims.

Used by make_golden.py to produce the committed fixtures; no test needs the checkout.
"""
import collections
import collections.abc
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REFERENCE = os.environ.get("SAFE_LEARNING_REFERENCE", "")


def _listify(fn):
    def wrapper(arrays, *args, **kwargs):
        if not isinstance(arrays, (list, tuple, np.ndarray)):
            arrays = list(arrays)        # numpy 2 rejects generators / map objects
        return fn(arrays, *args, **kwargs)
    return wrapper


def load_reference():
    """Returns the imported ``safe_learning`` reference module."""
    if not os.path.isdir(REFERENCE):
        raise RuntimeError("set SAFE_LEARNING_REFERENCE to a befelix/safe_learning checkout")
    # Python >= 3.10 / numpy >= 1.24 compatibility aliases the 2018 sources rely on
    for name in ("Sequence", "Mapping", "Iterable"):
        if not hasattr(collections, name):
            setattr(collections, name, getattr(collections.abc, name))
    for alias, target in (("int", int), ("float", float), ("bool", bool)):
        if alias not in np.__dict__:
            setattr(np, alias, target)
    # SURVEY.md Q2: lyapunov.py:512 sorts V with numpy's default (unstable) kind, so which of two
    # states with EQUAL V comes first -- and hence where the prefix is cut inside a tie group --
    # is an accident of the numpy version.  The build pins ties by flat index; the fixtures are
    # generated with the same tie-break so everything else is compared bit for bit.
    _argsort = np.argsort
    np.argsort = lambda a, axis=-1, kind=None, order=None, **kw: _argsort(
        a, axis=axis, kind="stable", order=order, **kw)
    np.column_stack = _listify(np.column_stack)
    np.hstack = _listify(np.hstack)
    np.vstack = _listify(np.vstack)
    shim = os.path.join(HERE, "tf1_shim")
    for path in (REFERENCE, shim):
        if path not in sys.path:
            sys.path.insert(0, path)
    import safe_learning
    assert safe_learning.__file__.startswith(os.path.abspath(REFERENCE))
    return safe_learning
