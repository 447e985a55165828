"""CPU oracle for the safe_learning region-of-attraction hot path.

TEST INFRASTRUCTURE ONLY.  This package is a numpy/scipy (fp64) restatement of the
reference algorithm (befelix/safe_learning @ f1aad5a); every function cites the
reference ``file:line`` it follows.  Only ``tests/``, ``__graft_entry__.smoke()``
and ``bench.py``'s CPU-baseline / ``--impl reference`` legs may import it -- and
there only as the checker or the timed CPU baseline, never as the product.  The
product package ``safe_learning_b200`` must never import ``oracle``.

Pinning status (see DESIGN.md "Oracle"):

* pinned by the reference's own known-answer tests: RBF GP posterior golden
  vector (``safe_learning/tests/test_functions.py:237-261``), ``update_safe_set``
  known answers (``tests/test_lyapunov.py:48-74``), safe-set initialisation
  (``:24-46``), quadratic values (``test_functions.py:264-282``), GridWorld round
  trips (``:313-367``), triangulation known answers (``:457-655``), ``dlqr``
  (``test_utilities.py:17-28``), ``r + gamma V`` (``test_rl.py:145-172``);
* pinned by outputs of the reference itself executed in the build container through
  a numpy-backed TF1/gpflow API shim (``tests/golden/make_golden.py`` ->
  ``tests/golden/*.npz``): GP-uncertain ``update_safe_set`` incl. multi-batch
  ``can_shrink`` behaviour and the ``c_max`` quirks, ``Triangulation`` evaluation,
  ``PolicyIteration.future_values`` / ``value_iteration`` /
  ``discrete_policy_optimization``;
* third-party arithmetic restated from its published algorithm (not under
  the upstream sources): ``gpflow==0.4.0`` ``kernels`` ``K/Kdiag`` (``requirements.txt:3``).  RBF is
  anchored by the golden vector above; Matern12/32/52, Linear, Constant, White, Add and Prod
  are PARITY UNPINNED as arithmetic (no vector of theirs exists upstream) -- the reference's
  own GP code around them runs on the fixture shim's restatement of the same formulae;
* PARITY UNPINNED: the adaptive-refinement branch (``lyapunov.py:445-487, 540-582``) -- no
  upstream test, and upstream tests the wrong tensor in the refined check; both readings are
  restated (``Lyapunov.refined_negative``).
"""

from .reference_path import *  # noqa: F401,F403
