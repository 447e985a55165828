"""safe_learning_b200 -- the region-of-attraction hot path of befelix/safe_learning on H100.

Drop-in for ``Lyapunov.update_safe_set`` / ``v_decrease_confidence`` / ``v_decrease_bound`` on a
``GridWorld`` with ``GaussianProcess`` / ``FunctionStack`` dynamics and the ``PolicyIteration``
Bellman sweep; the arithmetic runs in hand-written sm_90a CUDA (``libslb200.so``, C ABI in
``include/slb200.h``).  No CPU fallback.
"""

from .functions import config  # noqa: F401  (singleton, like safe_learning.config)
from .functions import *  # noqa: F401,F403
from .lyapunov import *  # noqa: F401,F403
from .reinforcement_learning import *  # noqa: F401,F403
from .rollout import *  # noqa: F401,F403
from . import utilities  # noqa: F401
from .utilities import compute_trajectory  # noqa: F401

__version__ = "0.1.0"
