"""numpy restatement of the reference's reverse-time Van der Pol plant (``examples/utilities.py:440-519``),
the checker of ``safe_learning_b200.VanDerPol``.

Called like the ``oracle`` plants (``vdp(states, actions)``, the action column ignored), so it slots into
``oracle.Lyapunov``, ``oracle.PolicyIteration`` and ``rollout_oracle``.  The normalisation is the
reference's ``tf.matmul(state, np.diag(T))``, a matrix product here too: an inf or NaN component of a
state makes the other column NaN.
"""
import numpy as np
import scipy.signal

from oracle.reference_path import hstack_inputs


class VanDerPol(object):
    """``examples/utilities.py:440-519``."""

    def __init__(self, damping=1, dt=0.01, normalization=None):
        self.damping, self.dt = damping, dt
        self.state_dim, self.action_dim = 2, 0
        self.normalization = normalization
        if normalization is not None:
            self.normalization = np.array(normalization, dtype=np.float64)
            self.inv_norm = self.normalization ** -1
        self.input_dim, self.output_dim = 3, 2

    def normalize(self, state):
        if self.normalization is None:
            return state
        return np.matmul(state, np.diag(self.inv_norm))

    def denormalize(self, state):
        if self.normalization is None:
            return state
        return np.matmul(state, np.diag(self.normalization))

    def linearize(self):
        A = np.array([[0, -1], [1, -1]], dtype=np.float64)
        if self.normalization is not None:
            A = np.linalg.multi_dot((np.diag(self.inv_norm), A, np.diag(self.normalization)))
        Ad, _, _, _, _ = scipy.signal.cont2discrete((A, np.zeros([2, 1]), 0, 0), self.dt, method="zoh")
        return Ad

    def ode(self, state):
        x, y = state[:, 0:1], state[:, 1:2]
        return np.concatenate((-y, x + self.damping * (x ** 2 - 1) * y), axis=1)

    def __call__(self, *inputs):
        sa = hstack_inputs(inputs)
        state = self.denormalize(sa[:, :2].copy())
        dt = self.dt / 10
        with np.errstate(over="ignore", invalid="ignore"):
            for _ in range(10):
                state = state + dt * self.ode(state)
            return self.normalize(state)
