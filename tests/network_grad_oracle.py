"""torch-CPU fp64 restatement of the networks and plants the reference trains through, written from
the reference (``safe_learning/functions.py:1702-1729`` NeuralNetwork, ``examples/utilities.py:48-104``
LyapunovNetwork, ``:242-289`` InvertedPendulum, ``:387-437`` CartPole), for autograd gradients.

Parameters are plain tensors in the reference's TF shapes: MLP kernels ``[in_i, out_i]`` and hidden
biases ``[out_i]``; LyapunovNetwork ``weights_posdef_i [hidden_i, in_i]`` and ``weights_i [out_i - in_i,
in_i]``.  Activations are given as 'tanh' | 'relu' | 'linear' (TF's gradients: relu' = 0 at 0).
"""

import numpy as np
import torch

ACT = {"tanh": torch.tanh, "relu": torch.relu, "linear": lambda v: v, None: lambda v: v}


def mlp(x, kernels, biases, acts, output_scale=1.0, use_bias=True):
    """``tf.layers.dense`` stack: hidden layers with bias when use_bias, output layer without."""
    net = x
    for i, w in enumerate(kernels[:-1]):
        net = net @ w
        if use_bias:
            net = net + biases[i]
        net = ACT[acts[i]](net)
    net = ACT[acts[-1]](net @ kernels[-1])
    return net * output_scale


def lyapunov_kernels(weights, input_dim, output_dims, eps=1e-6):
    """``[W^T W + eps I; W_extra]`` per layer from a flat [W_posdef_0, (W_0,) W_posdef_1, ...] list."""
    out, it = [], iter(weights)
    din = input_dim
    for dout in output_dims:
        w0 = next(it)
        k = w0.T @ w0 + eps * torch.eye(din, dtype=torch.float64)
        if dout > din:
            k = torch.cat([k, next(it)], dim=0)
        out.append(k)
        din = dout
    return out


def lyapunov_network(x, weights, input_dim, output_dims, acts, eps=1e-6):
    net = x
    for k, a in zip(lyapunov_kernels(weights, input_dim, output_dims, eps), acts):
        net = ACT[a](net @ k.T)
    return torch.sum(net * net, dim=1, keepdim=True)


def pendulum(z, mass, length, friction=0.0, dt=1 / 80, normalization=None):
    state, action = z[:, :2], z[:, 2:3]
    if normalization is not None:
        state = state * torch.as_tensor(normalization[0], dtype=torch.float64)
        action = action * torch.as_tensor(normalization[1], dtype=torch.float64)
    inertia = mass * length ** 2
    h = dt / 10
    for _ in range(10):
        angle, omega = state[:, :1], state[:, 1:2]
        x_ddot = 9.81 / length * torch.sin(angle) + action / inertia
        if friction > 0:
            x_ddot = x_ddot - friction / inertia * omega
        state = state + h * torch.cat([omega, x_ddot], dim=1)
    if normalization is not None:
        state = state * torch.as_tensor(np.asarray(normalization[0], dtype=np.float64) ** -1)
    return state


def cartpole(z, m, M, L, b=0.0, dt=0.01, normalization=None):
    state, action = z[:, :4], z[:, 4:5]
    if normalization is not None:
        state = state * torch.as_tensor(normalization[0], dtype=torch.float64)
        action = action * torch.as_tensor(normalization[1], dtype=torch.float64)
    g = 9.81
    h = dt / 10
    for _ in range(10):
        theta, v, omega = state[:, 1:2], state[:, 2:3], state[:, 3:4]
        det = L * (M + m * torch.sin(theta) ** 2)
        v_dot = (action - m * L * omega ** 2 * torch.sin(theta) - b * omega * torch.cos(theta)
                 + 0.5 * m * g * L * torch.sin(2 * theta)) * L / det
        omega_dot = (action * torch.cos(theta) - 0.5 * m * L * omega ** 2 * torch.sin(2 * theta)
                     - b * (m + M) * omega / (m * L) + (m + M) * g * torch.sin(theta)) / det
        state = state + h * torch.cat([v, omega, v_dot, omega_dot], dim=1)
    if normalization is not None:
        state = state * torch.as_tensor(np.asarray(normalization[0], dtype=np.float64) ** -1)
    return state


def central_difference(f, x, h=1e-6):
    """d sum(f(x)) / dx by central differences (x a float64 tensor, f -> tensor)."""
    g = torch.zeros_like(x)
    flat, gflat = x.view(-1), g.view(-1)
    for i in range(flat.numel()):
        old = flat[i].item()
        flat[i] = old + h
        up = f(x).sum().item()
        flat[i] = old - h
        down = f(x).sum().item()
        flat[i] = old
        gflat[i] = (up - down) / (2 * h)
    return g
