"""Workload definitions (BASELINE.json ``configs``; parameters from SURVEY.md §8d).

Each function returns the keyword arguments of ``MPCController(...)`` for one MPC instance.
Sources of the numbers (reference file:line):
  point_mass   /root/reference/examples/example_point_mass.py:11-71
  pendulum     /root/reference/examples/example_inverted_pendulum.py:10-69
  mimo         shape of /root/reference/test_scripts/cvx_mpc_reference_governor_du_mimo.py:15-62,
               SISO blocks in canonical form per test_scripts/reference_governor/system_dynamics.py:9-24
"""
import numpy as np


def point_mass():
    Ts, M, b = 0.2, 2.0, 0.3
    Ac = np.array([[0.0, 1.0], [0.0, -b / M]])
    Bc = np.array([[0.0], [1.0 / M]])
    return dict(Ad=np.eye(2) + Ac * Ts, Bd=Bc * Ts, Np=20,
                x0=np.array([0.1, 0.2]), xref=np.array([7.0, 0.0]), uminus1=np.array([0.0]),
                Qx=np.diag([0.5, 0.1]), QxN=np.diag([0.5, 0.1]), Qu=2.0 * np.eye(1), QDu=10.0 * np.eye(1),
                xmin=np.array([-100.0, -100.0]), xmax=np.array([100.0, 100.0]),
                umin=np.array([-1.2]), umax=np.array([1.2]),
                Dumin=np.array([-0.2]), Dumax=np.array([0.2]))


# cart-pole constants of the inverted-pendulum example: cart mass M, pole mass m, cart friction b, pole friction ftheta, pole
# length l, gravity g, sampling time Ts
CARTPOLE = (0.5, 0.2, 0.1, 0.1, 0.3, 9.81, 50e-3)


def pendulum():
    M, m, b, ftheta, l, g, Ts = CARTPOLE
    Ac = np.array([[0, 1, 0, 0],
                   [0, -b / M, -(g * m) / M, (ftheta * m) / M],
                   [0, 0, 0, 1],
                   [0, b / (M * l), (M * g + g * m) / (M * l), -(M * ftheta + ftheta * m) / (M * l)]])
    Bc = np.array([[0.0], [1.0 / M], [0.0], [-1 / (M * l)]])
    return dict(Ad=np.eye(4) + Ac * Ts, Bd=Bc * Ts, Np=20,
                x0=np.array([0.0, 0.0, 15 * 2 * np.pi / 360, 0.0]),
                xref=np.array([0.3, 0.0, 0.0, 0.0]), uminus1=np.array([0.0]),
                Qx=np.diag([0.3, 0.0, 1.0, 0.0]), QxN=np.diag([0.3, 0.0, 1.0, 0.0]),
                Qu=0.0 * np.eye(1), QDu=0.01 * np.eye(1),
                xmin=np.array([-1.0, -100.0, -100.0, -100.0]), xmax=np.array([0.3, 100.0, 100.0, 100.0]),
                umin=np.array([-20.0]), umax=np.array([20.0]),
                Dumin=np.array([-5.0]), Dumax=np.array([5.0]), eps_feas=1e3)


def pendulum_random(batch, seed=0):
    """Per-instance x0 / xref of BASELINE config 3 (SURVEY.md §8d): returns (X0[B,4], Xref[B,4])."""
    rng = np.random.default_rng(seed)
    X0 = np.stack([rng.uniform(-0.5, 0.25, batch), rng.uniform(-0.5, 0.5, batch),
                   rng.uniform(-15, 15, batch) * np.pi / 180, rng.uniform(-0.5, 0.5, batch)], axis=1)
    Xref = np.zeros((batch, 4))
    Xref[:, 0] = rng.uniform(-0.5, 0.3, batch)
    return X0, Xref


def _ops(X):
    """(sin, cos, stack) for numpy arrays or torch tensors"""
    if type(X).__module__.startswith("torch"):
        import torch
        return torch.sin, torch.cos, torch.stack
    return np.sin, np.cos, np.stack


def _cartpole_terms(X, U):
    M, m, b, ft, l, g, _ = CARTPOLE
    sin, cos, stack = _ops(X)
    v, th, om = X[..., 1], X[..., 2], X[..., 3]
    F = U[..., 0] if U.ndim == X.ndim else U
    s, c = sin(th), cos(th)
    D = M + m * s * s                                  # effective mass of the cart
    f = F - b * v                                      # force minus cart friction
    N1 = m * l * s * om * om - m * g * s * c + m * ft * c * om + f
    N3 = (M + m) * (g * s - ft * om) - m * l * om * om * s * c - f * c
    return stack, v, om, s, c, D, f, N1, N3


def cartpole_rhs(X, U):
    """Nonlinear cart-pole whose linearisation at the upright equilibrium is pendulum()'s model — the plant the inverted-pendulum
    example simulates in closed loop.  Batched: X [B,4] = (cart position, cart velocity v, pole angle theta from upright, angular
    velocity omega), U [B,1] or [B] = force on the cart; returns dX/dt [B,4].  Constants: CARTPOLE.  numpy arrays or torch tensors."""
    l = CARTPOLE[4]
    stack, v, om, s, c, D, f, N1, N3 = _cartpole_terms(X, U)
    return stack([v, N1 / D, om, N3 / (l * D)], -1)


def cartpole_linearised(X, U, Ts=CARTPOLE[6]):
    """Euler-discretised Jacobians of cartpole_rhs about each instance's (x, u): Ad = I + Ts df/dx [B,4,4], Bd = Ts df/du [B,4,1] —
    the model a successive-linearisation MPC hands to MPCController.update_system at every sample.  At the upright equilibrium
    (x = 0, u = 0) they are pendulum()'s Ad and Bd.  numpy arrays or torch tensors (the result lives where X does)."""
    M, m, b, ft, l, g, _ = CARTPOLE
    stack, v, om, s, c, D, f, N1, N3 = _cartpole_terms(X, U)
    dD = 2.0 * m * s * c                               # dD/dtheta
    av, aw = N1 / D, N3 / (l * D)
    # cart acceleration av = N1 / D
    dav_dv, dav_dom, dav_dF = -b / D, (2.0 * m * l * s * om + m * ft * c) / D, 1.0 / D
    dav_dth = (m * l * c * om * om - m * g * (c * c - s * s) - m * ft * s * om - av * dD) / D
    # angular acceleration aw = N3 / (l D)
    daw_dv, daw_dom, daw_dF = b * c / (l * D), (-(M + m) * ft - 2.0 * m * l * om * s * c) / (l * D), -c / (l * D)
    daw_dth = ((M + m) * g * c - m * l * om * om * (c * c - s * s) + f * s - aw * l * dD) / (l * D)
    z = v * 0.0
    o = z + 1.0
    Ad = stack([stack([o, z + Ts, z, z], -1),
                stack([z, 1.0 + Ts * dav_dv, Ts * dav_dth, Ts * dav_dom], -1),
                stack([z, z, o, z + Ts], -1),
                stack([z, Ts * daw_dv, Ts * daw_dth, 1.0 + Ts * daw_dom], -1)], -2)
    Bd = stack([z, Ts * dav_dF, z, Ts * daw_dF], -1)[..., None]
    return Ad, Bd


def mimo():
    r, ws = 0.9, [0.2, 0.4, 0.2, 0.4]
    nb = len(ws)
    Ad = np.zeros((2 * nb, 2 * nb)); Bd = np.zeros((2 * nb, nb)); C = np.zeros((nb, 2 * nb))
    xref = np.zeros(2 * nb)
    for i, w in enumerate(ws):
        kap = 1 - 2 * r * np.cos(w) + r * r
        Ad[2 * i:2 * i + 2, 2 * i:2 * i + 2] = [[2 * r * np.cos(w), -r * r], [1.0, 0.0]]
        Bd[2 * i, i] = 1.0
        C[i, 2 * i + 1] = kap
        xref[2 * i:2 * i + 2] = 1.0 / kap                      # steady state with C xref = 1
    Qx = C.T @ (20.0 * np.eye(nb)) @ C
    return dict(Ad=Ad, Bd=Bd, Np=40, x0=np.zeros(2 * nb), xref=xref, uminus1=np.zeros(nb),
                Qx=Qx, QxN=Qx, Qu=np.zeros((nb, nb)), QDu=0.5 * np.eye(nb),
                xmin=-100.0 * np.ones(2 * nb), xmax=100.0 * np.ones(2 * nb),
                umin=-1000.0 * np.ones(nb), umax=1000.0 * np.ones(nb),
                Dumin=-0.2 * np.ones(nb), Dumax=0.2 * np.ones(nb))


WORKLOADS = {"point_mass": point_mass, "pendulum": pendulum, "mimo": mimo}
