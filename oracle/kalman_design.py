"""scipy restatement of the Kalman design functions of pyMPC.kalman (/root/reference/pyMPC/kalman.py:24-106).  TEST
INFRASTRUCTURE.  The reference calls ``control.dare``; here the DARE is solved by ``scipy.linalg.solve_discrete_are``, a QZ
(generalised Schur) method, algorithmically independent of the structured doubling of pympc_b200 (csrc/bmpc_dare.cuh).
One system at a time (2-D arrays)."""
import numpy as np
import scipy.linalg


def dare(A, B, Q, R, S=None):
    """python-control's ``dare(A, B, Q, R, S)`` with E = I: returns (X, L, G) with
    X = A'XA - (A'XB + S)(R + B'XB)^-1 (B'XA + S') + Q,  G = (R + B'XB)^-1 (B'XA + S'),  L = eig(A - B G)."""
    A, B, Q, R = (np.asarray(a, float) for a in (A, B, Q, R))
    S = np.zeros(B.shape) if S is None else np.asarray(S, float)
    X = scipy.linalg.solve_discrete_are(A, B, Q, R, s=S)
    G = np.linalg.solve(R + B.T @ X @ B, B.T @ X @ A + S.T)
    return X, np.linalg.eigvals(A - B @ G), G


def kalman_design(A, B, C, D, Qn, Rn, Nn=None):
    """General design (kalman.py:44-70): the last nw = Qn.shape[0] columns of B and D carry the process noise w."""
    A, B, C, D, Qn, Rn = (np.asarray(a, float) for a in (A, B, C, D, Qn, Rn))
    nw = Qn.shape[0]; nu = B.shape[1] - nw; ny = C.shape[0]
    Nn = np.zeros((nw, ny)) if Nn is None else np.asarray(Nn, float)
    Bw, Dw = B[:, nu:], D[:, nu:]
    Hn = Dw @ Nn                                                   # kalman.py:58
    Rb = Rn + Hn + Hn.T + Dw @ Qn @ Dw.T                           # kalman.py:59
    Qb = Bw @ Qn @ Bw.T                                            # kalman.py:60
    Nb = Bw @ (Qn @ Dw.T + Nn)                                     # kalman.py:61
    Qb = (Qb + Qb.T) / 2; Rb = (Rb + Rb.T) / 2                     # kalman.py:64-65
    P, W, K = dare(A.T, C.T, Qb, Rb, Nb)                           # kalman.py:67 (E = I)
    return K.T, P, W                                               # kalman.py:69-70


def kalman_design_simple(A, B, C, D, Qn, Rn, type='filter'):
    """Simplified design (kalman.py:96-106); B and D are not used."""
    A, C, Qn, Rn = (np.asarray(a, float) for a in (A, C, Qn, Rn))
    P, W, _ = dare(A.T, C.T, Qn, Rn)                               # kalman.py:96
    Sinv = np.linalg.inv(C @ P @ C.T + Rn)
    if type == 'filter':
        L = P @ C.T @ Sinv                                         # kalman.py:100
    elif type == 'predictor':
        L = A @ P @ C.T @ Sinv                                     # kalman.py:102
    else:
        raise ValueError("Unknown Kalman design type. Specify either filter or predictor!")
    return L, P, W
