"""numpy Kalman filter: the oracle of the batched filter (csrc/bmpc_kf.cuh).  TEST INFRASTRUCTURE.

The model of kalman_design_simple (/root/reference/pyMPC/kalman.py:73-106): x+ = A x + B u + w, y = C x + v, E[ww'] = Qn,
E[vv'] = Rn.  The filter holds the a-priori estimate x[k|k-1] and its covariance P.  The update uses the plain covariance form
P <- P - K S K', independent of the Joseph form the library evaluates.  The matrices are attributes: assign them to change the
model between steps."""
import numpy as np


class KalmanFilter:
    def __init__(self, x0, A, B, C, Qn, Rn, P0):
        self.A, self.B, self.C, self.Qn, self.Rn = A, B, C, Qn, Rn
        self.x = np.copy(x0); self.y = C @ self.x; self.P = np.copy(P0); self.K = None

    def predict(self, u):
        self.x = self.A @ self.x + self.B @ u
        self.P = self.A @ self.P @ self.A.T + self.Qn
        self.y = self.C @ self.x
        return self.x

    def update(self, y_meas):
        S = self.C @ self.P @ self.C.T + self.Rn
        self.K = self.P @ self.C.T @ np.linalg.inv(S)
        self.x = self.x + self.K @ (y_meas - self.y)
        self.P = self.P - self.K @ S @ self.K.T
        return self.x
