"""numpy float64 restatement of the PLDA adaptation of DESIGN.md section 5.26 (vbx_b200/adapt.py's docstring), for the
tests.  It shares no code with vbx_b200: the covariances come from explicit inverses, and the generalised eigenproblem
C' v = lambda Sigma v is reduced by its own Cholesky factor Sigma = L L^T to the ordinary one of L^-1 C' L^-T."""
import numpy as np


def covariances(T, psi):
    """W = T^-1 T^-T, B = T^-1 diag(psi) T^-T."""
    Ti = np.linalg.inv(np.asarray(T, dtype=np.float64))
    return Ti @ Ti.T, Ti @ np.diag(np.asarray(psi, dtype=np.float64)) @ Ti.T


def adapt(mu, W, B, m, C, w=0.3, b=0.7, s=1.0):
    """(mu', W', B', lambda ascending): Delta = m - mu, C' = C + s Delta Delta^T, Sigma = W + B = L L^T;
    L^-1 C' L^-T = U diag(lambda) U^T, V = L^-T U; E = Sigma V diag(max(lambda - 1, 0)) V^T Sigma = L U diag(e) U^T L^T;
    W' = W + w E, B' = B + b E, mu' = m."""
    delta = np.asarray(m, dtype=np.float64) - np.asarray(mu, dtype=np.float64)
    Cp = np.asarray(C, dtype=np.float64) + s * np.outer(delta, delta)
    L = np.linalg.cholesky(W + B)
    Li = np.linalg.inv(L)
    A = Li @ Cp @ Li.T
    lam, U = np.linalg.eigh(0.5 * (A + A.T))
    LU = L @ U
    E = LU @ np.diag(np.maximum(lam - 1.0, 0.0)) @ LU.T
    return np.asarray(m, dtype=np.float64).copy(), W + w * E, B + b * E, lam


def stats(z):
    """Mean and covariance (scatter / N) of the rows z, float64."""
    z = np.asarray(z, dtype=np.float64)
    m = z.mean(0)
    zc = z - m[None, :]
    return m, zc.T @ zc / z.shape[0]
