"""fp64 restatement of the iLQR backward pass (fb_lqr; Tassa, Erez & Todorov 2012) in numpy, one problem at a time."""
import numpy as np


def backward(A, B, q, r, Q, R, Qf, mu):
    """A [T, nx, nx], B [T, nx, nu], q [T + 1, nx], r [T, nu], diagonal weights Q [nx], R [nu], Qf [nx], regularisation mu (added to
    Quu).  -> (K [T, nu, nx], k [T, nu], dV [2], status): status t + 1 when Quu is not positive definite at step t (the steps before it
    are not computed: their K and k are zero)."""
    A, B = np.asarray(A, np.float64), np.asarray(B, np.float64)
    T, nx, nu = B.shape
    K, k, dV = np.zeros((T, nu, nx)), np.zeros((T, nu)), np.zeros(2)
    s, P = np.array(q[T], np.float64), np.diag(np.asarray(Qf, np.float64))
    for t in range(T - 1, -1, -1):
        a, b = A[t], B[t]
        Qx, Qu = q[t] + a.T @ s, r[t] + b.T @ s
        Qxx = np.diag(Q) + a.T @ P @ a
        Quu = np.diag(R) + b.T @ P @ b + mu * np.eye(nu)
        Qux = b.T @ P @ a
        try:
            c = np.linalg.cholesky(Quu)
        except np.linalg.LinAlgError:
            return K, k, dV, t + 1
        solve = lambda y: -np.linalg.solve(c.T, np.linalg.solve(c, y))       # noqa: E731
        k[t], K[t] = solve(Qu), solve(Qux)
        dV += [k[t] @ Qu, 0.5 * k[t] @ Quu @ k[t]]
        s = Qx + K[t].T @ Quu @ k[t] + K[t].T @ Qu + Qux.T @ k[t]
        P = Qxx + K[t].T @ Quu @ K[t] + K[t].T @ Qux + Qux.T @ K[t]
        P = 0.5 * (P + P.T)
    return K, k, dV, 0
