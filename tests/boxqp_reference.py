"""fp64 restatement of control-limited DDP's backward pass (fb_lqr_box; Tassa, Mansard & Todorov 2014) in numpy, one problem at a time:
the projected Newton method of Tassa's boxQP with the constants and stop rules of csrc/fb_lqr.h, and the Riccati recursion around it."""
import numpy as np

MAX_ITER, MIN_GRAD, MIN_REL, STEP_DEC, MIN_STEP, ARMIJO = 100, 1e-8, 1e-8, 0.6, 1e-22, 0.1


def _clamped(x, g, lo, hi):
    return np.where((x == lo) & (g > 0), -1, np.where((x == hi) & (g < 0), 1, 0))


def boxqp(H, q, lo, hi):
    """min 1/2 x'Hx + q'x over lo <= x <= hi -> (x, clamped [n] (-1, +1, 0), chol of the free block (None: not positive definite),
    accepted steps, stop reason)"""
    n = len(q)
    f = lambda x: 0.5 * x @ H @ x + q @ x              # noqa: E731
    x = np.minimum(np.maximum(0.0, lo), hi)
    fx, steps, reason, cset, fac = f(x), 0, 1, None, None

    def factor(free):
        try:
            return np.linalg.cholesky(H[np.ix_(free, free)])
        except np.linalg.LinAlgError:
            return None

    for _ in range(MAX_ITER):
        g = q + H @ x
        c = _clamped(x, g, lo, hi)
        free = c == 0
        if not free.any():
            reason = 6
            break
        if cset is None or ((c != 0) != cset).any():
            fac, cset = factor(free), c != 0
            if fac is None:
                return x, c, None, steps, -1
        if np.linalg.norm(g[free]) < MIN_GRAD:
            reason = 5
            break
        dx = np.zeros(n)
        dx[free] = -np.linalg.solve(fac.T, np.linalg.solve(fac, g[free]))
        sdotg = dx @ g
        if not sdotg < 0:
            reason = 0
            break
        step, xt = 1.0, None
        while True:
            xc = np.minimum(np.maximum(x + step * dx, lo), hi)
            fc = f(xc)
            if (fc - fx) / (step * sdotg) >= ARMIJO:
                xt = xc
                break
            step *= STEP_DEC
            if step < MIN_STEP:
                break
        if xt is None:
            reason = 2
            break
        f0, x, fx = fx, xt, fc
        steps += 1
        if f0 - fx < MIN_REL * abs(f0):
            reason = 4
            break
    c = _clamped(x, q + H @ x, lo, hi)
    if cset is None or ((c != 0) != cset).any():
        fac = factor(c == 0) if (c == 0).any() else np.zeros((0, 0))
        if fac is None:
            return x, c, None, steps, -1
    return x, c, fac, steps, reason


def backward(A, B, q, r, Q, R, Qf, mu, lower, upper, record=None):
    """A [T, nx, nx], B [T, nx, nu], q [T + 1, nx], r [T, nu], diagonal weights Q [nx], R [nu], Qf [nx], mu (added to Quu), bounds
    lower, upper [T, nu] on du -> (K [T, nu, nx], k [T, nu], dV [2], status, clamped [T, nu], qp [T, 2]): status t + 1 when the free
    block of Quu is not positive definite at step t (the steps before it are not computed).  record: a dict that gets each step's QP,
    {t: (Quu, Qu)}."""
    A, B = np.asarray(A, np.float64), np.asarray(B, np.float64)
    T, nx, nu = B.shape
    K, k, dV = np.zeros((T, nu, nx)), np.zeros((T, nu)), np.zeros(2)
    clamped, qp = np.zeros((T, nu), np.int32), np.zeros((T, 2), np.int32)
    s, P = np.array(q[T], np.float64), np.diag(np.asarray(Qf, np.float64))
    for t in range(T - 1, -1, -1):
        a, b = A[t], B[t]
        Qx, Qu = q[t] + a.T @ s, r[t] + b.T @ s
        Qxx = np.diag(Q) + a.T @ P @ a
        Quu = np.diag(R) + b.T @ P @ b + mu * np.eye(nu)
        Qux = b.T @ P @ a
        if record is not None:
            record[t] = (Quu, Qu)
        x, c, fac, steps, reason = boxqp(Quu, Qu, lower[t], upper[t])
        clamped[t], qp[t] = c, (steps, reason)
        if fac is None:
            return K, k, dV, t + 1, clamped, qp
        free = c == 0
        k[t] = x
        if free.any():
            K[t][free] = -np.linalg.solve(fac.T, np.linalg.solve(fac, Qux[free]))
        dV += [k[t] @ Qu, 0.5 * k[t] @ Quu @ k[t]]
        s = Qx + K[t].T @ Quu @ k[t] + K[t].T @ Qu + Qux.T @ k[t]
        P = Qxx + K[t].T @ Quu @ K[t] + K[t].T @ Qux + Qux.T @ K[t]
        P = 0.5 * (P + P.T)
    return K, k, dV, 0, clamped, qp
