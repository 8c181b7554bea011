"""fp64 reference of the stepper's finite-difference inverse-dynamics Jacobians (fb_fd_inverse, flybody_b200.derivatives.inverse_fd),
for tests/test_inverse_fd.py and tools/gpu_inverse_fd.py.

It restates the definition on the oracle: inputs (dq, qvel, qacc), the same columns (input j nudged by +delta / -delta centred, +delta
forward against the nominal) and step (delta_j = eps max(1, |x_j|), x_j the hinge angle or the free joint's translation component, qvel
or qacc; rotational tangent coordinates eps: tests/fd_reference.py).  Per column the oracle is reset to the nudged (qpos, qvel) and runs
`forward()`, then the fp64 mj_inverse of tests/inverse_reference.py at the nudged qacc; the forces and the dense M are differenced, M
mapped to MuJoCo's sparse qM order through dof_Madr and the dof's ancestor chain.  Outputs are transposed as MuJoCo's: row i is the
derivative with respect to input i.  A model with a ball joint goes through the free-joint surrogate (tests/test_walk_on_ball.py).
Nothing here changes the oracle.
"""
import numpy as np

from oracle import fly_oracle as fo

import fd_reference as fr
import inverse_reference as ir


def sparse_index(m):
    """(row, col) of every entry of the sparse qM: entry dof_Madr[i] + t is M[i, t-th ancestor of i] (t = 0: the diagonal)"""
    rows, cols = np.zeros(int(m.nM), np.int64), np.zeros(int(m.nM), np.int64)
    for i in range(m.nv):
        t, k = 0, i
        while k >= 0:
            rows[int(m.dof_Madr[i]) + t], cols[int(m.dof_Madr[i]) + t] = i, k
            k, t = int(m.dof_parentid[k]), t + 1
    return rows, cols


class Inverse:
    """the oracle's mj_inverse of states of model m: (qpos, qvel, qacc) -> (qfrc_inverse [nv], dense M [nv, nv], oracle); a ball model
    through its free-joint surrogate"""

    def __init__(self, m):
        self.m, self.ball = m, any(int(t) == fr.BALL for t in m.jnt_type)
        if self.ball:
            from test_walk_on_ball import free_surrogate, to_surrogate_q
            self.mo = free_surrogate(m)
            self.to_q = lambda q: to_surrogate_q(m, q)
        else:
            self.mo, self.to_q = m, lambda q: q
        self.o = fo.Oracle(self.mo, tolerance=1e-12)

    def __call__(self, q, v, a):
        k = 3 if self.ball else 0
        self.o.reset(self.to_q(q), np.concatenate([np.zeros(k), v]))
        self.o.forward()
        r = ir.inverse(self.mo, self.o, np.concatenate([np.zeros(k), a]))
        return r['qfrc_inverse'][k:], r['M'][k:, k:]


def steps(m, q, v, a, eps, centered):
    """per input j of (dq, qvel, qacc): (plus step, minus step), the minus step 0 forward (fd_reference's step rule; qacc like qvel)"""
    out = fr.steps(m, (q, v, np.zeros(m.na), np.zeros(m.nu)), eps, centered)[:2 * m.nv]
    for x in a:
        d = eps * max(1.0, abs(x))
        out.append((d, -d if centered else 0.0))
    return out


def nudge(m, q, v, a, j, step):
    """(q, v, a) with input j moved by step (fd_reference._nudge: mj_integratePos for dq)"""
    if j < 2 * m.nv:
        q, v, _, _ = fr._nudge(m, (q, v, np.zeros(m.na), np.zeros(m.nu)), j, step)
        return q, v, a.copy()
    a = a.copy()
    a[j - 2 * m.nv] += step
    return q.copy(), v.copy(), a


def inverse_fd(m, qpos, qvel, qacc, eps=1e-3, centered=True, run=None):
    """fp64 dict of DfDq, DfDv, DfDa [nv, nv], DmDq [nv, nM] (transposed: row i = d / d input i) and the nominal qfrc_inverse"""
    q, v, a = (np.asarray(x, np.float64) for x in (qpos, qvel, qacc))
    run = run or Inverse(m)
    f0, M0 = run(q, v, a)
    rows, cols = sparse_index(m)
    nv = m.nv
    F, S = np.zeros((3 * nv, nv)), np.zeros((nv, int(m.nM)))
    for j, (dp, dm) in enumerate(steps(m, q, v, a, eps, centered)):
        fb, Mb = run(*nudge(m, q, v, a, j, dp))
        fa, Ma = run(*nudge(m, q, v, a, j, dm)) if dm else (f0, M0)
        F[j] = (fb - fa) / (dp - dm)
        if j < nv:
            S[j] = (Mb - Ma)[rows, cols] / (dp - dm)
    return dict(DfDq=F[:nv], DfDv=F[nv:2 * nv], DfDa=F[2 * nv:], DmDq=S, qfrc_inverse=f0)
