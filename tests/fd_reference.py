"""fp64 reference of the stepper's finite-difference transition Jacobians (fb_fd_transition, flybody_b200.derivatives), for
tests/test_transition_fd.py and tools/gpu_fd.py.

It restates the definition on the oracle: the same columns (column 0 the nominal; input j nudged by +delta / -delta centred, +delta
forward), the same step delta_j = eps max(1, |x_j|) (x_j the hinge angle or the free joint's translation component, qvel, act or ctrl;
rotational tangent coordinates eps) and MuJoCo's ctrl-limit rule.  The nudge of a dq coordinate is fp64 mj_integratePos, every column is
stepped n_substeps times by the oracle (mj_step2; mj_step1 with ctrl held fixed), and the next states are differenced with fp64
mj_differentiatePos (inverse_dynamics._differentiate_pos).  A model with a ball joint is stepped through the free-joint surrogate the
ball tests use (tests/test_walk_on_ball.py).  Nothing here changes the oracle.
"""
import numpy as np

from flybody_b200.inverse_dynamics import _differentiate_pos
from flybody_b200.synthetic import mult_quat
from oracle import fly_oracle as fo

FREE, BALL, HINGE = 0, 1, 3


def inputs(m):
    return 2 * m.nv + m.na + m.nu


def dof_coordinate(m, k):
    """(qpos address, rotation axis or -1) of dof k: the hinge or translation coordinate, or the quaternion of a rotational dof"""
    j = int(m.dof_jntid[k])
    t, qa, c = int(m.jnt_type[j]), int(m.jnt_qposadr[j]), k - int(m.jnt_dofadr[j])
    if t == FREE:
        return (qa + c, -1) if c < 3 else (qa + 3, c - 3)
    if t == BALL:
        return qa, c
    return qa, -1


def _nudge(m, x, j, step):
    """x = (q, v, act, ctrl) with input j moved by step (mj_integratePos for the dq inputs: mju_quatIntegrate normalises first)"""
    q, v, a, u = (y.copy() for y in x)
    if j < m.nv:
        qa, axis = dof_coordinate(m, j)
        if axis < 0:
            q[qa] += step
        else:
            quat = q[qa:qa + 4] / np.linalg.norm(q[qa:qa + 4])
            rot = np.zeros(4)
            rot[0], rot[1 + axis] = np.cos(step / 2), np.sin(step / 2)
            quat = mult_quat(quat, rot)
            q[qa:qa + 4] = quat / np.linalg.norm(quat)
    elif j < 2 * m.nv:
        v[j - m.nv] += step
    elif j < 2 * m.nv + m.na:
        a[j - 2 * m.nv] += step
    else:
        u[j - 2 * m.nv - m.na] += step
    return q, v, a, u


def steps(m, x, eps, centered):
    """per input j: (plus step, minus step), 0 where that side is not nudged; MuJoCo's ctrl-limit rule"""
    q, v, a, u = x
    out = []
    for j in range(inputs(m)):
        if j < m.nv:
            qa, axis = dof_coordinate(m, j)
            xj = 0.0 if axis >= 0 else q[qa]
        elif j < 2 * m.nv:
            xj = v[j - m.nv]
        elif j < 2 * m.nv + m.na:
            xj = a[j - 2 * m.nv]
        else:
            xj = u[j - 2 * m.nv - m.na]
        d = eps * max(1.0, abs(xj))
        if j < 2 * m.nv + m.na:
            out.append((d, -d if centered else 0.0))
            continue
        i = j - 2 * m.nv - m.na
        lo, hi = m.actuator_ctrlrange[i]

        def ok(p, r):
            return not m.actuator_ctrllimited[i] or (lo <= p <= hi and lo <= r <= hi)
        fwd = ok(xj, xj + d)
        back = (centered or not fwd) and ok(xj - d, xj)
        out.append((d if fwd else 0.0, -d if back else 0.0))
    return out


class Stepper:
    """the oracle stepping states of model m (a ball model through its free-joint surrogate)"""

    def __init__(self, m):
        self.m, self.ball = m, any(int(t) == BALL for t in m.jnt_type)
        if self.ball:
            from test_walk_on_ball import free_surrogate, to_surrogate_q
            self.o, self.to_q = fo.Oracle(free_surrogate(m), tolerance=1e-12), lambda q: to_surrogate_q(m, q)
        else:
            self.o, self.to_q = fo.Oracle(m, tolerance=1e-12), lambda q: q

    def __call__(self, x, n_substeps):
        q, v, a, u = x
        o, k = self.o, 3 if self.ball else 0
        o.reset(self.to_q(q), np.concatenate([np.zeros(k), v]))
        if self.m.na:
            o.set(fo.ACT, a)
        o.set(fo.CTRL, u)
        o.control_step(n_substeps)
        return o.qpos[k:], o.qvel[k:], o.get(fo.ACT) if self.m.na else np.zeros(0)


def transition_fd(m, qpos, qvel, act, ctrl, eps=1e-3, centered=True, n_substeps=1, stepper=None):
    """fp64 A [nx, nx], B [nx, nu] and the nominal next state (qpos, qvel, act) of one state"""
    x = tuple(np.asarray(y, np.float64) for y in (qpos, qvel, act if act is not None else np.zeros(m.na), ctrl))
    run = stepper or Stepper(m)
    nominal = run(x, n_substeps)
    sides = steps(m, x, eps, centered)
    nin, nx = inputs(m), 2 * m.nv + m.na
    qa_, qb_, va, vb, aa, ab, den = [], [], [], [], [], [], np.zeros(nin)
    for j, (dp, dm) in enumerate(sides):
        plus = run(_nudge(m, x, j, dp), n_substeps) if dp else nominal
        minus = run(_nudge(m, x, j, dm), n_substeps) if dm else nominal
        den[j] = dp - dm
        qa_.append(minus[0]); qb_.append(plus[0]); va.append(minus[1]); vb.append(plus[1]); aa.append(minus[2]); ab.append(plus[2])
    dq = _differentiate_pos(m, np.array(qa_), np.array(qb_), 1.0)
    cols = np.concatenate([dq, np.array(vb) - np.array(va), (np.array(ab) - np.array(aa)).reshape(nin, m.na)], 1)   # [nin, nx]
    cols = np.divide(cols, den[:, None], out=np.zeros_like(cols), where=den[:, None] != 0)
    return cols[:nx].T.copy(), cols[nx:].T.copy(), nominal
