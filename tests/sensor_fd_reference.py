"""fp64 reference of the sensor outputs of the dynamics queries (fb_query_sensors), for tests/test_sensor_fd.py.

- Transition, C = ds/dx and D = ds/du: s is the sensordata of x itself, which the oracle's `forward()` gives (step1 + step2 without the
  integration).  The columns and steps are tests/fd_reference.py's; every column is one forward of the nudged state.
- Inverse sensordata at a given qacc: the oracle's sensors are those of its forward qacc and solver forces, so the acceleration-stage
  sensors are restated as their change from there.  At a fixed position / velocity state they are affine in (qacc, efc_force):
    accelerometer = forward's + R_site^T J_site (qacc - qacc_fwd)            (J_site: the site's translational Jacobian)
    force         = forward's + R_site^T [ sum over the subtree of m_c J_com,c (qacc - qacc_fwd) - (ext(f) - ext(f_fwd)) ]
  with ext the linear contact force on the subtree (orc_sensors_acc's cfrc_ext), f the efc_force of tests/inverse_reference.py.  The
  Jacobians come from the oracle's body poses and the model's joint axes; touch is restated with the ray test of orc_sensors_acc.
  Gyro and velocimeter are forward's.
- Inverse Jacobians DsDq / DsDv / DsDa: tests/inverse_fd_reference.py's columns of the sensordata above.
A ball model goes through the free-joint surrogate (tests/test_walk_on_ball.py).  Nothing here changes the oracle.
"""
import numpy as np

from oracle import fly_oracle as fo

import fd_reference as fr
import inverse_fd_reference as ifr
import inverse_reference as ir

TOUCH, ACCELEROMETER, VELOCIMETER, GYRO, FORCE = range(5)
CAPSULE = 3


def stage_rows(m):
    """(velocity-stage rows, accelerometer rows, force rows, touch rows) of the sensordata"""
    out = {t: [] for t in range(5)}
    for s in range(len(m.sensor_type)):
        a = int(m.sensor_adr[s])
        out[int(m.sensor_type[s])] += list(range(a, a + int(m.sensor_dim[s])))
    return (np.array(out[GYRO] + out[VELOCIMETER], int), np.array(out[ACCELEROMETER], int), np.array(out[FORCE], int),
            np.array(out[TOUCH], int))


def force_subtree_mass(m):
    """the largest mass of a force sensor's subtree"""
    parent, out = np.asarray(m.body_parentid, int), 0.0
    for s in range(len(m.sensor_type)):
        if int(m.sensor_type[s]) != FORCE:
            continue
        b = int(m.site_bodyid[int(m.sensor_objid[s])])
        tot = 0.0
        for c in range(1, m.nbody):
            k = c
            while k > 0 and k != b:
                k = parent[k]
            tot += float(m.body_mass[c]) if k == b else 0.0
        out = max(out, tot)
    return out


# ---- transition -------------------------------------------------------------------------------------------------------------------------
class Forward:
    """the oracle's sensordata of states x = (q, v, act, ctrl) of model m (a ball model through its free-joint surrogate)"""

    def __init__(self, m):
        self.st = fr.Stepper(m)
        self.m, self.o = m, self.st.o

    def __call__(self, x):
        q, v, a, u = x
        k = 3 if self.st.ball else 0
        self.o.reset(self.st.to_q(q), np.concatenate([np.zeros(k), v]))
        if self.m.na:
            self.o.set(fo.ACT, a)
        self.o.set(fo.CTRL, u)
        self.o.forward()
        return self.o.get(fo.SENSORDATA)


def transition_sensors_fd(m, qpos, qvel, act, ctrl, eps=1e-3, centered=True, run=None):
    """fp64 C [nsd, nx], D [nsd, nu] and the sensordata of the state"""
    x = tuple(np.asarray(y, np.float64) for y in (qpos, qvel, act if act is not None else np.zeros(m.na), ctrl))
    run = run or Forward(m)
    s0 = run(x)
    cols = []
    for j, (dp, dm) in enumerate(fr.steps(m, x, eps, centered)):
        if dp == dm:
            cols.append(np.zeros_like(s0))
            continue
        sb = run(fr._nudge(m, x, j, dp)) if dp else s0
        sa = run(fr._nudge(m, x, j, dm)) if dm else s0
        cols.append((sb - sa) / (dp - dm))
    cols = np.array(cols).T
    nx = 2 * m.nv + m.na
    return cols[:, :nx].copy(), cols[:, nx:].copy(), s0


# ---- inverse ----------------------------------------------------------------------------------------------------------------------------
def point_jacobian(m, xpos, xmat, b, p):
    """[3, nv] d(velocity of world point p fixed to body b) / d qvel"""
    J = np.zeros((3, m.nv))
    while b > 0:
        for k in range(int(m.body_dofadr[b]), int(m.body_dofadr[b]) + int(m.body_dofnum[b])):
            j = int(m.dof_jntid[k])
            t, c = int(m.jnt_type[j]), k - int(m.jnt_dofadr[j])
            R = xmat[b]
            anchor = xpos[b] + R @ m.jnt_pos[j]
            if t == fr.FREE and c < 3:
                J[c, k] = 1.0
                continue
            axis = R[:, c - 3] if t == fr.FREE else (R[:, c] if t == fr.BALL else R @ m.jnt_axis[j])
            J[:, k] = np.cross(axis, p - anchor)
        b = int(m.body_parentid[b])
    return J


def _ray_quad(a, b, c):
    det = b * b - a * c
    if det < 1e-30:
        return -1.0, (-1.0, -1.0)
    det = np.sqrt(det)
    x0, x1 = (-b - det) / a, (-b + det) / a
    return (x0 if x0 >= 0 else (x1 if x1 >= 0 else -1.0)), (x0, x1)


def _ray_capsule(pos, mat, size, pnt, vec):
    dif = pnt - pos
    ssz = size[0] + size[1]
    if _ray_quad(vec @ vec, vec @ dif, dif @ dif - ssz * ssz)[0] < 0:
        return -1.0
    lp, lv = mat.T @ dif, mat.T @ vec
    x = -1.0
    sol, _ = _ray_quad(lv[0] ** 2 + lv[1] ** 2, lv[0] * lp[0] + lv[1] * lp[1], lp[0] ** 2 + lp[1] ** 2 - size[0] ** 2)
    if sol >= 0 and abs(lp[2] + sol * lv[2]) <= size[1]:
        x = sol
    for sgn in (1, -1):
        ld = np.array([lp[0], lp[1], lp[2] - sgn * size[1]])
        _, xx = _ray_quad(lv @ lv, lv @ ld, ld @ ld - size[0] ** 2)
        for t in xx:
            if t >= 0 and sgn * (lp[2] + t * lv[2]) >= size[1] and (x < 0 or t < x):
                x = t
    return x


def inverse_sensors(m, o, qacc, efc_force=None):
    """the sensordata of mj_inverse at the oracle's current state (after forward()) and accelerations qacc [nv]; efc_force: the
    inverse's (default: tests/inverse_reference.py's at qacc)"""
    qacc = np.asarray(qacc, np.float64)
    f = ir.inverse(m, o, qacc)['efc_force'] if efc_force is None else np.asarray(efc_force, np.float64)
    s = o.get(fo.SENSORDATA)
    dqa = qacc - o.get(fo.QACC)
    f_fwd = o.get(fo.EFC_FORCE)
    xpos, xmat = o.get(fo.XPOS).reshape(-1, 3), o.get(fo.XMAT).reshape(-1, 3, 3)
    spos, smat = o.get(fo.SITE_XPOS).reshape(-1, 3), o.get(fo.SITE_XMAT).reshape(-1, 3, 3)
    ncon = int(o.get(fo.NCON)[0])
    con = o.get(fo.CONTACT).reshape(-1, 16)[:ncon] if ncon else np.zeros((0, 16))
    parent = np.asarray(m.body_parentid, int)

    def in_subtree(c, b):
        while c > 0 and c != b:
            c = parent[c]
        return c == b and b > 0

    def contact_force(row, forces):
        adr, dim = int(row[12]), int(row[9])
        n, t1 = row[4:7], row[13:16]
        frame = [n, t1, np.cross(n, t1)]
        return sum(frame[r] * forces[adr + r] for r in range(3 if dim >= 3 else 1))

    out = s.copy()
    for k in range(len(m.sensor_type)):
        tp, site, adr = int(m.sensor_type[k]), int(m.sensor_objid[k]), int(m.sensor_adr[k])
        b = int(m.site_bodyid[site])
        if tp == ACCELEROMETER:
            out[adr:adr + 3] = s[adr:adr + 3] + smat[site].T @ (point_jacobian(m, xpos, xmat, b, spos[site]) @ dqa)
        elif tp == FORCE:
            lin = np.zeros(3)
            for c in range(1, m.nbody):
                if in_subtree(c, b):
                    com = xpos[c] + xmat[c] @ m.body_ipos[c]
                    lin += m.body_mass[c] * (point_jacobian(m, xpos, xmat, c, com) @ dqa)
            for row in con:
                if row[12] < 0:
                    continue
                b1, b2 = int(m.geom_bodyid[int(row[7])]), int(m.geom_bodyid[int(row[8])])
                dF = contact_force(row, f) - contact_force(row, f_fwd)
                lin += (dF if in_subtree(b1, b) else 0) - (dF if in_subtree(b2, b) else 0)
            out[adr:adr + 3] = s[adr:adr + 3] + smat[site].T @ lin
        elif tp == TOUCH:
            total = 0.0
            for row in con:
                ea = int(row[12])
                if ea < 0:
                    continue
                b1, b2 = int(m.geom_bodyid[int(row[7])]), int(m.geom_bodyid[int(row[8])])
                if b not in (b1, b2) or f[ea] <= 0:
                    continue
                ray = row[4:7] / np.linalg.norm(row[4:7]) * (-1.0 if b == b2 else 1.0)
                size = np.asarray(m.site_size[site], np.float64)
                if int(m.site_type[site]) == CAPSULE:
                    hit = _ray_capsule(spos[site], smat[site], size, row[1:4], ray)
                else:
                    dif = row[1:4] - spos[site]
                    hit = _ray_quad(ray @ ray, ray @ dif, dif @ dif - size[0] ** 2)[0]
                if hit >= 0:
                    total += f[ea]
            out[adr] = total
    return out


class InverseSensors:
    """the reference of `inverse_dynamics.inverse(..., sensors=True)` of states of model m: (qpos, qvel, qacc) -> sensordata"""

    def __init__(self, m):
        self.inv = ifr.Inverse(m)
        self.m = m

    def __call__(self, q, v, a):
        inv = self.inv
        k = 3 if inv.ball else 0
        inv.o.reset(inv.to_q(q), np.concatenate([np.zeros(k), v]))
        inv.o.forward()
        return inverse_sensors(inv.mo, inv.o, np.concatenate([np.zeros(k), a]))


def inverse_sensors_fd(m, qpos, qvel, qacc, eps=1e-3, centered=True, run=None):
    """fp64 dict of DsDq, DsDv, DsDa [nv, nsd] (transposed: row i = d / d input i) and the nominal sensordata"""
    q, v, a = (np.asarray(x, np.float64) for x in (qpos, qvel, qacc))
    run = run or InverseSensors(m)
    s0 = run(q, v, a)
    nv = m.nv
    S = np.zeros((3 * nv, len(s0)))
    for j, (dp, dm) in enumerate(ifr.steps(m, q, v, a, eps, centered)):
        sb = run(*ifr.nudge(m, q, v, a, j, dp))
        sa = run(*ifr.nudge(m, q, v, a, j, dm)) if dm else s0
        S[j] = (sb - sa) / (dp - dm)
    return dict(DsDq=S[:nv], DsDv=S[nv:2 * nv], DsDa=S[2 * nv:], sensordata=s0)
