"""fp64 reference of the applied-force term (MuJoCo mj_xfrcAccumulate / mj_applyFT), restated in numpy for the tests at the oracle's state
(fp64 kinematics of the model compiler): the smooth force of a state with applied forces is the oracle's smooth force of that state plus
qfrc_applied + J^T xfrc_applied (both terms are linear and leave every other stage unchanged), and, in a state without constraint rows,
qacc = M^-1 qfrc_smooth (mj_forward), so the oracle's qacc plus M^-1 of the same term."""
import numpy as np

from oracle import fly_oracle as fo


def kinematics(m, o):
    """(xpos [nbody, 3], xmat [nbody, 3, 3], xipos [nbody, 3], dof axis [nv, 3], dof anchor [nv, 3], dof is a translation [nv]) in the world
    frame at the oracle's qpos, fp64, from the compiler's own forward kinematics (the joints of a body applied in order: a joint's axis
    is the frame before the body's later joints turn it, as mj_kinematics has it)"""
    from flybody_b200.compiler.compile_model import kinematics0
    from flybody_b200.compiler.quat import q2mat
    xpos, xquat, axis, anchor, trans = kinematics0(dict(m.a), o.get(fo.QPOS))
    xmat = np.stack([q2mat(x) for x in xquat])
    return xpos, xmat, xpos + np.einsum('bij,bj->bi', xmat, m.body_ipos), axis, anchor, trans


def frames(m, o):
    """(xpos, xmat, xipos) of kinematics()"""
    return kinematics(m, o)[:3]


def apply_ft(m, o, body, point, force, torque):
    """J^T [force at world `point`; torque] of `body`: the dofs of its ancestor chain, fp64 [nv]"""
    _, _, _, axis, anchor, trans = kinematics(m, o)
    out = np.zeros(m.nv)
    point, force, torque = (np.asarray(x, np.float64) for x in (point, force, torque))
    d = int(m.body_lastdof[body])
    while d >= 0:
        out[d] = force @ axis[d] if trans[d] else force @ np.cross(axis[d], point - anchor[d]) + torque @ axis[d]
        d = int(m.dof_parentid[d])
    return out


def applied_term(m, o, qfrc=None, xfrc=None):
    """qfrc_applied + J^T xfrc_applied at the oracle's current state, fp64 [nv]"""
    out = np.zeros(m.nv) if qfrc is None else np.asarray(qfrc, np.float64).copy()
    if xfrc is not None:
        _, _, xi = frames(m, o)
        w = np.asarray(xfrc, np.float64).reshape(m.nbody, 6)
        for b in range(1, m.nbody):
            if w[b].any():
                out += apply_ft(m, o, b, xi[b], w[b, :3], w[b, 3:])
    return out
