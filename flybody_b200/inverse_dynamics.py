"""Batched inverse dynamics on the device (MuJoCo `mj_inverse`, continuous time), and the finite differences that feed it.

The second half of the tracking pipeline: tracked keypoints -> `inverse_kinematics.qpos_from_site_xpos` -> joint angles ->
`differentiate` -> qvel, qacc -> `inverse` -> joint torques and ground-contact forces -> `joint_forces`.  With dm_control this is
`mjlib.mj_inverse(physics.model.ptr, physics.data.ptr)` followed by `physics.data.qfrc_inverse` and `efc_force`.

`inverse` runs one problem per env, one warp each, on the CUDA stepper (`fb_inverse`), in chunks of 4096 problems.  There is no CPU
fallback: without the CUDA library the call raises `StepperError`.  What it returns excludes applied and actuator forces:
qfrc_inverse = M qacc + qfrc_bias - qfrc_passive - qfrc_constraint, so for the qacc a forward pass produced it equals
qfrc_applied + J^T xfrc_applied + qfrc_actuator.  Noslip is not inverted: the contact forces are the soft constraint model's.
"""
from collections import namedtuple

import numpy as np

from . import stepper as st
from .inverse_kinematics import CHUNK, HINGE, _differentiate_pos

InverseResult = namedtuple('InverseResult', ['qfrc_inverse', 'qfrc_constraint', 'qfrc_bias', 'qfrc_passive', 'contacts'])
InverseSensorResult = namedtuple('InverseSensorResult', InverseResult._fields + ('sensordata',))
# per problem: the contacts that have constraint rows; force holds mj_contactForce's six numbers for an elliptic cone (contact frame:
# normal, then the two tangent directions, then torques, which the fly's condim <= 3 contacts leave at 0)
Contacts = namedtuple('Contacts', ['geom', 'pos', 'normal', 'force'])


def inverse(model, qpos, qvel, qacc, device=0, lib_path=None, sensors=False):
    """mj_inverse of B states: qpos [B, nq], qvel [B, nv], qacc [B, nv] (or one state without the batch dimension).

    Returns InverseResult(qfrc_inverse, qfrc_constraint, qfrc_bias, qfrc_passive, contacts): four [B, nv] fp64 arrays of the device's
    fp32 values, and per problem a `Contacts` of its k contacts with rows: geom [k, 2] geom ids, pos [k, 3] world position, normal
    [k, 3], force [k, 6] in the contact frame.  sensors=True returns InverseSensorResult, the same followed by sensordata [B, nsd]
    (columns in the model's sensor_adr order), evaluated as mj_inverse does: gyro and velocimeter of the state, accelerometer, force
    and touch at the given qacc and the inverse's contact forces (xfrc_applied does not enter the force sensors, as in the step)."""
    def run(sim, rows, n):
        q, v, a = rows
        pad = np.minimum(np.arange(sim.n_envs), n - 1)         # the chunk's states, the last one repeated
        sim.set(st.QPOS, q[pad])
        sim.set(st.QVEL, v[pad])
        sim.inverse(a)
        qi, qc, f = sim.inverse_read()
        sd = (sim.inverse_sensor_read(),) if sensors else ()
        con, ncon = sim.get(st.CONTACT).reshape(sim.n_envs, st.MAXCON, 16), sim.get(st.NCON)[:, 0].astype(int)
        contacts = []
        for i in range(n):
            c = con[i, :ncon[i]]
            c = c[c[:, 12] >= 0]
            force = np.zeros((len(c), 6))
            for k, row in enumerate(c):
                adr, dim = int(row[12]), int(row[9])
                force[k, :dim] = f[i, adr:adr + dim]
            contacts.append(Contacts(c[:, 7:9].astype(np.int64), c[:, 1:4].astype(np.float64), c[:, 4:7].astype(np.float64), force))
        return (qi, qc, sim.get(st.QFRC_BIAS)[:n], sim.get(st.QFRC_PASSIVE)[:n], contacts) + sd

    single, out = st._batched(model, [('qpos', qpos, (model.nq,)), ('qvel', qvel, (model.nv,)), ('qacc', qacc, (model.nv,))], run, CHUNK,
                              setup=(lambda sim: sim.query_sensors(True)) if sensors else None, device=device, lib_path=lib_path)
    kind = InverseSensorResult if sensors else InverseResult
    res = kind(*(x.astype(np.float64) for x in out[:4]), out[4], *(x.astype(np.float64) for x in out[5:]))
    return kind(*(x[0] for x in res)) if single else res


def differentiate(model, qpos_track, dt):
    """(qvel, qacc) [T - 2, nv] of frames 1 .. T-2 of a pose track [T, nq] sampled every dt seconds, fp64 central differences:
    qvel_t = differentiatePos(q_{t-1}, q_{t+1}) / 2 dt,  qacc_t = (differentiatePos(q_t, q_{t+1}) - differentiatePos(q_{t-1}, q_t)) / dt^2
    (mj_differentiatePos per joint).  Both are second-order accurate in dt for smooth motion."""
    q = np.asarray(qpos_track, np.float64)
    if q.ndim != 2 or q.shape[0] < 3 or q.shape[1] != model.nq:
        raise ValueError(f'a track [T >= 3, {model.nq}] is needed, got {q.shape}')
    qvel = _differentiate_pos(model, q[:-2], q[2:], 2 * dt)
    fwd = _differentiate_pos(model, q[:-1], q[1:], dt)
    return qvel, (fwd[1:] - fwd[:-1]) / dt


def joint_forces(model, qfrc, joint_names):
    """the generalized forces of hinge joints by name: qfrc [..., nv] -> [..., len(joint_names)]"""
    ids = [model.jnt_id(j) for j in joint_names]
    bad = [n for n, j in zip(joint_names, ids) if int(model.jnt_type[j]) != HINGE]
    if bad:
        raise ValueError(f'not hinge joints: {bad}')
    return np.asarray(qfrc)[..., model.jnt_dofadr[ids]]
