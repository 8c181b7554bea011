"""Batched rollouts on the device (MuJoCo `mujoco.rollout.rollout`).

`rollout` steps B initial states through a control sequence each and returns the trajectories: the primitive that MPPI / CEM sampling,
iLQR forward passes, TVLQR tracking and system identification all loop over.  Every control step of every rollout runs on the device
(`fb_rollout`): an input kernel writes the step's ctrl (and applied forces), the step graph advances n_substeps substeps, a record kernel
stores the state, so a horizon has no host round trip.  There is no CPU fallback: without the CUDA library the call raises
`StepperError`.

Optional linear feedback: with x_ref [T, nq + nv + na] and K [T, nu, nx] (nx = 2 nv + na), step t applies
ctrl_t + K_t (x_t - x_ref_t), the difference in the tangent space of `derivatives.transition_fd` (mj_differentiatePos for qpos), so
gains from a Riccati recursion on its A and B apply as they are.  x_ref and K are shared by all rollouts, or x_ref [L, T, .] and
K [L, T, nu, nx] are a bank of L laws and law [B] says which one each rollout applies (`trajopt.ilqr`'s line search: one law per
problem, many rollouts per law).

As in `derivatives`, every rollout starts from a cold solver warm start (the state is written and `forward` run with the first control),
and no heightfield program is set up, so the vision model runs without terrain contacts.
"""
from collections import namedtuple

import numpy as np

from . import stepper as st
from .derivatives import _batch_values, _value_inputs, _write_values, compiled_params

ENVS = 4096          # envs of a handle: rollouts beyond it run in chunks

Rollout = namedtuple('Rollout', ['qpos', 'qvel', 'act', 'ctrl', 'time', 'flags'])
RolloutSensors = namedtuple('RolloutSensors', Rollout._fields + ('sensordata', 'sensor_mean'))


def rollout(model, qpos, qvel, ctrl, act=None, n_substeps=1, qfrc_applied=None, xfrc_applied=None, params=None, x_ref=None, K=None,
            law=None, sensors=False, device=0, lib_path=None):
    """Roll B initial states qpos [B, nq], qvel [B, nv], act [B, na] (zeros when None) through ctrl [B, T, nu], or one state
    without the batch dimension (ctrl [T, nu]); each control step is n_substeps substeps with ctrl held.

    qfrc_applied [B, T, nv] / xfrc_applied [B, T, nbody, 6]: applied forces written at each control step (world-frame force, then
    torque, at each body's CoM); without them the rollouts run without applied forces.  params {name: [B, size] or [size]}: per-rollout
    values of the per-env model parameters (`stepper.PARAMS`; MuJoCo rollout's one model per rollout), the others as compiled.
    x_ref [T, nq + nv + na] and K [T, nu, 2 nv + na]: the feedback law above (both or neither); or a bank x_ref [L, T, nq + nv + na],
    K [L, T, nu, 2 nv + na] with law [B] (ints in [0, L); default arange(B) when L == B): rollout b applies law law[b].

    Returns Rollout(qpos [B, T, nq], qvel [B, T, nv], act [B, T, na], ctrl [B, T, nu], time [B, T], flags [B, T]): row t is the state
    after control step t and the ctrl it applied, fp64 arrays of the device's fp32 values (flags: the env's int32 flag word).
    sensors=True returns RolloutSensors, adding sensordata and sensor_mean [B, T, nsd] after each step (the substep mean a policy
    observes)."""
    m = model
    if (x_ref is None) != (K is None):
        raise ValueError('feedback needs both x_ref and K')
    T = np.shape(ctrl)[-2]
    bank = x_ref is not None and np.ndim(x_ref) == 3
    if law is not None and not bank:
        raise ValueError('law picks laws of a bank: x_ref [L, T, nq + nv + na] and K [L, T, nu, nx]')
    if x_ref is not None:
        x_ref, K = np.asarray(x_ref, np.float64), np.asarray(K, np.float64)
        lead = x_ref.shape[:1] if bank else ()
        want = (lead + (T, m.nq + m.nv + m.na), lead + (T, m.nu, 2 * m.nv + m.na))
        if x_ref.shape != want[0] or K.shape != want[1]:
            raise ValueError(f'x_ref {x_ref.shape} and K {K.shape} against {want[0]} and {want[1]} (the horizon of ctrl)')
    laws = []
    if bank:
        n_laws, n_roll = x_ref.shape[0], np.reshape(qpos, (-1, m.nq)).shape[0]
        if law is None and n_laws != n_roll:
            raise ValueError(f'a bank of {n_laws} laws for {n_roll} rollouts needs law')
        law = np.arange(n_roll) if law is None else np.asarray(law)
        if not np.issubdtype(law.dtype, np.integer) or law.size != n_roll or (law < 0).any() or (law >= n_laws).any():
            raise ValueError(f'law: {n_roll} ints in [0, {n_laws})')
        laws = [('law', law.reshape(np.shape(qpos)[:-1]), ())]
    vals = _value_inputs(m, params)
    given = _batch_values(qpos, vals)
    names = [n for n, _, _ in given]
    applied = [(name, x, shape) for name, x, shape in (('qfrc_applied', qfrc_applied, (T, m.nv)), ('xfrc_applied', xfrc_applied,
                                                                                                   (T, m.nbody, 6))) if x is not None]

    def setup(sim):
        if given:
            sim.param_set('gravity', compiled_params(m, 'gravity'))     # the overlay before the bank (the rows carry it)
        if applied:
            sim.applied_ptrs()                                           # the applied-force arrays before the bank (the rows carry them)
        sim.state_bank(sim.n_envs)
        if sensors:
            sim.query_sensors(True)
        if x_ref is not None and not bank:
            sim.rollout_feedback(x_ref, K)

    def run(sim, rows, k):
        q, v, u, a = rows[:4]
        ins = dict(zip([n for n, _, _ in applied] + names, rows[4:]))
        pad = np.minimum(np.arange(sim.n_envs), k - 1)
        sim.reset(q[pad], v[pad])
        if m.na:
            sim.set(st.ACT, a[pad])
        sim.set_control(u[pad, 0])
        if given:
            _write_values(sim, m, [(n, ins.get(n)) for n, _, _ in vals], k)
        sim.forward()
        sim.save_state(slots=np.arange(k), env_ids=np.arange(k))
        if bank:
            sim.rollout_feedback_bank(x_ref, K, rows[-1].astype(np.int32))
        sim.rollout(np.arange(k), u, n_substeps, ins.get('qfrc_applied'), ins.get('xfrc_applied'))
        return sim.rollout_read() + (sim.rollout_sensor_read() if sensors else ())

    act = np.zeros(np.shape(qpos)[:-1] + (m.na,)) if act is None else act
    single, out = st._batched(m, [('qpos', qpos, (m.nq,)), ('qvel', qvel, (m.nv,)), ('ctrl', ctrl, (T, m.nu)), ('act', act, (m.na,))]
                              + applied + given + laws, run, ENVS, setup=setup, device=device, lib_path=lib_path)
    out = [x if x.dtype == np.int32 else x.astype(np.float64) for x in out]
    kind = RolloutSensors if sensors else Rollout
    return kind(*(x[0] for x in out)) if single else kind(*out)
