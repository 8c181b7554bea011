"""Batched finite-difference transition Jacobians on the device (MuJoCo `mjd_transitionFD`; dm_control `mjlib.mjd_transitionFD`).

`transition_fd` linearises the stepper around a batch of states: A = dx'/dx and B = dx'/du, with x = (dq, qvel, act) (dq: the tangent of
qpos, as MuJoCo's) and u = ctrl, for the transition of n_substeps substeps with ctrl held fixed -- n_substeps = 1 is mjd_transitionFD,
the task's substep count the transition a policy sees over one control step.  This is what LQR stabilisers, iLQR / MPC around a gait and
system identification are built on.

Every nudged copy of a state is one env of one batched step (`fb_fd_transition`): a centred Jacobian of the walking fly takes
1 + 2 (nx + nu) = 693 envs, so one handle runs several problems per launch.  There is no CPU fallback: without the CUDA library the call
raises `StepperError`.

Two deliberate differences from MuJoCo:
- the step is relative: coordinate j is nudged by eps max(1, |x_j|) (rotational tangent coordinates by eps), because the stepper is
  fp32 and the flight model's wings move at ~1e3 rad/s, where an absolute step would carry the rounding of the coordinate itself;
  MuJoCo's absolute step is the case |x_j| <= 1, and its usual eps of 1e-6 means nothing in fp32.  The default 1e-2 is where a sweep
  against the fp64 limit (DESIGN section 6) put the error lowest: on contact states it is lowest there, on constraint-free flight states
  within 3x of the lowest (3e-2);
- no heightfield program is set up, so the vision model is stepped without terrain contacts (as `inverse_dynamics.inverse` steps it).
Every column starts from a cold solver warm start: the states are written and `forward` run on a fresh handle.

`inverse_fd` differentiates the inverse dynamics (MuJoCo `mjd_inverseFD` with flg_actuation = 0; `fb_fd_inverse`): the Jacobians of
`inverse_dynamics.inverse`'s qfrc_inverse = M qacc + qfrc_bias - qfrc_passive - qfrc_constraint with respect to (dq, qvel, qacc), and of
the sparse inertia qM with respect to dq.  They are what Gauss-Newton needs to make a tracked trajectory dynamically consistent (drive the
root's "ghost force" to zero), and what direct trajectory optimisation and system identification from inverse dynamics use.  The
columns and the relative step are transition_fd's; the outputs are transposed as MuJoCo's (row i: the derivative with respect to input
i), the transpose of transition_fd's row-major A and B.  The vision model runs without terrain contacts here too.
"""
from collections import namedtuple

import numpy as np

from . import stepper as st

ENVS = 4096          # envs of the handle: max(1, ENVS // columns) problems per launch

Transition = namedtuple('Transition', ['A', 'B', 'qpos_next', 'qvel_next', 'act_next'])
InverseJacobians = namedtuple('InverseJacobians', ['DfDq', 'DfDv', 'DfDa', 'DmDq', 'qfrc_inverse'])
TransitionSensors = namedtuple('TransitionSensors', Transition._fields + ('C', 'D', 'sensordata'))
InverseSensorJacobians = namedtuple('InverseSensorJacobians', InverseJacobians._fields + ('DsDq', 'DsDv', 'DsDa', 'sensordata'))


def transition_fd(model, qpos, qvel, ctrl, act=None, eps=1e-2, centered=True, n_substeps=1, device=0, lib_path=None, sensors=False):
    """A = dx'/dx [B, nx, nx] and B = dx'/du [B, nx, nu] (row-major, as MuJoCo's) of B states qpos [B, nq], qvel [B, nv], ctrl [B, nu],
    act [B, na] (zeros when None), or of one state without the batch dimension; nx = 2 nv + na.

    Returns Transition(A, B, qpos_next, qvel_next, act_next) as fp64 arrays of the device's fp32 values; *_next is the unperturbed
    state after the n_substeps substeps.  sensors=True returns TransitionSensors, the same followed by MuJoCo's C = ds/dx [B, nsd, nx],
    D = ds/du [B, nsd, nu] and the nominal sensordata [B, nsd], s the sensors of x, the state before the step (columns in the model's
    sensor_adr order).  That holds for every n_substeps: C and D are not derivatives of the substep-mean sensors a policy observes."""
    m = model
    ncol = 1 + (2 if centered else 1) * (2 * m.nv + m.na + m.nu)
    per = max(1, ENVS // ncol)

    def run(sim, rows, k):
        q, v, u, a = rows
        pad = np.minimum(np.arange(sim.n_envs), k - 1)         # the chunk's states in envs 0 .. k-1, the last one repeated
        sim.reset(q[pad], v[pad])
        if m.na:
            sim.set(st.ACT, a[pad])
        sim.set_control(u[pad])
        sim.forward()
        sim.save_state(slots=np.arange(k), env_ids=np.arange(k))
        sim.fd_transition(np.arange(k), eps=eps, centered=centered, n_substeps=n_substeps)
        return sim.fd_read() + (sim.fd_sensor_read() if sensors else ())

    act = np.zeros(np.shape(qpos)[:-1] + (m.na,)) if act is None else act
    single, out = st._batched(m, [('qpos', qpos, (m.nq,)), ('qvel', qvel, (m.nv,)), ('ctrl', ctrl, (m.nu,)), ('act', act, (m.na,))], run,
                              per, n_envs=per * ncol, setup=lambda sim: _setup(sim, per, sensors), device=device, lib_path=lib_path)
    kind = TransitionSensors if sensors else Transition
    res = kind(*(x.astype(np.float64) for x in out))
    return kind(*(x[0] for x in res)) if single else res


def _setup(sim, slots, sensors):
    sim.state_bank(slots)
    if sensors:
        sim.query_sensors(True)


def inverse_fd(model, qpos, qvel, qacc, eps=1e-2, centered=True, device=0, lib_path=None, sensors=False):
    """The inverse-dynamics Jacobians of B states qpos [B, nq], qvel [B, nv], qacc [B, nv], or of one state without the batch dimension.

    Returns InverseJacobians(DfDq, DfDv, DfDa, DmDq, qfrc_inverse) as fp64 arrays of the device's fp32 values, transposed as MuJoCo's
    mjd_inverseFD: DfDq [B, nv, nv] with DfDq[p, i, j] = d qfrc_inverse_j / d dq_i (dq: the tangent of qpos), DfDv and DfDa likewise
    for qvel and qacc, DmDq [B, nv, nM] = d qM / d dq_i in MuJoCo's sparse qM order (the diagonal at dof_Madr, then the ancestors), and
    the unperturbed qfrc_inverse [B, nv].  centered=False is MuJoCo's forward difference.  sensors=True returns InverseSensorJacobians,
    the same followed by DsDq, DsDv, DsDa [B, nv, nsd] (transposed alike: DsDq[p, i, k] = d sensordata_k / d dq_i) of the sensordata
    `inverse_dynamics.inverse(..., sensors=True)` returns, and the nominal sensordata [B, nsd]."""
    m = model
    ncol = 1 + (2 if centered else 1) * 3 * m.nv
    per = max(1, ENVS // ncol)

    def run(sim, rows, k):
        sim.fd_inverse(*rows, eps=eps, centered=centered)
        return sim.fd_inverse_read() + (sim.fd_inverse_sensor_read() if sensors else ())

    single, out = st._batched(m, [('qpos', qpos, (m.nq,)), ('qvel', qvel, (m.nv,)), ('qacc', qacc, (m.nv,))], run, per, n_envs=per * ncol,
                              setup=(lambda sim: sim.query_sensors(True)) if sensors else None, device=device, lib_path=lib_path)
    kind = InverseSensorJacobians if sensors else InverseJacobians
    res = kind(*(x.astype(np.float64) for x in out))
    return kind(*(x[0] for x in res)) if single else res
