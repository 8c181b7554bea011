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

`parameter_fd` and `inverse_parameter_fd` differentiate the same two quantities with respect to the per-env model parameters
(`fb_fd_param_*`): dx'/dtheta and d qfrc_inverse / dtheta along element directions (one value of a field) or scale directions (`Scale`:
a set of values multiplied by one factor), at each problem's own parameter values.  They are the Jacobians system identification needs
to fit masses, damping, actuator gains or fluid coefficients to recorded motion or to inverse dynamics.
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
        _bank_rows(sim, m, rows, k)
        sim.fd_transition(np.arange(k), eps=eps, centered=centered, n_substeps=n_substeps)
        return sim.fd_read() + (sim.fd_sensor_read() if sensors else ())

    act = np.zeros(np.shape(qpos)[:-1] + (m.na,)) if act is None else act
    single, out = st._batched(m, [('qpos', qpos, (m.nq,)), ('qvel', qvel, (m.nv,)), ('ctrl', ctrl, (m.nu,)), ('act', act, (m.na,))], run,
                              per, n_envs=per * ncol, setup=lambda sim: _setup(sim, per, sensors), device=device, lib_path=lib_path)
    return _result(TransitionSensors if sensors else Transition, single, out)


def _setup(sim, slots, sensors):
    sim.state_bank(slots)
    if sensors:
        sim.query_sensors(True)


def _bank_rows(sim, model, rows, k, vals=()):
    """the chunk's k states (qpos, qvel, ctrl, act) into envs 0 .. k-1 (the last one repeated over the handle), each parameter of vals
    (name, rows or None: compiled) into those envs, forward, then bank rows 0 .. k-1"""
    q, v, u, a = rows[:4]
    pad = np.minimum(np.arange(sim.n_envs), k - 1)
    sim.reset(q[pad], v[pad])
    if model.na:
        sim.set(st.ACT, a[pad])
    sim.set_control(u[pad])
    _write_values(sim, model, vals, k)
    sim.forward()
    sim.save_state(slots=np.arange(k), env_ids=np.arange(k))


def _result(kind, single, out, labels=None):
    """the device's fp32 outputs as fp64 arrays in the namedtuple `kind` (one state: without the batch dimension); labels: its
    `columns`"""
    out = [x.astype(np.float64) for x in out]
    if single:
        out = [x[0] for x in out]
    if labels is not None:
        out.insert(kind._fields.index('columns'), list(labels))
    return kind(*out)


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
    return _result(InverseSensorJacobians if sensors else InverseJacobians, single, out)


# ---- parameter Jacobians (fb_fd_param_*): derivatives with respect to the per-env model parameters, for system identification --------
ParamTransition = namedtuple('ParamTransition', ['dxdp', 'qpos_next', 'qvel_next', 'act_next', 'columns'])
ParamTransitionSensors = namedtuple('ParamTransitionSensors', ParamTransition._fields + ('dsdp', 'sensordata'))
InverseParamJacobians = namedtuple('InverseParamJacobians', ['DfDp', 'qfrc_inverse', 'columns'])
InverseParamSensorJacobians = namedtuple('InverseParamSensorJacobians', InverseParamJacobians._fields + ('DsDp', 'sensordata'))

# the FlyModel array of each parameter (stepper.PARAMS)
_FIELD = {'body_mass': 'body_mass', 'body_inertia': 'body_inertia', 'dof_armature': 'dof_armature', 'dof_damping': 'dof_damping',
          'jnt_stiffness': 'jnt_stiffness', 'geom_friction': 'geom_friction', 'actuator_gainprm': 'actuator_gainprm',
          'actuator_biasprm': 'actuator_biasprm', 'gravity': 'opt_gravity', 'wind': 'opt_wind', 'density': 'opt_density',
          'viscosity': 'opt_viscosity'}
_HINGE = 3


class Scale:
    """a scale direction: every element of the named fields (jnt_stiffness: its hinge joints) multiplied by one factor s; idx picks a
    subset of a single field's elements.  Its column is d / ds at s = 1."""

    def __init__(self, *fields, idx=None):
        if not fields or any(f not in _FIELD for f in fields):
            raise ValueError(f'Scale takes parameter names ({", ".join(st.PARAMS)}), not {fields}')
        if idx is not None and len(fields) != 1:
            raise ValueError('an index subset needs a single field')
        self.fields, self.idx = tuple(fields), None if idx is None else [int(i) for i in np.reshape(idx, -1)]

    def __repr__(self):
        return f'Scale({", ".join(map(repr, self.fields))}{"" if self.idx is None else f", idx={self.idx}"})'


def compiled_params(model, name):
    """the compiled values of parameter `name` as the stepper counts its elements (fp64)"""
    return np.asarray(model.a[_FIELD[name]], np.float64).reshape(-1)


def _elements(model, name):
    n = len(compiled_params(model, name))
    if name == 'jnt_stiffness':
        return [j for j in range(n) if int(model.jnt_type[j]) == _HINGE]
    return list(range(n))


def _directions(model, params, floors):
    """params (see parameter_fd) -> (the program's directions for BatchedStepper.fd_param_program, one label each)"""
    floors = floors or {}

    def floor_of(name, i):
        if name in floors:
            return float(np.broadcast_to(np.asarray(floors[name], np.float64).reshape(-1), (len(compiled_params(model, name)),))[i])
        v = np.abs(compiled_params(model, name))
        return float(v[v > 0].mean()) if (v > 0).any() else 1.0

    dirs, labels = [], []
    for item in ([params] if isinstance(params, (str, Scale)) else params):
        if isinstance(item, Scale):
            entries = [(f, i) for f in item.fields for i in (_elements(model, f) if item.idx is None else item.idx)]
            dirs.append((st.FD_SCALE, entries, None))
            sub = '' if item.idx is None else f'[{",".join(map(str, item.idx))}]'
            labels.append(f'scale({",".join(item.fields)}{sub})')
            continue
        name, idx = (item, None) if isinstance(item, str) else (item[0], [int(i) for i in np.reshape(item[1], -1)])
        if name not in _FIELD:
            raise KeyError(f'{name!r} is not a per-env model parameter ({", ".join(st.PARAMS)})')
        for i in (_elements(model, name) if idx is None else idx):
            dirs.append((st.FD_ELEMENT, [(name, i)], [floor_of(name, i)]))
            labels.append(f'{name}[{i}]')
    if not dirs:
        raise ValueError('no parameter directions')
    return dirs, labels


def _value_inputs(model, values):
    """values {name: [B, size] or [size]} -> _batched inputs of per-problem rows (each parameter not given: its compiled values)"""
    values = values or {}
    unknown = set(values) - set(_FIELD)
    if unknown:
        raise KeyError(f'{sorted(unknown)} are not per-env model parameters ({", ".join(st.PARAMS)})')
    return [(name, values.get(name), len(compiled_params(model, name))) for name in st.PARAMS]


def _write_values(sim, model, vals, k):
    """each parameter's rows (None: compiled) into envs 0 .. k-1 (the handle's other envs are overwritten by the fan-out)"""
    for name, v in vals:
        sim.param_set(name, compiled_params(model, name) if v is None else v, env_ids=np.arange(k))


def _param_setup(sim, model, dirs, sensors, slots=None):
    sim.param_set('gravity', compiled_params(model, 'gravity'))        # the overlay (the rows carry it; allocating it drops the bank)
    if slots:
        sim.state_bank(slots)
    if sensors:
        sim.query_sensors(True)
    sim.fd_param_program(dirs)


def _batch_values(rows_first, val_inputs):
    """broadcast [size] values to the B problems of the first input"""
    B = np.asarray(rows_first).reshape(-1, np.shape(rows_first)[-1]).shape[0]
    return [(name, v, (k,)) for name, v, k in
            ((n, np.broadcast_to(np.asarray(v, np.float64).reshape(-1, k), (B, k)), k) for n, v, k in val_inputs if v is not None)]


def parameter_fd(model, qpos, qvel, ctrl, act=None, *, params, values=None, floors=None, eps=1e-2, centered=True, n_substeps=1,
                 sensors=False, device=0, lib_path=None):
    """dx'/dtheta [B, nx, k] of B states qpos [B, nq], qvel [B, nv], ctrl [B, nu], act [B, na] (zeros when None), or of one state
    without the batch dimension, along k parameter directions; x' as transition_fd's (n_substeps substeps, ctrl held).

    params: a list of
      'dof_damping'            one element direction per element (jnt_stiffness: per hinge joint);
      ('dof_damping', idx)     element directions for the listed elements;
      Scale('dof_damping') / Scale('body_mass', 'body_inertia') / Scale('dof_damping', idx=...)   one scale direction.
    An element direction is nudged by eps max(|theta_i|, floor_i), its column d / d theta_i in the parameter's units; floors {name:
    scalar or [size]} default to the mean |value| of the field's nonzero compiled elements (else 1).  A scale direction multiplies its
    elements by (1 +- eps) (eps < 1), its column d / ds at s = 1.  values {name: [B, size] or [size]}: each problem's parameters
    (default: compiled), the point the Jacobian is taken at.  Derived constants hold as compiled (no mj_setConst).

    Returns ParamTransition(dxdp, qpos_next, qvel_next, act_next, columns) as fp64 arrays of the device's fp32 values; columns: one
    label per direction.  sensors=True returns ParamTransitionSensors, adding dsdp [B, nsd, k] and the nominal sensordata [B, nsd] of
    the sensors of x, the state before the step (as transition_fd's C and D).  The default eps is where a sweep against the fp64 limit
    put the error lowest (DESIGN section 6)."""
    m = model
    dirs, labels = _directions(m, params, floors)
    ncol = 1 + (2 if centered else 1) * len(dirs)
    per = max(1, ENVS // ncol)
    vals = _value_inputs(m, values)
    given = _batch_values(qpos, vals)
    names = [n for n, _, _ in given]

    def run(sim, rows, k):
        chunk = dict(zip(names, rows[4:]))
        _bank_rows(sim, m, rows, k, [(n, chunk.get(n)) for n, _, _ in vals])
        sim.fd_param_transition(np.arange(k), eps=eps, centered=centered, n_substeps=n_substeps)
        return sim.fd_param_read() + (sim.fd_param_sensor_read() if sensors else ())

    act = np.zeros(np.shape(qpos)[:-1] + (m.na,)) if act is None else act
    single, out = st._batched(m, [('qpos', qpos, (m.nq,)), ('qvel', qvel, (m.nv,)), ('ctrl', ctrl, (m.nu,)), ('act', act, (m.na,))] + given,
                              run, per, n_envs=per * ncol, setup=lambda sim: _param_setup(sim, m, dirs, sensors, per), device=device,
                              lib_path=lib_path)
    return _result(ParamTransitionSensors if sensors else ParamTransition, single, out, labels)


def inverse_parameter_fd(model, qpos, qvel, qacc, *, params, values=None, floors=None, eps=1e-2, centered=True, sensors=False, device=0,
                         lib_path=None):
    """d qfrc_inverse / dtheta of B states qpos [B, nq], qvel [B, nv], qacc [B, nv] (or one state), along parameter directions; params,
    values, floors and eps as parameter_fd's.  qfrc_inverse is inverse_dynamics.inverse's (M qacc + qfrc_bias - qfrc_passive -
    qfrc_constraint, no actuation: actuator gain / bias columns are 0).

    Returns InverseParamJacobians(DfDp, qfrc_inverse, columns): DfDp [B, k, nv] transposed as inverse_fd's DfDq (DfDp[p, j, i] =
    d qfrc_inverse_i / d direction j), the nominal qfrc_inverse [B, nv] and one label per direction.  sensors=True returns
    InverseParamSensorJacobians, adding DsDp [B, k, nsd] of the inverse's sensordata and the nominal sensordata [B, nsd]."""
    m = model
    dirs, labels = _directions(m, params, floors)
    ncol = 1 + (2 if centered else 1) * len(dirs)
    per = max(1, ENVS // ncol)
    vals = _value_inputs(m, values)
    given = _batch_values(qpos, vals)
    names = [n for n, _, _ in given]

    def run(sim, rows, k):
        chunk = dict(zip(names, rows[3:]))
        _write_values(sim, m, [(n, chunk.get(n)) for n, _, _ in vals], k)      # problem i takes env i's parameters
        sim.fd_param_inverse(*rows[:3], eps=eps, centered=centered)
        return sim.fd_param_inverse_read() + (sim.fd_param_inverse_sensor_read() if sensors else ())

    single, out = st._batched(m, [('qpos', qpos, (m.nq,)), ('qvel', qvel, (m.nv,)), ('qacc', qacc, (m.nv,))] + given, run, per,
                              n_envs=per * ncol, setup=lambda sim: _param_setup(sim, m, dirs, sensors), device=device, lib_path=lib_path)
    return _result(InverseParamSensorJacobians if sensors else InverseParamJacobians, single, out, labels)
