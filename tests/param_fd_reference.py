"""fp64 reference of the parameter Jacobians (fb_fd_param_*), for tests/test_param_fd.py.

A direction is (kind, [(parameter name, element)], floors), as flybody_b200.derivatives._directions gives it: an element direction has one, nudged by +-eps max(|theta|, floor) (the
non-negative fields skip a side that would go below 0, as the device does); a scale direction multiplies its entries by (1 +- eps).
Each side is a `FlyModel.copy()` with the raw fields replaced and the derived constants as compiled (test_model_params.patched, the
overlay's semantics), run through the oracle:
- transition: fd_reference.Stepper (n_substeps substeps, ctrl held), mj_differentiatePos for the dq rows; sensors of x through
  sensor_fd_reference.Forward;
- inverse: inverse_fd_reference.Inverse (qfrc_inverse) and sensor_fd_reference.InverseSensors.
Nothing here changes the oracle.
"""
import numpy as np

from flybody_b200 import stepper as st
from flybody_b200.derivatives import compiled_params
from flybody_b200.inverse_dynamics import _differentiate_pos

import fd_reference as fr
import inverse_fd_reference as ifr
import sensor_fd_reference as sr
from test_model_params import patched

NONNEG = {'body_mass', 'body_inertia', 'dof_armature', 'dof_damping', 'jnt_stiffness', 'geom_friction', 'density', 'viscosity'}


def _values(m, values):
    return {name: np.array(values[name], np.float64).reshape(-1) if values and name in values else compiled_params(m, name).copy()
            for name in st.PARAMS}


def sides(vals, direction, eps, centered):
    """-> (plus step, minus step) of a direction (kind, entries, floors) as derivatives._directions gives it"""
    kind, entries, floors = direction
    if kind == st.FD_SCALE:
        return eps, (-eps if centered else 0.0)
    (name, i), = entries
    x = vals[name][i]
    d = eps * max(abs(x), floors[0])
    nn = name in NONNEG
    fwd = not nn or x + d >= 0
    back = (centered or not fwd) and (not nn or x - d >= 0)
    if centered:
        return (d if fwd else 0.0), (-d if back else 0.0)
    return (d if fwd else (-d if back else 0.0)), 0.0


def moved(vals, direction, step):
    kind, entries, _ = direction
    out = {k: v.copy() for k, v in vals.items()}
    for name, i in entries:
        out[name][i] = out[name][i] * (1 + step) if kind == st.FD_SCALE else out[name][i] + step
    return out


def _columns(m, values, directions, eps, centered, run):
    """per direction (run(plus model) - run(minus model)) / (plus - minus) for a run returning a tuple of arrays; and the nominal"""
    vals = _values(m, values)
    nominal = run(patched(m, vals))
    cols = []
    for dr in directions:
        dp, dm = sides(vals, dr, eps, centered)
        b = run(patched(m, moved(vals, dr, dp))) if dp else nominal
        a = run(patched(m, moved(vals, dr, dm))) if dm else nominal
        cols.append((a, b, dp - dm))
    return nominal, cols


def transition(m, qpos, qvel, act, ctrl, directions, values=None, eps=1e-2, centered=True, n_substeps=1, sensors=False):
    """fp64 dxdp [nx, k], the nominal next state and, with sensors, dsdp [nsd, k] and the sensordata of x"""
    x = tuple(np.asarray(y, np.float64) for y in (qpos, qvel, act if act is not None else np.zeros(m.na), ctrl))

    def run(mp):
        nxt = fr.Stepper(mp)(x, n_substeps)
        return nxt + ((sr.Forward(mp)(x),) if sensors else ())
    nominal, cols = _columns(m, values, directions, eps, centered, run)
    dxdp, dsdp = [], []
    for a, b, den in cols:
        dq = _differentiate_pos(m, a[0][None], b[0][None], 1.0)[0]
        dxdp.append(np.concatenate([dq, b[1] - a[1], b[2] - a[2]]) / den)
        if sensors:
            dsdp.append((b[3] - a[3]) / den)
    out = dict(dxdp=np.array(dxdp).T, next=nominal[:3])
    if sensors:
        out.update(dsdp=np.array(dsdp).T.reshape(m.nsensordata, len(directions)), sensordata=nominal[3])
    return out


def inverse(m, qpos, qvel, qacc, directions, values=None, eps=1e-2, centered=True, sensors=False):
    """fp64 DfDp [k, nv], the nominal qfrc_inverse and, with sensors, DsDp [k, nsd] and the nominal sensordata"""
    q, v, a = (np.asarray(y, np.float64) for y in (qpos, qvel, qacc))

    def run(mp):
        f = ifr.Inverse(mp)(q, v, a)[0]
        return (f,) + ((sr.InverseSensors(mp)(q, v, a),) if sensors else ())
    nominal, cols = _columns(m, values, directions, eps, centered, run)
    out = dict(DfDp=np.array([(b[0] - a[0]) / den for a, b, den in cols]), qfrc_inverse=nominal[0])
    if sensors:
        out.update(DsDp=np.array([(b[1] - a[1]) / den for a, b, den in cols]).reshape(len(directions), m.nsensordata), sensordata=nominal[1])
    return out
