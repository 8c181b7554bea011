"""Smooth-dynamics states for tests/test_smooth_gates.py: the constraint-free model copy, the pinned table of states that reach the
edges of the smooth half of the step, and the per-element fp64 gates.

The fly's inertia spans six decades (walk: qM's diagonal runs from 1e-6 to 1), so a field-max gate such as
tests/parity_common.compare_stage_fields' cannot see an error in most of its entries.  The gates here are per element and scale-aware:
qM per entry in the metric of its own diagonal, generalised forces per dof in the inertia metric, positions relative to the body's
distance from the root, sensors per sensor.  `free_model` drops every collision pair and joint limit, so nefc = 0 on both sides and
qacc = M^-1 qfrc_smooth, one substep's qvel change = h (M + hD)^-1 qfrc_smooth: the two factorisations and their triangular sweeps are
compared on their own, without the constraint solve in between.
"""
import os

import numpy as np
import pytest

from flybody_b200 import stepper as st
from flybody_b200.flymodel import load_model, model_for
from oracle import fly_oracle as fo
from oracle import variants as ov
from parity_common import SENSOR_FLOOR, random_act, reset_qpos

FREE, BALL, HINGE = 0, 1, 3
DEFAULT_MODELS = ['walk', 'flight', 'vision', 'ball']
MODELS = DEFAULT_MODELS + list(ov.VARIANTS)
WING_NAMES = [f'walker/wing_{a}_{s}' for s in ('left', 'right') for a in ('yaw', 'roll', 'pitch')]
TERMINAL_LINVEL, TERMINAL_ANGVEL = 50.0, 200.0      # the flight task's termination limits (cm/s, rad/s), flybody_b200/synthetic.py
POS_FLOOR = 1e-2                    # cm: distance floor of the position gates (the root body itself)
U32 = 2.0 ** -24                    # fp32 unit roundoff
NEAR = 10.0                         # cm: world points closer than this to the origin are gated relative to their distance from the root
BACK_FLOOR = 1e-3                   # floor of the backward-error denominators, relative to their largest entry in the inertia metric


def base_model(name):
    """a shipped model ('walk', 'flight', 'vision', 'ball') or a FruitFly variant of oracle/variants.py (skips where it is not built)"""
    if name in DEFAULT_MODELS:
        return load_model(name)
    p = ov.variant_path(name)
    if not os.path.exists(p):
        pytest.skip(f'{p} is missing: build() compiles it where the reference fruitfly.xml is reachable (oracle/variants.py)')
    task, kw = ov.VARIANTS[name]
    return model_for(task, cache_dir=ov.VARIANT_DIR, **kw)


def free_model(m, fluid=True, springs=True):
    """copy of `m` without collision pairs and joint limits (nefc = 0 in every state); fluid=False also turns the medium off
    (opt_density = opt_viscosity = 0), springs=False the joint springs and dampers: with both edits on both sides, qfrc_passive with
    the medium on minus the same with it off is the fluid part alone, and without springs and dampers it is not the difference of
    two larger forces (a wing's damper at wing-beat speed is larger than its drag)"""
    a = m.copy()
    if not springs:
        a.a['jnt_stiffness'] = np.zeros_like(a.jnt_stiffness)
        a.a['dof_damping'] = np.zeros_like(a.dof_damping)
    a.a['pair_geom1'] = np.zeros(0, np.int32)
    a.a['pair_geom2'] = np.zeros(0, np.int32)
    a.a['npair'] = a.meta['npair'] = 0
    a.a['jnt_limited'] = np.zeros_like(a.jnt_limited)
    if not fluid:
        for k in ('opt_density', 'opt_viscosity'):
            a.a[k] = a.meta[k] = 0.0
    return a.rebuild()


def wing_beat(row):
    """(wing angles [6], wing speeds [6]) at control row `row` of the flight task's base-frequency wing-beat table: the angles of the
    table and their central difference at 218 Hz (the table is sampled every control step, 2e-4 s)"""
    from flybody_b200.fly_envs import BatchedWingBeatPatternGenerator
    wb = BatchedWingBeatPatternGenerator(1)
    k = int(np.abs(wb.beat_freqs - wb.base_beat_freq).argmin())
    tab = wb.traj[k, :wb.lengths[k]]
    n = len(tab)
    return tab[row % n], (tab[(row + 1) % n] - tab[(row - 1) % n]) / (2 * wb._dt)


def _uniform_quat(rs):
    q = rs.normal(size=4)
    return q / np.linalg.norm(q)


def _joints(m, kind):
    return [j for j in range(m.njnt) if m.jnt_type[j] == kind]


# name -> (seed, recipe).  Recipe keys: quat ('random' | 'w0' | state name to copy and scale), qscale (factor on the copied quaternion,
# negative: -q), far ((x, y) cm added to the root), wings (wing-beat table row: wings at real flight angles and speeds), body (root
# moves at the termination limits), still ('joints': no joint velocity but the wings'; 'all': none but the root's), needs (free root /
# wing joints).  Every state has hinges uniform over their full range and a random activation.
STATES = {
    'quat_a':      (1, dict(quat='random')),
    'quat_b':      (2, dict(quat='random')),
    'quat_w0':     (3, dict(quat='w0')),
    'quat_neg':    (1, dict(quat='quat_a', qscale=-1.0)),
    'quat_half':   (1, dict(quat='quat_a', qscale=0.5)),
    'quat_double': (1, dict(quat='quat_a', qscale=2.0)),
    'far_1e2':     (1, dict(quat='quat_a', far=(173.25, -121.5), needs='free')),
    'far_1e3':     (1, dict(quat='quat_a', far=(-871.5, 642.75), needs='free')),
    'wings_only':  (4, dict(quat='random', wings=9, still='joints', needs='wings')),
    'body_only':   (5, dict(quat='random', body=True, still='all', needs='free')),
    'flight':      (6, dict(quat='random', wings=3, body=True, needs=('wings', 'free'))),
}
FLUID_STATES = ('wings_only', 'body_only')


def applies(m, name):
    need = STATES[name][1].get('needs', ())
    need = (need,) if isinstance(need, str) else need
    return ('free' not in need or bool(_joints(m, FREE))) and ('wings' not in need or all(n in m.meta['jnt_names'] for n in WING_NAMES))


def state_names(m):
    return [k for k in STATES if applies(m, k)]


def _quat_of(m, name, rs, k):
    recipe = STATES[name][1]
    if recipe['quat'] == 'random':
        return _uniform_quat(rs)
    if recipe['quat'] == 'w0':                       # a 180-degree turn about a random axis
        ax = rs.normal(size=3)
        return np.concatenate([[1e-4], ax / np.linalg.norm(ax) * np.sqrt(1 - 1e-8)])
    src = recipe['quat']
    q = _quat_of(m, src, np.random.RandomState(STATES[src][0] * 1000 + 7 + 31 * k), k)
    return q * recipe.get('qscale', 1.0)


def state_inputs(m, name):
    """qpos, qvel, act, ctrl of pinned state `name` on `m`, rounded to fp32 so that both sides start from the same numbers"""
    seed, recipe = STATES[name]
    rs = np.random.RandomState(seed)
    q = reset_qpos(m)
    v = np.zeros(m.nv)
    for j in _joints(m, HINGE):                    # hinges across their whole range (unlimited ones: a full turn)
        lo, hi = m.jnt_range[j] if m.jnt_range[j][1] > m.jnt_range[j][0] else (-np.pi, np.pi)
        q[m.jnt_qposadr[j]] = rs.uniform(lo, hi)
        v[m.jnt_dofadr[j]] = rs.uniform(-2.0, 2.0)
    rot = _joints(m, FREE)[:1] + _joints(m, BALL)  # the walker's root (not the ghost) and every ball joint
    for k, j in enumerate(rot):
        qa, da = m.jnt_qposadr[j], m.jnt_dofadr[j]
        off = 3 if m.jnt_type[j] == FREE else 0
        # the orientation is drawn from its own stream: states that copy another's quaternion get exactly that quaternion
        q[qa + off:qa + off + 4] = _quat_of(m, name, np.random.RandomState(seed * 1000 + 7 + 31 * k), k)
        v[da:da + off + 3] = rs.uniform(-1.0, 1.0, off + 3)
    if 'far' in recipe:
        # the whole scene moves: the ghost (the second free joint of walk and flight) tracks the walker in the tasks, and the kernels
        # take one reference point for all trees, the walker's root (kpos_p0)
        for j in _joints(m, FREE):
            q[m.jnt_qposadr[j]:m.jnt_qposadr[j] + 2] += recipe['far']
    wing_q = [m.jnt_qposadr_of(n) for n in WING_NAMES] if applies(m, 'wings_only') else []
    wing_v = [m.jnt_dofadr_of(n) for n in WING_NAMES] if wing_q else []
    still = recipe.get('still')
    if still == 'joints':
        v[:] = 0.0
    elif still == 'all':
        keep = np.zeros(m.nv, bool)
        for j in _joints(m, FREE)[:1]:
            keep[m.jnt_dofadr[j]:m.jnt_dofadr[j] + 6] = True
        v[~keep] = 0.0
    if 'wings' in recipe and wing_q:
        wq, wv = wing_beat(recipe['wings'])
        q[wing_q], v[wing_v] = wq, wv
    if recipe.get('body'):
        j = _joints(m, FREE)[0]
        da = m.jnt_dofadr[j]
        lin, ang = rs.normal(size=3), rs.normal(size=3)
        v[da:da + 3] = lin / np.linalg.norm(lin) * TERMINAL_LINVEL
        v[da + 3:da + 6] = ang / np.linalg.norm(ang) * TERMINAL_ANGVEL
    act = random_act(m, seed)
    ctrl = np.random.RandomState(seed + 100).uniform(-0.5, 0.5, m.nu)
    return tuple(np.asarray(x, np.float64).astype(np.float32).astype(np.float64) for x in (q, v, act, ctrl))


def describe(m, name):
    """the edge a state reaches, from its inputs alone"""
    q, v, act, _ = state_inputs(m, name)
    out = {}
    rot = _joints(m, FREE)[:1] + _joints(m, BALL)
    if rot:
        j = rot[0]
        off = 3 if m.jnt_type[j] == FREE else 0
        qa = m.jnt_qposadr[j] + off
        quat = q[qa:qa + 4]
        out.update(quat_norm=float(np.linalg.norm(quat)), quat_w=float(quat[0] / np.linalg.norm(quat)))
        if m.jnt_type[j] == FREE:
            out['root_xy'] = float(np.abs(q[m.jnt_qposadr[j]:m.jnt_qposadr[j] + 2]).max())
            da = m.jnt_dofadr[j]
            out.update(linvel=float(np.linalg.norm(v[da:da + 3])), angvel=float(np.linalg.norm(v[da + 3:da + 6])))
    hinge = _joints(m, HINGE)
    lim = [j for j in hinge if m.jnt_range[j][1] > m.jnt_range[j][0]]
    if lim:     # the largest fraction of its half-range a limited hinge reaches from the range's centre
        c = m.jnt_range[lim].mean(1)
        h = 0.5 * (m.jnt_range[lim][:, 1] - m.jnt_range[lim][:, 0])
        out['range_reach'] = float(np.max(np.abs(q[m.jnt_qposadr[lim]] - c) / h))
    if applies(m, 'wings_only'):
        out['wing_speed'] = float(np.abs(v[[m.jnt_dofadr_of(n) for n in WING_NAMES]]).max())
    hv = v[[m.jnt_dofadr[j] for j in hinge]]
    out['hinge_speed'] = float(np.abs(hv).max()) if len(hv) else 0.0
    out['min_act'] = float(np.abs(act).min()) if m.na else 1.0
    return out


# ----------------------------------------------------------------------------------------------------------------- both sides

FIELDS = (('xpos', fo.XPOS), ('xmat', fo.XMAT), ('site_xpos', fo.SITE_XPOS), ('site_xmat', fo.SITE_XMAT),
          ('subtree_com', fo.SUBTREE_COM), ('qM', fo.QM_DENSE), ('qfrc_bias', fo.QFRC_BIAS), ('qfrc_passive', fo.QFRC_PASSIVE),
          ('qfrc_actuator', fo.QFRC_ACTUATOR), ('qfrc_smooth', fo.QFRC_SMOOTH), ('qacc', fo.QACC), ('sensordata', fo.SENSORDATA))


def oracle_fields(m, name, step=True):
    """the oracle's fields of one state after forward(); step=True also takes one substep and adds its qvel change as 'dqvel'.  The
    oracle has no ball joint: a model with one is stepped as tests/test_walk_on_ball.py's surrogate (the ball's joint a free joint whose
    translation carries a huge armature, so that it decouples), and its leading three dofs are dropped again."""
    q, v, act, ctrl = state_inputs(m, name)
    ball = bool(_joints(m, BALL))
    o = fo.Oracle(m, tolerance=1e-12)
    if ball:
        from test_walk_on_ball import free_surrogate, to_surrogate_q
        o = fo.Oracle(free_surrogate(m), tolerance=1e-12)
        o.reset(to_surrogate_q(m, q), np.concatenate([np.zeros(3), v]))
    else:
        o.reset(q, v)
    if m.na:
        o.set(fo.ACT, act)
    o.set(fo.CTRL, ctrl)
    o.forward()
    out = {k: o.get(f) for k, f in FIELDS}
    out['nefc'] = int(o.get(fo.NEFC)[0])
    if ball:
        n = m.nv + 3
        out['qM'] = out['qM'].reshape(n, n)[3:, 3:].ravel()
        for k in ('qfrc_bias', 'qfrc_passive', 'qfrc_actuator', 'qfrc_smooth', 'qacc'):
            out[k] = out[k][3:]
    if step:
        o.step()
        out['qvel1'] = o.qvel[3:] if ball else o.qvel
        out['dqvel'] = out['qvel1'] - v
    return out


def device_fields(m, sim, names, assign, step=True):
    """reset env i of `sim` to state names[assign[i]], one forward (and one substep): per env, the same fields as oracle_fields"""
    inputs = [state_inputs(m, k) for k in names]
    q, v, act, ctrl = (np.array([inputs[a][c] for a in assign]) for c in range(4))
    sim.reset(q, v)
    if m.na:
        sim.set(st.ACT, act)
    sim.set_control(ctrl)
    sim.forward()
    got = {k: np.asarray(sim.get(f), np.float64) for k, f in FIELDS}
    nefc, flags = sim.get(st.NEFC)[:, 0], sim.get(st.FLAGS)[:, 0]
    if step:
        sim.step(1)
        qvel1 = np.asarray(sim.get(st.QVEL), np.float64)
    out = []
    for i in range(sim.n_envs):
        d = {k: got[k][i] for k, _ in FIELDS}
        d.update(nefc=int(nefc[i]), flags=int(flags[i]))
        if step:
            d['dqvel'] = qvel1[i] - v[i]
            d['qvel1'] = qvel1[i]
        out.append(d)
    return out


# ----------------------------------------------------------------------------------------------------------------- the gates

def _metric(M):
    return np.sqrt(np.maximum(np.diag(M), 1e-300))


def qm_entry_error(M_dev, M_ora):
    """max over entries |dM_ij| / sqrt(M_ii M_jj)"""
    s = _metric(M_ora)
    return float((np.abs(M_dev - M_ora) / np.outer(s, s)).max())


def force_error(f_dev, f_ora, M_ora):
    """per dof in the inertia metric: max_i |df_i| / sqrt(M_ii) relative to max_j |f_j| / sqrt(M_jj)"""
    s = _metric(M_ora)
    scale = float((np.abs(f_ora) / s).max())
    if scale == 0.0:
        return 0.0
    return float((np.abs(f_dev - f_ora) / s).max() / scale)


def solve_errors(A, x_dev, x_ora, b, x_res=None):
    """(backward, forward) error of the device's solution of A x = b.  Backward: max_i |(A x_dev - b)_i| / (|A| |x_dev| + |b|)_i, the
    denominator floored at BACK_FLOOR of its largest entry in the inertia metric (a dof whose terms all vanish, such as the force-free
    ghost's, is then measured on the scale of the others).  Forward: max_i |dx_i| sqrt(A_ii) relative to max_j |x_j| sqrt(A_jj).
    x_res: per-entry resolution of the device's x (the fp32 rounding of the quantity x was read from), added to |x_dev| in the
    backward denominator and taken off |dx| in the forward error"""
    absA = np.abs(A)
    xr = np.zeros_like(x_dev) if x_res is None else x_res
    s = _metric(A)
    den = absA @ (np.abs(x_dev) + xr) + np.abs(b)
    den = den + BACK_FLOOR * s * (den / s).max()
    back = float((np.abs(A @ x_dev - b) / (den + 1e-300)).max())
    fwd = float((np.maximum(np.abs(x_dev - x_ora) - xr, 0.0) * s).max() / ((np.abs(x_ora) * s).max() + 1e-300))
    return back, fwd


def position_error(x_dev, x_ora, x_root):
    """(relative, ulps) of a set of world points.  relative: max |dx| / (|x - x_root| + POS_FLOOR), the error relative to the point's
    distance from the root, over the points the device's fp32 world coordinates can resolve to that level (|x| < NEAR cm: the kernels
    work relative to the root, but fb_get adds the root position back in fp32); ulps: max |dx| in units of 2^-24 max(|x|, 1), every point"""
    xd, xo = x_dev.reshape(-1, 3), x_ora.reshape(-1, 3)
    err = np.linalg.norm(xd - xo, axis=1)
    near = np.abs(xo).max(1) < NEAR
    rel = err / (np.linalg.norm(xo - x_root, axis=1) + POS_FLOOR)
    return float(rel[near].max()) if near.any() else 0.0, float((err / (U32 * np.maximum(np.abs(xo).max(1), 1.0))).max())


def sensor_error(m, s_dev, s_ora):
    """max over sensors |ds| / (max |s| + SENSOR_FLOOR[type])"""
    worst = 0.0
    for s in range(m.nsensor):
        a, n = int(m.sensor_adr[s]), int(m.sensor_dim[s])
        ref = s_ora[a:a + n]
        worst = max(worst, float(np.abs(s_dev[a:a + n] - ref).max() / (np.abs(ref).max() + SENSOR_FLOOR[int(m.sensor_type[s])])))
    return worst


def root_xpos(m, fields):
    """the walker's root body position (the first body with a free joint; the world origin without one)"""
    free = _joints(m, FREE)
    if not free:
        return np.zeros(3)
    return fields['xpos'].reshape(-1, 3)[m.jnt_bodyid[free[0]]]


def errors(m, dev, ora):
    """every per-element gate of one state (dev, ora: device_fields / oracle_fields entries)"""
    nv = m.nv
    M = ora['qM'].reshape(nv, nv)
    Md = dev['qM'].reshape(nv, nv)
    r0 = root_xpos(m, ora)
    e = dict(qM=qm_entry_error(Md, M))
    for k in ('qfrc_bias', 'qfrc_passive', 'qfrc_actuator', 'qfrc_smooth'):
        e[k] = force_error(dev[k], ora[k], M)
    for k in ('xpos', 'site_xpos', 'subtree_com'):
        e[k], e[k + '_ulps'] = position_error(dev[k], ora[k], r0)
    e['xmat'] = float(max(np.abs(dev['xmat'] - ora['xmat']).max(), np.abs(dev['site_xmat'] - ora['site_xmat']).max()))
    e['sensor'] = sensor_error(m, dev['sensordata'], ora['sensordata'])
    if 'qacc' in dev and ora['nefc'] == 0:
        e['qacc_back'], e['qacc_fwd'] = solve_errors(M, dev['qacc'], ora['qacc'], ora['qfrc_smooth'])
    if 'dqvel' in dev and ora['nefc'] == 0:
        h = float(m.opt_timestep)
        Ae = M + h * np.diag(m.dof_damping)
        res = U32 * np.abs(ora['qvel1']) / h             # the fp32 rounding of the qvel the change is read from
        e['dv_back'], e['dv_fwd'] = solve_errors(Ae, dev['dqvel'] / h, ora['dqvel'] / h, ora['qfrc_smooth'], res)
    return e


def probe_solve_errors(m, sim, names, assign, seed=0):
    """per-dof errors of both solves on a right-hand side built so that every dof's solution has the same size in the inertia metric:
    env i holds state names[assign[i]] plus qfrc_applied = M x* - qfrc_smooth (oracle's M and forces), x*_i = +-1 / sqrt(M_ii).  The
    reference is the fp64 solve of the oracle's M (and M + hD) against the qfrc_smooth the stepper itself solved (read back; the kernels
    solve exactly those fp32 numbers), so force errors drop out and a dof that the natural forces leave nearly at rest is measured on
    its own scale.  Per env: (max_i |dqacc_i| sqrt(M_ii), max_i |d(dqvel / h)_i| sqrt((M + hD)_ii) less the fp32 resolution of qvel),
    both relative to the dof's own |x_i| sqrt(A_ii) (about 1)"""
    rs = np.random.RandomState(seed)
    inputs = [state_inputs(m, k) for k in names]
    ora = {a: oracle_fields(m, names[a], step=False) for a in set(assign)}
    nv, h = m.nv, float(m.opt_timestep)
    M = {a: o['qM'].reshape(nv, nv) for a, o in ora.items()}
    signs = rs.choice([-1.0, 1.0], size=(len(assign), nv))
    app = np.array([M[a] @ (signs[i] / np.sqrt(np.diag(M[a]))) - ora[a]['qfrc_smooth'] for i, a in enumerate(assign)])
    q, v, act, ctrl = (np.array([inputs[a][c] for a in assign]) for c in range(4))
    sim.reset(q, v)
    if m.na:
        sim.set(st.ACT, act)
    sim.set_control(ctrl)
    sim.set_applied(qfrc=app)
    sim.forward()
    qacc, fs = np.asarray(sim.get(st.QACC), np.float64), np.asarray(sim.get(st.QFRC_SMOOTH), np.float64)
    Md = np.asarray(sim.get(st.QM_DENSE), np.float64).reshape(-1, nv, nv)
    sim.step(1)
    qvel1 = np.asarray(sim.get(st.QVEL), np.float64)
    sim.clear_applied()
    out = []
    for i, a in enumerate(assign):
        damp = np.float32(h) * m.dof_damping.astype(np.float32)         # the kernel's fp32 h * damping on the diagonal
        A, Ae = Md[i], Md[i] + np.diag(damp.astype(np.float64))
        s, se = np.sqrt(np.diag(A)), np.sqrt(np.diag(Ae))
        x, xe = np.linalg.solve(A, fs[i]), np.linalg.solve(Ae, fs[i])
        ea = float((np.abs(qacc[i] - x) * s / np.maximum(np.abs(x) * s, 0.5)).max())
        res = U32 * np.abs(qvel1[i]) / h
        dv = (qvel1[i] - v[i]) / h
        ee = float((np.maximum(np.abs(dv - xe) - res, 0.0) * se / np.maximum(np.abs(xe) * se, 0.5)).max())
        out.append((ea, ee))
    return out
