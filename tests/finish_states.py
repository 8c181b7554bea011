"""Finish-stage states and fp64 restatements for tests/test_finish_gates.py.

The finish kernel (fb_constraint.h kfin_f1 .. kfin_f10) turns the solver's forces into qacc = L^-1 (D^-1 u + D^-1/2 Z^T f) and
qfrc_constraint = J^T f, builds the contact wrenches and the delta accelerations behind the accelerometer, force and touch sensors,
and takes the semi-implicit Euler step.  One substep leaves every input and output of that kernel readable: fb_get returns the
stage of the substep (M, qfrc_smooth, the rows, efc_force, qacc, the contacts, the site poses and the sensors of the state the step
started from) next to the integrated qpos, qvel, act and time.  So the restatements here take the device's own upstream numbers, and
solver and collision error drop out of them.

States: the 14 pinned solver states (tests/solver_states.py, analytic walk model) and EXTRA_STATES: pinned cases on model copies
that reach the branches of the touch ray test the solver states never do (a positive-force contact whose ray misses the claw site,
the claw geom as geom1 of a claw-leg contact inside, outside and missing the site), the template model and the flight model with
joint limits only, and the ball model (walk_on_ball) with the claws on the moving ball.
"""
import numpy as np

import solver_states as ss
from flybody_b200 import stepper as st
from flybody_b200.flymodel import load_model
from oracle import fly_oracle as fo
from sensor_fd_reference import ACCELEROMETER, CAPSULE, FORCE, TOUCH, inverse_sensors

SPHERE = 2
FREE, BALL, HINGE = 0, 1, 3
U32 = 2.0 ** -24
# touch: a contact whose fp64 ray passes within TOUCH_BAND x (site radius) of the site's surface is counted and printed, not gated; the
# kernel's fp32 decision and the fp64 one part within 1e-6 radii (test_finish_gates.py band_sweep measures it)
TOUCH_BAND = 1e-3

# name -> (model, (seed, pos_scale, vel_scale)) of parity_common.random_state, found once by a search with the oracle; the model is a
# key of MODELS.  test_finish_states_keep_their_properties asserts what each one reaches.
EXTRA_STATES = {
    'miss_one':       ('shifted_site', (65, 0.1, 1.0)),     # one_contact with the site moved off the claw: a positive force, missed
    'miss_rows64':    ('shifted_site', (114, 0.1, 1.0)),    # rows64 likewise: misses on the generic path
    'geom1_inside':   ('walk', (47, 1.0, 1.0)),             # a claw-leg contact with the claw geom as geom1, inside the site
    'geom1_outside':  ('side_site', (47, 1.0, 1.0)),        # the same contact outside the side-shifted site, its ray hitting
    'geom1_miss':     ('shifted_site', (47, 1.0, 1.0)),     # ... and missing
    'template':       ('template', (2, 0.5, 1.0)),          # the template task's model
    'flight_limits':  ('flight', (1, 0.5, 1.0)),            # the flight model: joint limits only, accelerometer without contacts
    # the ball model: the claws press on the moving ball (the ball geom is geom1), so both trees get a contact wrench and contact rows
    # span the fly's tree and the ball's, whose ball joint is integrated under the contact forces (state_inputs: a random ball turn)
    'ball_rest':      ('ball', (0, 0.0, 1.0)),              # the legs at the task's reset pose: four claws on the ball
    'ball_few':       ('ball', (4, 0.1, 1.0)),              # nefc 7: the register solve path
    'ball_many':      ('ball', (1, 0.3, 1.0)),              # nefc 88: the generic solve path
}


def walk_model(noslip=None):
    return ss.analytic_model(load_model('walk'), noslip=noslip)


def touch_sites(m):
    return [int(m.sensor_objid[s]) for s in range(m.nsensor) if int(m.sensor_type[s]) == TOUCH]


def site_shift_model(shift, noslip=None):
    """the analytic walk model with every touch site moved by `shift` (cm, in its body's frame)"""
    a = walk_model(noslip).copy()
    pos = a.site_pos.copy()
    for s in touch_sites(a):
        pos[s] += shift
    a.a['site_pos'] = pos
    return a.rebuild()


# shifted_site: every touch site 0.02 cm along its body's z (4x the claw site's half-length), so the claw's own contacts fall outside
# it and their rays miss; side_site: 0.004 cm along -x (twice the site radius), where a claw-leg contact's outward ray still
# crosses the site while the opposite ray would not
MODELS = {
    'walk': walk_model,
    'shifted_site': lambda noslip=None: site_shift_model((0.0, 0.0, 0.02), noslip),
    'side_site': lambda noslip=None: site_shift_model((-0.004, 0.0, 0.0), noslip),
    'template': lambda noslip=None: ss.analytic_model(load_model('template'), noslip=noslip),
    'flight': lambda noslip=None: ss.analytic_model(load_model('flight'), noslip=noslip),
    'ball': lambda noslip=None: ss.analytic_model(load_model('ball'), noslip=noslip),
}


def state_inputs(m, model_key, t):
    """qpos, qvel, ctrl of pinned state t = (seed, pos_scale, vel_scale) on model `model_key` (solver_states.state_inputs); on the
    ball model the ball is also turned to a uniformly random orientation, so that its quaternion step is not the identity's"""
    q, v, c = ss.state_inputs(m, *t)
    if model_key == 'ball':
        quat = np.random.RandomState(t[0] + 300).normal(size=4)
        q = q.copy()
        q[0:4] = (quat / np.linalg.norm(quat)).astype(np.float32).astype(np.float64)
    return q, v, c


def all_states():
    """name -> (model key, (seed, pos_scale, vel_scale)): the solver states on the walk model, then EXTRA_STATES"""
    out = {k: ('walk', v[0]) for k, v in ss.STATES.items()}
    out.update(EXTRA_STATES)
    return out


# ---------------------------------------------------------------------------------------------------------- both sides

STAGE = (('qM', st.QM_DENSE), ('qfrc_smooth', st.QFRC_SMOOTH), ('qfrc_constraint', st.QFRC_CONSTRAINT), ('qacc', st.QACC),
         ('efc_force', st.EFC_FORCE), ('contact', st.CONTACT), ('site_xpos', st.SITE_XPOS), ('site_xmat', st.SITE_XMAT),
         ('sensordata', st.SENSORDATA))
SOLVED = ('qfrc_constraint', 'qacc', 'efc_force')       # what the substep's own constraint solve and finish kernel rewrite


def device_step(m, sim, inputs, act=None, xfrc=None):
    """reset env i of `sim` to inputs[i] = (qpos, qvel, ctrl), optionally act [n, na] and xfrc_applied; one forward, then one substep.  Per env: the
    stage (M, qfrc_smooth, qfrc_constraint, efc_force, qacc, contacts, site poses, sensors) and the state after the substep.

    A substep runs the constraint and finish kernels on the position / velocity stage that forward() left, then the position and
    velocity stages of the new state, so the stage is read after forward(); the substep's own solve must give the same bits
    (asserted on SOLVED), so the stage is exactly what its Euler step integrated."""
    q, v, c = (np.array([x[k] for x in inputs]) for k in range(3))
    sim.reset(q, v)
    if act is not None:
        sim.set(st.ACT, act)
    if xfrc is not None:
        sim.set_applied(xfrc=xfrc)
    sim.set_control(c)
    act0 = np.asarray(sim.get(st.ACT), np.float64) if m.na else np.zeros((sim.n_envs, 0))
    time0 = np.asarray(sim.get(st.TIME), np.float64)[:, 0]
    sim.forward()
    g = {k: np.asarray(sim.get(f), np.float64) for k, f in STAGE}
    nefc, ncon, flags = sim.get(st.NEFC)[:, 0], sim.get(st.NCON)[:, 0], sim.get(st.FLAGS)[:, 0]
    sim.step(1)
    for k, f in STAGE:
        if k in SOLVED:
            assert np.array_equal(np.asarray(sim.get(f), np.float64), g[k]), f'the substep solved {k} differently from forward()'
    g.update({k: np.asarray(sim.get(f), np.float64) for k, f in (('qpos1', st.QPOS), ('qvel1', st.QVEL), ('act1', st.ACT),
                                                                  ('time1', st.TIME))})
    out = []
    for i in range(sim.n_envs):
        ne, nc = int(nefc[i]), int(ncon[i])
        d = {k: x[i] for k, x in g.items()}
        d.update(nefc=ne, ncon=nc, flags=int(flags[i]), qpos0=q[i].astype(np.float64), qvel0=v[i].astype(np.float64),
                 ctrl=c[i].astype(np.float64), act0=act0[i], time0=float(time0[i]), qM=d['qM'].reshape(m.nv, m.nv),
                 force=d['efc_force'][:ne], con=d['contact'].reshape(-1, 16)[:nc], time1=float(d['time1'][0]))
        out.append(d)
    return out


def oracle_stage(m, inputs):
    """the oracle's forward() at inputs = (qpos, qvel, ctrl), its rows, and its state after one step, on the ball model's dofs.  The
    oracle has no ball joint: a ball model is stepped as tests/test_walk_on_ball.py's free-joint surrogate (the ball's joint a free
    joint whose translation carries a huge armature), whose leading three dofs (and qpos entries) are dropped again; `model`, `oracle`
    and `k` (the number of dropped dofs) are what sensor_restatement needs"""
    q, v, c = inputs
    mo, k, qo = m, 0, q
    if any(int(t) == BALL for t in m.jnt_type):
        from test_walk_on_ball import free_surrogate, to_surrogate_q
        mo, k, qo = free_surrogate(m), 3, to_surrogate_q(m, q)
    vo = np.concatenate([np.zeros(k), v])
    o = fo.Oracle(mo, tolerance=1e-12)
    o.reset(qo, vo)
    o.set(fo.CTRL, c)
    o.forward()
    ncon = int(o.get(fo.NCON)[0])
    efc = o.efc()
    efc['J'] = efc['J'][:, k:]
    r = dict(nefc=int(o.get(fo.NEFC)[0]), ncon=ncon, efc=efc, force=o.get(fo.EFC_FORCE),
             con=o.get(fo.CONTACT).reshape(-1, 16)[:ncon] if ncon else np.zeros((0, 16)), oracle=o, model=mo, k=k)
    for key, f in (('qM', fo.QM_DENSE), ('qfrc_smooth', fo.QFRC_SMOOTH), ('qfrc_constraint', fo.QFRC_CONSTRAINT), ('qacc', fo.QACC),
                   ('sensordata', fo.SENSORDATA), ('site_xpos', fo.SITE_XPOS), ('site_xmat', fo.SITE_XMAT)):
        r[key] = o.get(f)
    r['qM'] = r['qM'].reshape(m.nv + k, m.nv + k)[k:, k:]
    for key in ('qfrc_smooth', 'qfrc_constraint', 'qacc'):
        r[key] = r[key][k:]
    s = fo.Oracle(mo, tolerance=1e-12)
    s.reset(qo, vo)
    s.set(fo.CTRL, c)
    s.step()
    r.update(qpos1=s.qpos[k:], qvel1=s.qvel[k:], act1=s.get(fo.ACT) if m.na else np.zeros(0))
    return r


def sensor_restatement(o, qacc, force):
    """sensor_fd_reference.inverse_sensors about the oracle's forward state (oracle_stage's `o`) at the ball model's qacc"""
    return inverse_sensors(o['model'], o['oracle'], np.concatenate([np.zeros(o['k']), qacc]), force)


# ---------------------------------------------------------------------------------------------------------- touch

def _segment_distance(p, r, c, axis, hl):
    """distance from the half-line p + t r (t >= 0) to the segment c + s axis (|s| <= hl): golden-section search of the convex
    distance over t in [0, T], T past every point of the segment"""
    r = r / np.linalg.norm(r)

    def dist(t):
        x = p + t * r - c
        s = np.clip(x @ axis, -hl, hl)
        return np.linalg.norm(x - s * axis)

    lo, hi = 0.0, np.linalg.norm(p - c) + 2 * hl + 1.0
    g = (np.sqrt(5) - 1) / 2
    for _ in range(120):
        a, b = hi - g * (hi - lo), lo + g * (hi - lo)
        if dist(a) <= dist(b):
            hi = b
        else:
            lo = a
    return min(dist(0.5 * (lo + hi)), dist(0.0))


def touch_contacts(m, site, con, force, spos, smat):
    """the contacts of the touch site's body with rows, each as a dict: index, fn, side (1: the body is geom1's, 2: geom2's),
    inside (the point is inside the site), margin (distance of the fp64 ray from the site's surface relative to the site radius;
    <= 0: it hits), hit"""
    b = int(m.site_bodyid[site])
    size = np.asarray(m.site_size[site], np.float64)
    c = spos.reshape(-1, 3)[site]
    R = smat.reshape(-1, 3, 3)[site]
    out = []
    for i, row in enumerate(con):
        ea = int(row[12])
        if ea < 0:
            continue
        b1, b2 = int(m.geom_bodyid[int(row[7])]), int(m.geom_bodyid[int(row[8])])
        if b not in (b1, b2):
            continue
        ray = row[4:7] * (-1.0 if b == b2 else 1.0)
        p = row[1:4]
        hl = size[1] if int(m.site_type[site]) == CAPSULE else 0.0
        axis = R[:, 2]
        s = np.clip((p - c) @ axis, -hl, hl)
        inside = np.linalg.norm(p - c - s * axis) < size[0]
        margin = (_segment_distance(p, ray, c, axis, hl) - size[0]) / size[0]
        out.append(dict(index=i, fn=float(force[ea]), side=1 if b == b1 else 2, inside=bool(inside), margin=float(margin),
                        hit=bool(margin <= 0)))
    return out


def site_radius_model(m, radii):
    """copy of `m` with the touch sites' radii set: radii {site: radius} (fp32 values); contacts and dynamics are unchanged"""
    a = m.copy()
    size = a.site_size.copy()
    for site, r in radii.items():
        size[site, 0] = r
    a.a['site_size'] = size
    return a.rebuild()


def touch_reference(m, con, force, spos, smat):
    """per touch sensor: (fp64 sum of the positive normal forces of the hitting contacts, number of positive-force contacts in the
    TOUCH_BAND band), on the given contacts, forces and site poses"""
    out = []
    for s in range(m.nsensor):
        if int(m.sensor_type[s]) != TOUCH:
            continue
        site = int(m.sensor_objid[s])
        cs = [c for c in touch_contacts(m, site, con, force, spos, smat) if c['fn'] > 0]
        out.append((int(m.sensor_adr[s]), sum(c['fn'] for c in cs if c['hit']),
                    sum(1 for c in cs if abs(c['margin']) < TOUCH_BAND)))
    return out


def touch_branches(m, con, force, spos, smat):
    """which branches of the ray test the contacts reach: counts of miss, hit-outside, inside, geom1, zero-force"""
    n = dict(miss=0, outside_hit=0, inside=0, geom1=0, zero_force=0)
    for site in touch_sites(m):
        for c in touch_contacts(m, site, con, force, spos, smat):
            if c['fn'] <= 0:
                n['zero_force'] += 1
                continue
            n['geom1'] += c['side'] == 1
            if c['inside']:
                n['inside'] += 1
            elif c['hit']:
                n['outside_hit'] += 1
            else:
                n['miss'] += 1
    return n


# ---------------------------------------------------------------------------------------------------------- tier 1

def _metric(M):
    return np.sqrt(np.maximum(np.diag(M), 1e-300))


def constraint_force_error(d, J):
    """qfrc_constraint against fp64 J^T f_dev, per dof in the inertia metric relative to the largest dof"""
    ref = J.T @ d['force'] if len(d['force']) else np.zeros(len(d['qfrc_constraint']))
    s = _metric(d['qM'])
    scale = float((np.abs(ref) / s).max())
    return float((np.abs(d['qfrc_constraint'] - ref) / s).max() / scale) if scale > 0 else float(np.abs(d['qfrc_constraint']).max())


def solve_error_pair(A, x_dev, b, res=None):
    """(backward, forward) error of x_dev as the solution of A x = b (the fp64 solve of the same numbers as the reference);
    smooth_states.solve_errors"""
    from smooth_states import solve_errors
    return solve_errors(A, x_dev, np.linalg.solve(A, b), b, res)


def euler_matrix(m, M):
    h = np.float32(m.opt_timestep)
    return M + np.diag((h * m.dof_damping.astype(np.float32)).astype(np.float64))


def quat_mul(a, b):
    w1, x1, y1, z1 = a
    w2, x2, y2, z2 = b
    return np.array([w1 * w2 - x1 * x2 - y1 * y2 - z1 * z2, w1 * x2 + x1 * w2 + y1 * z2 - z1 * y2,
                     w1 * y2 - x1 * z2 + y1 * w2 + z1 * x2, w1 * z2 + x1 * y2 - y1 * x2 + z1 * w2])


def quat_integrate(q, w, h):
    """q (x) exp(w h / 2), w in the body frame, normalised (MuJoCo mju_quatIntegrate)"""
    ang = np.linalg.norm(w) * h
    if ang > 0:
        ax = w / np.linalg.norm(w)
        q = quat_mul(q, np.concatenate([[np.cos(ang / 2)], np.sin(ang / 2) * ax]))
    return q / np.linalg.norm(q)


def integrate_reference(m, qpos0, qvel1):
    """fp64 qpos after one Euler substep from the device's qpos0 and its qvel after the step, and per qpos entry the scale of its
    fp32 ulps: max(|qpos1|, |h qvel|) for positions and hinge angles, 1 for quaternion entries"""
    h = float(np.float32(m.opt_timestep))
    q1, scale = qpos0.copy(), np.ones(m.nq)
    for j in range(m.njnt):
        t, qa, da = int(m.jnt_type[j]), int(m.jnt_qposadr[j]), int(m.jnt_dofadr[j])
        if t == FREE:
            q1[qa:qa + 3] = qpos0[qa:qa + 3] + h * qvel1[da:da + 3]
            scale[qa:qa + 3] = np.maximum(np.abs(q1[qa:qa + 3]), np.abs(h * qvel1[da:da + 3]))
            q1[qa + 3:qa + 7] = quat_integrate(qpos0[qa + 3:qa + 7], qvel1[da + 3:da + 6], h)
        elif t == BALL:
            q1[qa:qa + 4] = quat_integrate(qpos0[qa:qa + 4], qvel1[da:da + 3], h)
        else:
            q1[qa] = qpos0[qa] + h * qvel1[da]
            scale[qa] = max(abs(q1[qa]), abs(h * qvel1[da]))
    return q1, np.maximum(scale, 1e-30)


def act_reference(m, act0, ctrl):
    """fp64 act after one substep: act0 + h (clamp(ctrl) - act0) / tau for every filter actuator, and its ulp scale"""
    h = float(np.float32(m.opt_timestep))
    a1 = act0.copy()
    for i in range(m.nu):
        a = int(m.actuator_actadr[i])
        if a < 0:
            continue
        assert int(m.actuator_dyntype[i]) == 2, 'only filter dynamics are restated'
        u = ctrl[i]
        if m.actuator_ctrllimited[i]:
            u = np.clip(u, *m.actuator_ctrlrange[i])
        tau = max(float(np.float32(m.actuator_dynprm[i][0])), 1e-15)
        a1[a] = act0[a] + h * (u - act0[a]) / tau
    return a1, np.maximum(np.maximum(np.abs(a1), np.abs(act0)), 1e-30)


def acc_sensor_errors(m, sens_dev, sens_ref, floor):
    """worst per-sensor error of the accelerometers and force sensors: |ds| / (max |s| + floor[type])"""
    out = {ACCELEROMETER: 0.0, FORCE: 0.0}
    for s in range(m.nsensor):
        tp = int(m.sensor_type[s])
        if tp not in out:
            continue
        a, n = int(m.sensor_adr[s]), int(m.sensor_dim[s])
        ref = sens_ref[a:a + n]
        out[tp] = max(out[tp], float(np.abs(sens_dev[a:a + n] - ref).max() / (np.abs(ref).max() + floor[tp])))
    return out[ACCELEROMETER], out[FORCE]


def touch_error(m, sens, ref, floor):
    """worst per-sensor touch error |ds| / (|s| + floor) over the sensors without a contact in the band, and the band count"""
    worst, band = 0.0, 0
    for adr, s, nb in ref:
        if nb:
            band += nb
            continue
        worst = max(worst, abs(sens[adr] - s) / (abs(s) + floor))
    return worst, band


def errors(m, d, o=None):
    """every finish gate of one state.  Tier 1 (the device's own inputs): qfrc_constraint against J^T f_dev (J: the oracle's rows),
    qacc and one substep's dqvel / h against fp64 solves of the device's M (and M + hD) and qfrc_smooth + qfrc_constraint, qpos / act
    after the substep in fp32 ulps, the accelerometers and force sensors against sensor_fd_reference.inverse_sensors at
    (qacc_dev, f_dev), touch against the fp64 ray test on the device's contacts.  Tier 2 (with `o`, oracle_stage): the same fields
    against the oracle's forward() and one step.  d: a device_step entry; o=None: the oracle-free gates only"""
    from parity_common import SENSOR_FLOOR
    from smooth_states import sensor_error
    h = float(np.float32(m.opt_timestep))
    e = {}
    rhs = d['qfrc_smooth'] + d['qfrc_constraint']
    e['qacc_back'], e['qacc_fwd'] = solve_error_pair(d['qM'], d['qacc'], rhs)
    res = U32 * np.abs(d['qvel1']) / h           # the fp32 rounding of the qvel the change is read from
    e['dv_fwd'] = solve_error_pair(euler_matrix(m, d['qM']), (d['qvel1'] - d['qvel0']) / h, rhs, res)[1]
    q1, sc = integrate_reference(m, d['qpos0'], d['qvel1'])
    e['qpos_ulps'] = float((np.abs(d['qpos1'] - q1) / sc).max() / U32)
    if m.na:
        a1, sa = act_reference(m, d['act0'], d['ctrl'])
        e['act_ulps'] = float((np.abs(d['act1'] - a1) / sa).max() / U32)
    e['time'] = abs(d['time1'] - float(np.float32(d['time0'] + np.float32(h))))
    tr = touch_reference(m, d['con'], d['force'], d['site_xpos'], d['site_xmat'])
    e['touch'], e['band'] = touch_error(m, d['sensordata'], tr, SENSOR_FLOOR[TOUCH])
    if o is None:
        return e
    assert (d['nefc'], d['ncon']) == (o['nefc'], o['ncon']), (d['nefc'], o['nefc'], d['ncon'], o['ncon'])
    assert np.array_equal(d['con'][:, 7:10], o['con'][:, 7:10]) and np.array_equal(d['con'][:, 12], o['con'][:, 12])
    e['qfrc_constraint'] = constraint_force_error(d, o['efc']['J'])
    sref = sensor_restatement(o, d['qacc'], d['force'])
    e['accelerometer'], e['force'] = acc_sensor_errors(m, d['sensordata'], sref, SENSOR_FLOOR)
    # tier 2
    s = _metric(o['qM'])
    rel = lambda a, b: float((np.abs(a - b) * s).max() / ((np.abs(b) * s).max() + 1e-300))       # noqa: E731
    e['t2_qfrc_constraint'] = float((np.abs(d['qfrc_constraint'] - o['qfrc_constraint']) / s).max()
                                    / ((np.abs(o['qfrc_constraint']) / s).max() + 1e-300))
    e['t2_qacc'] = rel(d['qacc'], o['qacc'])
    e['t2_dqvel'] = rel(d['qvel1'] - d['qvel0'], o['qvel1'] - d['qvel0'])
    e['t2_qpos'] = float(np.abs(d['qpos1'] - o['qpos1']).max())
    e['t2_accelerometer'], e['t2_force'] = acc_sensor_errors(m, d['sensordata'], o['sensordata'], SENSOR_FLOOR)
    tt = [(a, o['sensordata'][a], 0) for a, _, _ in tr]
    e['t2_touch'] = touch_error(m, d['sensordata'], tt, SENSOR_FLOOR[TOUCH])[0]
    e['t2_sensor'] = sensor_error(m, d['sensordata'], o['sensordata'])
    return e
