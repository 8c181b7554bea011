"""Parameter Jacobians (fb_fd_param_*): dx'/dtheta and d qfrc_inverse/dtheta (and their sensor rows) along element and scale directions of
the per-env model parameters.  Mechanics bit for bit against one-env handles of patched models; exact zeros; the inverse's exact linear
answers; accuracy against the fp64 restatement of tests/param_fd_reference.py; the fits they exist for (Gauss-Newton on one-step
predictions, one least-squares step on inverse dynamics); isolation, determinism and refusals.  CPU tier: the host-emulation build of the
kernel source; GPU tier (-m gpu): the same through the CUDA library on 4096-env handles.  "Bit-identical" compares uint32 views.

The Jacobian error is test_transition_fd's per-column error (col_errors).  Tolerances are 2.5 x the larger of the host-emulation and
H100 measurements (the worst case is named beside each constant)."""
import numpy as np
import pytest

import __graft_entry__ as ge
from flybody_b200 import derivatives as dv, stepper as st
from flybody_b200.flymodel import load_model

import param_fd_reference as pr
import sensor_fd_reference as sr
import smooth_states as ss
from test_model_params import patched, random_params, start_state
from test_sensor_fd import free_cases, solver_cases, stack
from test_transition_fd import col_errors
from flybody_b200.inverse_dynamics import _differentiate_pos

# ---- gates (measured: host emulation / H100 80GB HBM3 at a 700 W power limit; worst case) -------------------------------------------
LINEAR = 1e-3              # the inverse's linear columns (armature, damping, stiffness against their exact values; gravity, mass and
                           # inertia against the fp64 regressor), per column relative to its largest entry: measured 1.7e-4 emu / 2.1e-4 H100
FREE_ERR = 0.2             # constraint-free flight states, worst column over dxdp / dsdp / DfDp / DsDp: measured 7.6e-3 emu (one state, DfDp)
                           # / 7.8e-2 H100 (three states, dsdp)
CONTACT_ERR = 0.24         # template contact states one_contact and nefc31_zones, noslip on and off: measured 8.0e-2 emu (one substep, dsdp)
                           # / 9.6e-2 H100 (1 and 10 substeps, dsdp); DsDp 2.5e-3 on both
BALL_ERR = 2.1e-3          # walk_on_ball constraint-free states: measured 6.1e-4 emu / 8.2e-4 H100 (dsdp)
MASS_FORCE = 2.8e-5        # force rows of a body_mass scale against the nominal force rows (accuracy's known answer (b)), relative to
                           # the largest: measured 5.4e-6 emu / 1.1e-5 H100
GN_TOL, GN_ITERS = 1e-3, 6
LS_TOL = 1e-4

EPS = 1e-2


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


@pytest.fixture(scope='module')
def emu():
    ge.build()
    return ge.EMU


@pytest.fixture
def small(monkeypatch):
    """the front ends on handles sized to the problems (the emulation runs every env)"""
    monkeypatch.setattr(dv, 'ENVS', 64)


MECH_PARAMS = [dv.Scale('body_mass', 'body_inertia'), ('dof_damping', [6]), ('geom_friction', [0]), dv.Scale('actuator_gainprm'),
               ('gravity', [2]), dv.Scale('dof_damping')]


def den32(vals, direction, eps, centered=True):
    """the device's step difference of a direction at fp32 values (centred)"""
    kind, entries, floors = direction
    if kind == st.FD_SCALE:
        return np.float32(eps) - np.float32(-eps)
    (name, i), = entries
    x = np.float32(vals[name][i])
    d = np.float32(eps) * np.maximum(np.abs(x), np.float32(floors[0]))
    return d if name in pr.NONNEG and x - d < 0 else d - (-d)         # (a side below 0 is skipped: the nominal takes its place)


# ---- 1. mechanics, bit for bit --------------------------------------------------------------------------------------------------------
def check_mechanics(lib, variant, n_envs=None, n_sub=2):
    m = load_model(variant)
    p = random_params(m, 3)
    dirs, _ = dv._directions(m, MECH_PARAMS, None)
    ncol = 1 + 2 * len(dirs)
    sim = st.BatchedStepper(m, n_envs or max(ncol, 1 + 2 * m.nv + m.na + m.nu), lib_path=lib)
    sim.query_sensors(True)
    for name in st.PARAMS:
        sim.param_set(name, p[name])
    q, v = start_state(m, 4)
    u = np.random.RandomState(5).uniform(-0.5, 0.5, m.nu)
    sim.reset(q, v)
    sim.set_control(u)
    sim.state_bank(2)
    sim.save_state([1], [0])
    sim.fd_param_program(dirs)
    assert sim.fd_param_columns(True) == ncol and sim.fd_param_columns(False) == 1 + len(dirs)
    sim.fd_param_transition([1], eps=EPS, centered=True, n_substeps=n_sub)
    got = [sim.get(f) for f in (st.QPOS, st.QVEL, st.ACT)]
    vals = {name: sim.param_get(name) for name in st.PARAMS}
    dxdp, qn, vn, an = sim.fd_param_read()
    dsdp, sd0 = sim.fd_param_sensor_read()
    for name in st.PARAMS:
        assert np.array_equal(vals[name][0], p[name]), name                     # the nominal column: the row's own parameters
    assert not np.array_equal(vals['dof_damping'][3], p['dof_damping'])       # (a dof_damping direction: the M_damp slot moves too)
    for c in range(ncol):
        one = st.BatchedStepper(patched(m, {k: x[c] for k, x in vals.items()}), 1, lib_path=lib)
        one.reset(q, v)
        one.set_control(u)
        one.step(n_sub)
        for x, f in zip(got, (st.QPOS, st.QVEL, st.ACT)):
            assert np.array_equal(bits(x[c]), bits(one.get(f)[0])), (variant, c, f)
        one.close()
    # the nominal column is fb_fd_transition's nominal next state of the same row
    # (and its sensordata, the sensors of x, is fb_fd_transition's)
    sim.fd_transition([1], eps=EPS, centered=False, n_substeps=n_sub)
    _, _, q2, v2, a2 = sim.fd_read()
    assert np.array_equal(bits(q2), bits(qn)) and np.array_equal(bits(v2), bits(vn)) and np.array_equal(bits(a2), bits(an))
    assert np.array_equal(bits(sim.fd_sensor_read()[2]), bits(sd0))
    # dsdp (kfd_diff's sensor block): column j is the difference of its two columns' sensors of x over their steps
    sd = []
    for c in range(ncol):
        one = st.BatchedStepper(patched(m, {k: x[c] for k, x in vals.items()}), 1 + 2 * m.nv + m.na + m.nu, lib_path=lib)
        one.query_sensors(True)
        one.reset(q, v)
        one.set_control(u)
        one.state_bank(1)
        one.save_state([0], [0])
        one.fd_transition([0], eps=EPS, centered=False, n_substeps=1)     # its nominal sensordata: the sensors of x on this model
        sd.append(one.fd_sensor_read()[2][0])
        one.close()
    assert np.array_equal(bits(sd[0]), bits(sd0[0]))
    for j, dr in enumerate(dirs):
        want = (sd[1 + 2 * j] - sd[2 + 2 * j]) / den32({k: x[0] for k, x in vals.items()}, dr, EPS)
        assert np.array_equal(bits(dsdp[0, :, j]), bits(want)), (variant, j)
    assert np.isfinite(dxdp).all() and np.abs(dxdp).max() > 0
    sim.close()


def check_inverse_mechanics(lib, variant, n_envs=None):
    m = load_model(variant)
    p = random_params(m, 8)
    dirs, _ = dv._directions(m, MECH_PARAMS + [('dof_armature', [7]), ('jnt_stiffness', [dv._elements(m, 'jnt_stiffness')[3]])], None)
    ncol = 1 + 2 * len(dirs)
    sim = st.BatchedStepper(m, n_envs or ncol, lib_path=lib)
    sim.query_sensors(True)
    for name in st.PARAMS:
        sim.param_set(name, p[name], env_ids=[0])
    q, v = start_state(m, 2)
    qa = np.random.RandomState(4).uniform(-100, 100, m.nv)
    sim.fd_param_program(dirs)
    sim.fd_param_inverse(q[None], v[None], qa[None], eps=EPS, centered=True)
    DfDp, f0 = sim.fd_param_inverse_read()
    DsDp, sd0 = sim.fd_param_inverse_sensor_read()
    vals = {name: sim.param_get(name) for name in st.PARAMS}
    ref = st.BatchedStepper(m, 1, lib_path=lib)                  # fb_inverse with the same parameters
    ref.query_sensors(True)
    for name in st.PARAMS:
        ref.param_set(name, p[name])
    ref.reset(q, v)
    ref.inverse(qa[None])
    assert np.array_equal(bits(ref.inverse_read()[0][0]), bits(f0[0]))
    assert np.array_equal(bits(ref.inverse_sensor_read()[0]), bits(sd0[0]))
    for j, dr in enumerate(dirs):
        f, sd = [], []
        for c in (1 + 2 * j, 2 + 2 * j):
            one = st.BatchedStepper(patched(m, {k: x[c] for k, x in vals.items()}), 1, lib_path=lib)
            one.query_sensors(True)
            one.reset(q, v)
            one.inverse(qa[None])
            f.append(one.inverse_read()[0][0])
            sd.append(one.inverse_sensor_read()[0])
            one.close()
        den = den32({k: x[0] for k, x in vals.items()}, dr, EPS)
        assert np.array_equal(bits(DfDp[0, j]), bits((f[0] - f[1]) / den)), (variant, j)
        assert np.array_equal(bits(DsDp[0, j]), bits((sd[0] - sd[1]) / den)), (variant, j)
    sim.close()


@pytest.mark.parametrize('variant', ['template', 'flight'])
def test_mechanics_under_emulation(emu, variant):
    check_mechanics(emu, variant)
    check_inverse_mechanics(emu, variant)


# ---- 2. exact zeros, 3. exact linear answers --------------------------------------------------------------------------------------------
def check_zeros(lib):
    m = load_model('template')
    q, v = start_state(m, 4)
    u = np.random.RandomState(5).uniform(-0.5, 0.5, m.nu)
    probe = st.BatchedStepper(m, 1, lib_path=lib)
    probe.reset(q, v)
    con = probe.get(st.CONTACT).reshape(st.MAXCON, 16)[:int(probe.get(st.NCON)[0, 0])]
    probe.close()
    touching = set(con[:, 7].astype(int)) | set(con[:, 8].astype(int))
    assert touching
    g_on = sorted(touching)[-1]
    g_off = [g for g in range(m.ngeom) if g not in touching and m.geom_bodyid[g] > 0][-1]
    params = [('geom_friction', [3 * g_on, 3 * g_on + 1, 3 * g_on + 2, 3 * g_off]), dv.Scale('actuator_gainprm'),
              dv.Scale('actuator_biasprm'), dv.Scale('body_mass'), ('dof_damping', [6])]
    act = np.random.RandomState(6).uniform(-0.5, 0.5, m.na)      # (the actuators' input is act: at act = 0 the gain does not act)
    T = dv.parameter_fd(m, q, v, u, act, params=params, eps=EPS, lib_path=lib)
    cols = T.columns
    assert cols[:4] == [f'geom_friction[{3 * g_on}]', f'geom_friction[{3 * g_on + 1}]', f'geom_friction[{3 * g_on + 2}]', f'geom_friction[{3 * g_off}]']
    assert not T.dxdp[2 * m.nv:].any()                          # act rows: the activation dynamics read no parameter
    assert not T.dxdp[:, 1:4].any()                             # friction entries 1-2 (the step reads column 0 at condim <= 3), a geom in no contact
    assert np.abs(T.dxdp[:, 0]).max() > 0 and np.abs(T.dxdp[:, 4:]).max(0).min() > 0
    qa = np.random.RandomState(1).uniform(-50, 50, m.nv)
    inv = dv.inverse_parameter_fd(m, q, v, qa, params=params, eps=EPS, lib_path=lib)
    assert not inv.DfDp[1:3].any() and not inv.DfDp[4:6].any()      # no actuation in qfrc_inverse
    assert np.abs(inv.DfDp[6:]).max(1).min() > 0
    mf, cases = free_cases('flight')
    qf, vf, _, _, af = stack(cases, range(5))
    free = dv.inverse_parameter_fd(mf, qf[:2], vf[:2], af[:2], params=[('geom_friction', [0, 3, 4]), dv.Scale('geom_friction')], eps=EPS, lib_path=lib)
    assert not free.DfDp.any()                                  # constraint-free: friction does not reach qfrc_inverse


def test_exact_zeros_under_emulation(emu, small):
    check_zeros(emu)


def linear_columns(lib, m, q, v, qa):
    """the inverse's columns that are linear in the parameters against their exact values: -> the worst column error"""
    hinges = dv._elements(m, 'jnt_stiffness')
    js = hinges[:4]
    dofs = [int(m.jnt_dofadr[j]) for j in js]
    params = [('dof_armature', dofs), ('dof_damping', dofs), ('jnt_stiffness', js), 'gravity', dv.Scale('body_mass'), dv.Scale('body_inertia'),
              ('body_mass', [5])]
    values = {'density': np.zeros((len(q), 1)), 'viscosity': np.zeros((len(q), 1))}
    inv = dv.inverse_parameter_fd(m, q, v, qa, params=params, values=values, eps=EPS, lib_path=lib)
    k = len(dofs)
    err = 0.0
    for p in range(len(q)):
        exact = np.zeros((3 * k, m.nv))
        for t, (d, j) in enumerate(zip(dofs, js)):
            exact[t, d] = qa[p, d]
            exact[k + t, d] = v[p, d]
            exact[2 * k + t, d] = q[p, int(m.jnt_qposadr[j])] - m.qpos_spring[int(m.jnt_qposadr[j])]
        dirs, _ = dv._directions(m, params[3:], None)
        ref = pr.inverse(m, q[p], v[p], qa[p], dirs, values={n: x[p] for n, x in values.items()}, eps=EPS)['DfDp']
        err = max(err, col_errors(inv.DfDp[p, :3 * k].T, exact.T).max(), col_errors(inv.DfDp[p, 3 * k:].T, ref.T).max())
    return err


def check_linear(lib):
    m, cases = solver_cases(0, ['one_contact', 'nefc31_zones'])
    q, v, _, a = stack(cases, range(4))
    mf, fc = free_cases('walk')
    qf, vf, _, _, af = stack(fc, range(5))
    e = max(linear_columns(lib, m, q, v, a), linear_columns(lib, mf, qf[:2], vf[:2], af[:2]))
    print(f'linear columns {e:.1e}')
    assert e <= LINEAR


def test_exact_linear_answers_under_emulation(emu, small):
    check_linear(emu)


# ---- 4. accuracy against fp64 ---------------------------------------------------------------------------------------------------------
# parameters the inverse's sensordata does not read: at fixed (qpos, qvel, qacc) the sensors are kinematics, the bodies' masses and
# the contact forces (whose soft-model terms use the derived constants, held), so these DsDp columns are exactly 0 on the device
JOINT_SPACE = {'dof_armature', 'dof_damping', 'jnt_stiffness', 'actuator_gainprm', 'actuator_biasprm'}


def accuracy(lib, m, cases, params, n_sub, free, values=None):
    """-> {output: worst column error over the states} against the fp64 reference, and the worst force-row error of a mass scale
    against its known answer on constraint-free states (see below).

    Two parts of DsDp are checked by known answers instead of the reference, which restates the inverse's sensors as forward()'s plus
    their change from forward's qacc (tests/sensor_fd_reference.py): (a) the JOINT_SPACE columns, which must be exactly 0 and are; the
    restatement gives them its own cancellation residual (forward's sensors move with forward's qacc, ~1e2 rad/s^2 per nudge), which
    alone made the worst column read 1.0; (b) on constraint-free states, the force rows: the reference's own nominal force sensors
    disagree with fb_inverse's there (test_sensor_fd leaves the force rows out of that nominal for the same reason), and without
    contacts a force sensor is linear in the body masses and blind to their inertia, so a scale of every body_mass has the nominal
    force rows as its column"""
    q, v, u, act, a = cases
    T = dv.parameter_fd(m, q, v, u, act if free else None, params=params, values=values, eps=EPS, n_substeps=n_sub, sensors=True, lib_path=lib)
    I = dv.inverse_parameter_fd(m, q, v, a, params=params, values=values, eps=EPS, sensors=True, lib_path=lib)
    dirs, labels = dv._directions(m, params, None)
    silent = [j for j, (_, ent, _) in enumerate(dirs) if all(n in JOINT_SPACE for n, _ in ent)]
    assert not I.DsDp[:, silent].any()
    keep = [j for j in range(len(dirs)) if j not in silent]
    _, _, frc, _ = sr.stage_rows(m)
    rows = np.setdiff1d(np.arange(m.nsensordata), frc) if free else np.arange(m.nsensordata)
    mass = [j for j, (k, ent, _) in enumerate(dirs) if k == st.FD_SCALE and {n for n, _ in ent} <= {'body_mass', 'body_inertia'}
            and len([1 for n, _ in ent if n == 'body_mass']) == m.nbody]
    err, known = {}, 0.0
    for p in range(len(q)):
        R = pr.transition(m, q[p], v[p], act[p] if free else None, u[p], dirs, eps=EPS, n_substeps=n_sub, sensors=True)
        Ri = pr.inverse(m, q[p], v[p], a[p], dirs, eps=EPS, sensors=True)
        for name, dev, ref in (('dxdp', T.dxdp[p], R['dxdp']), ('dsdp', T.dsdp[p], R['dsdp']), ('DfDp', I.DfDp[p].T, Ri['DfDp'].T),
                               ('DsDp', I.DsDp[p][keep][:, rows].T, Ri['DsDp'][keep][:, rows].T)):
            e = col_errors(dev, ref)
            err[name] = max(err.get(name, 0.0), float(e.max()))
        if free and len(frc):
            f0 = I.sensordata[p, frc]
            for j in mass:
                known = max(known, float(np.abs(I.DsDp[p, j, frc] - f0).max() / np.abs(f0).max()))
    return err, known


def free_params(m):
    out = [dv.Scale('dof_damping'), dv.Scale('actuator_gainprm'), dv.Scale('body_mass', 'body_inertia'), ('dof_damping', [7]), ('gravity', [2])]
    return out + ([dv.Scale('density')] if float(m.opt_density) > 0 else [])


def run_accuracy(tag, lib, m, c, params, n_subs, free):
    res = [accuracy(lib, m, c, params, n, free) for n in n_subs]
    err = {k: max(r[0][k] for r in res) for k in res[0][0]}
    known = max(r[1] for r in res)
    print(tag, {k: f'{x:.1e}' for k, x in err.items()}, f'force rows of the mass scale {known:.1e}')
    return max(err.values()), known


def check_free(lib, n_states, n_subs=(1, 10)):
    m, cases = free_cases('flight')
    c = [x[:n_states] for x in stack(cases, range(5))]
    err, _ = run_accuracy('flight', lib, m, c, free_params(m), n_subs, True)
    assert err <= FREE_ERR


def contact_params(lib, m, q, v):
    probe = st.BatchedStepper(m, len(q), lib_path=lib)
    probe.reset(q, v)
    con = probe.get(st.CONTACT).reshape(len(q), st.MAXCON, 16)[0, :int(probe.get(st.NCON)[0, 0])]
    probe.close()
    g = int(con[0, 7]) if m.geom_bodyid[int(con[0, 7])] > 0 else int(con[0, 8])
    return [dv.Scale('dof_damping'), dv.Scale('body_mass', 'body_inertia'), ('geom_friction', [3 * g]), ('dof_armature', [8]), ('gravity', [2])]


def check_contacts(lib, noslip, names, n_subs=(1, 10)):
    m, cases = solver_cases(noslip, names)
    q, v, u, a = stack(cases, range(4))
    err, _ = run_accuracy(f'contacts noslip={noslip}', lib, m, (q, v, u, np.zeros((len(q), m.na)), a), contact_params(lib, m, q, v), n_subs, False)
    assert err <= CONTACT_ERR


def check_ball(lib, n_states):
    m, cases = free_cases('ball')
    c = [x[:n_states] for x in stack(cases, range(5))]
    err, known = run_accuracy('ball', lib, m, c, [dv.Scale('dof_damping'), dv.Scale('body_mass', 'body_inertia'), dv.Scale('body_mass'),
                                                   ('gravity', [2])], (1,), True)
    assert err <= BALL_ERR and known <= MASS_FORCE


def test_constraint_free_under_emulation(emu, small):
    check_free(emu, 1, (1,))


@pytest.mark.parametrize('noslip', [0, None])
def test_contacts_under_emulation(emu, small, noslip):
    check_contacts(emu, noslip, ['one_contact', 'nefc31_zones'], (1,))


def test_ball_under_emulation(emu, small):
    check_ball(emu, 2)


# ---- 5. the fits the Jacobians exist for ---------------------------------------------------------------------------------------------
GROUPS = ('dof_damping', 'actuator_gainprm', 'body_mass', 'density')


def check_gauss_newton(lib, n_pairs=64, n_sub=4):
    """one-control-step predictions of a flight handle whose overlay scales the four groups by s*: Gauss-Newton from s = 1 on dxdp"""
    m = load_model('flight')
    s_true = np.array([1.15, 0.9, 1.1, 0.85])
    rs = np.random.RandomState(0)
    q, v = (np.array(x) for x in zip(*[start_state(m, 100 + k) for k in range(n_pairs)]))
    u = rs.uniform(-0.5, 0.5, (n_pairs, m.nu))
    base = {g: dv.compiled_params(m, g) for g in GROUPS}
    data = st.BatchedStepper(m, n_pairs, lib_path=lib)
    for g, s in zip(GROUPS, s_true):
        data.param_set(g, base[g] * s)
    data.reset(q, v)
    data.set_control(u)
    data.step(n_sub)
    qd, vd = data.get(st.QPOS).astype(np.float64), data.get(st.QVEL).astype(np.float64)
    data.close()
    w = 1.0 / np.maximum(np.abs(np.concatenate([np.zeros_like(vd[:, :m.nv]) + 1e-3, vd], 1)).max(0), 1e-3)      # per-row scaling

    def step(s):
        T = dv.parameter_fd(m, q, v, u, params=[dv.Scale(g) for g in GROUPS], values={g: base[g] * sg for g, sg in zip(GROUPS, s)},
                            eps=EPS, n_substeps=n_sub, lib_path=lib)
        r = np.concatenate([_differentiate_pos(m, T.qpos_next, qd, 1.0), vd - T.qvel_next], 1)        # [B, nx]
        J = (T.dxdp / s[None, None, :] * w[None, :, None]).reshape(-1, 4)   # d / ds_g at the estimate (the column is d / d(relative scale))
        return np.linalg.lstsq(J, (r * w[None]).reshape(-1), rcond=None)[0], J
    s = np.ones(4)
    for it in range(GN_ITERS):
        s = s + step(s)[0]
        if np.abs(s / s_true - 1).max() < GN_TOL:
            break
    print('Gauss-Newton', it + 1, s, np.abs(s / s_true - 1).max())
    # the floor of the fit: the step taken from the true scales (its residual is the fp32 rounding of the device's predictions) and the
    # conditioning of the weighted Jacobian there
    ds, J = step(s_true)
    print('from s*: step', ds, 'singular values', np.linalg.svd(J, compute_uv=False), 'column norms', np.linalg.norm(J, axis=0))
    assert np.abs(s / s_true - 1).max() < GN_TOL and it + 1 <= GN_ITERS


def check_least_squares(lib):
    """template walking states with contacts: qfrc_inverse at scales s* of armature, damping and gravity is linear in the scales; one
    least-squares step on DfDp recovers them"""
    m, cases = solver_cases(0, ['one_contact', 'nefc31_zones', 'nefc33'])
    q, v, _, a = stack(cases, range(4))
    groups, s_true = ('dof_armature', 'dof_damping', 'gravity'), np.array([1.2, 0.8, 1.05])
    data = st.BatchedStepper(m, len(q), lib_path=lib)
    for g, s in zip(groups, s_true):
        data.param_set(g, dv.compiled_params(m, g) * s)
    data.reset(q, v)
    data.inverse(a)
    fd = data.inverse_read()[0].astype(np.float64)
    data.close()
    inv = dv.inverse_parameter_fd(m, q, v, a, params=[dv.Scale(g) for g in groups], eps=EPS, lib_path=lib)
    J = np.transpose(inv.DfDp, (0, 2, 1)).reshape(-1, 3)
    ds = np.linalg.lstsq(J, (fd - inv.qfrc_inverse).reshape(-1), rcond=None)[0]
    s = 1 + ds
    print('least squares', s)
    assert np.abs(s / s_true - 1).max() < LS_TOL


def test_fits_under_emulation(emu):
    check_least_squares(emu)


# ---- 6. isolation and determinism; 7. refusals ------------------------------------------------------------------------------------------
FIELDS = (st.QPOS, st.QVEL, st.ACT, st.QACC, st.SENSORDATA, st.EFC_FORCE)


def check_isolation(lib, n_big):
    """a program changes no other query's bits; a problem's outputs do not depend on its slot or on n; the sensor switch changes no
    other output"""
    m, cases = free_cases('flight')
    q, v, u, act, a = stack(cases, range(5))
    q, v, u, a = q[:3], v[:3], u[:3], a[:3]
    dirs, _ = dv._directions(m, free_params(m), None)
    out = {}
    for prog in (False, True):
        sim = st.BatchedStepper(m, n_big, lib_path=lib)
        if prog:
            sim.fd_param_program(dirs)
        rows = np.arange(n_big) % 3
        sim.reset(q[rows], v[rows]); sim.set_control(u[rows]); sim.step(2)
        r = [sim.get(f) for f in FIELDS]
        sim.inverse(a)
        r += list(sim.inverse_read())
        sim.fd_inverse(q, v, a, eps=EPS, centered=False)
        r += list(sim.fd_inverse_read())
        sim.state_bank(3); sim.save_state([0, 1, 2], [0, 1, 2])
        r += [sim.read_states([0, 1, 2])]
        sim.fd_transition([0, 1, 2], eps=EPS, centered=False)
        r += list(sim.fd_read())
        out[prog] = r
        sim.close()
    for x, y in zip(out[False], out[True]):
        assert np.array_equal(bits(x), bits(y))
    # slot, n and the sensor switch
    res = {}
    for tag, n_p, order, sens in (('one', 1, [1], False), ('many', None, [2, 0, 1], False), ('sens', None, [2, 0, 1], True)):
        ncol = 1 + 2 * len(dirs)
        sim = st.BatchedStepper(m, n_big if n_p is None else ncol, lib_path=lib)
        sim.param_set('gravity', dv.compiled_params(m, 'gravity'))
        sim.query_sensors(sens)
        sim.fd_param_program(dirs)
        rows = np.array(order + [order[-1]] * (sim.n_envs - len(order)))
        sim.reset(q[rows], v[rows]); sim.set_control(u[rows])
        per = sim.n_envs // ncol
        slots = np.arange(len(order))[::-1] if n_p is None else [0]
        sim.state_bank(len(order)); sim.save_state(slots, np.arange(len(order)))
        sim.fd_param_transition(slots[:per], eps=EPS, n_substeps=2)
        t = sim.fd_param_read()
        if sens:
            assert [x.shape for x in sim.fd_param_sensor_read()] == [(len(slots[:per]), m.nsensordata, len(dirs)), (len(slots[:per]), m.nsensordata)]
        else:
            with pytest.raises(st.StepperError, match='sensors off'):
                sim.fd_param_sensor_read()
        for name in st.PARAMS:                                  # (the transition left nudged parameters in its columns' envs)
            sim.param_set(name, dv.compiled_params(m, name))
        sim.fd_param_inverse(q[order], v[order], a[order], eps=EPS, n=min(per, len(order)))
        i = sim.fd_param_inverse_read()
        res[tag] = (t, i, list(slots[:per]), order)
        sim.close()
    (t1, i1, _, _), (tm, im, sl, order) = res['one'], res['many']
    k = order.index(1)                                          # problem k: slot sl[k], saved from env k, which held state 1
    for x, y in zip(t1, tm):
        assert np.array_equal(bits(x[0]), bits(y[k]))
    for x, y in zip(i1, im):
        assert np.array_equal(bits(x[0]), bits(y[order.index(1)]))
    for x, y in zip(res['many'][0] + res['many'][1], res['sens'][0] + res['sens'][1]):
        assert np.array_equal(bits(x), bits(y))


def test_isolation_under_emulation(emu):
    check_isolation(emu, 3 * (1 + 3 * 48) + 7)


def check_refusals(lib):
    m = load_model('flight')
    sim = st.BatchedStepper(m, 8, lib_path=lib)
    lib_, h = sim._lib, sim._h
    q, v = start_state(m, 1)
    a = np.zeros(m.nv)
    for read, what in ((sim.fd_param_read, 'no parameter Jacobians'), (sim.fd_param_sensor_read, 'no parameter Jacobians'),
                       (sim.fd_param_inverse_read, 'no parameter Jacobians'), (sim.fd_param_inverse_sensor_read, 'no parameter Jacobians')):
        sim._fdp_n = sim._fdpi_n = (1, 1)
        with pytest.raises(st.StepperError, match=what):
            read()
    sim.fd_param_program([(st.FD_SCALE, [('dof_damping', 0)], None)])
    with pytest.raises(st.StepperError, match='no parameter overlay'):
        sim.fd_param_inverse(q[None], v[None], a[None])
    sim.state_bank(1)
    with pytest.raises(st.StepperError, match='no parameter overlay'):
        sim.fd_param_transition([0])
    sim.param_set('gravity', dv.compiled_params(m, 'gravity'))
    sim.fd_param_program([])                                   # k = 0 clears
    with pytest.raises(st.StepperError, match='no direction program'):
        sim.fd_param_inverse(q[None], v[None], a[None])
    with pytest.raises(st.StepperError, match='no direction program'):
        sim.fd_param_columns()
    ge_ = (st.FD_ELEMENT, [('dof_damping', 0)], [1.0])
    bad = [([(2, [('dof_damping', 0)], None)], 'kind'),
           ([(st.FD_ELEMENT, [('dof_damping', 0), ('dof_damping', 1)], [1.0, 1.0])], 'one entry'),
           ([(st.FD_ELEMENT, [('dof_damping', m.nv)], [1.0])], 'out of range'),
           ([(st.FD_ELEMENT, [('dof_damping', -1)], [1.0])], 'out of range'),
           ([(st.FD_ELEMENT, [('dof_damping', 0)], [0.0])], 'floor'),
           ([(st.FD_ELEMENT, [('dof_damping', 0)], [np.nan])], 'floor'),
           ([(st.FD_SCALE, [('dof_damping', 0), ('dof_damping', 0)], None)], 'twice'),
           ([(st.FD_SCALE, [('jnt_stiffness', [j for j in range(m.njnt) if m.jnt_type[j] != 3][0])], None)], 'not a hinge'),
           ([ge_, (st.FD_SCALE, [], None)], 'no entries')]
    for prog, msg in bad:
        with pytest.raises(st.StepperError, match=msg):
            sim.fd_param_program(prog)
    arr = np.zeros(4, np.int32)
    assert lib_.fb_fd_param_program(h, -1, *[arr.ctypes.data] * 4, arr.ctypes.data) == -1 and 'k >= 1' in lib_.fb_last_error(h).decode()
    assert lib_.fb_fd_param_program(h, 1, None, *[arr.ctypes.data] * 3, arr.ctypes.data) == -1 and 'NULL' in lib_.fb_last_error(h).decode()
    assert lib_.fb_fd_param_program(h, 999, 0, 0, 0, 0, 0) == -1
    unknown = np.array([0, 1], np.int32)
    assert lib_.fb_fd_param_program(h, 1, arr.ctypes.data, unknown.ctypes.data, np.array([12], np.int32).ctypes.data, arr.ctypes.data,
                                    np.ones(1, np.float32).ctypes.data) == -1 and 'unknown parameter' in lib_.fb_last_error(h).decode()
    sim.fd_param_program([ge_, (st.FD_SCALE, [('dof_damping', 0), ('body_mass', 1)], None)])
    assert sim.fd_param_columns() == 5 and sim.fd_param_columns(False) == 3
    for eps, msg in ((0.0, 'positive'), (np.inf, 'positive'), (1.0, 'eps < 1'), (-1e-2, 'positive')):
        with pytest.raises(st.StepperError, match=msg):
            sim.fd_param_inverse(q[None], v[None], a[None], eps=eps)
    with pytest.raises(st.StepperError, match='n_envs'):
        sim.fd_param_inverse(np.tile(q, (2, 1)), np.tile(v, (2, 1)), np.tile(a, (2, 1)))
    sim.state_bank(2)
    sim.save_state([0], [0])
    with pytest.raises(st.StepperError, match='n_envs'):
        sim.fd_param_transition([0, 0])
    with pytest.raises(st.StepperError, match='never written'):
        sim.fd_param_transition([1])
    with pytest.raises(st.StepperError, match='non-finite'):
        sim.fd_param_inverse(np.full((1, m.nq), np.nan), v[None], a[None])
    sim.fd_param_transition([0])
    sim.fd_param_inverse(q[None], v[None], a[None])
    with pytest.raises(st.StepperError, match='sensors off'):
        sim.fd_param_sensor_read()
    with pytest.raises(st.StepperError, match='sensors off'):
        sim.fd_param_inverse_sensor_read()
    with pytest.raises(st.StepperError, match='overlay'):       # fb_fd_inverse keeps refusing overlays
        sim.fd_inverse(q[None], v[None], a[None])
    sim.close()


def test_refusals_under_emulation(emu):
    check_refusals(emu)


def test_python_front_ends(emu, small):
    m, cases = free_cases('flight')
    q, v, u, act, a = stack(cases, range(5))
    T = dv.parameter_fd(m, q[:2], v[:2], u[:2], params=['gravity', dv.Scale('dof_damping', idx=[0, 1])], eps=EPS, lib_path=emu)
    assert type(T) is dv.ParamTransition and T.dxdp.shape == (2, 2 * m.nv + m.na, 4) and T.dxdp.dtype == np.float64
    assert T.columns == ['gravity[0]', 'gravity[1]', 'gravity[2]', 'scale(dof_damping[0,1])']
    t1 = dv.parameter_fd(m, q[1], v[1], u[1], params=['gravity', dv.Scale('dof_damping', idx=[0, 1])], eps=EPS, lib_path=emu, sensors=True)
    assert np.array_equal(t1.dxdp, T.dxdp[1]) and t1.dsdp.shape == (m.nsensordata, 4) and t1._fields[-2:] == ('dsdp', 'sensordata')
    tm = load_model('template')
    assert dv.parameter_fd(tm, tm.qpos0, np.zeros(tm.nv), np.zeros(tm.nu), params=['jnt_stiffness'], lib_path=emu).columns == \
        [f'jnt_stiffness[{j}]' for j in range(tm.njnt) if tm.jnt_type[j] == 3]
    I = dv.inverse_parameter_fd(m, q[:2], v[:2], a[:2], params=[('dof_armature', [3])], values={'dof_armature': np.full(m.nv, 2e-3)},
                                eps=EPS, lib_path=emu, sensors=True)
    assert type(I) is dv.InverseParamSensorJacobians and I.DfDp.shape == (2, 1, m.nv) and I.DsDp.shape == (2, 1, m.nsensordata)
    with pytest.raises(ValueError, match='single field'):
        dv.Scale('dof_damping', 'body_mass', idx=[0])
    with pytest.raises(KeyError):
        dv.parameter_fd(m, q[0], v[0], u[0], params=['body_pos'], lib_path=emu)


# ---- GPU tier ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize('variant', ['template', 'flight'])
def test_gpu_mechanics(variant):
    ge.build()
    check_mechanics(None, variant, 4096)
    check_inverse_mechanics(None, variant, 4096)


@pytest.mark.gpu
def test_gpu_zeros_and_linear_answers():
    ge.build()
    check_zeros(None)
    check_linear(None)


@pytest.mark.gpu
def test_gpu_accuracy_free():
    ge.build()
    check_free(None, 3)


@pytest.mark.gpu
@pytest.mark.parametrize('noslip', [0, None])
def test_gpu_accuracy_contacts(noslip):
    ge.build()
    check_contacts(None, noslip, ['one_contact', 'nefc31_zones'])


@pytest.mark.gpu
def test_gpu_accuracy_ball():
    ge.build()
    check_ball(None, 2)


@pytest.mark.gpu
@pytest.mark.xfail(strict=True, reason='finding: six iterations recover the dof_damping, actuator_gainprm and body_mass scales to '
                   '1.3e-4, 4.9e-5 and 1.3e-3, but density ends at 0.978 against 0.85.  The density column agrees with fp64 at s = 1 and '
                   'the predictions at s* reproduce the data bit for bit, but near s* the predicted response to a 1 % density change is '
                   'not smooth (DESIGN section 6)')
def test_gpu_gauss_newton():
    ge.build()
    check_gauss_newton(None)


@pytest.mark.gpu
def test_gpu_least_squares():
    ge.build()
    check_least_squares(None)


@pytest.mark.gpu
def test_gpu_isolation_and_refusals():
    ge.build()
    check_isolation(None, 4096)
    check_refusals(None)
