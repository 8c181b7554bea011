"""Sensors in the dynamics queries (fb_query_sensors): the inverse's sensordata, the transition's C and D and the inverse's DsDq / DsDv /
DsDa, against the fp64 restatement of tests/sensor_fd_reference.py; known answers that pin "the sensors of x"; bits that the switch does
not change; determinism, refusals, a model without sensors and the Python front ends.  CPU tier: the host-emulation build of the kernel
source; GPU tier (-m gpu): the same through the CUDA library on full-size handles.  "Bit-identical" compares uint32 views.

The Jacobian error is test_transition_fd's per-column error: per input, the largest entry error relative to the column's largest reference
entry, floored at 1e-3 of the matrix's largest entry.  Touch and force rows on contact states are not smooth in the inputs (a nudge moves
a contact across a cone zone or its activation), so contact states are gated on the worst and on the median column, as the other FD
tests do.  Sensordata itself is gated per value relative to the largest value of its sensor type.

Tolerances are 2.5 x the larger of the host-emulation and H100 measurements (the worst case is named beside each constant)."""
import numpy as np
import pytest

import __graft_entry__ as ge
from flybody_b200 import derivatives as dv, inverse_dynamics as idy, stepper as st
from flybody_b200.flymodel import load_model

import inverse_fd_reference as ifr
import sensor_fd_reference as sr
import smooth_states as ss
import solver_states as sv
from test_transition_fd import col_errors

# ---- gates (measured: host emulation / H100 80GB HBM3 at a 700 W power limit; worst case) -------------------------------------------------
SENS_VALUE = 2.8e-4        # sensordata against the reference, per value relative to its type's largest: measured 5.3e-5 emu / 1.1e-4 H100
                           # (the nominal of the contact states)
STEP_MATCH = 2.3e-2        # the inverse's sensordata at the device's forward qacc against the step's of the same state, force and touch
                           # relative to the contact-force scale: measured 9.2e-3 emu / 7.3e-3 H100 (the fp32 solver's efc_force against
                           # the inverse's at its own qacc; velocity and accelerometer rows agree to rounding)
LINEAR = 3.5e-3            # the linear blocks (velocity sensors in qvel, accelerometer in qacc) against exact unit differences: measured
                           # 8.5e-4 emu ('flight') / 1.4e-3 H100 ('walk')
FREE_ERR = 105.0           # constraint-free states, worst column of C / D / DsD*: measured 42 emu / 42 H100 ('ball' 'quat_w0'), the fp32
                           # rounding of a large term over the step in a column whose reference entries are small (test_inverse_fd's FREE_ERR)
CONTACT_ERR = 24.0         # contact states, worst column: measured 0.97 emu / 9.4 H100 ('condim13', forward)
CONTACT_MEDIAN = 2.4e-3    # contact states, per state the median column: measured 5.1e-4 emu / 9.3e-4 H100

EPS = 1e-3                 # the eps the gates were measured at


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def rounded(x):
    return np.asarray(x, np.float64).astype(np.float32).astype(np.float64)


@pytest.fixture(scope='module')
def emu():
    ge.build()
    return ge.EMU


def value_error(dev, ref, m, contact_scale=False, force=True):
    """per value, |dev - ref| relative to the largest |ref| of its sensor type (at least 1e-3).  A force sensor reads the small
    difference of its subtree's m a and weight: its floor is the heaviest force-sensor subtree's mass times the largest accelerometer
    reading.  contact_scale: force and touch rows relative to the largest of either (the contact forces both are made of); force=False
    leaves the force rows out"""
    dev, ref = np.asarray(dev, np.float64), np.asarray(ref, np.float64)
    vel, acc, frc, touch = sr.stage_rows(m)
    groups = [vel, acc, np.concatenate([frc, touch])] if contact_scale else [vel, acc, frc if force else frc[:0], touch]
    floor = {id(frc): sr.force_subtree_mass(m) * np.abs(ref[..., acc]).max()} if len(frc) and len(acc) else {}
    err = 0.0
    for rows in groups:
        if len(rows):
            scale = max(np.abs(ref[..., rows]).max(), 1e-3, floor.get(id(rows), 0.0))
            err = max(err, float(np.abs(dev[..., rows] - ref[..., rows]).max() / scale))
    return err


_ANALYTIC = {}


def analytic(noslip=0):
    if noslip not in _ANALYTIC:
        _ANALYTIC[noslip] = sv.analytic_model(load_model('walk'), noslip=noslip)
    return _ANALYTIC[noslip]


def forward_qacc(run, q, v, ctrl=None, act=None):
    k = 3 if run.ball else 0
    run.o.reset(run.to_q(q), np.concatenate([np.zeros(k), v]))
    if act is not None and run.m.na:
        run.o.set(ifr.fo.ACT, act)
    if ctrl is not None:
        run.o.set(ifr.fo.CTRL, ctrl)
    run.o.forward()
    return rounded(run.o.qacc[k:])


def solver_cases(noslip, names=None):
    """analytic-walk states: name -> (q, v, ctrl, forward qacc)"""
    m = analytic(noslip)
    run = ifr.Inverse(m)
    out = {}
    for k in names or list(sv.STATES):
        q, v, ctrl = sv.state_inputs(m, *sv.STATES[k][0])
        out[k] = (q, v, ctrl, forward_qacc(run, q, v, ctrl))
    return m, out


def free_cases(name):
    """constraint-free states of a model: name -> (q, v, ctrl, act, forward qacc)"""
    m = ss.free_model(ss.base_model(name))
    run = ifr.Inverse(m)
    out = {}
    for k in ss.state_names(m):
        q, v, act, ctrl = ss.state_inputs(m, k)
        out[k] = (q, v, ctrl, act, forward_qacc(run, q, v, ctrl, act))
    return m, out


def stack(cases, idx):
    return [np.array([c[i] for c in cases.values()]) for i in idx]


# ---- 1. isolation: the switch changes no other output ---------------------------------------------------------------------------------
FIELDS = (st.QPOS, st.QVEL, st.QACC, st.SENSORDATA, st.XPOS, st.SITE_XPOS, st.NCON, st.NEFC, st.QFRC_BIAS, st.QFRC_PASSIVE,
          st.CONTACT, st.EFC_FORCE, st.QM_DENSE)


def check_isolation(lib):
    m, cases = solver_cases(0, ['one_contact', 'nefc31_zones'])
    q, v, u, a = stack(cases, range(4))
    res = {}
    for on in (False, True):
        sim = st.BatchedStepper(m, 2, lib_path=lib)
        sim.query_sensors(on)
        sim.reset(q, v)
        sim.set_control(u)
        l0 = sim.launch_count
        sim.inverse(a)
        launches = sim.launch_count - l0
        res[on] = dict(inv=sim.inverse_read(), rec=[sim.get(f) for f in FIELDS], launches=launches)
        sim.close()
    assert res[False]['launches'] == 5 and res[True]['launches'] == 6
    for x, y in zip(res[False]['inv'] + tuple(res[False]['rec']), res[True]['inv'] + tuple(res[True]['rec'])):
        assert np.array_equal(bits(x), bits(y))
    # the FD calls: on / off give the same A, B, next state, DfD*, DmDq; fb_inverse_read and the bank are untouched
    ncol_t, ncol_i = 1 + 2 * m.nv + m.na + m.nu, 1 + 3 * m.nv
    out = {}
    for on in (False, True):
        sim = st.BatchedStepper(m, 2 * max(ncol_t, ncol_i), lib_path=lib)
        sim.query_sensors(on)
        rows = np.minimum(np.arange(sim.n_envs), 1)
        sim.reset(q[rows], v[rows])
        sim.set_control(u[rows])
        sim.forward()
        sim.inverse(a)
        before = sim.inverse_read()
        sim.state_bank(2)
        sim.save_state(slots=[0, 1], env_ids=[0, 1])
        bank = sim.read_states([0, 1])
        l0 = sim.launch_count
        sim.fd_transition([0, 1], eps=EPS, centered=False, n_substeps=3)
        l1 = sim.launch_count
        fd = sim.fd_read()
        sim.fd_inverse(q, v, a, eps=EPS, centered=False)
        l2 = sim.launch_count
        fdi = sim.fd_inverse_read()
        assert all(np.array_equal(bits(x), bits(y)) for x, y in zip(before, sim.inverse_read()))
        assert np.array_equal(sim.read_states([0, 1]), bank)
        out[on] = (fd, fdi, l1 - l0, l2 - l1)
        sim.close()
    for x, y in zip(out[False][0] + out[False][1], out[True][0] + out[True][1]):
        assert np.array_equal(bits(x), bits(y))
    # sensors on adds the two snapshots of x (transition) and kinv_sensors (inverse); the sensor differences are in the one diff launch
    assert out[True][2] == out[False][2] + 2 and out[True][3] == out[False][3] + 1


def test_isolation_and_launch_counts_under_emulation(emu):
    check_isolation(emu)


# ---- 2. known answers ------------------------------------------------------------------------------------------------------------------
def check_known_answers(lib, name='flight'):
    """constraint-free states: D's and DsDa's velocity-sensor rows are exactly 0, touch rows of C, D, DsD* are exactly 0; the velocity
    sensors are linear in qvel and the accelerometer in qacc, so those blocks equal exact fp64 unit differences"""
    m, cases = free_cases(name)
    vel, accel, _, touch = sr.stage_rows(m)
    q, v, u, act, a = stack(cases, range(5))
    T = dv.transition_fd(m, q, v, u, act, eps=EPS, centered=True, lib_path=lib, sensors=True)
    I = dv.inverse_fd(m, q, v, a, eps=EPS, centered=True, lib_path=lib, sensors=True)
    assert not T.D[:, vel].any() and not I.DsDa[:, :, vel].any()
    if len(touch):
        assert not T.C[:, touch].any() and not T.D[:, touch].any()
        assert not any(x[:, :, touch].any() for x in (I.DsDq, I.DsDv, I.DsDa))
    run, inv = sr.Forward(m), sr.InverseSensors(m)
    err = 0.0
    for p, (q0, v0, u0, a0, qa0) in enumerate(cases.values()):
        base = run((q0, np.zeros(m.nv), a0, u0))
        unit = np.array([run((q0, np.eye(m.nv)[j], a0, u0)) - base for j in range(m.nv)])      # [nv, nsd]
        ref = unit[:, vel]
        err = max(err, col_errors(T.C[p][vel][:, m.nv:2 * m.nv], ref.T).max(), col_errors(I.DsDv[p][:, vel].T, ref.T).max())
        if len(accel):
            b0 = inv(q0, v0, np.zeros(m.nv))
            acc = np.array([inv(q0, v0, np.eye(m.nv)[j]) - b0 for j in range(m.nv)])[:, accel]
            err = max(err, col_errors(I.DsDa[p][:, accel].T, acc.T).max())
    print(f'{name}: linear blocks {err:.1e}')
    assert err <= LINEAR


def test_known_answers_under_emulation(emu):
    check_known_answers(emu, 'flight')


# ---- 3. the inverse's sensordata ------------------------------------------------------------------------------------------------------
def check_inverse_sensordata(lib, noslip=0, names=None):
    """against the reference at forward's qacc and at a perturbed qacc; at the device's own forward qacc (noslip off) against the step's
    sensordata of the state (fb_forward): the two differ only by the inverse's efc_force against the solver's"""
    m, cases = solver_cases(noslip, names)
    q, v, u, a = stack(cases, range(4))
    rs = np.random.RandomState(5)
    a2 = rounded(a + rs.normal(size=a.shape) * np.abs(a).max(axis=1, keepdims=True) * 1e-2)
    ref = sr.InverseSensors(m)
    out = {}
    for tag, acc in (('fwd', a), ('perturbed', a2)):
        r = idy.inverse(m, q, v, acc, lib_path=lib, sensors=True)
        want = np.array([ref(*x) for x in zip(q, v, acc)])
        out[tag] = value_error(r.sensordata, want, m)
        if tag == 'fwd' and noslip == 0:
            sim = st.BatchedStepper(m, len(q), lib_path=lib)
            sim.query_sensors(True)
            sim.reset(q, v)
            sim.set_control(u)
            sim.forward()
            step = sim.get(st.SENSORDATA)
            sim.inverse(sim.get(st.QACC))
            out['step'] = value_error(sim.inverse_sensor_read(), step, m, contact_scale=True)
            sim.close()
    print(f'noslip={noslip}: {out}')
    assert out['fwd'] <= SENS_VALUE and out['perturbed'] <= SENS_VALUE and out.get('step', 0.0) <= STEP_MATCH


@pytest.mark.parametrize('noslip', [0, None])
def test_inverse_sensordata_under_emulation(emu, noslip):
    check_inverse_sensordata(emu, noslip, ['one_contact', 'nefc31_zones', 'nefc33'])


# ---- 4. the Jacobians against the reference ------------------------------------------------------------------------------------------
def jac_errors(lib, m, cases, centered, free, force=True):
    """per state: (worst column, median column) over C, D, DsDq, DsDv, DsDa; and the nominal sensordata's value error over the states"""
    q, v, u, act = stack(cases, range(4))
    a = np.array([c[-1] for c in cases.values()])
    T = dv.transition_fd(m, q, v, u, act if free else None, eps=EPS, centered=centered, lib_path=lib, sensors=True)
    I = dv.inverse_fd(m, q, v, a, eps=EPS, centered=centered, lib_path=lib, sensors=True)
    run, inv = sr.Forward(m), sr.InverseSensors(m)
    out, nom = {}, []
    for p, k in enumerate(cases):
        c = cases[k]
        C, D, s0 = sr.transition_sensors_fd(m, c[0], c[1], c[3] if free else None, c[2], eps=EPS, centered=centered, run=run)
        R = sr.inverse_sensors_fd(m, c[0], c[1], c[-1], eps=EPS, centered=centered, run=inv)
        e = [col_errors(T.C[p], C), col_errors(T.D[p], D)] + [col_errors(getattr(I, n)[p].T, R[n].T) for n in ('DsDq', 'DsDv', 'DsDa')]
        e = np.concatenate(e)
        out[k] = (float(e.max()), float(np.median(e)))
        nom.append((s0, R['sensordata']))
    s0, sr0 = (np.array(x) for x in zip(*nom))
    return out, max(value_error(T.sensordata, s0, m, force=force), value_error(I.sensordata, sr0, m, force=force))


def report(tag, out, nominal):
    print(tag, {k: f'worst {a:.1e} median {b:.1e}' for k, (a, b) in out.items()}, f'nominal {nominal:.1e}')


def check_free(lib, name, centered, n_states=None):
    m, cases = free_cases(name)
    cases = {k: (c[0], c[1], c[2], c[3], c[4]) for k, c in list(cases.items())[:n_states]}
    # the nominal without the force rows: with no contacts a tarsus force sensor is the small difference of its subtree's m a and weight,
    # and at these states' accelerations that difference lies near the fp32 rounding of its terms; the contact states gate it
    out, nominal = jac_errors(lib, m, cases, centered, True, force=False)
    report(f'{name} centered={centered}', out, nominal)
    assert max(x[0] for x in out.values()) <= FREE_ERR and nominal <= SENS_VALUE


def check_contacts(lib, noslip, centered, names=None):
    m, cases = solver_cases(noslip, names)
    cases = {k: (c[0], c[1], c[2], np.zeros(m.na), c[3]) for k, c in cases.items()}
    out, nominal = jac_errors(lib, m, cases, centered, False)
    report(f'contacts noslip={noslip} centered={centered}', out, nominal)
    assert max(x[0] for x in out.values()) <= CONTACT_ERR and max(x[1] for x in out.values()) <= CONTACT_MEDIAN and nominal <= SENS_VALUE


@pytest.mark.parametrize('name', ['flight', 'ball'])
def test_constraint_free_states_under_emulation(emu, name):
    check_free(emu, name, False)


@pytest.mark.parametrize('noslip', [0, None])
def test_contact_states_under_emulation(emu, noslip):
    check_contacts(emu, noslip, False, ['one_contact', 'nefc31_zones'])


# ---- 5. determinism ------------------------------------------------------------------------------------------------------------------
def check_positions(lib, n_big):
    """a problem's bits alone on a one-problem handle and at other positions of a larger handle with padding envs"""
    m, cases = free_cases('flight')
    q, v, u, act, a = stack(cases, range(5))
    q, v, u, act, a = q[:3], v[:3], u[:3], act[:3], a[:3]
    ncol_i, ncol_t = 1 + 3 * m.nv, 1 + 2 * m.nv + m.na + m.nu
    one = st.BatchedStepper(m, max(ncol_i, ncol_t), lib_path=lib)
    one.query_sensors(True)
    one.fd_inverse(q[1:2], v[1:2], a[1:2], eps=EPS, centered=False)
    xi = one.fd_inverse_sensor_read()
    rows = [1] * one.n_envs
    one.reset(q[rows], v[rows])
    one.set(st.ACT, act[rows])
    one.set_control(u[rows])
    one.forward()
    one.state_bank(1)
    one.save_state(slots=[0], env_ids=[0])
    one.fd_transition([0], eps=EPS, centered=False, n_substeps=2)
    xt = one.fd_sensor_read()
    one.reset(q[rows], v[rows])
    one.inverse(a[1:2])
    xs = one.inverse_sensor_read()
    one.close()
    big = st.BatchedStepper(m, n_big, lib_path=lib)
    big.query_sensors(True)
    per_i, per_t = n_big // ncol_i, n_big // ncol_t
    order = [2, 0] + [1] * (per_i - 2)
    big.fd_inverse(q[order], v[order], a[order], eps=EPS, centered=False)
    yi = big.fd_inverse_sensor_read()
    ot = [2, 1] + [0] * (big.n_envs - 2)
    big.reset(q[ot], v[ot])
    big.set(st.ACT, act[ot])
    big.set_control(u[ot])
    big.forward()
    big.state_bank(per_t)
    big.save_state(slots=np.arange(per_t), env_ids=np.arange(per_t))
    big.fd_transition(np.arange(per_t), eps=EPS, centered=False, n_substeps=2)
    yt = big.fd_sensor_read()
    oi = [0] * 5 + [1]
    big.reset(q[oi + [0] * (big.n_envs - 6)], v[oi + [0] * (big.n_envs - 6)])
    big.inverse(a[oi])
    ys = big.inverse_sensor_read()
    big.close()
    assert n_big > per_i * ncol_i and n_big > per_t * ncol_t
    for s, t in zip(xi, yi):
        for p in [i for i, k in enumerate(order) if k == 1]:
            assert np.array_equal(bits(s[0]), bits(t[p]))
    for s, t in zip(xt, yt):
        assert np.array_equal(bits(s[0]), bits(t[1]))
    assert np.array_equal(bits(xs[0]), bits(ys[5]))


def test_positions_under_emulation(emu):
    check_positions(emu, 2 * 145 + 7 + 300)


# ---- 6. refusals, a model without sensors, Python ---------------------------------------------------------------------------------------
def no_sensor_model():
    a = load_model('flight').copy()
    for k in ('sensor_type', 'sensor_objid', 'sensor_adr', 'sensor_dim'):
        a.a[k] = np.zeros(0, np.int32)
    for k in ('nsensor', 'nsensordata'):
        a.a[k] = a.meta[k] = 0
    return a.rebuild()


def check_refusals(lib):
    m, cases = free_cases('flight')
    q, v, u, act, a = stack(cases, range(5))
    sim = st.BatchedStepper(m, 2 * (1 + 3 * m.nv), lib_path=lib)
    for read, what in ((sim.inverse_sensor_read, 'no inverse'), (sim.fd_sensor_read, 'no transition'), (sim.fd_inverse_sensor_read, 'no Jacobians')):
        with pytest.raises(st.StepperError, match=what):
            read()
    sim.inverse(a[:2])
    sim.fd_inverse(q[:2], v[:2], a[:2], eps=EPS, centered=False)
    sim.state_bank(1)
    sim.save_state(slots=[0], env_ids=[0])
    sim.fd_transition([0], eps=EPS, centered=False)
    for read in (sim.inverse_sensor_read, sim.fd_sensor_read, sim.fd_inverse_sensor_read):
        with pytest.raises(st.StepperError, match='sensors off'):
            read()
    sim.query_sensors(True)
    with pytest.raises(st.StepperError, match='non-finite qacc'):
        sim.inverse(np.full((2, m.nv), np.nan))
    with pytest.raises(st.StepperError, match='NULL'):
        sim._check(sim._lib.fb_inverse(sim._h, 2, None, 0), 'fb_inverse')
    with pytest.raises(st.StepperError, match='sensors off'):
        sim.inverse_sensor_read()                              # a refused call leaves the last call's state
    sim.inverse(a[:2])
    assert sim.inverse_sensor_read().shape == (2, m.nsensordata)
    sim._check(sim._lib.fb_inverse_sensor_read(sim._h, None, 0), 'fb_inverse_sensor_read')
    sim.close()
    # nsensordata == 0: valid, nothing more launched, empty outputs
    z = no_sensor_model()
    assert z.nsensordata == 0
    sim = st.BatchedStepper(z, 1 + 3 * z.nv, lib_path=lib)
    sim.query_sensors(True)
    sim.reset(q[:1], v[:1])
    l0 = sim.launch_count
    sim.inverse(a[:1])
    assert sim.launch_count - l0 == 5
    assert sim.inverse_sensor_read().shape == (1, 0)
    sim.fd_inverse(q[:1], v[:1], a[:1], eps=EPS, centered=False)
    assert [x.shape for x in sim.fd_inverse_sensor_read()] == [(1, z.nv, 0)] * 3 + [(1, 0)]
    sim.close()
    T = dv.transition_fd(z, q[0], v[0], u[0], act[0], eps=EPS, centered=False, lib_path=lib, sensors=True)
    assert T.C.shape == (0, 2 * z.nv + z.na) and T.D.shape == (0, z.nu) and T.sensordata.shape == (0,)


def test_refusals_under_emulation(emu):
    check_refusals(emu)


def test_python_front_ends(emu):
    m, cases = solver_cases(0, ['one_contact', 'nefc31_zones', 'nefc33'])
    q, v, u, a = stack(cases, range(4))
    plain = idy.inverse(m, q, v, a, lib_path=emu)
    withs = idy.inverse(m, q, v, a, lib_path=emu, sensors=True)
    assert type(plain) is idy.InverseResult and withs._fields == idy.InverseResult._fields + ('sensordata',)
    for x, y in zip(plain[:4], withs[:4]):
        assert np.array_equal(x, y)
    assert withs.sensordata.shape == (3, m.nsensordata) and withs.sensordata.dtype == np.float64
    one = idy.inverse(m, q[1], v[1], a[1], lib_path=emu, sensors=True)
    assert np.array_equal(one.sensordata, withs.sensordata[1])
    T0 = dv.transition_fd(m, q[:2], v[:2], u[:2], eps=EPS, centered=False, lib_path=emu)
    T1 = dv.transition_fd(m, q[:2], v[:2], u[:2], eps=EPS, centered=False, lib_path=emu, sensors=True)
    assert type(T0) is dv.Transition and T1._fields == dv.Transition._fields + ('C', 'D', 'sensordata')
    assert all(np.array_equal(x, y) for x, y in zip(T0, T1[:5]))
    assert T1.C.shape == (2, m.nsensordata, 2 * m.nv + m.na) and T1.D.shape == (2, m.nsensordata, m.nu)
    t1 = dv.transition_fd(m, q[1], v[1], u[1], eps=EPS, centered=False, lib_path=emu, sensors=True)
    assert np.array_equal(t1.C, T1.C[1]) and np.array_equal(t1.sensordata, T1.sensordata[1])
    I0 = dv.inverse_fd(m, q, v, a, eps=EPS, centered=False, lib_path=emu)
    I1 = dv.inverse_fd(m, q, v, a, eps=EPS, centered=False, lib_path=emu, sensors=True)
    assert type(I0) is dv.InverseJacobians and I1._fields == dv.InverseJacobians._fields + ('DsDq', 'DsDv', 'DsDa', 'sensordata')
    assert all(np.array_equal(x, y) for x, y in zip(I0, I1[:5]))
    assert I1.DsDq.shape == (3, m.nv, m.nsensordata)
    # the nominal sensordata of the inverse FD is the inverse's
    assert np.array_equal(I1.sensordata, withs.sensordata.astype(np.float32).astype(np.float64))


# ---- GPU tier ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_gpu_isolation_launch_counts_determinism_and_refusals():
    ge.build()
    check_isolation(None)
    check_positions(None, 4096)
    check_refusals(None)


@pytest.mark.gpu
def test_gpu_known_answers():
    ge.build()
    for name in ('flight', 'walk'):
        check_known_answers(None, name)


@pytest.mark.gpu
@pytest.mark.parametrize('noslip', [0, None])
def test_gpu_inverse_sensordata(noslip):
    ge.build()
    check_inverse_sensordata(None, noslip)


@pytest.mark.gpu
@pytest.mark.parametrize('centered', [False, True])
@pytest.mark.parametrize('name', ss.DEFAULT_MODELS)
def test_gpu_constraint_free_states(name, centered):
    ge.build()
    check_free(None, name, centered, 4)


GPU_CONTACT_STATES = ['one_contact', 'one_limit', 'nefc31_zones', 'condim13']     # the fp64 reference costs 3 (nx + nu) forwards per state


@pytest.mark.gpu
@pytest.mark.parametrize('centered', [False, True])
@pytest.mark.parametrize('noslip', [0, None])
def test_gpu_contact_states(noslip, centered):
    ge.build()
    check_contacts(None, noslip, centered, GPU_CONTACT_STATES)
