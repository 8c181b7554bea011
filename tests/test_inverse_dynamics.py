"""Batched inverse dynamics (fb_inverse, flybody_b200.inverse_dynamics) against an fp64 restatement of MuJoCo's mj_inverse at the oracle's
state (tests/inverse_reference.py), the forward solve against its own inverse, isolation from the step, and the Python front end.
CPU tier: the host-emulation build of the kernel source; GPU tier (-m gpu): the same comparisons through the CUDA library, at 4096
problems.  "Bit-identical" compares uint32 views.

Tolerances are 2.5 x the larger of the host-emulation and H100 measurements (the worst state is named beside each constant)."""
import ctypes as C

import numpy as np
import pytest

import __graft_entry__ as ge
from flybody_b200 import inverse_dynamics as invd, inverse_kinematics as ik, stepper as st
from flybody_b200.flymodel import load_model
from oracle import fly_oracle as fo

import inverse_reference as ir
import smooth_states as ss
import solver_states as sv

# ---- gates (measured: host emulation / H100 80GB HBM3 at a 700 W power limit, 4096-env batches; worst state) ------------------------------
# The contact gates are set by the fp32 evaluation of jar = J qacc - aref, not by the kernel's arithmetic: where a row's terms cancel,
# its force can only be resolved to about 2^-24 of them times its stiffness (tests/solver_states.py: jar_resolution).  The consistency
# gate is the fp32 forward solve's own convergence.
ORACLE_SELF = 2.5e-12      # oracle forward (tolerance 1e-12), then its own inverse, per dof in the inertia metric: measured 8.7e-13 ('one_contact')
FREE_FORCE = 2.5e-6        # qfrc_inverse per dof, inertia metric, constraint-free states: measured 9.3e-7 emu / 9.8e-7 H100 ('walk_force' flight)
CONTACT_MAXREL = 7.1e-4    # efc_force, max over rows relative to the state's largest force: measured 9.2e-5 emu ('reg_cols24') / 2.8e-4 H100 ('reg_cols25')
CONTACT_PER = 3.8e-3       # efc_force per contact / limit row (FLOOR convention of tests/solver_states.py): measured 1.3e-3 emu / 1.5e-3 H100 ('middle_mu1_a', noslip)
CONTACT_FORCE = 1.8e-3     # qfrc_constraint and qfrc_inverse per dof, inertia metric: measured 4.1e-4 emu ('nefc32') / 7.2e-4 H100 ('nefc31_zones')
CONSISTENCY = 0.14         # stepper forward -> inverse against applied + actuator, inertia metric (see consistency_errors): measured 5.0e-2 emu ('middle_mu1_b') / 5.6e-2 H100 ('rows105')

FREE_MODELS = ss.DEFAULT_MODELS


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


@pytest.fixture(scope='module')
def emu():
    ge.build()
    return ge.EMU


_ANALYTIC = {}


def analytic(noslip):
    if noslip not in _ANALYTIC:
        _ANALYTIC[noslip] = sv.analytic_model(load_model('walk'), noslip=noslip)
    return _ANALYTIC[noslip]


def rounded(x):
    return np.asarray(x, np.float64).astype(np.float32).astype(np.float64)


def device_inverse(sim, q, v, qacc, act=None, ctrl=None):
    """reset the first len(q) envs (the rest keep theirs) to states (q, v[, act, ctrl]) and run the inverse of qacc on them"""
    n = len(q)
    Q, V = sim.get(st.QPOS).astype(np.float64), sim.get(st.QVEL).astype(np.float64)
    Q[:n], V[:n] = q, v
    sim.reset(Q, V)
    if act is not None:
        A = sim.get(st.ACT); A[:n] = act; sim.set(st.ACT, A)
    if ctrl is not None:
        U = sim.get(st.CTRL); U[:n] = ctrl; sim.set_control(U)
    sim.inverse(np.asarray(qacc, np.float32), n=n)
    qi, qc, f = sim.inverse_read()
    return qi.astype(np.float64), qc.astype(np.float64), f.astype(np.float64)


# ---- 1. the reference against the oracle's own forward solve -------------------------------------------------------------------------
def oracle_self_error(name, noslip=0):
    m = analytic(noslip)
    o = fo.Oracle(m, tolerance=1e-12)
    q, v, ctrl = sv.state_inputs(m, *sv.STATES[name][0])
    o.reset(q, v)
    o.set(fo.CTRL, ctrl)
    o.forward()
    r = ir.inverse(m, o, o.qacc)
    # the oracle has no applied-force input: the forward's non-constraint force is the actuation alone
    return ss.force_error(r['qfrc_inverse'], o.get(fo.QFRC_ACTUATOR), r['M'])


@pytest.mark.parametrize('name', list(sv.STATES))
def test_oracle_inverse_returns_the_forward_forces(name):
    err = oracle_self_error(name)
    print(f'{name}: oracle forward -> inverse {err:.2e}')
    assert err <= ORACLE_SELF


# ---- 2. known answer --------------------------------------------------------------------------------------------------------------------
def check_known_answer(lib):
    m = ss.free_model(load_model('flight'))
    sim = st.BatchedStepper(m, 4, lib_path=lib)
    sim.reset(m.qpos0)
    sim.inverse(np.zeros((4, m.nv), np.float32))
    qi, qc, f = sim.inverse_read()
    bias, passive = sim.get(st.QFRC_BIAS), sim.get(st.QFRC_PASSIVE)
    assert np.array_equal(bits(qi), bits(bias - passive)) and not qc.any() and not f.any()
    root = [j for j in range(m.njnt) if m.jnt_type[j] == ss.FREE][0]
    rb, da = int(m.jnt_bodyid[root]), int(m.jnt_dofadr[root])
    sub = [b for b in range(m.nbody) if any(a == rb for a in _ancestors(m, b))]
    weight = -m.body_mass[sub].sum() * np.asarray(m.opt_gravity, np.float64)
    sim.close()
    # the weight held up, to fp32 rounding of the composite inertia
    assert np.abs(qi[:, da:da + 3] - weight).max() <= 1e-5 * np.abs(weight).max(), (qi[0, da:da + 3], weight)


def _ancestors(m, b):
    while b > 0:
        yield b
        b = int(m.body_parentid[b])


def test_known_answer_weight_held_up(emu):
    check_known_answer(emu)


# ---- 3. constraint-free states ------------------------------------------------------------------------------------------------------
def random_qacc(qacc, seed):
    """a random acceleration of the size of the state's own: qacc (1 + N(0, 1/2)), rounded to fp32"""
    rs = np.random.RandomState(seed)
    return rounded(qacc * (1 + 0.5 * rs.normal(size=qacc.shape)) + 1e-3 * rs.normal(size=qacc.shape))


def oracle_free_inverse(m, name, seed=0):
    """the oracle's inverse of state `name` on the free model m, for a random fp32 qacc; ball joints through the free surrogate"""
    q, v, act, ctrl = ss.state_inputs(m, name)
    ball = bool(ss._joints(m, ss.BALL))
    if ball:
        from test_walk_on_ball import free_surrogate, to_surrogate_q
        mo = free_surrogate(m)
        o = fo.Oracle(mo, tolerance=1e-12)
        o.reset(to_surrogate_q(m, q), np.concatenate([np.zeros(3), v]))
    else:
        mo, o = m, fo.Oracle(m, tolerance=1e-12)
        o.reset(q, v)
    if m.na:
        o.set(fo.ACT, act)
    o.set(fo.CTRL, ctrl)
    o.forward()
    qacc = random_qacc(o.qacc[3:] if ball else o.qacc, seed)
    r = ir.inverse(mo, o, np.concatenate([np.zeros(3), qacc]) if ball else qacc)
    if ball:
        r = {k: (x[3:] if k != 'M' else x[3:, 3:]) for k, x in r.items() if k in ('qfrc_inverse', 'M')}
    return (q, v, act, ctrl), qacc, r


def free_errors(name_model, lib, n_envs=None):
    m = ss.free_model(ss.base_model(name_model))
    names = ss.state_names(m)
    cases = [oracle_free_inverse(m, k, seed=i) for i, k in enumerate(names)]
    sim = st.BatchedStepper(m, n_envs or len(names), lib_path=lib)
    reps = (n_envs or len(names)) // len(names)
    idx = np.tile(np.arange(len(names)), reps)
    qi, _, _ = device_inverse(sim, *[np.array([cases[i][0][c] for i in idx]) for c in (0, 1)], np.array([cases[i][1] for i in idx]),
                              act=np.array([cases[i][0][2] for i in idx]) if m.na else None)
    sim.close()
    errs = {}
    for e, i in enumerate(idx):
        r = cases[i][2]
        errs[names[i]] = max(errs.get(names[i], 0.0), ss.force_error(qi[e], r['qfrc_inverse'], r['M']))
    return errs


@pytest.mark.parametrize('name', FREE_MODELS + list(ss.ov.VARIANTS))
def test_constraint_free_states_under_emulation(emu, name):
    errs = free_errors(name, emu)
    print(name, {k: f'{v:.1e}' for k, v in errs.items()})
    assert max(errs.values()) <= FREE_FORCE


# ---- 4. contact states ------------------------------------------------------------------------------------------------------------------
def contact_case(name, noslip):
    """the oracle's fp64 inverse of solver state `name` at the forward solve's qacc (rounded to fp32): inputs and reference"""
    m = analytic(noslip)
    o = fo.Oracle(m, tolerance=1e-12)
    q, v, ctrl = sv.state_inputs(m, *sv.STATES[name][0])
    o.reset(q, v)
    o.set(fo.CTRL, ctrl)
    o.forward()
    qacc = rounded(o.qacc)
    r = ir.inverse(m, o, qacc)
    ncon = int(o.get(fo.NCON)[0])
    con = o.get(fo.CONTACT).reshape(-1, 16)[:ncon] if ncon else np.zeros((0, 16))
    r.update(nefc=len(r['efc_force']), con=con, force=r['efc_force'])
    return (q, v, ctrl, qacc), r


def contact_errors(noslip, lib, names=None, reps=1):
    names = names or list(sv.STATES)
    m = analytic(noslip)
    cases = [contact_case(k, noslip) for k in names]
    idx = np.tile(np.arange(len(names)), reps)
    sim = st.BatchedStepper(m, len(idx), lib_path=lib)
    qi, qc, f = device_inverse(sim, *[np.array([cases[i][0][c] for i in idx]) for c in (0, 1)], np.array([cases[i][0][3] for i in idx]),
                               ctrl=np.array([cases[i][0][2] for i in idx]))
    nefc, ncon, con = sim.get(st.NEFC)[:, 0].astype(int), sim.get(st.NCON)[:, 0].astype(int), sim.get(st.CONTACT)
    sim.close()
    out = {}
    for e, i in enumerate(idx):
        r = cases[i][1]
        dev = dict(nefc=nefc[e], con=con[e].astype(np.float64).reshape(-1, 16)[:ncon[e]], force=f[e, :nefc[e]])
        assert dev['nefc'] == r['nefc'], names[i]
        g = sv.errors(dev, r)
        assert not g['zone_mismatch'], (names[i], g['zone_mismatch'])
        assert not f[e, nefc[e]:].any()
        fe = max(ss.force_error(qc[e], r['qfrc_constraint'], r['M']), ss.force_error(qi[e], r['qfrc_inverse'], r['M']))
        prev = out.get(names[i], (0, 0, 0))
        out[names[i]] = (max(prev[0], g['maxrel']), max(prev[1], g['per']), max(prev[2], fe))
    return out


@pytest.mark.parametrize('noslip', [0, None])
def test_contact_states_under_emulation(emu, noslip):
    out = contact_errors(noslip, emu)
    for k, (a, b, c) in out.items():
        print(f'{k} noslip={noslip}: efc_force maxrel {a:.1e} per-contact {b:.1e} qfrc {c:.1e}')
    assert max(a for a, _, _ in out.values()) <= CONTACT_MAXREL
    assert max(b for _, b, _ in out.values()) <= CONTACT_PER
    assert max(c for _, _, c in out.values()) <= CONTACT_FORCE


# ---- 5. forward -> inverse on the stepper -----------------------------------------------------------------------------------------------
def consistency_errors(lib, names=None):
    names = names or list(sv.STATES)
    m = analytic(0)
    n = len(names)
    ins = [sv.state_inputs(m, *sv.STATES[k][0]) for k in names]
    rs = np.random.RandomState(7)
    sim = st.BatchedStepper(m, n, lib_path=lib)
    sim.reset(np.array([x[0] for x in ins]), np.array([x[1] for x in ins]))
    sim.set_control(np.array([x[2] for x in ins]))
    sim.set_applied(qfrc=rs.normal(size=(n, m.nv)) * 1e-3, xfrc=rs.normal(size=(n, m.nbody, 6)) * 1e-3)
    sim.forward()
    want = (sim.get(st.QFRC_SMOOTH) - sim.get(st.QFRC_PASSIVE) + sim.get(st.QFRC_BIAS)).astype(np.float64)   # applied + actuator
    qc = sim.get(st.QFRC_CONSTRAINT).astype(np.float64)
    M = sim.get(st.QM_DENSE).astype(np.float64).reshape(n, m.nv, m.nv)
    sim.inverse(sim.get(st.QACC))
    qi, _, _ = sim.inverse_read()
    sim.close()
    # per dof in the inertia metric, relative to the larger of the applied + actuator force and the forward's constraint force: M qacc
    # carries both, and the fp32 forward solve converges to a tolerance relative to the constraint forces
    out = {}
    for e, k in enumerate(names):
        s = np.sqrt(np.diag(M[e]))
        scale = max((np.abs(want[e]) / s).max(), (np.abs(qc[e]) / s).max())
        out[k] = float((np.abs(qi[e] - want[e]) / s).max() / scale)
    return out


def test_forward_inverse_consistency_under_emulation(emu):
    errs = consistency_errors(emu)
    for k, v in errs.items():
        print(f'{k}: forward -> inverse residual {v:.2e}')
    assert max(errs.values()) <= CONSISTENCY


# ---- 6. determinism and isolation ---------------------------------------------------------------------------------------------------
def record_bytes(sim):
    """the raw records of every env (host-emulation build: the device pointer is host memory; qpos opens the record)"""
    p = np.zeros(1, np.int64)
    sim._check(sim._lib.fb_get(sim._h, st.QPOS, p.ctypes.data, 1), 'fb_get')
    n = sim._lib.fb_n_envs_padded(sim._h) * sim._lib.fb_record_stride(sim._h) * 4
    return C.string_at(int(p[0]), n)


def walking_states(m, n, seed=0):
    q, v, ctrl = zip(*[sv.state_inputs(m, *sv.STATES[k][0]) for k in sv.STATES])
    idx = np.random.RandomState(seed).randint(0, len(q), n)
    return np.array(q)[idx], np.array(v)[idx], np.array(ctrl)[idx]


def check_slots_and_batches(lib, n_big):
    m = analytic(0)
    q, v, ctrl = walking_states(m, n_big)
    qacc = np.random.RandomState(3).normal(size=(n_big, m.nv)).astype(np.float32) * 10
    big = st.BatchedStepper(m, n_big, lib_path=lib)
    a = device_inverse(big, q, v, qacc, ctrl=ctrl)
    big.close()
    for s in sorted({0, 1, 5, n_big // 2, n_big - 1}):
        one = st.BatchedStepper(m, 3, lib_path=lib)
        k = 2 if s % 2 else 0                      # the same problem in another slot of a smaller batch
        qq, vv, aa = (np.repeat(x[s:s + 1], 3, 0) for x in (q, v, qacc))
        qq[1 - k // 2] = q[(s + 1) % n_big]
        b = device_inverse(one, qq, vv, aa)
        one.close()
        for x, y in zip(a, b):
            assert np.array_equal(bits(x[s]), bits(y[k])), s


def test_slots_and_batches_under_emulation(emu):
    check_slots_and_batches(emu, 24)


def check_isolation(lib, n, raw):
    """the record unchanged by an inverse on a current state, and the next control step unchanged; launches: step1's plus one"""
    m = analytic(0)
    q, v, ctrl = walking_states(m, n, seed=1)
    sims = [st.BatchedStepper(m, n, lib_path=lib) for _ in range(2)]
    for s in sims:
        s.reset(q, v)
        s.set_control(ctrl)
        s.step(2)
        s.step(2)
    a, b = sims
    fields = [f for f in range(25) if f not in (st.QACC_WARMSTART,)]
    before = record_bytes(a) if raw else {f: a.get(f).copy() for f in fields}
    l0 = a.launch_count
    a.inverse(np.random.RandomState(4).normal(size=(n, m.nv)).astype(np.float32))
    step1 = 4 + 0                                  # pos, col, proj, vel (no heightfield on this model)
    assert a.launch_count - l0 == step1 + 1
    after = record_bytes(a) if raw else {f: a.get(f) for f in fields}
    if raw:
        assert before == after
    else:
        for f in fields:
            assert np.array_equal(bits(before[f]), bits(after[f])), f
    l0, l1 = a.launch_count, b.launch_count
    for s in sims:
        s.step(2)
    assert a.launch_count - l0 == b.launch_count - l1
    for f in fields:
        assert np.array_equal(bits(a.get(f)), bits(b.get(f))), f
    for s in sims:
        s.close()


def test_isolation_under_emulation(emu):
    check_isolation(emu, 8, raw=True)


# ---- 7. refusals ------------------------------------------------------------------------------------------------------------------------
def check_refusals(lib):
    m = analytic(0)
    sim = st.BatchedStepper(m, 4, lib_path=lib)
    with pytest.raises(st.StepperError, match='no inverse to read'):
        sim._check(sim._lib.fb_inverse_read(sim._h, None, None, None, 0), 'fb_inverse_read')
    good = np.zeros((4, m.nv), np.float32)
    for n in (0, 5, -1):
        with pytest.raises(st.StepperError, match='1 <= n <= n_envs'):
            sim._check(sim._lib.fb_inverse(sim._h, n, good.ctypes.data, 0), 'fb_inverse')
    with pytest.raises(st.StepperError, match='qacc is NULL'):
        sim._check(sim._lib.fb_inverse(sim._h, 2, None, 0), 'fb_inverse')
    for bad in (np.nan, np.inf):
        q = good.copy(); q[1, 3] = bad
        with pytest.raises(st.StepperError, match='non-finite qacc'):
            sim.inverse(q)
    sim.inverse(good[:2])
    qi, qc, f = sim.inverse_read()
    assert qi.shape == (2, m.nv) and f.shape == (2, st.MAXEFC)
    sim._check(sim._lib.fb_inverse_read(sim._h, None, None, None, 0), 'fb_inverse_read')      # every pointer may be NULL
    sim.close()


def test_refusals_under_emulation(emu):
    check_refusals(emu)


# ---- 8. Python ------------------------------------------------------------------------------------------------------------------------
def analytic_track(m, dt, T=9):
    """an fp64 track: hinges q_j(t) = a_j sin(w_j t + p_j), the root moving at constant world velocity and turning at a constant
    body-frame rate; -> (qpos [T, nq], qvel, qacc [T, nv]) analytic"""
    rs = np.random.RandomState(0)
    t = np.arange(T) * dt
    q = np.repeat(m.qpos0[None].astype(np.float64), T, 0)
    qv, qa = np.zeros((T, m.nv)), np.zeros((T, m.nv))
    for j in range(m.njnt):
        qadr, dadr = int(m.jnt_qposadr[j]), int(m.jnt_dofadr[j])
        if m.jnt_type[j] == ss.HINGE:
            a, w, p = rs.uniform(0.1, 0.5), rs.uniform(5, 40), rs.uniform(0, 2 * np.pi)
            q[:, qadr] += a * np.sin(w * t + p)
            qv[:, dadr] = a * w * np.cos(w * t + p)
            qa[:, dadr] = -a * w * w * np.sin(w * t + p)
        elif m.jnt_type[j] == ss.FREE:
            lin, om = rs.normal(size=3), rs.normal(size=3) * 3
            q[:, qadr:qadr + 3] += t[:, None] * lin
            ang = np.linalg.norm(om)
            ax = om / ang
            dq = np.concatenate([np.cos(ang * t / 2)[:, None], np.sin(ang * t / 2)[:, None] * ax], 1)
            q0 = q[0, qadr + 3:qadr + 7] / np.linalg.norm(q[0, qadr + 3:qadr + 7])
            from flybody_b200.synthetic import mult_quat
            q[:, qadr + 3:qadr + 7] = mult_quat(np.broadcast_to(q0, (T, 4)), dq)      # body-frame rate om
            qv[:, dadr:dadr + 3], qv[:, dadr + 3:dadr + 6] = lin, om
    return q, qv, qa


def test_differentiate_is_second_order():
    m = load_model('template')
    errs = []
    for dt in (2e-3, 1e-3):
        q, qv, qa = analytic_track(m, dt)
        v, a = invd.differentiate(m, q, dt)
        assert v.shape == (len(q) - 2, m.nv) == a.shape
        errs.append((np.abs(v - qv[1:-1]).max(), np.abs(a - qa[1:-1]).max()))
    # halving dt quarters both errors (second order), and the root's constant turn has zero acceleration
    assert errs[1][0] < 0.3 * errs[0][0] and errs[1][1] < 0.3 * errs[0][1], errs
    assert errs[1][0] < 1e-2 and errs[1][1] < 5.0, errs


def test_inverse_chunks_and_readme_chain(emu, monkeypatch):
    m = load_model('template')
    q, _, _ = analytic_track(m, 2e-3, T=12)
    v, a = invd.differentiate(m, q, 2e-3)
    q = q[1:-1]
    whole = invd.inverse(m, q, v, a, lib_path=emu)
    monkeypatch.setattr(ik, 'CHUNK', 4)
    monkeypatch.setattr(invd, 'CHUNK', 4)
    parts = invd.inverse(m, q, v, a, lib_path=emu)
    for k in ('qfrc_inverse', 'qfrc_constraint', 'qfrc_bias', 'qfrc_passive'):
        assert np.array_equal(getattr(whole, k), getattr(parts, k)), k
    for x, y in zip(whole.contacts, parts.contacts):
        assert all(np.array_equal(xa, ya) for xa, ya in zip(x, y))
    hinges = [j for j in m.meta['observable_joints'] if 'T1_left' in j]
    tau = invd.joint_forces(m, whole.qfrc_inverse, hinges)
    assert tau.shape == (len(q), len(hinges)) and np.isfinite(tau).all()
    one = invd.inverse(m, q[0], v[0], a[0], lib_path=emu)
    assert np.array_equal(one.qfrc_inverse, whole.qfrc_inverse[0])
    with pytest.raises(ValueError):
        invd.joint_forces(m, whole.qfrc_inverse, ['walker/'])


def test_readme_chain_from_keypoints(emu):
    """qpos_from_site_xpos -> differentiate -> inverse -> joint_forces on the template model"""
    m = load_model('template')
    sim = st.BatchedStepper(m, 1, lib_path=emu)
    sim.reset(m.qpos0)
    sites = ['walker/claw_T1_left', 'walker/claw_T2_left', 'walker/claw_T3_left', 'walker/thorax']
    sid = [m.site_id(s) for s in sites]
    keys = []
    for t in range(5):
        keys.append(sim.get(st.SITE_XPOS)[0].reshape(-1, 3)[sid].astype(np.float64))
        sim.set_control(np.full(m.nu, 0.1))
        sim.step(2)
    sim.close()
    hinges = [j for j in m.meta['observable_joints'] if 'T1_left' in j and 'tarsus' not in j]
    fit = ik.qpos_from_site_xpos(m, sites, np.stack(keys), ['walker/'] + hinges, max_steps=300, lib_path=emu)
    qvel, qacc = invd.differentiate(m, fit.qpos, 2e-3)
    res = invd.inverse(m, fit.qpos[1:-1], qvel, qacc, lib_path=emu)
    tau = invd.joint_forces(m, res.qfrc_inverse, hinges)
    assert tau.shape == (3, len(hinges)) and np.isfinite(tau).all()
    assert len(res.contacts) == 3 and all(c.force.shape[1] == 6 for c in res.contacts)


# ---- GPU tier ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_gpu_known_answer_and_refusals():
    ge.build()
    check_known_answer(None)
    check_refusals(None)


@pytest.mark.gpu
@pytest.mark.parametrize('name', FREE_MODELS + list(ss.ov.VARIANTS))
def test_gpu_constraint_free_states(name):
    ge.build()
    errs = free_errors(name, None, n_envs=4096 - 4096 % len(ss.state_names(ss.free_model(ss.base_model(name)))))
    print(name, {k: f'{v:.1e}' for k, v in errs.items()})
    assert max(errs.values()) <= FREE_FORCE


@pytest.mark.gpu
@pytest.mark.parametrize('noslip', [0, None])
def test_gpu_contact_states(noslip):
    ge.build()
    out = contact_errors(noslip, None, reps=4096 // len(sv.STATES))
    for k, (a, b, c) in out.items():
        print(f'{k} noslip={noslip}: efc_force maxrel {a:.1e} per-contact {b:.1e} qfrc {c:.1e}')
    assert max(a for a, _, _ in out.values()) <= CONTACT_MAXREL
    assert max(b for _, b, _ in out.values()) <= CONTACT_PER
    assert max(c for _, _, c in out.values()) <= CONTACT_FORCE


@pytest.mark.gpu
def test_gpu_forward_inverse_consistency():
    ge.build()
    errs = consistency_errors(None)
    for k, v in errs.items():
        print(f'{k}: forward -> inverse residual {v:.2e}')
    assert max(errs.values()) <= CONSISTENCY


@pytest.mark.gpu
def test_gpu_determinism_and_isolation():
    ge.build()
    check_slots_and_batches(None, 4096)
    check_isolation(None, 4096, raw=False)
