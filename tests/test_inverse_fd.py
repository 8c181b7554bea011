"""Finite-difference inverse-dynamics Jacobians (fb_fd_inverse, flybody_b200.derivatives.inverse_fd) against an fp64 restatement of
the same definition on the oracle (tests/inverse_fd_reference.py), known answers of the inverse dynamics, determinism, isolation from
fb_inverse and the state bank, refusals and the Python front end.  CPU tier: the host-emulation build of the kernel source; GPU tier
(-m gpu): the same through the CUDA library on full-size handles.  "Bit-identical" compares uint32 views.

The outputs are transposed (row i: the derivative with respect to input i), so the error measure is test_transition_fd's per-column
error of the transposes: per input, the largest entry error relative to the row's largest reference entry, floored at 1e-3 of the
matrix's largest entry.  The nominal qfrc_inverse is gated per dof in the inertia metric (tests/smooth_states.py force_error).

Tolerances are 2.5 x the larger of the host-emulation and H100 measurements (the worst case is named beside each constant)."""
import numpy as np
import pytest

import __graft_entry__ as ge
from flybody_b200 import derivatives as dv, stepper as st
from flybody_b200.flymodel import load_model

import inverse_fd_reference as ifr
import smooth_states as ss
import solver_states as sv
from test_transition_fd import col_errors

# ---- gates (measured: host emulation / H100 80GB HBM3 at a 700 W power limit; worst case) -------------------------------------------------
REF_ORDER = 5e-5           # fp64 reference, centred eps 1e-4 against 1e-6, worst row of the four outputs: measured 2.0e-5 ('flight', 'vision'); eps 1e-5 gives
                           # the same distance, so this is the fp64 rounding of the 1e-6 side (the root's DfDv rows), the 1e-4 truncation lies below it
DFDA_M = 2.4e-3            # constraint-free DfDa against the nominal M (FB_QM_DENSE), per row: measured 9.5e-4 emu / 9.5e-4 H100 (flight states)
DFDA_SYM = 6.5e-5          # the same, max |DfDa - DfDa^T| relative to max |M|: measured 2.6e-5 emu / 2.6e-5 H100
LINEAR_ZONE = 1.9e-2       # one_limit / one_contact: DfDa against M + J^T D J, per row: measured 7.7e-3 emu / 3.0e-3 H100 ('one_contact')
DAMPING = 4.3e-3           # qvel = 0, fluid off, centred: DfDv against diag(dof_damping), relative to its largest entry: measured 1.7e-3 emu / 1.7e-3 H100
FREE_ERR = 98.0            # constraint-free states, eps 1e-3, worst row of DfDq / DfDv / DfDa / DmDq: measured 39 emu / 36 H100 ('ball' 'wings_only',
                           # forward): one fp32 ulp of a large force over the step, in a row whose reference entries are small
FREE_FORCE = 3.8e-6        # the nominal qfrc_inverse, inertia metric: measured 5.9e-7 emu ('ball' 'wings_only') / 1.5e-6 H100 ('walk_force' 'flight')
CONTACT_ERR = 3.5          # contact states, worst row: measured 0.14 emu ('nefc31_zones') / 1.4 H100 ('one_limit', forward; a template rollout state 1.4)
CONTACT_MEDIAN = 4.8e-3    # contact states, per state the median row over the four outputs: measured 3.0e-4 emu / 1.9e-3 H100 (template rollout, forward)
CONTACT_FORCE = 1.8e-3     # the nominal qfrc_inverse of the contact states, inertia metric: measured 4.0e-4 emu / 7.2e-4 H100 ('nefc31_zones')

EPS = 1e-3                 # the eps the gates were measured at (derivatives.inverse_fd defaults to 1e-2: DESIGN section 6)
OUTS = ('DfDq', 'DfDv', 'DfDa', 'DmDq')


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def rounded(x):
    return np.asarray(x, np.float64).astype(np.float32).astype(np.float64)


@pytest.fixture(scope='module')
def emu():
    ge.build()
    return ge.EMU


def row_errors(dev, ref):
    """per row (input): test_transition_fd.col_errors of the transposes"""
    return col_errors(np.asarray(dev).T, np.asarray(ref).T)


def errors(dev, ref):
    """per output: the rows' errors"""
    return {k: row_errors(dev[k], ref[k]) for k in OUTS}


def device(r, p):
    return {k: getattr(r, k)[p] for k in OUTS + ('qfrc_inverse',)}


_ANALYTIC = {}


def analytic(noslip=0):
    if noslip not in _ANALYTIC:
        _ANALYTIC[noslip] = sv.analytic_model(load_model('walk'), noslip=noslip)
    return _ANALYTIC[noslip]


def forward_qacc(run, q, v, ctrl=None, act=None):
    """the oracle's forward acceleration of a state, rounded to fp32 (a ball model: without the surrogate's dofs)"""
    k = 3 if run.ball else 0
    run.o.reset(run.to_q(q), np.concatenate([np.zeros(k), v]))
    if act is not None and run.m.na:
        run.o.set(ifr.fo.ACT, act)
    if ctrl is not None:
        run.o.set(ifr.fo.CTRL, ctrl)
    run.o.forward()
    return rounded(run.o.qacc[k:])


def free_cases(m, names, run):
    out = []
    for k in names:
        q, v, act, ctrl = ss.state_inputs(m, k)
        out.append((q, v, forward_qacc(run, q, v, ctrl, act)))
    return out


# ---- 1. the reference itself ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('name', ss.DEFAULT_MODELS)
def test_reference_is_second_order(name):
    m = ss.free_model(ss.base_model(name))
    run = ifr.Inverse(m)
    q, v, a = free_cases(m, ss.state_names(m)[:1], run)[0]
    r4 = ifr.inverse_fd(m, q, v, a, eps=1e-4, run=run)
    r6 = ifr.inverse_fd(m, q, v, a, eps=1e-6, run=run)
    err = max(row_errors(r4[k], r6[k]).max() for k in OUTS)
    print(f'{name}: centred eps 1e-4 against 1e-6 {err:.1e}')
    assert err <= REF_ORDER


# ---- 2. known answers on the stepper --------------------------------------------------------------------------------------------------
def check_dfda_is_m(lib, centered):
    """constraint-free: the inverse is linear in qacc, DfDa = M (the nominal's FB_QM_DENSE) and symmetric"""
    m = ss.free_model(load_model('flight'))
    run = ifr.Inverse(m)
    names = ss.state_names(m)
    cases = free_cases(m, names, run)
    q, v, a = (np.array([c[i] for c in cases]) for i in range(3))
    r = dv.inverse_fd(m, q, v, a, eps=EPS, centered=centered, lib_path=lib)
    sim = st.BatchedStepper(m, len(names), lib_path=lib)
    sim.reset(q, v)
    sim.forward()
    M = sim.get(st.QM_DENSE).astype(np.float64).reshape(-1, m.nv, m.nv)
    sim.close()
    rel = max(row_errors(r.DfDa[p], M[p]).max() for p in range(len(names)))
    sym = max(np.abs(r.DfDa[p] - r.DfDa[p].T).max() / np.abs(M[p]).max() for p in range(len(names)))
    return rel, sym


def check_linear_zone(lib, centered):
    """one active limit row / one contact in the bottom zone: f = -D jar on every row, so DfDa = M + J^T D J (J, D from the oracle)"""
    m = analytic()
    out = {}
    for name in ('one_limit', 'one_contact'):
        run = ifr.Inverse(m)
        q, v, ctrl = sv.state_inputs(m, *sv.STATES[name][0])
        a = forward_qacc(run, q, v, ctrl)
        e = run.o.efc()
        want = run.o.get(ifr.fo.QM_DENSE).reshape(m.nv, m.nv) + e['J'].T @ (e['D'][:, None] * e['J'])
        ref = ifr.inverse_fd(m, q, v, a, eps=EPS, centered=centered, run=run)
        assert row_errors(ref['DfDa'], want).max() < 1e-6, name          # the nudges stay in the linear zone
        r = dv.inverse_fd(m, q, v, a, eps=EPS, centered=centered, lib_path=lib)
        out[name] = float(row_errors(r.DfDa, want).max())
    return out


def check_damping(lib):
    """qvel = 0, fluid off, centred: qfrc_bias is quadratic in qvel, so DfDv = -d qfrc_passive / d qvel.  The oracle's passive force
    (orc_passive) is joint springs - dof_damping qvel + fluid forces; the model has no tendons: DfDv = diag(dof_damping)"""
    m = ss.free_model(load_model('flight'), fluid=False)
    out = {}
    for name in ('quat_a', 'flight'):
        q, _, _, _ = ss.state_inputs(m, name)
        a = rounded(np.random.RandomState(3).normal(size=m.nv))
        r = dv.inverse_fd(m, q, np.zeros(m.nv), a, eps=EPS, centered=True, lib_path=lib)
        want = np.diag(np.asarray(m.dof_damping, np.float64))
        out[name] = float(np.abs(r.DfDv - want).max() / np.abs(want).max())
    return out


def check_known_answers(lib):
    rel, sym = zip(*[check_dfda_is_m(lib, c) for c in (False, True)])
    lin = {**{f'{k} fwd': x for k, x in check_linear_zone(lib, False).items()},
           **{f'{k} ctr': x for k, x in check_linear_zone(lib, True).items()}}
    damp = check_damping(lib)
    print(f'DfDa = M: {max(rel):.1e}  symmetric: {max(sym):.1e}  linear zone: {lin}  damping: {damp}')
    assert max(rel) <= DFDA_M and max(sym) <= DFDA_SYM
    assert max(lin.values()) <= LINEAR_ZONE and max(damp.values()) <= DAMPING


def test_known_answers_under_emulation(emu):
    check_known_answers(emu)


# ---- 3. constraint-free states against the reference -----------------------------------------------------------------------------------
def free_errors(name, lib, centered, names=None):
    m = ss.free_model(ss.base_model(name))
    run = ifr.Inverse(m)
    names = names or ss.state_names(m)
    cases = free_cases(m, names, run)
    r = dv.inverse_fd(m, *[np.array([c[i] for c in cases]) for i in range(3)], eps=EPS, centered=centered, lib_path=lib)
    out = {}
    for p, (k, c) in enumerate(zip(names, cases)):
        ref = ifr.inverse_fd(m, *c, eps=EPS, centered=centered, run=run)
        M = run(*c)[1]
        out[k] = (max(e.max() for e in errors(device(r, p), ref).values()), ss.force_error(r.qfrc_inverse[p], ref['qfrc_inverse'], M))
    return out


def report(tag, out):
    print(tag, {k: f'{a:.1e} / {b:.1e}' for k, (a, b) in out.items()})


@pytest.mark.parametrize('centered', [False, True])
@pytest.mark.parametrize('name', ['flight', 'ball'])
def test_constraint_free_states_under_emulation(emu, name, centered):
    out = free_errors(name, emu, centered)
    report(f'{name} centered={centered}: worst row / nominal force', out)
    assert max(a for a, _ in out.values()) <= FREE_ERR and max(b for _, b in out.values()) <= FREE_FORCE


# ---- 4. contact states -----------------------------------------------------------------------------------------------------------------
def contact_errors(lib, centered, m, cases):
    """cases: name -> (q, v, qacc); per state the worst row, the median row over the four outputs, and the nominal force error"""
    names = list(cases)
    r = dv.inverse_fd(m, *[np.array([cases[k][i] for k in names]) for i in range(3)], eps=EPS, centered=centered, lib_path=lib)
    run = ifr.Inverse(m)
    out = {}
    for p, k in enumerate(names):
        ref = ifr.inverse_fd(m, *cases[k], eps=EPS, centered=centered, run=run)
        e = np.concatenate(list(errors(device(r, p), ref).values()))
        out[k] = (float(e.max()), float(np.median(e)), ss.force_error(r.qfrc_inverse[p], ref['qfrc_inverse'], run(*cases[k])[1]))
    return out


def solver_cases(noslip, names=None):
    m = analytic(noslip)
    run = ifr.Inverse(m)
    out = {}
    for k in names or list(sv.STATES):
        q, v, ctrl = sv.state_inputs(m, *sv.STATES[k][0])
        out[k] = (q, v, forward_qacc(run, q, v, ctrl))
    return m, out


def check_contacts(out):
    print({k: f'worst {a:.1e} median {b:.1e} force {c:.1e}' for k, (a, b, c) in out.items()})
    assert max(a for a, _, _ in out.values()) <= CONTACT_ERR
    assert max(b for _, b, _ in out.values()) <= CONTACT_MEDIAN
    assert max(c for _, _, c in out.values()) <= CONTACT_FORCE


@pytest.mark.parametrize('noslip', [0, None])
def test_contact_states_under_emulation(emu, noslip):
    m, cases = solver_cases(noslip, ['one_contact', 'nefc31_zones', 'nefc33'])
    check_contacts(contact_errors(emu, False, m, cases))


# ---- 5. determinism and isolation ---------------------------------------------------------------------------------------------------
def flight_problems(n):
    m = ss.free_model(load_model('flight'))
    run = ifr.Inverse(m)
    names = ss.state_names(m)
    cases = free_cases(m, [names[i % len(names)] for i in range(n)], run)
    return m, [np.array([c[i] for c in cases]) for i in range(3)]


def check_positions(lib, n_big):
    """a problem's bits alone on a one-problem handle, at other positions of a larger batch, with padding envs"""
    m, (q, v, a) = flight_problems(3)
    ncol = 1 + 3 * m.nv
    one = st.BatchedStepper(m, ncol, lib_path=lib)
    one.fd_inverse(q[1:2], v[1:2], a[1:2], eps=EPS, centered=False)
    x = one.fd_inverse_read()
    one.close()
    per = n_big // ncol
    order = [2, 0] + [1] * (per - 2) if per > 2 else [2, 1]
    big = st.BatchedStepper(m, n_big, lib_path=lib)
    big.fd_inverse(q[order], v[order], a[order], eps=EPS, centered=False)
    y = big.fd_inverse_read()
    big.close()
    assert n_big > per * ncol                                    # padding envs
    for s, t in zip(x, y):
        for p in [i for i, k in enumerate(order) if k == 1]:
            assert np.array_equal(bits(s[0]), bits(t[p]))


def check_isolation(lib):
    """fb_inverse_read returns the last fb_inverse after an FD call; the state bank is untouched; the launches are perturb + step1 +
    inverse + diff"""
    m, cases = solver_cases(0, ['one_contact', 'nefc32'])
    q, v, a = (np.array([c[i] for c in cases.values()]) for i in range(3))
    ncol = 1 + 3 * m.nv
    sim = st.BatchedStepper(m, 2 * ncol, lib_path=lib)
    rows = np.minimum(np.arange(sim.n_envs), 1)
    sim.reset(q[rows], v[rows])
    sim.inverse(a)
    before = sim.inverse_read()
    sim.state_bank(2)
    sim.save_state(slots=[0, 1], env_ids=[0, 1])
    bank = sim.read_states([0, 1])
    l0 = sim.launch_count
    sim.fd_inverse(q, v, a, eps=EPS, centered=False)
    assert sim.launch_count - l0 == 1 + 4 + 1 + 1
    after = sim.inverse_read()
    for x, y in zip(before, after):
        assert np.array_equal(bits(x), bits(y))
    assert np.array_equal(sim.read_states([0, 1]), bank)
    sim.close()


def test_positions_and_isolation_under_emulation(emu):
    check_positions(emu, 2 * 145 + 7)
    check_isolation(emu)


# ---- 6. refusals ------------------------------------------------------------------------------------------------------------------------
def check_refusals(lib):
    m, (q, v, a) = flight_problems(2)
    ncol = 1 + 3 * m.nv
    sim = st.BatchedStepper(m, 2 * ncol, lib_path=lib)
    assert sim.fd_inverse_columns(False) == ncol == 145 and sim.fd_inverse_columns(True) == 1 + 6 * m.nv
    with pytest.raises(st.StepperError, match='no Jacobians to read'):
        sim.fd_inverse_read()
    f32 = [np.ascontiguousarray(x, np.float32) for x in (q, v, a)]
    ptrs = [x.ctypes.data for x in f32]
    for n in (0, -1, 3):
        with pytest.raises(st.StepperError, match='n_envs'):
            sim._check(sim._lib.fb_fd_inverse(sim._h, n, *ptrs, 1e-3, 0, 0), 'fb_fd_inverse')
    with pytest.raises(st.StepperError, match='n_envs'):
        sim.fd_inverse(q, v, a, centered=True)
    for k in range(3):
        p = list(ptrs)
        p[k] = None
        with pytest.raises(st.StepperError, match='NULL'):
            sim._check(sim._lib.fb_fd_inverse(sim._h, 2, *p, 1e-3, 0, 0), 'fb_fd_inverse')
    for k, what in enumerate(('qpos', 'qvel', 'qacc')):
        for bad in (np.nan, np.inf):
            x = [y.copy() for y in (q, v, a)]
            x[k][1, 2] = bad
            with pytest.raises(st.StepperError, match=f'non-finite {what}'):
                sim.fd_inverse(*x, centered=False)
    for eps in (0.0, -1e-3, np.inf, np.nan):
        with pytest.raises(st.StepperError, match='eps'):
            sim.fd_inverse(q, v, a, eps=eps, centered=False)
    sim.fd_inverse(q, v, a, centered=False)
    out = sim.fd_inverse_read()
    assert [x.shape for x in out] == [(2, m.nv, m.nv)] * 3 + [(2, m.nv, m.nM), (2, m.nv)]
    sim._check(sim._lib.fb_fd_inverse_read(sim._h, None, None, None, None, None, 0), 'fb_fd_inverse_read')      # every pointer may be NULL
    sim.close()


def test_refusals_under_emulation(emu):
    check_refusals(emu)


# ---- 7. Python ------------------------------------------------------------------------------------------------------------------------
def test_python_shapes_chunks_and_readme(emu, monkeypatch):
    m, (q, v, a) = flight_problems(3)
    with pytest.raises(ValueError):
        dv.inverse_fd(m, q, v[:2], a, lib_path=emu)
    whole = dv.inverse_fd(m, q, v, a, centered=False, lib_path=emu)
    assert whole.DfDq.shape == (3, m.nv, m.nv) and whole.DmDq.shape == (3, m.nv, m.nM) and whole.qfrc_inverse.shape == (3, m.nv)
    assert whole.DfDa.dtype == np.float64
    monkeypatch.setattr(dv, 'ENVS', 2 * (1 + 3 * m.nv))
    parts = dv.inverse_fd(m, q, v, a, centered=False, lib_path=emu)
    for x, y in zip(whole, parts):
        assert np.array_equal(x, y)
    one = dv.inverse_fd(m, q[2], v[2], a[2], centered=False, lib_path=emu)
    assert one.DfDq.shape == (m.nv, m.nv) and all(np.array_equal(x, y[2]) for x, y in zip(one, whole))
    monkeypatch.setattr(dv, 'ENVS', 4096)
    # README: the inverse-dynamics Jacobians of a walking state (qacc from fb_forward)
    w = load_model('template')
    sim = st.BatchedStepper(w, 1, lib_path=emu)
    sim.reset(w.qpos0)
    sim.set_control(np.full(w.nu, 0.1))
    sim.step(2)
    qpos, qvel, qacc = (sim.get(f)[0] for f in (st.QPOS, st.QVEL, st.QACC))
    sim.close()
    J = dv.inverse_fd(w, qpos, qvel, qacc, centered=False, lib_path=emu)
    assert J.DfDq.shape == (w.nv, w.nv) and all(np.isfinite(x).all() for x in J)


# ---- GPU tier ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_gpu_known_answers():
    ge.build()
    check_known_answers(None)


@pytest.mark.gpu
@pytest.mark.parametrize('centered', [False, True])
@pytest.mark.parametrize('name', ss.MODELS)
def test_gpu_constraint_free_states(name, centered):
    ge.build()
    out = free_errors(name, None, centered)
    report(f'{name} centered={centered}: worst row / nominal force', out)
    assert max(a for a, _ in out.values()) <= FREE_ERR and max(b for _, b in out.values()) <= FREE_FORCE


@pytest.mark.gpu
@pytest.mark.parametrize('centered', [False, True])
@pytest.mark.parametrize('noslip', [0, None])
def test_gpu_solver_states(noslip, centered):
    ge.build()
    m, cases = solver_cases(noslip)
    check_contacts(contact_errors(None, centered, m, cases))


def template_cases(n, steps=40, seed=0):
    """n states of a rollout of the analytic-contact template model (tests/solver_states.py: the oracle and the stepper find the same
    contacts) from qpos0 with random ctrl, with ground contacts and the forward qacc"""
    m = sv.analytic_model(load_model('template'))
    sim = st.BatchedStepper(m, n)
    sim.reset(m.qpos0)
    rs = np.random.RandomState(seed)
    for _ in range(steps):
        sim.set_control(rs.uniform(-0.3, 0.3, (n, m.nu)))
        sim.step(10)
    q, v, a = (sim.get(f).astype(np.float64) for f in (st.QPOS, st.QVEL, st.QACC))
    ncon = sim.get(st.NCON)[:, 0]
    sim.close()
    return m, {f'rollout{i} ({int(ncon[i])} contacts)': (q[i], v[i], a[i]) for i in range(n)}


@pytest.mark.gpu
@pytest.mark.parametrize('centered', [False, True])
def test_gpu_rollout_template_states(centered):
    ge.build()
    m, cases = template_cases(4)
    check_contacts(contact_errors(None, centered, m, cases))


@pytest.mark.gpu
def test_gpu_determinism_isolation_and_refusals():
    ge.build()
    check_positions(None, 4096)
    check_isolation(None)
    check_refusals(None)
