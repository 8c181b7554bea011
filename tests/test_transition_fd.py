"""Finite-difference transition Jacobians (fb_fd_transition, flybody_b200.derivatives) against an fp64 restatement of the same
definition on the oracle (tests/fd_reference.py), known answers of the step, determinism, isolation from the state bank, and the Python
front end.  CPU tier: the host-emulation build of the kernel source; GPU tier (-m gpu): the same through the CUDA library on full-size
handles.  "Bit-identical" compares uint32 views.

Error measure (`col_error`): per column of A or B, the largest entry error relative to the column's largest reference entry, floored at
1e-3 of the matrix's largest entry (a column the input barely reaches is not gated on its own round-off).  In fp32 a column's error is
the rounding of the next state over the step: one ulp of a wing's qvel of ~500 rad/s over 2 eps is ~1.5e-2.

Tolerances are 2.5 x the larger of the host-emulation and H100 measurements (the worst case is named beside each constant)."""
import numpy as np
import pytest

import __graft_entry__ as ge
from flybody_b200 import derivatives as dv, stepper as st
from flybody_b200.flymodel import load_model

import fd_reference as fr
import smooth_states as ss
import solver_states as sv

# ---- gates (measured: host emulation / H100 80GB HBM3 at a 700 W power limit; worst case) -------------------------------------------------
REF_ORDER = 2.2e-7         # fp64 reference, centred eps 1e-4 against 1e-6, col_error: measured 8.7e-8 ('flight', 'vision')
FREE_ERR = 0.45            # constraint-free states, eps 1e-3, col_error: measured 6.8e-2 emu ('flight' state, forward) / 1.8e-1 H100 ('flight_legs' 'flight', forward)
CONTACT_ERR = 40.0         # analytic-walk contact states, eps 1e-3, col_error: measured 1.9 emu ('nefc31_zones', forward) / 16 H100 ('middle_mu1_b', forward, 1 substep);
                           # the fp32 solve's convergence over the step, and nudges that move contacts across cone zones, set it
CONTACT_MEDIAN = 0.85      # the same states, per state the median over the columns of A and B: measured 3.4e-2 emu ('nefc31_zones') / 0.34 H100
                           # ('condim13', forward, 1 substep)
ONE_ROW_ERR = 0.25         # the states with a single contact or a single limit row ('one_contact', 'one_limit'), col_error: measured 5.8e-2 emu /
                           # 0.10 H100 ('one_contact', forward, 10 substeps)
FILTER_REL = 1.2e-2        # d act' / d ctrl = h / tau and d act' / d act = 1 - h / tau, relative: measured 4.6e-3 emu / 4.6e-3 H100 (forward)
EULER_ERR = 5e-4           # hinge rows: max |A[q_i] - e_i - h A[v_i]| (the rounding of q' over the step): measured 2.0e-4 emu / 2.0e-4 H100 (forward)

EPS = 1e-3                 # the eps the gates were measured at (derivatives.transition_fd defaults to 1e-2: DESIGN section 6)


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


@pytest.fixture(scope='module')
def emu():
    ge.build()
    return ge.EMU


def col_errors(dev, ref):
    """per column: max_i |dev - ref| / max(max_i |ref|, 1e-3 max |ref|)"""
    scale = np.maximum(np.abs(ref).max(0), 1e-3 * max(np.abs(ref).max(), 1e-30))
    return np.abs(dev - ref).max(0) / scale


def col_error(dev, ref):
    """the worst column of col_errors"""
    return float(col_errors(dev, ref).max())


_ANALYTIC = {}


def analytic():
    if 'm' not in _ANALYTIC:
        _ANALYTIC['m'] = sv.analytic_model(load_model('walk'))
    return _ANALYTIC['m']


# ---- 1. the reference itself ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('name', ss.DEFAULT_MODELS)
def test_reference_is_second_order(name):
    m = ss.free_model(ss.base_model(name))
    q, v, act, ctrl = ss.state_inputs(m, ss.state_names(m)[0])
    run = fr.Stepper(m)
    A4, B4, _ = fr.transition_fd(m, q, v, act, ctrl, eps=1e-4, stepper=run)
    A6, B6, _ = fr.transition_fd(m, q, v, act, ctrl, eps=1e-6, stepper=run)
    err = max(col_error(A4, A6), col_error(B4, B6) if m.nu else 0.0)
    print(f'{name}: centred eps 1e-4 against 1e-6 {err:.1e}')
    assert err <= REF_ORDER


def filter_rates(m, x, eps):
    """h / tau per actuator with a filter activation whose ctrl lies inside its range, nudged both ways (act address, actuator)"""
    out = []
    sides = fr.steps(m, x, eps, True)[2 * m.nv + m.na:]
    for i in range(m.nu):
        a = int(m.actuator_actadr[i])
        if a >= 0 and sides[i][0] and sides[i][1]:
            out.append((a, i, float(m.opt_timestep) / float(m.actuator_dynprm[i][0])))
    return out


def test_reference_act_rows_are_the_filter():
    m = ss.free_model(load_model('walk'))
    q, v, act, ctrl = ss.state_inputs(m, 'quat_a')
    A, B, _ = fr.transition_fd(m, q, v, act, ctrl, eps=1e-4)
    r = 2 * m.nv
    rates = filter_rates(m, (q, v, act, ctrl), 1e-4)
    assert len(rates) > m.na // 2
    for a, i, k in rates:
        assert abs(B[r + a, i] - k) <= 1e-9 and abs(A[r + a, r + a] - (1 - k)) <= 1e-9


# ---- 2. known answers on the stepper --------------------------------------------------------------------------------------------------
def template_case():
    m = ss.free_model(load_model('template'))
    q, v, act, ctrl = ss.state_inputs(m, 'quat_a')
    # an upper bound fp32 represents exactly, so that the device and the reference see the same ctrl on it
    lim = [i for i in range(m.nu) if m.actuator_ctrllimited[i]]
    at_top = [i for i in lim if np.float32(m.actuator_ctrlrange[i][1]) == m.actuator_ctrlrange[i][1]][0]
    outside = [i for i in lim if i != at_top][0]
    ctrl = ctrl.copy()
    ctrl[at_top] = m.actuator_ctrlrange[at_top][1]
    ctrl[outside] = m.actuator_ctrlrange[outside][1] + 0.25
    return m, (q, v, act, np.float64(np.float32(ctrl))), at_top, outside


def check_known_answers(lib, centered):
    m, (q, v, act, ctrl), at_top, outside = template_case()
    r = dv.transition_fd(m, q, v, ctrl, act, eps=EPS, centered=centered, lib_path=lib)
    nv, na = m.nv, m.na
    # ctrl reaches the force only through act, and act is integrated after the force is taken
    assert not r.B[:2 * nv].any()
    # the activation filter: act' = act + h (ctrl - act) / tau
    rel = 0.0
    for a, i, k in filter_rates(m, (q, v, act, ctrl), EPS):
        rel = max(rel, abs(r.B[2 * nv + a, i] - k) / k, abs(r.A[2 * nv + a, 2 * nv + a] - (1 - k)) / (1 - k))
    # semi-implicit Euler on hinge rows: q_i' = q_i + h v_i'
    h = float(m.opt_timestep)
    hinge = [int(m.jnt_dofadr[j]) for j in range(m.njnt) if m.jnt_type[j] == ss.HINGE]
    euler = np.abs(r.A[hinge] - np.eye(2 * nv + na)[hinge] - h * r.A[[nv + k for k in hinge]]).max()
    # a ctrl at its upper bound: the reference's backward difference; a ctrl outside its range: a zero column
    A, B, _ = fr.transition_fd(m, q, v, act, ctrl, eps=EPS, centered=centered)
    assert not r.B[:, outside].any() and not B[:, outside].any()
    assert np.abs(r.B[:, at_top]).max() > 0
    top = np.abs(r.B[:, at_top] - B[:, at_top]).max() / np.abs(B[:, at_top]).max()
    free = max(col_error(r.A, A), col_error(r.B, B))
    return rel, euler, top, free


@pytest.mark.parametrize('centered', [False, True])
def test_known_answers_under_emulation(emu, centered):
    rel, euler, top, free = check_known_answers(emu, centered)
    print(f'centered={centered}: filter {rel:.1e}  euler {euler:.1e}  ctrl at its bound {top:.1e}  template against the reference {free:.1e}')
    assert rel <= FILTER_REL and euler <= EULER_ERR and top <= FREE_ERR and free <= FREE_ERR


# ---- 3. against the fp64 reference ---------------------------------------------------------------------------------------------------
def free_errors(name, lib, centered, names=None):
    m = ss.free_model(ss.base_model(name))
    names = names or ss.state_names(m)
    xs = [ss.state_inputs(m, k) for k in names]
    r = dv.transition_fd(m, *[np.array([x[c] for x in xs]) for c in (0, 1, 3, 2)], eps=EPS, centered=centered, lib_path=lib)
    run = fr.Stepper(m)
    out = {}
    for p, (k, x) in enumerate(zip(names, xs)):
        A, B, nom = fr.transition_fd(m, *x, eps=EPS, centered=centered, stepper=run)
        out[k] = max(col_error(r.A[p], A), col_error(r.B[p], B))
    return out


@pytest.mark.parametrize('centered', [False, True])
def test_constraint_free_flight_under_emulation(emu, centered):
    errs = free_errors('flight', emu, centered, names=['quat_a', 'flight'])
    print(centered, {k: f'{v:.1e}' for k, v in errs.items()})
    assert max(errs.values()) <= FREE_ERR


def contact_errors(lib, centered, n_substeps, names):
    m = analytic()
    xs = [sv.state_inputs(m, *sv.STATES[k][0]) for k in names]
    q, v, ctrl = (np.array([x[c] for x in xs]) for c in range(3))
    r = dv.transition_fd(m, q, v, ctrl, eps=EPS, centered=centered, n_substeps=n_substeps, lib_path=lib)
    run = fr.Stepper(m)
    out = {}
    for p, k in enumerate(names):
        A, B, _ = fr.transition_fd(m, q[p], v[p], None, ctrl[p], eps=EPS, centered=centered, n_substeps=n_substeps, stepper=run)
        ea, eb = col_errors(r.A[p], A), col_errors(r.B[p], B)
        out[k] = (float(ea.max()), float(eb.max()), float(np.median(np.concatenate([ea, eb]))))
    return out


def test_contact_states_under_emulation(emu):
    out = contact_errors(emu, False, 1, ['one_contact', 'nefc31_zones'])
    print({k: f'A {a:.1e} B {b:.1e} median {c:.1e}' for k, (a, b, c) in out.items()})
    assert max(max(a, b) for a, b, _ in out.values()) <= CONTACT_ERR
    assert max(c for _, _, c in out.values()) <= CONTACT_MEDIAN
    assert max(max(a, b) for k, (a, b, _) in out.items() if k in ('one_contact', 'one_limit')) <= ONE_ROW_ERR


# ---- 4. determinism and isolation ---------------------------------------------------------------------------------------------------
def flight_states(n, seed=0):
    m = ss.free_model(load_model('flight'))
    names = ss.state_names(m)
    xs = [ss.state_inputs(m, names[i % len(names)]) for i in range(n)]
    return m, [np.array([x[c] for x in xs]) for c in range(4)]


def fd_on(sim, q, v, act, ctrl, slots_order, n_slots, eps=EPS, centered=False, n_substeps=1):
    """write states k -> envs k, save them to slots k, run fd_transition on the listed slots"""
    m, n = sim.model, len(q)
    rows = np.minimum(np.arange(sim.n_envs), n - 1)
    sim.reset(q[rows], v[rows])
    if m.na:
        sim.set(st.ACT, act[rows])
    sim.set_control(ctrl[rows])
    sim.forward()
    sim.state_bank(n_slots)
    sim.save_state(slots=np.arange(n), env_ids=np.arange(n))
    sim.fd_transition(slots_order, eps=eps, centered=centered, n_substeps=n_substeps)
    return sim.fd_read()


def check_positions(lib, n_big):
    """a problem's bits alone, at another position of a batch, with padding envs"""
    m, (q, v, act, ctrl) = flight_states(3)
    ncol = 1 + 2 * m.nv + m.na + m.nu
    one = st.BatchedStepper(m, ncol, lib_path=lib)
    a = fd_on(one, q[1:2], v[1:2], act[1:2], ctrl[1:2], [0], 1)
    one.close()
    per = n_big // ncol
    big = st.BatchedStepper(m, n_big, lib_path=lib)
    order = [2, 0] + [1] * (per - 2) if per > 2 else [2, 1]
    b = fd_on(big, q, v, act, ctrl, order, 3)
    big.close()
    for x, y in zip(a, b):
        for p in [i for i, s in enumerate(order) if s == 1]:
            assert np.array_equal(bits(x[0]), bits(y[p]))


def test_positions_and_padding_under_emulation(emu):
    check_positions(emu, 2 * 108 + 5)


def check_nominal_and_bank(lib, n_substeps):
    """the nominal next state equals fb_state_load + fb_step of the row on another handle (xfrc_applied in the row); the bank is
    unchanged; the launches are fan-out + perturb + step1 + fb_step's + diff"""
    m = analytic()
    names = ['one_contact', 'nefc32']
    xs = [sv.state_inputs(m, *sv.STATES[k][0]) for k in names]
    q, v, ctrl = (np.array([x[c] for x in xs]) for c in range(3))
    ncol = 1 + 2 * m.nv + m.na + m.nu
    rs = np.random.RandomState(5)
    xfrc = rs.normal(size=(2, m.nbody, 6)) * 1e-3
    a, b = sims = [st.BatchedStepper(m, n, lib_path=lib) for n in (2 * ncol, 2)]
    rows = np.minimum(np.arange(a.n_envs), 1)
    a.set_applied(xfrc=xfrc[rows])
    b.set_applied(xfrc=xfrc)
    a.reset(q[rows], v[rows])
    a.set_control(ctrl[rows])
    a.forward()
    a.state_bank(2)
    a.save_state(slots=[0, 1], env_ids=[0, 1])
    bank = a.read_states([0, 1])
    l0 = a.launch_count
    a.fd_transition([0, 1], eps=EPS, centered=False, n_substeps=n_substeps)
    assert a.launch_count - l0 == 1 + 1 + 4 + 7 * n_substeps + 1
    _, _, qn, vn, an = a.fd_read()
    assert np.array_equal(a.read_states([0, 1]), bank)
    b.state_bank(2)
    b.write_states([0, 1], bank)
    b.load_state(slots=[0, 1], env_ids=[0, 1])
    b.step(n_substeps)
    for x, f in ((qn, st.QPOS), (vn, st.QVEL), (an, st.ACT)):
        assert np.array_equal(bits(x), bits(b.get(f)))
    for s in sims:
        s.close()


def test_nominal_and_bank_under_emulation(emu):
    check_nominal_and_bank(emu, 2)


# ---- 5. refusals and wiring ------------------------------------------------------------------------------------------------------
def check_refusals(lib):
    m, (q, v, act, ctrl) = flight_states(2)
    ncol = 1 + 2 * m.nv + m.na + m.nu
    assert (ncol, 1 + 2 * (ncol - 1)) == (108, 215)
    sim = st.BatchedStepper(m, 2 * ncol, lib_path=lib)
    assert sim.fd_columns(False) == 108 and sim.fd_columns(True) == 215
    with pytest.raises(st.StepperError, match='no transition to read'):
        sim.fd_read()
    with pytest.raises(st.StepperError, match='no state bank'):
        sim.fd_transition([0], centered=False)
    sim.state_bank(3)
    sim.save_state(slots=[0, 1], env_ids=[0, 1])
    for slots, msg in (([3], 'out of range'), ([-1], 'out of range'), ([2], 'never written'), ([0, 1, 0], 'n_envs'), ([], 'n_envs')):
        with pytest.raises(st.StepperError, match=msg):
            sim.fd_transition(slots, centered=False)
    with pytest.raises(st.StepperError, match='n_envs'):
        sim.fd_transition([0, 1], centered=True)
    for eps in (0.0, -1e-3, np.inf, np.nan):
        with pytest.raises(st.StepperError, match='eps'):
            sim.fd_transition([0], eps=eps, centered=False)
    with pytest.raises(st.StepperError, match='n_substeps'):
        sim.fd_transition([0], centered=False, n_substeps=0)
    sim.reset_hold([1], q[0])
    sim.save_state(slots=[2], env_ids=[1])
    with pytest.raises(st.StepperError, match='held for a reset'):
        sim.fd_transition([2], centered=False)
    sim.fd_transition([0, 1], centered=False)
    A, B, qn, vn, an = sim.fd_read()
    assert A.shape == (2, 96, 96) and B.shape == (2, 96, 11) and qn.shape == (2, m.nq) and an.shape == (2, 0)
    sim._check(sim._lib.fb_fd_read(sim._h, None, None, None, None, None, 0), 'fb_fd_read')      # every pointer may be NULL
    sim.close()


def test_refusals_under_emulation(emu):
    check_refusals(emu)


def test_python_shapes_chunks_and_readme(emu, monkeypatch):
    m, (q, v, act, ctrl) = flight_states(3)
    with pytest.raises(ValueError):
        dv.transition_fd(m, q, v[:2], ctrl, lib_path=emu)
    whole = dv.transition_fd(m, q, v, ctrl, centered=False, lib_path=emu)
    assert whole.A.shape == (3, 96, 96) and whole.B.shape == (3, 96, 11) and whole.A.dtype == np.float64
    monkeypatch.setattr(dv, 'ENVS', 2 * 108)
    parts = dv.transition_fd(m, q, v, ctrl, centered=False, lib_path=emu)
    for x, y in zip(whole, parts):
        assert np.array_equal(x, y)
    one = dv.transition_fd(m, q[2], v[2], ctrl[2], centered=False, lib_path=emu)
    assert one.A.shape == (96, 96) and np.array_equal(one.A, whole.A[2]) and np.array_equal(one.qvel_next, whole.qvel_next[2])
    # README: the transition of one control step of the walking fly (10 substeps), at a state of a rollout
    w = load_model('template')
    sim = st.BatchedStepper(w, 1, lib_path=emu)
    sim.reset(w.qpos0)
    sim.set_control(np.full(w.nu, 0.1))
    sim.step(2)
    qpos, qvel, act, u = (sim.get(f)[0] for f in (st.QPOS, st.QVEL, st.ACT, st.CTRL))
    sim.close()
    monkeypatch.setattr(dv, 'ENVS', 4096)
    lin = dv.transition_fd(w, qpos, qvel, u, act, centered=False, n_substeps=10, lib_path=emu)
    assert lin.A.shape == (2 * w.nv + w.na,) * 2 and np.isfinite(lin.A).all() and np.isfinite(lin.B).all()


# ---- GPU tier ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize('centered', [False, True])
def test_gpu_known_answers(centered):
    ge.build()
    rel, euler, top, free = check_known_answers(None, centered)
    print(f'centered={centered}: filter {rel:.1e}  euler {euler:.1e}  ctrl at its bound {top:.1e}  template against the reference {free:.1e}')
    assert rel <= FILTER_REL and euler <= EULER_ERR and top <= FREE_ERR and free <= FREE_ERR


@pytest.mark.gpu
@pytest.mark.parametrize('centered', [False, True])
@pytest.mark.parametrize('name', ss.DEFAULT_MODELS + list(ss.ov.VARIANTS))
def test_gpu_constraint_free_states(name, centered):
    ge.build()
    errs = free_errors(name, None, centered)
    print(name, centered, {k: f'{v:.1e}' for k, v in errs.items()})
    assert max(errs.values()) <= FREE_ERR


@pytest.mark.gpu
@pytest.mark.parametrize('n_substeps', [1, 10])
@pytest.mark.parametrize('centered', [False, True])
def test_gpu_contact_states(centered, n_substeps):
    ge.build()
    names = list(sv.STATES) if n_substeps == 1 else ['one_contact', 'nefc31_zones', 'rows64', 'middle_mu1_a']
    out = contact_errors(None, centered, n_substeps, names)
    print(centered, n_substeps, {k: f'A {a:.1e} B {b:.1e} median {c:.1e}' for k, (a, b, c) in out.items()})
    assert max(max(a, b) for a, b, _ in out.values()) <= CONTACT_ERR
    assert max(c for _, _, c in out.values()) <= CONTACT_MEDIAN
    assert max(max(a, b) for k, (a, b, _) in out.items() if k in ('one_contact', 'one_limit')) <= ONE_ROW_ERR


@pytest.mark.gpu
def test_gpu_determinism_bank_and_refusals():
    ge.build()
    check_positions(None, 4096)
    check_nominal_and_bank(None, 10)
    check_refusals(None)
