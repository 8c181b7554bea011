"""System identification (fb_sid_accumulate / fb_sid_read, flybody_b200.sysid): the device's normal equations against the fp64 restatement
of tests/sysid_reference.py on the outputs of the same parameter-Jacobian query; their bit invariance (split across calls, interleaved
with other problems, weight 0 against left out); the bad-state mark; the refusals; and the Levenberg-Marquardt fits they exist for.
CPU tier: the host-emulation build of the kernel source on small handles; GPU tier (-m gpu): the CUDA library on 4096-env handles.
"Bit-identical" compares the bytes.

Tolerances are 2.5 x the larger of the host-emulation and H100 measurements (the worst case is named beside each constant)."""
import numpy as np
import pytest

import __graft_entry__ as ge
from flybody_b200 import derivatives as dv, stepper as st, sysid
from flybody_b200.flymodel import load_model

import sysid_reference as sr
from test_model_params import start_state
from test_sensor_fd import free_cases, solver_cases, stack

# ---- gates (measured: host emulation / H100 80GB HBM3 at a 700 W power limit; worst case) -------------------------------------------
H_TOL = 1e-12              # H against fp64 from the same fp32 J, relative to max|H| (both sum the same products): measured 3.4e-16 emu /
                           # 4.2e-16 H100 (flight); kept at 1e-12, far above both, as the bound a fixed-order fp64 sum must meet
G_TOL = 7.5e-7             # g and cost, relative to max|g| / max cost: the fp32 quaternion residual rows (fd_subquat) against fp64's:
                           # measured 3.0e-7 emu / 1.5e-7 H100 (flight, cost)
FIT_TOL = 2e-3             # recovered scales, relative (the fit's target): measured 4.2e-4 emu / 3.4e-4 H100 (flight), template 8.5e-5 /
                           # 1.1e-4
INV_TOL = 1e-4             # the inverse fit (check_least_squares through the library): measured 1.1e-7 emu / 1.4e-7 H100

EPS = 1e-2
FREE_DIRS = [dv.Scale('dof_damping'), dv.Scale('actuator_gainprm'), dv.Scale('body_mass', 'body_inertia'), ('dof_damping', [7]),
             ('gravity', [2])]


def raw(a):
    return np.ascontiguousarray(a).view(np.uint8)


def same(x, y):
    return all(np.array_equal(raw(a), raw(b)) for a, b in zip(x, y))


@pytest.fixture(scope='module')
def emu():
    ge.build()
    return ge.EMU


@pytest.fixture
def small(monkeypatch):
    monkeypatch.setattr(sysid, 'ENVS', 64)


def unit_quats(m, q):
    """q [n, nq] with its free and ball joints' quaternions normalised"""
    q = q.copy()
    for j in range(m.njnt):
        t, a = int(m.jnt_type[j]), int(m.jnt_qposadr[j])
        if t in (0, 1):
            a += 3 if t == 0 else 0
            q[:, a:a + 4] /= np.linalg.norm(q[:, a:a + 4], axis=1, keepdims=True)
    return q


def transition_query(lib, m, q, v, u, act, dirs, n_envs=None, n_sub=1):
    """a handle whose last call is fb_fd_param_transition of the n states (bank rows 0 .. n - 1)"""
    dirs, _ = dv._directions(m, dirs, None)
    n, ncol = len(q), 1 + 2 * len(dirs)
    sim = st.BatchedStepper(m, n_envs or n * ncol, lib_path=lib)
    dv._param_setup(sim, m, dirs, False, n)
    dv._bank_rows(sim, m, (q, v, u, act), n)
    sim.fd_param_transition(np.arange(n), eps=EPS, n_substeps=n_sub)
    return sim


def observed(m, pred, seed):
    """recorded next states near the predictions [n, nq + nv + na]: every coordinate moved by ~1e-2, quaternions kept unit (fp32)"""
    x = pred + np.random.RandomState(seed).normal(0, 1e-2, pred.shape)
    x[:, :m.nq] = unit_quats(m, x[:, :m.nq])
    return x.astype(np.float32)


# ---- 1. the normal equations against fp64 ---------------------------------------------------------------------------------------------
def errors(got, ref):
    (H, g, c, n, b), (Hr, gr, cr, nr, br) = got, ref
    assert np.array_equal(n, nr) and np.array_equal(b, br)
    return (np.abs(H - Hr).max() / np.abs(Hr).max(), np.abs(g - gr).max() / np.abs(gr).max(), np.abs(c - cr).max() / cr.max())


def check_normal(lib, m, cases, dirs, L=3, n_envs=None):
    q, v, u, act, qa = cases
    n = len(q)
    nx = 2 * m.nv + m.na
    rs = np.random.RandomState(7)
    problem = np.arange(n) % (L + 1) - 1                        # every fit problem, and skipped transitions
    sw = rs.uniform(0.5, 2.0, n).astype(np.float32)
    sw[min(2, n - 1)] = 0
    sim = transition_query(lib, m, q, v, u, act, dirs, n_envs)
    dxdp, qn, vn, an = sim.fd_param_read()
    pred = np.concatenate([qn, vn, an], 1)
    obs = observed(m, pred, 3)
    W = rs.uniform(0.5, 2.0, nx)
    W[0] = 0
    sim.sid_accumulate(st.SID_TRANSITION, L, problem, W, target=obs, sample_weight=sw)
    err = errors(sim.sid_read(), sr.normal_equations(dxdp, sr.transition_residual(m, pred, obs), W, problem, L, sw))
    # the inverse on the same handle: qfrc_inverse against a target near it
    sim.fd_param_inverse(q, v, qa, eps=EPS)
    DfDp, f0 = sim.fd_param_inverse_read()
    target = (f0 + rs.normal(0, 1e-2, f0.shape) * np.abs(f0).max()).astype(np.float32)
    Wv = rs.uniform(0.5, 2.0, m.nv)
    sim.sid_accumulate(st.SID_INVERSE, L, problem, Wv, target=target, sample_weight=sw)
    ei = errors(sim.sid_read(), sr.normal_equations(np.transpose(DfDp, (0, 2, 1)), f0.astype(np.float64) - target, Wv, problem, L, sw))
    sim.close()
    return tuple(max(a, b) for a, b in zip(err, ei))


def normal_cases(lib, n_envs=None):
    out = {}
    m, c = free_cases('flight')
    out['flight'] = check_normal(lib, m, stack(c, range(5)), FREE_DIRS, n_envs=n_envs)
    m, c = solver_cases(0, ['one_contact', 'nefc31_zones', 'nefc33'])
    q, v, u, a = stack(c, range(4))
    out['template'] = check_normal(lib, m, (q, v, u, np.zeros((len(q), m.na)), a),
                                   [dv.Scale('dof_damping'), dv.Scale('body_mass', 'body_inertia'), ('gravity', [2])], n_envs=n_envs)
    m, c = free_cases('walk')
    out['walk'] = check_normal(lib, m, stack(c, range(5)), FREE_DIRS, n_envs=n_envs)
    m, c = free_cases('ball')
    out['ball'] = check_normal(lib, m, stack(c, range(5)), [dv.Scale('dof_damping'), dv.Scale('body_mass'), ('gravity', [2])],
                               n_envs=n_envs)
    print({k: 'H {:.1e} g {:.1e} cost {:.1e}'.format(*e) for k, e in out.items()})
    assert max(e[0] for e in out.values()) <= H_TOL
    assert max(max(e[1], e[2]) for e in out.values()) <= G_TOL


def test_normal_equations_under_emulation(emu):
    normal_cases(emu)


# ---- 2. bit invariance, 3. the bad-state mark ------------------------------------------------------------------------------------------
def check_invariance(lib, n_envs=None):
    m, c = free_cases('flight')
    q, v, u, act = (x[:5] for x in stack(c, range(4)))
    n, nx = len(q), 2 * m.nv + m.na
    sim = transition_query(lib, m, q, v, u, act, FREE_DIRS, n_envs)
    _, qn, vn, an = sim.fd_param_read()
    obs = observed(m, np.concatenate([qn, vn, an], 1), 4)
    W = np.random.RandomState(2).uniform(0.5, 2.0, nx)
    sw = np.random.RandomState(3).uniform(0.5, 2.0, n).astype(np.float32)

    def run(slots, problem, L, weights=sw, parts=None):
        for j, part in enumerate(parts or [np.arange(len(slots))]):
            sim.fd_param_transition(np.asarray(slots)[part], eps=EPS)
            sim.sid_accumulate(st.SID_TRANSITION, L, np.asarray(problem)[part], W, target=obs[np.asarray(slots)[part]],
                               sample_weight=weights[np.asarray(slots)[part]], reset=j == 0)
        return [x.copy() for x in sim.sid_read()]

    whole = run(range(n), [0] * n, 1)
    assert np.isfinite(whole[2]).all() and whole[3][0] == n and np.abs(whole[0]).max() > 0
    assert np.array_equal(whole[0], whole[0][0].T[None])        # both triangles
    assert same(whole, run(range(n), [0] * n, 1, parts=[[0, 1], [2, 3, 4]]))
    assert same(whole, run(range(n), [0] * n, 1, parts=[[0], [1, 2, 3], [4]]))
    mixed = run(range(n), [1, 0, 2, 0, 0], 3)                  # problem 0 interleaved with two others, at another index and L
    alone = run([1, 3, 4], [0, 0, 0], 1)
    assert same([x[:1] for x in mixed[:3]], alone[:3]) and mixed[3][0] == 3
    moved = run(range(n), [2, 1, 0, 1, 1], 3)
    assert same([x[1:2] for x in moved[:3]], alone[:3])
    zero = sw.copy()
    zero[2] = 0
    assert same(run(range(n), [0] * n, 1, weights=zero), run(range(n), [0, 0, -1, 0, 0], 1))
    sim.close()
    # a bad-state transition: +inf and bad, nothing in H or g
    vb = v.copy()
    vb[1, 6:] = 1e18
    sim = transition_query(lib, m, q, vb, u, act, FREE_DIRS, n_envs)
    sim.sid_accumulate(st.SID_TRANSITION, 2, [0, 0, 1, 1, 1], W, target=obs, sample_weight=sw)
    H, g, cost, count, bad = sim.sid_read()
    assert cost[0] == np.inf and bad[0] == 1 and count[0] == 2 and np.isfinite(cost[1]) and bad[1] == 0
    assert np.isfinite(H).all() and np.isfinite(g).all()
    sim.fd_param_transition(np.arange(n), eps=EPS)
    sim.sid_accumulate(st.SID_TRANSITION, 2, [0, -1, 1, 1, 1], W, target=obs, sample_weight=sw)
    H2, g2, cost2, _, bad2 = sim.sid_read()
    assert same((H, g, cost[1:]), (H2, g2, cost2[1:])) and np.isfinite(cost2[0]) and bad2[0] == 0
    sim.close()


def test_bit_invariance_under_emulation(emu):
    check_invariance(emu)


# ---- 4. refusals -----------------------------------------------------------------------------------------------------------------------
def check_refusals(lib):
    m, c = free_cases('flight')
    q, v, u, act = (x[:2] for x in stack(c, range(4)))
    nx = 2 * m.nv + m.na
    W = np.ones(nx)
    fresh = st.BatchedStepper(m, 4, lib_path=lib)
    with pytest.raises(st.StepperError, match='no sums to read'):
        fresh.sid_read()
    with pytest.raises(st.StepperError, match='no parameter Jacobians'):
        fresh.sid_accumulate(st.SID_TRANSITION, 1, [0, 0], W, target=np.zeros((2, m.nq + m.nv + m.na)))
    fresh.close()
    sim = transition_query(lib, m, q, v, u, act, FREE_DIRS)
    obs = np.zeros((2, m.nq + m.nv + m.na), np.float32)
    lib_, h = sim._lib, sim._h
    bad = [(dict(query=st.SID_INVERSE, W=np.ones(m.nv), target=None), 'no parameter Jacobians'), (dict(query=7, target=None), 'query is'), (dict(L=0), 'L >= 1'),
           (dict(problem=[0, 0, 0], target=np.zeros((3, obs.shape[1]), np.float32)), 'n = 3'), (dict(problem=[0, 2]), r'not in \[-1, L\)'), (dict(problem=[-2, 0]), r'not in \[-1, L\)'),
           (dict(target=None), 'needs its target'), (dict(W=np.r_[-1.0, W[1:]]), '>= 0 and finite'),
           (dict(W=np.r_[np.nan, W[1:]]), '>= 0 and finite'), (dict(sw=[1.0, -1.0]), 'sample weights'),
           (dict(sw=[1.0, np.inf]), 'sample weights'), (dict(target=np.full_like(obs, np.nan)), 'non-finite target'),
           (dict(reset=False), 'no sums to add to')]
    for kw, msg in bad:
        a = dict(query=st.SID_TRANSITION, L=2, problem=[0, 1], W=W, target=obs, sw=None, reset=True)
        a.update(kw)
        with pytest.raises(st.StepperError, match=msg):
            sim.sid_accumulate(a['query'], a['L'], a['problem'], a['W'], target=a['target'], sample_weight=a['sw'], reset=a['reset'])
    assert lib_.fb_sid_accumulate(h, st.SID_TRANSITION, 2, None, 2, obs.ctypes.data, W.ctypes.data, None, 1, 0) == -1
    assert 'must not be NULL' in lib_.fb_last_error(h).decode()
    sim.sid_accumulate(st.SID_TRANSITION, 2, [0, 1], W, target=obs)
    sim.fd_param_transition([0, 1], eps=EPS)
    with pytest.raises(st.StepperError, match='without reset, L and k'):
        sim.sid_accumulate(st.SID_TRANSITION, 3, [0, 1], W, target=obs, reset=False)
    sim.forward()
    with pytest.raises(st.StepperError, match='launched kernels since'):
        sim.sid_accumulate(st.SID_TRANSITION, 2, [0, 1], W, target=obs, reset=False)
    sim.fd_param_transition([0, 1], eps=EPS)
    sim.sid_accumulate(st.SID_TRANSITION, 2, [0, 1], W, target=obs, reset=False)
    with pytest.raises(st.StepperError, match='launched kernels since'):     # the accumulate's own launches count too: one query, once
        sim.sid_accumulate(st.SID_TRANSITION, 2, [0, 1], W, target=obs, reset=False)
    assert sim.sid_read()[3].tolist() == [2, 2]
    sim.close()
    # the front ends
    groups = [dv.Scale('dof_damping'), dv.Scale('body_mass')]
    x3 = lambda x: x[None, :2]                                             # noqa: E731
    with pytest.raises(ValueError, match='share the element'):
        sysid.fit_transitions(m, x3(q), x3(v), x3(u), x3(q), x3(v), np.ones(nx), params=groups + [('dof_damping', [3])], lib_path=lib)
    with pytest.raises(ValueError, match='excludes actuation'):
        sysid.fit_inverse(m, x3(q), x3(v), x3(v), np.ones(m.nv), params=[dv.Scale('actuator_gainprm')], lib_path=lib)
    with pytest.raises(ValueError, match='weights'):
        sysid.fit_transitions(m, x3(q), x3(v), x3(u), x3(q), x3(v), -np.ones(nx), params=groups, lib_path=lib)
    with pytest.raises(ValueError, match='qvel_next'):
        sysid.fit_transitions(m, x3(q), x3(v), x3(u), x3(q), x3(v)[:, :1], np.ones(nx), params=groups, lib_path=lib)
    with pytest.raises(ValueError, match='sample_weight'):
        sysid.fit_inverse(m, x3(q), x3(v), x3(v), np.ones(m.nv), params=groups, sample_weight=-np.ones((1, 2)), lib_path=lib)
    with pytest.raises(ValueError, match='max_iter'):
        sysid.fit_inverse(m, x3(q), x3(v), x3(v), np.ones(m.nv), params=groups, max_iter=-1, lib_path=lib)


def test_refusals_under_emulation(emu):
    check_refusals(emu)


# ---- 5. the fits ---------------------------------------------------------------------------------------------------------------------
def transitions(lib, m, groups, s_true, q, v, u, n_sub):
    """the next states of states q [L, T, nq], v, u after n_sub substeps on handles whose groups are scaled by s_true [L, G]: the data a
    fit at s* reproduces bit for bit (set the parameters, reset, step)"""
    L, T = q.shape[:2]
    data = st.BatchedStepper(m, L * T, lib_path=lib)
    for l in range(L):
        for g, s in zip(groups, s_true[l]):
            for name in g.fields:
                data.param_set(name, dv.compiled_params(m, name) * s, env_ids=np.arange(l * T, (l + 1) * T))
    data.reset(q.reshape(L * T, -1), v.reshape(L * T, -1))
    data.set_control(u.reshape(L * T, -1))
    data.step(n_sub)
    out = [data.get(f).reshape(L, T, -1).astype(np.float64) for f in (st.QPOS, st.QVEL)]
    data.close()
    return out


def row_weights(m, vd):
    """per-row scaling as check_gauss_newton's: 1e3 on the dq rows, 1 / max|qvel_j| on the qvel rows"""
    return np.r_[np.full(m.nv, 1e3), 1.0 / np.maximum(np.abs(vd).reshape(-1, m.nv).max(0), 1e-3), np.ones(m.na)]


def scales(m, fit, groups):
    """-> [L, G] the fitted scale of each group: its values over the compiled ones at the largest compiled element"""
    out = []
    for g in groups:
        name = g.fields[0]
        base = dv.compiled_params(m, name)
        j = int(np.argmax(np.abs(base)))
        out.append(fit.values[name][:, j] / base[j])
    return np.stack(out, 1)


def check_history(fit):
    for h in fit.cost:
        h = h[np.isfinite(h)]
        assert (np.diff(h) <= 0).all()
    assert (fit.status >= 0).all()


def flight_fit(lib, L, T, n_sub=4, groups=('dof_damping', 'actuator_gainprm', 'body_mass'), seed=0, **kw):
    m = load_model('flight')
    groups = [dv.Scale(g) for g in groups]
    rs = np.random.RandomState(seed)
    s_true = rs.uniform(0.85, 1.15, (L, len(groups)))
    qv = [start_state(m, 100 + k) for k in range(L * T)]
    q = np.array([x[0] for x in qv]).reshape(L, T, m.nq)
    v = np.array([x[1] for x in qv]).reshape(L, T, m.nv)
    u = rs.uniform(-0.5, 0.5, (L, T, m.nu))
    qd, vd = transitions(lib, m, groups, s_true, q, v, u, n_sub)
    fit = sysid.fit_transitions(m, q, v, u, qd, vd, row_weights(m, vd), params=groups, n_substeps=n_sub, lib_path=lib, **kw)
    return m, groups, s_true, fit, (q, v, u, qd, vd)


def check_flight(lib, L, T):
    m, groups, s_true, fit, _ = flight_fit(lib, L, T)
    s = scales(m, fit, groups)
    err = np.abs(s / s_true - 1).max()
    print('flight one-step: iterations', fit.iterations, 'status', fit.status, 'worst relative error', f'{err:.1e}')
    check_history(fit)
    assert (fit.status == sysid.CONVERGED).all() and err <= FIT_TOL
    assert fit.H.shape == (L, 3, 3) and fit.count.tolist() == [T] * L and fit.columns == [f'scale({g.fields[0]})' for g in groups]


def check_template(lib, n_sub):
    m, cases = solver_cases(0, ['one_contact', 'nefc31_zones', 'nefc33'])
    q, v, u, _ = stack(cases, range(4))
    groups = [dv.Scale('dof_damping'), dv.Scale('body_mass', 'body_inertia')]
    s_true = np.array([[1.1, 0.9], [0.9, 1.12]])
    L, T = len(s_true), len(q)
    Q, V, U = (np.broadcast_to(x, (L,) + x.shape).copy() for x in (q, v, u))
    qd, vd = transitions(lib, m, groups, s_true, Q, V, U, n_sub)
    fit = sysid.fit_transitions(m, Q, V, U, qd, vd, row_weights(m, vd), params=groups, n_substeps=n_sub, lib_path=lib)
    s = scales(m, fit, groups)
    err = np.abs(s / s_true - 1)
    print(f'template one-step ({n_sub} substeps): iterations', fit.iterations, 'status', fit.status, 'relative error per group',
          err.max(0))
    check_history(fit)
    return fit, err


def check_inverse_fit(lib):
    """check_least_squares through the library: template contact states, armature, damping and gravity scales, two problems"""
    m, cases = solver_cases(0, ['one_contact', 'nefc31_zones', 'nefc33'])
    q, v, _, a = stack(cases, range(4))
    names, s_true = ('dof_armature', 'dof_damping', 'gravity'), np.array([[1.2, 0.8, 1.05], [0.9, 1.1, 0.97]])
    L = len(s_true)
    tgt = []
    for l in range(L):
        data = st.BatchedStepper(m, len(q), lib_path=lib)
        for g, s in zip(names, s_true[l]):
            data.param_set(g, dv.compiled_params(m, g) * s)
        data.reset(q, v)
        data.inverse(a)
        tgt.append(data.inverse_read()[0].astype(np.float64))
        data.close()
    groups = [dv.Scale(g) for g in names]
    Q, V, A = (np.broadcast_to(x, (L,) + x.shape).copy() for x in (q, v, a))
    fit = sysid.fit_inverse(m, Q, V, A, np.ones(m.nv), params=groups, target=np.array(tgt), lib_path=lib)
    err = np.abs(scales(m, fit, groups) / s_true - 1).max()
    print('inverse fit: iterations', fit.iterations, 'status', fit.status, f'worst relative error {err:.1e}')
    check_history(fit)
    assert (fit.status == sysid.CONVERGED).all() and err <= INV_TOL


def test_flight_fit_under_emulation(emu, small):
    check_flight(emu, 2, 6)


def test_inverse_fit_under_emulation(emu, small):
    check_inverse_fit(emu)


def test_template_fit_under_emulation(emu, small):
    fit, err = check_template(emu, 1)
    assert (fit.status == sysid.CONVERGED).all() and err.max() <= FIT_TOL


# ---- 6. LM bookkeeping -------------------------------------------------------------------------------------------------------------
def test_lm_bookkeeping():
    """the host loop on a synthetic sweep: a rejected trial leaves the values as they were, the history never rises, a trial that would
    make a non-negative field negative or a scale <= 0 is refused without a sweep, a zero diagonal is held"""
    m = load_model('flight')
    j = int(np.argmax(dv.compiled_params(m, 'dof_damping')))
    dirs, _ = dv._directions(m, [dv.Scale('dof_damping'), ('gravity', [2]), ('body_mass', [1])], None)
    vals = {n: np.tile(dv.compiled_params(m, n), (2, 1)) for n in st.PARAMS}
    d0 = vals['dof_damping'][0, j]
    unit = np.array([1.0, vals['gravity'][0, 2], vals['body_mass'][0, 1]])
    target, scale = np.array([[1.3, 0.98, 1.01], [0.9, 1.02, 0.99]]) * unit, 1.0 / np.abs(unit)
    events = []

    def state(tv, p):
        return np.array([tv['dof_damping'][p][j] / d0, tv['gravity'][p][2], tv['body_mass'][p][1]])

    def sweep(idx, tv):                 # least squares plus a wall past a damping scale of 1.2: the full steps of problem 0 overshoot
        cost, H, g = np.zeros(len(idx)), np.zeros((len(idx), 3, 3)), np.zeros((len(idx), 3))
        for p, l in enumerate(idx):
            x = state(tv, p)
            wall = np.sqrt(2e3) * max(0.0, x[0] - 1.2)
            r = np.r_[(x - target[l]) * scale, wall]
            J = np.r_[np.diag(scale * np.array([x[0], 1.0, 1.0])), [[np.sqrt(2e3) * x[0] * (wall > 0), 0.0, 0.0]]]
            cost[p] = 0.5 * r @ r
            H[p], g[p] = J.T @ J, J.T @ r
            events.append((l, x, cost[p]))
        return cost, H, g, np.ones(len(idx), np.int32)

    J, H, g, count, hist, iters, status = sysid._lm(dirs, vals, 2, sweep, 50, 1e-9, sysid._Clock(None))
    rejected = 0
    for l in range(2):
        mine = [(x, c) for k, x, c in events if k == l]
        x_acc, c_acc = mine[0]
        for x, c in mine[1:]:
            if c < c_acc:
                x_acc, c_acc = x, c
            else:
                rejected += 1
        assert np.array_equal(state(vals, l), x_acc) and J[l] == c_acc == hist[l][np.isfinite(hist[l])][-1]
        h = hist[l][np.isfinite(hist[l])]
        assert (np.diff(h) < 0).all() and len(h) == iters[l] + 1
    assert rejected > 0 and (status == sysid.CONVERGED).all()
    assert abs(state(vals, 0)[0] - 1.2) < 1e-3 and abs(state(vals, 1)[0] - 0.9) < 1e-6
    assert sysid._trial(dirs, vals, 0, np.array([0.0, 0.0, -1.0])) is None           # body_mass < 0
    assert sysid._trial(dirs, vals, 0, np.array([-1.0, 0.0, 0.0])) is None           # a scale to 0
    t = sysid._trial(dirs, vals, 0, np.array([-0.5, 2e3, 0.0]))                      # gravity may change sign
    assert t['gravity'][2] > 0 and np.array_equal(t['dof_damping'], vals['dof_damping'][0] * 0.5)
    d = sysid._step(np.diag([2.0, 0.0, 1.0]), np.array([1.0, 5.0, 1.0]), 0.0)
    assert d[1] == 0 and np.allclose(d, [-0.5, 0.0, -1.0])
    with pytest.raises(ValueError, match='share the element'):
        sysid._prepare(m, [dv.Scale('body_mass'), ('body_mass', [1])], None, None, 1, False)


def check_fit_bits(lib, monkeypatch, envs, L=2, T=3):
    """a fit's bits alone, in a batch and under another sysid.ENVS"""
    fits = []
    for e in envs:
        monkeypatch.setattr(sysid, 'ENVS', e)
        m, groups, _, fit, (q, v, u, qd, vd) = flight_fit(lib, L, T, groups=('dof_damping', 'body_mass'), max_iter=3)
        fits.append(fit)
    alone = sysid.fit_transitions(m, q[1:], v[1:], u[1:], qd[1:], vd[1:], row_weights(m, vd), params=groups, n_substeps=4, lib_path=lib,
                                  max_iter=3)
    a = fits[0]
    for b in fits[1:]:
        assert same([a.values[n] for n in sorted(a.values)], [b.values[n] for n in sorted(b.values)])
        assert same((a.cost, a.H, a.g, a.iterations, a.status, a.count), (b.cost, b.H, b.g, b.iterations, b.status, b.count))
    assert same([a.values[n][1:] for n in sorted(a.values)], [alone.values[n] for n in sorted(alone.values)])
    assert same((a.H[1:], a.g[1:], a.iterations[1:], a.cost[1:, :alone.cost.shape[1]]), (alone.H, alone.g, alone.iterations, alone.cost))
    assert np.isnan(a.cost[1:, alone.cost.shape[1]:]).all()


def test_fit_bits_alone_batched_and_envs_under_emulation(emu, monkeypatch):
    check_fit_bits(emu, monkeypatch, (64, 24))


# ---- GPU tier ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_gpu_normal_equations():
    ge.build()
    normal_cases(None, 4096)


@pytest.mark.gpu
def test_gpu_invariance_and_refusals():
    ge.build()
    check_invariance(None, 4096)
    check_refusals(None)


@pytest.mark.gpu
def test_gpu_flight_fit():
    ge.build()
    check_flight(None, 4, 64)


@pytest.mark.gpu
def test_gpu_template_fit():
    ge.build()
    for n_sub in (1, 10):
        fit, err = check_template(None, n_sub)
        assert (fit.status == sysid.CONVERGED).all() and err.max() <= FIT_TOL


@pytest.mark.gpu
def test_gpu_inverse_fit():
    ge.build()
    check_inverse_fit(None)


@pytest.mark.gpu
def test_gpu_flight_density():
    """(d) the flight fit with the density scale added, the direction plain Gauss-Newton does not recover (test_param_fd's xfail):
    the cost history never rises and every problem ends with a status; the recovered density is printed, not gated"""
    ge.build()
    m, groups, s_true, fit, _ = flight_fit(None, 4, 64, groups=('dof_damping', 'actuator_gainprm', 'body_mass', 'density'))
    check_history(fit)
    s = scales(m, fit, groups)
    print('flight with density: iterations', fit.iterations, 'status', fit.status, 'fitted / true', (s / s_true).round(4).tolist())
    assert set(fit.status.tolist()) <= {sysid.CONVERGED, sysid.ITER_CAP, sysid.LAMBDA_CAP}


@pytest.mark.gpu
def test_gpu_fit_bits(monkeypatch):
    ge.build()
    check_fit_bits(None, monkeypatch, (4096, 512), L=3, T=8)
