"""Batched rollouts (fb_rollout*, flybody_b200.rollout): mechanics bit for bit against the host loop of set_control / step / get on the
same stepper; independence of position, batch size and repeated slots, and isolation of the bank and the other queries; the feedback
law exactly (K = 0 and a nominal equal to the state give the open loop bit for bit; the recorded ctrl against an fp64 restatement) and
its convention to first order against transition_fd's A and B; a TVLQR run; the front end.  CPU tier: the host-emulation build of the
kernel source on small handles; GPU tier (-m gpu): the same through the CUDA library on 4096-env handles, which also runs the step
graph.  "Bit for bit" compares uint32 views.

Gates are 2.5 x the larger of the host-emulation and H100 measurements (both named beside each constant)."""
import numpy as np
import pytest

import __graft_entry__ as ge
import fd_reference as fr
import smooth_states as ss
from flybody_b200 import derivatives as dv, rollout as ro, stepper as st
from flybody_b200.flymodel import load_model
from flybody_b200.inverse_kinematics import _differentiate_pos
from test_model_params import patched, random_params, start_state

# ---- gates (measured: host emulation / H100 80GB HBM3 at a 700 W power limit; worst case) -------------------------------------------
CTRL_GATE = 5e-7           # recorded ctrl against u + K (x - xref) in fp64, relative to |u| + |K| |dx|: measured 1.3e-7 emu / 2.0e-7 H100 (flight)
FIRST_ORDER = 4.8e-4       # closed-loop deviation after one control step against (A + B K) d0, relative: measured 1.8e-4 emu / 1.9e-4 H100

SUBSTEPS = {'walk': 10, 'flight': 4, 'template': 10, 'ball': 10}     # the tasks' control steps
GPU_ENVS = 4096


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


@pytest.fixture(scope='module')
def emu():
    ge.build()
    return ge.EMU


def gpu_lib():
    ge.build()
    return None


def fill_bank(sim, m, states, params=None, applied=False, sensors=True, seed=0):
    """bank rows 0 .. len(states)-1 of (q, v) states at a cold warm start (env k -> slot k; the envs past them repeat the last);
    params: one random parameter set per row; applied: allocate the applied-force arrays first.  -> the rows' (qpos, qvel, act)"""
    n = len(states)
    pad = np.minimum(np.arange(sim.n_envs), n - 1)
    if params:
        p = [random_params(m, seed + k) for k in range(n)]
        for name in st.PARAMS:
            sim.param_set(name, np.array([p[k][name] for k in pad]))
    if applied:
        sim.applied_ptrs()
    sim.reset(np.array([s[0] for s in states])[pad], np.array([s[1] for s in states])[pad])
    sim.forward()
    sim.state_bank(max(n, 2))
    sim.save_state(slots=np.arange(n), env_ids=np.arange(n))
    if sensors:
        sim.query_sensors(True)
    return sim.get(st.QPOS)[:n], sim.get(st.QVEL)[:n], sim.get(st.ACT)[:n]


def inputs(m, n, T, seed, applied=False):
    rs = np.random.RandomState(seed)
    u = rs.uniform(-0.5, 0.5, (n, T, m.nu)).astype(np.float32)
    if not applied:
        return u, None, None
    qf = rs.uniform(-1e-3, 1e-3, (n, T, m.nv)).astype(np.float32)
    xf = rs.uniform(-1e-3, 1e-3, (n, T, m.nbody, 6)).astype(np.float32)
    return u, qf, xf


def host_loop(sim, slots, u, nsub, qf=None, xf=None, sensors=True):
    """the hand-written loop the rollout replaces: load, then per step set_control (set_applied), step and the reads"""
    n, T = u.shape[:2]
    pad = np.minimum(np.arange(sim.n_envs), n - 1)
    sim.load_state(slots=slots, env_ids=np.arange(n))
    out = [[] for _ in range(8 if sensors else 6)]
    for t in range(T):
        sim.set_control(u[pad, t])
        if qf is not None:
            sim.set_applied(qfrc=qf[pad, t], xfrc=xf[pad, t])
        sim.step(nsub)
        got = [sim.get(f)[:n] for f in (st.QPOS, st.QVEL, st.ACT, st.CTRL)] + [sim.get(st.TIME)[:n, 0], sim.get(st.FLAGS)[:n, 0].astype(np.int32)]
        if sensors:
            got += [sim.get(st.SENSORDATA)[:n], sim.get(st.SENSOR_MEAN)[:n]]
        for o, g in zip(out, got):
            o.append(g)
    return [np.stack(o, 1) for o in out]


def assert_records_equal(a, b, what):
    for k, (x, y) in enumerate(zip(a, b)):
        assert x.shape == y.shape, (what, k, x.shape, y.shape)
        assert np.array_equal(bits(x) if x.dtype != np.int32 else x, bits(y) if y.dtype != np.int32 else y), (what, k)


def read_all(sim, sensors=True):
    return list(sim.rollout_read()) + (list(sim.rollout_sensor_read()) if sensors else [])


# ---- 1. mechanics against the hand-written loop ----------------------------------------------------------------------------------------
def check_mechanics(lib, variant, nsub, n_envs, n, extras, T=3):
    m = load_model(variant)
    sim = st.BatchedStepper(m, n_envs, lib_path=lib)
    states = [start_state(m, s) for s in range(3)]
    fill_bank(sim, m, states, params=extras, applied=extras)
    slots = np.arange(n) % len(states)
    u, qf, xf = inputs(m, n, T, 7, applied=extras)
    sim.rollout(slots, u, nsub, qf, xf)
    got = read_all(sim)
    assert np.array_equal(got[3], u)                             # ctrl as written: not clamped
    want = host_loop(sim, slots, u, nsub, qf, xf)
    assert_records_equal(got, want, (variant, nsub, n_envs, n, extras))
    sim.close()


MECH = [(v, nsub, full, extras) for v in SUBSTEPS for nsub, full, extras in ((1, False, False), (SUBSTEPS[v], True, True))]


@pytest.mark.parametrize('variant,nsub,full,extras', MECH)
def test_mechanics_under_emulation(emu, variant, nsub, full, extras):
    check_mechanics(emu, variant, nsub, 4, 4 if full else 3, extras)


@pytest.mark.gpu
@pytest.mark.parametrize('variant,nsub,full,extras', MECH)
def test_gpu_mechanics(variant, nsub, full, extras):
    check_mechanics(gpu_lib(), variant, nsub, GPU_ENVS, GPU_ENVS if full else 1000, extras, T=4)


# ---- 2. independence and isolation -----------------------------------------------------------------------------------------------------
def check_independence(lib, variant, n_envs):
    m = load_model(variant)
    nsub, T = SUBSTEPS[variant], 3
    n_envs = max(n_envs, 1 + 2 * m.nv + m.na + m.nu)             # room for a forward-difference transition
    sim = st.BatchedStepper(m, n_envs, lib_path=lib)
    states = [start_state(m, s) for s in range(3)]
    fill_bank(sim, m, states)
    rows = sim.read_states([0, 1, 2])
    # the other queries' results, before the rollouts
    sim.fd_transition([1], centered=False, n_substeps=1)
    fd0 = sim.fd_read()
    sim.inverse(np.zeros((1, m.nv), np.float32))
    inv0 = sim.inverse_read()
    u, _, _ = inputs(m, 4, T, 3)
    slots = [2, 0, 1, 0]
    sim.rollout(slots, u, nsub)
    full = read_all(sim)
    sim.rollout([0], u[3:4], nsub)                               # one rollout alone, at another position
    assert_records_equal(read_all(sim), [x[3:4] for x in full], 'alone')
    small = st.BatchedStepper(m, 2, lib_path=lib)                # another batch size, rows moved across
    small.state_bank(3)
    small.write_states([0, 1, 2], rows)
    small.query_sensors(True)
    small.rollout([1, 2], u[[2, 0]], nsub)
    assert_records_equal(read_all(small), [x[[2, 0]] for x in full], 'small handle')
    # the bank and the other queries are untouched
    assert np.array_equal(sim.read_states([0, 1, 2]), rows)
    for a, b in zip(sim.fd_read(), fd0):
        assert np.array_equal(bits(a), bits(b))
    for a, b in zip(sim.inverse_read(), inv0):
        assert np.array_equal(bits(a), bits(b))
    # a step afterwards is a step of a handle that never ran a rollout
    fresh = st.BatchedStepper(m, n_envs, lib_path=lib)
    fresh.state_bank(3)
    fresh.write_states([0, 1, 2], rows)
    for h in (sim, fresh):
        h.load_state(slots=[1, 0, 2], env_ids=[0, 1, 2])
        h.set_control(np.full(m.nu, 0.1, np.float32))
        h.step(nsub)
    for f in (st.QPOS, st.QVEL, st.ACT, st.SENSORDATA, st.SENSOR_MEAN):
        assert np.array_equal(bits(sim.get(f)[:3]), bits(fresh.get(f)[:3])), f
    for h in (sim, small, fresh):
        h.close()


@pytest.mark.parametrize('variant', ['template', 'flight'])
def test_independence_under_emulation(emu, variant):
    check_independence(emu, variant, 6)


@pytest.mark.gpu
@pytest.mark.parametrize('variant', ['walk', 'flight'])
def test_gpu_independence(variant):
    check_independence(gpu_lib(), variant, GPU_ENVS)


# ---- 3. feedback, exactly --------------------------------------------------------------------------------------------------------------
def state_rows(m, q, v, a, rec):
    """x_t, the state each step starts from: the initial state, then the records"""
    x0 = np.concatenate([q, v, a], -1)[:, None]
    xr = np.concatenate([rec[0], rec[1], rec[2]], -1)
    return np.concatenate([x0, xr[:, :-1]], 1)


def tangent(m, x, xref):
    """transition_fd's tangent x - xref in fp64 (mj_differentiatePos(xref qpos, qpos), then qvel and act)"""
    nq, nv = m.nq, m.nv
    x = np.asarray(x, np.float64)
    x, xref = x.reshape(-1, x.shape[-1]), np.broadcast_to(np.asarray(xref, np.float64), x.shape).reshape(-1, x.shape[-1])
    dq = _differentiate_pos(m, xref[:, :nq], x[:, :nq], 1.0)
    return np.concatenate([dq, x[:, nq:nq + nv] - xref[:, nq:nq + nv], x[:, nq + nv:] - xref[:, nq + nv:]], -1)


def check_feedback(lib, variant, n_envs, n, measure=None):
    m = load_model(variant)
    nsub, T, nx = SUBSTEPS[variant], 4, 2 * m.nv + m.na
    sim = st.BatchedStepper(m, n_envs, lib_path=lib)
    q0, v0, a0 = fill_bank(sim, m, [start_state(m, 5)])
    u, _, _ = inputs(m, 1, T, 11)
    u = np.repeat(u, n, 0)
    slots = np.zeros(n, np.int32)
    sim.rollout(slots, u, nsub)
    open_loop = read_all(sim)
    rs = np.random.RandomState(2)
    # K = 0 and any nominal: the open loop
    xref = rs.uniform(-1, 1, (T, m.nq + m.nv + m.na)).astype(np.float32)
    sim.rollout_feedback(xref, np.zeros((T, m.nu, nx), np.float32))
    sim.rollout(slots, u, nsub)
    assert_records_equal(read_all(sim), open_loop, 'K = 0')
    # the nominal the open loop's own trajectory and random K: the tangent is exactly 0
    xs = state_rows(m, q0, v0, a0, [x[:1] for x in open_loop[:3]])[0].astype(np.float32)
    K = rs.uniform(-1, 1, (T, m.nu, nx)).astype(np.float32)
    sim.rollout_feedback(xs, K)
    sim.rollout(slots, u, nsub)
    assert_records_equal(read_all(sim), open_loop, 'xref = x')
    # a nominal off the trajectory: the recorded ctrl is u + K (x - xref), x the recorded state before the step
    xref = xs.copy()
    xref[:, m.nq:] += rs.uniform(-0.05, 0.05, (T, m.nv + m.na)).astype(np.float32)
    qa = [int(m.jnt_qposadr[j]) for j in range(m.njnt) if int(m.jnt_type[j]) == 3]
    xref[:, qa] += rs.uniform(-0.05, 0.05, (T, len(qa))).astype(np.float32)
    K = (rs.uniform(-1, 1, (T, m.nu, nx)) / nx).astype(np.float32)
    sim.rollout_feedback(xref, K)
    sim.rollout(slots, u, nsub)
    rec = read_all(sim)
    x = state_rows(m, q0[:1].repeat(n, 0), v0[:1].repeat(n, 0), a0.repeat(n, 0), rec[:3])
    dx = tangent(m, x, np.broadcast_to(xref, x.shape)).reshape(n, T, nx)
    want = u + np.einsum('tux,ntx->ntu', K.astype(np.float64), dx)
    scale = np.abs(u) + np.einsum('tux,ntx->ntu', np.abs(K.astype(np.float64)), np.abs(dx))
    err = (np.abs(rec[3] - want) / scale).max()
    assert np.abs(dx).max() > 1e-3
    if measure is not None:
        measure.append(err)
    assert err < CTRL_GATE, (variant, err)
    sim.rollout_feedback()                                       # cleared: the open loop again
    sim.rollout(slots, u, nsub)
    assert_records_equal(read_all(sim), open_loop, 'cleared')
    sim.close()


@pytest.mark.parametrize('variant', ['walk', 'flight', 'ball'])
def test_feedback_exactly_under_emulation(emu, variant):
    check_feedback(emu, variant, 3, 3)


@pytest.mark.gpu
@pytest.mark.parametrize('variant', ['walk', 'flight', 'ball'])
def test_gpu_feedback_exactly(variant):
    check_feedback(gpu_lib(), variant, GPU_ENVS, GPU_ENVS)


# ---- 4. the convention against transition_fd, to first order; a TVLQR run ------------------------------------------------------------
def perturbed(m, q, v, d):
    """(q, v) moved by the tangent d [2 nv] (mj_integratePos one dof after the other)"""
    x = (q.astype(np.float64), v.astype(np.float64), np.zeros(m.na), np.zeros(m.nu))
    for j in range(2 * m.nv):
        x = fr._nudge(m, x, j, d[j])
    return x[0].astype(np.float32), x[1].astype(np.float32)


def rollout_rows(sim, m, states, u, nsub, xref=None, K=None):
    """each (q, v) state rolled through u [T, nu] from a cold warm start (the rows of a fresh bank), with the feedback law (xref, K)
    -> (the initial states [n, nq + nv + na] as the envs hold them, the records)"""
    n = len(states)
    x0 = np.concatenate(fill_bank(sim, m, states, sensors=False), -1)
    sim.rollout_feedback(xref, K)
    sim.rollout(np.arange(n), np.repeat(u[None], n, 0), nsub)
    return x0, sim.rollout_read()


def check_first_order(lib, n_envs, measure=None):
    m = ss.free_model(load_model('flight'))
    nsub, nx, n = SUBSTEPS['flight'], 2 * m.nv, 6
    q0, v0 = (x.astype(np.float32) for x in start_state(m, 3))
    u0 = np.random.RandomState(4).uniform(-0.5, 0.5, (1, m.nu)).astype(np.float32)
    rs = np.random.RandomState(6)
    K = (rs.uniform(-1, 1, (1, m.nu, nx)) * 10 / nx).astype(np.float32)
    scale = np.concatenate([np.ones(m.nv), np.maximum(1, np.abs(v0))])
    states = [(q0, v0)] + [perturbed(m, q0, v0, 1e-3 * rs.uniform(-1, 1, nx) * scale) for _ in range(n - 1)]
    sim = st.BatchedStepper(m, n_envs, lib_path=lib)
    x0, rec = rollout_rows(sim, m, states[:1], u0, nsub)            # the nominal's initial state as the env holds it: the law's xref
    x0, rec = rollout_rows(sim, m, states, u0, nsub, x0[:1], K)
    r = dv.transition_fd(m, x0[0, :m.nq], x0[0, m.nq:], u0[0], n_substeps=nsub, lib_path=lib)
    d0 = tangent(m, x0, x0[:1])
    x1 = np.concatenate([rec[0][:, 0], rec[1][:, 0]], -1)
    d1 = tangent(m, x1, x1[:1])
    pred = d0 @ (r.A + r.B @ K[0].astype(np.float64)).T
    open_pred = d0 @ r.A.T
    err = max(np.linalg.norm(d1[k] - pred[k]) / np.linalg.norm(pred[k]) for k in range(1, n))
    assert min(np.linalg.norm(pred[k] - open_pred[k]) / np.linalg.norm(pred[k]) for k in range(1, n)) > 10 * FIRST_ORDER   # K matters
    if measure is not None:
        measure.append(err)
    assert err < FIRST_ORDER, err
    sim.close()


def test_first_order_convention_under_emulation(emu):
    check_first_order(emu, 6)


@pytest.mark.gpu
def test_gpu_first_order_convention():
    check_first_order(gpu_lib(), GPU_ENVS)


def check_tvlqr(lib, n_envs):
    """TVLQR from a Riccati recursion on transition_fd along a nominal rollout: from seeded perturbations of the initial state the
    closed loop ends closer to the nominal than the open loop"""
    m = ss.free_model(load_model('flight'))
    nsub, T, nx, seeds = SUBSTEPS['flight'], 6, 2 * m.nv, 5
    q0, v0 = (x.astype(np.float32) for x in start_state(m, 8))
    u = np.random.RandomState(9).uniform(-0.3, 0.3, (T, m.nu)).astype(np.float32)
    sim = st.BatchedStepper(m, n_envs, lib_path=lib)
    x0, nom = rollout_rows(sim, m, [(q0, v0)], u, nsub)
    xs = np.concatenate([x0, np.concatenate([nom[0][0], nom[1][0]], -1)], 0)          # x_0 .. x_T
    r = dv.transition_fd(m, xs[:T, :m.nq], xs[:T, m.nq:], u, n_substeps=nsub, lib_path=lib)
    scale = np.concatenate([np.ones(m.nv), np.maximum(1, np.abs(v0))])
    Q, R = np.diag(1 / scale ** 2), 1e-2 * np.eye(m.nu)
    P, K = Q, np.zeros((T, m.nu, nx))
    for t in range(T - 1, -1, -1):
        A, B = r.A[t], r.B[t]
        K[t] = -np.linalg.solve(R + B.T @ P @ B, B.T @ P @ A)
        P = Q + A.T @ P @ (A + B @ K[t])
    rs = np.random.RandomState(10)
    states = [perturbed(m, q0, v0, 1e-2 * rs.uniform(-1, 1, nx) * scale) for _ in range(seeds)]
    end = {}
    for name, gains in (('open', None), ('closed', K.astype(np.float32))):
        _, rec = rollout_rows(sim, m, states, u, nsub, None if gains is None else xs[:T], gains)
        d = tangent(m, np.concatenate([rec[0][:, -1], rec[1][:, -1]], -1), np.broadcast_to(xs[T], (seeds, len(xs[T]))))
        end[name] = np.sqrt(np.einsum('ki,ij,kj->k', d, Q, d))
    assert (end['closed'] < end['open']).all(), end
    sim.close()


def test_tvlqr_under_emulation(emu):
    check_tvlqr(emu, 5)


@pytest.mark.gpu
def test_gpu_tvlqr():
    check_tvlqr(gpu_lib(), GPU_ENVS)


# ---- 5. the front end --------------------------------------------------------------------------------------------------------------
def test_front_end_shapes_chunks_and_params(emu, monkeypatch):
    m = load_model('template')
    B, T, nsub = 3, 2, 2
    st0 = [start_state(m, s) for s in range(B)]
    q, v = np.array([s[0] for s in st0]), np.array([s[1] for s in st0])
    u, qf, xf = inputs(m, B, T, 1, applied=True)
    whole = ro.rollout(m, q, v, u, n_substeps=nsub, qfrc_applied=qf, xfrc_applied=xf, sensors=True, lib_path=emu)
    assert isinstance(whole, ro.RolloutSensors)
    shapes = [(B, T, m.nq), (B, T, m.nv), (B, T, m.na), (B, T, m.nu), (B, T), (B, T), (B, T, m.nsensordata), (B, T, m.nsensordata)]
    assert [x.shape for x in whole] == shapes and whole.flags.dtype == np.int32
    monkeypatch.setattr(ro, 'ENVS', 2)                           # chunked: the same bits
    parts = ro.rollout(m, q, v, u, n_substeps=nsub, qfrc_applied=qf, xfrc_applied=xf, sensors=True, lib_path=emu)
    assert_records_equal(list(parts), list(whole), 'chunks')
    one = ro.rollout(m, q[1], v[1], u[1], n_substeps=nsub, qfrc_applied=qf[1], xfrc_applied=xf[1], sensors=True, lib_path=emu)
    assert_records_equal([x[None] for x in one], [x[1:2] for x in whole], 'single')
    plain = ro.rollout(m, q[1], v[1], u[1], n_substeps=nsub, lib_path=emu)
    assert isinstance(plain, ro.Rollout) and plain.qpos.shape == (T, m.nq)
    # params: each rollout as a one-env handle of its patched model
    p = [random_params(m, 20 + k) for k in range(B)]
    params = {name: np.array([x[name] for x in p]) for name in ('body_mass', 'dof_damping', 'actuator_gainprm')}
    got = ro.rollout(m, q, v, u, n_substeps=nsub, params=params, lib_path=emu)
    for k in range(B):
        pm = patched(m, {name: x[k] for name, x in params.items()})
        want = ro.rollout(pm, q[k], v[k], u[k], n_substeps=nsub, lib_path=emu)
        assert_records_equal([x[k] for x in got], list(want), ('params', k))
    shared = ro.rollout(m, q, v, u, n_substeps=nsub, params={'dof_damping': params['dof_damping'][0]}, lib_path=emu)
    pm = patched(m, {'dof_damping': params['dof_damping'][0]})
    assert_records_equal(list(shared), list(ro.rollout(pm, q, v, u, n_substeps=nsub, lib_path=emu)), 'shared params')
    # feedback through the front end: a zero gain is the open loop
    nx = 2 * m.nv + m.na
    fb = ro.rollout(m, q, v, u, n_substeps=nsub, x_ref=np.zeros((T, m.nq + m.nv + m.na)), K=np.zeros((T, m.nu, nx)), lib_path=emu)
    assert_records_equal(list(fb), list(ro.rollout(m, q, v, u, n_substeps=nsub, lib_path=emu)), 'front-end K = 0')


def test_refusals(emu):
    m = load_model('flight')
    nx = 2 * m.nv + m.na
    q, v = start_state(m, 0)
    u = np.zeros((2, 3, m.nu), np.float32)
    with pytest.raises(ValueError):
        ro.rollout(m, q[None].repeat(2, 0), v[None].repeat(2, 0), u[:1], lib_path=emu)            # bad shapes
    with pytest.raises(ValueError):
        ro.rollout(m, q, v, u[0], x_ref=np.zeros((2, m.nq + m.nv)), K=np.zeros((2, m.nu, nx)), lib_path=emu)   # wrong horizon
    with pytest.raises(ValueError):
        ro.rollout(m, q, v, u[0], x_ref=np.zeros((3, m.nq + m.nv)), lib_path=emu)                  # x_ref without K
    sim = st.BatchedStepper(m, 2, lib_path=emu)
    with pytest.raises(st.StepperError, match='no state bank'):
        sim.rollout([0], u[:1])
    sim.reset(q, v)
    sim.state_bank(3)
    sim.save_state([0], [0])
    with pytest.raises(st.StepperError, match='never written'):
        sim.rollout([1], u[:1])
    with pytest.raises(st.StepperError, match='n_envs'):
        sim.rollout([0, 0, 0], np.zeros((3, 3, m.nu)))
    with pytest.raises(st.StepperError, match='T >= 1'):
        sim.rollout([0], np.zeros((1, 0, m.nu)))
    with pytest.raises(st.StepperError, match='n_substeps'):
        sim.rollout([0], u[:1], n_substeps=0)
    with pytest.raises(st.StepperError, match='non-finite'):
        sim.rollout([0], np.full((1, 3, m.nu), np.nan))
    with pytest.raises(st.StepperError, match='applied-force arrays'):
        sim.rollout([0], u[:1], qfrc_applied=np.zeros((1, 3, m.nv)))
    with pytest.raises(st.StepperError, match='no rollout'):
        sim.rollout_read()
    sim.rollout_feedback(np.zeros((2, m.nq + m.nv)), np.zeros((2, m.nu, nx)))
    with pytest.raises(st.StepperError, match='feedback law has 2 steps'):
        sim.rollout([0], u[:1])
    with pytest.raises(st.StepperError, match='non-finite'):
        sim.rollout_feedback(np.full((2, m.nq + m.nv), np.inf), np.zeros((2, m.nu, nx)))
    sim.rollout_feedback()
    sim.rollout([0], u[:1])
    with pytest.raises(st.StepperError, match='sensors off'):
        sim.rollout_sensor_read()
    sim.reset_hold([0], q)                                       # a row saved while its env is held
    sim.save_state([2], [0])
    with pytest.raises(st.StepperError, match='held'):
        sim.rollout([2], u[:1])
    sim.close()


@pytest.mark.gpu
def test_gpu_torch_inputs_and_outputs_by_pointer():
    import torch
    lib = gpu_lib()
    m = load_model('walk')
    nsub, T, n, nx = SUBSTEPS['walk'], 3, 512, 2 * m.nv + m.na
    sim = st.BatchedStepper(m, GPU_ENVS, lib_path=lib)
    fill_bank(sim, m, [start_state(m, s) for s in range(3)], applied=True)
    slots = np.arange(n) % 3
    u, qf, xf = inputs(m, n, T, 5, applied=True)
    rs = np.random.RandomState(1)
    xref = rs.uniform(-0.1, 0.1, (T, m.nq + m.nv + m.na)).astype(np.float32)
    K = (rs.uniform(-1, 1, (T, m.nu, nx)) / nx).astype(np.float32)
    sim.rollout_feedback(xref, K)
    sim.rollout(slots, u, nsub, qf, xf)
    host = read_all(sim)
    dev = [torch.from_numpy(x).cuda() for x in (u, qf, xf, xref, K)]
    sim.rollout_feedback(dev[3].data_ptr(), dev[4].data_ptr(), T=T, is_device=True)
    sim.rollout(slots, dev[0].data_ptr(), nsub, dev[1].data_ptr(), dev[2].data_ptr(), T=T, is_device=True)
    out = [torch.zeros(x.shape, dtype=torch.int32 if x.dtype == np.int32 else torch.float32, device='cuda') for x in host]
    sim.rollout_read(out=out[:6])
    sim.rollout_sensor_read(out=out[6:])
    assert_records_equal([x.cpu().numpy() for x in out], host, 'torch')
    sim.close()
