"""Applied forces (mjData.qfrc_applied / xfrc_applied, fb_set / fb_write_state / fb_applied_ptrs / fb_clear_applied): the smooth force of
the step gains qfrc_applied + J^T xfrc_applied, held against the fp64 oracle's kinematics and smooth force plus the fp64 restatement of
the term in applied_reference.py; two known answers; persistence, reset and clear semantics.  CPU tier: the host-emulation build of the
kernel source.  GPU tier (-m gpu): the same on the H100."""
import numpy as np
import pytest

import __graft_entry__ as ge
from flybody_b200 import stepper as st
from flybody_b200.flymodel import load_model
from oracle import fly_oracle as fo
from parity_common import random_state, rel_err, STAGE_TOL
from applied_reference import apply_ft, applied_term, frames


@pytest.fixture(scope='module')
def emu():
    ge.build()
    return ge.EMU


def random_applied(m, seed, bodies=6):
    """qfrc [nv] and xfrc [nbody, 6] on `bodies` random bodies (forces ~ the fly's weight, torques ~ weight x body length)"""
    rs = np.random.RandomState(seed)
    weight = float(m.body_subtreemass[1]) * abs(float(m.opt_gravity[2]))
    qfrc = rs.uniform(-1, 1, m.nv) * 0.1 * weight
    xfrc = np.zeros((m.nbody, 6))
    for b in rs.choice(np.arange(1, m.nbody), bodies, replace=False):
        xfrc[b, :3] = rs.uniform(-1, 1, 3) * weight
        xfrc[b, 3:] = rs.uniform(-1, 1, 3) * weight * 0.05
    return qfrc.astype(np.float32).astype(np.float64), xfrc.astype(np.float32).astype(np.float64)


def free_state(m, seed):
    """the template pose lifted 2 cm, turned to a random orientation, random velocities: no constraint rows (the oracle's nefc is 0)"""
    rs = np.random.RandomState(seed)
    root = m.jnt_id('walker/')
    rq = int(m.jnt_qposadr[root])
    q, v = random_state(m, seed, 0.0, 1.0)
    quat = rs.normal(size=4)
    q[rq + 2] += 2.0
    q[rq + 3:rq + 7] = (quat / np.linalg.norm(quat)).astype(np.float32)
    return q, v


def applied_parity(m, sim, seed, qfrc=None, xfrc=None, env=0, free=False):
    """forward on a random state with the given applied forces -> relative errors of qfrc_smooth and (free=True: a state without
    constraint rows, where qacc = M^-1 qfrc_smooth) of qacc, against the oracle without them plus the fp64 term; and that reference"""
    o = fo.Oracle(m, tolerance=1e-12)
    q, v = free_state(m, seed) if free else random_state(m, seed, 0.1, 1.0)
    ctrl = np.random.RandomState(seed + 100).uniform(-0.5, 0.5, m.nu)
    o.reset(q, v)
    sim.reset(q, v)                        # (a reset zeroes applied forces: set them afterwards)
    o.set(fo.CTRL, ctrl)
    sim.set_control(ctrl)
    sim.set_applied(qfrc, xfrc)
    o.forward()
    sim.forward()
    term = applied_term(m, o, qfrc, xfrc)
    smooth = o.get(fo.QFRC_SMOOTH) + term
    e_s = rel_err(smooth, sim.get(st.QFRC_SMOOTH)[env])
    assert int(o.get(fo.NEFC)[0]) == int(sim.get(st.NEFC)[env, 0])
    e_a = None
    if free:
        assert int(o.get(fo.NEFC)[0]) == 0
        qacc = o.get(fo.QACC) + np.linalg.solve(o.get(fo.QM_DENSE).reshape(m.nv, m.nv), term)
        e_a = rel_err(qacc, sim.get(st.QACC)[env])
    return e_s, e_a, smooth


@pytest.mark.parametrize('seed', [0, 1])
def test_qfrc_applied_matches_oracle(emu, seed):
    m = load_model('walk')
    qfrc, _ = random_applied(m, seed)
    e_s, _, _ = applied_parity(m, st.BatchedStepper(m, 2, lib_path=emu), seed, qfrc=qfrc)
    assert e_s < STAGE_TOL['smooth'], e_s
    e_s, e_a, _ = applied_parity(m, st.BatchedStepper(m, 2, lib_path=emu), seed, qfrc=qfrc, free=True)
    assert e_s < STAGE_TOL['smooth'] and e_a < STAGE_TOL['smooth'], (e_s, e_a)


@pytest.mark.parametrize('seed', [0, 1])
def test_xfrc_applied_matches_oracle(emu, seed):
    m = load_model('walk')
    qfrc, xfrc = random_applied(m, seed, bodies=8)
    for kw in (dict(xfrc=xfrc), dict(qfrc=qfrc, xfrc=xfrc)):
        e_s, _, _ = applied_parity(m, st.BatchedStepper(m, 2, lib_path=emu), seed, **kw)
        assert e_s < STAGE_TOL['smooth'], (sorted(kw), e_s)
        e_s, e_a, _ = applied_parity(m, st.BatchedStepper(m, 2, lib_path=emu), seed, free=True, **kw)
        assert e_s < STAGE_TOL['smooth'] and e_a < STAGE_TOL['smooth'], (sorted(kw), e_s, e_a)


def test_reference_jacobian_matches_finite_differences():
    """the fp64 J^T of applied_reference against a finite difference of the oracle's kinematics: a body point moved by dof k"""
    m = load_model('walk')
    o = fo.Oracle(m, tolerance=1e-12)
    q, _ = random_state(m, 9, 0.1, 0.0)
    o.reset(q)
    b = m.body_id('walker/tarsus_T2_left')
    xp, _, xi = frames(m, o)
    assert np.abs(xp - o.get(fo.XPOS).reshape(-1, 3)).max() < 1e-12      # the reference's kinematics are the oracle's
    local = o.get(fo.XMAT).reshape(-1, 3, 3)[b].T @ (xi[b] - o.get(fo.XPOS).reshape(-1, 3)[b])
    f = np.array([0.3, -0.7, 0.2])
    jt = apply_ft(m, o, b, xi[b], f, np.zeros(3))
    chain, d = [], int(m.body_lastdof[b])
    while d >= 0:
        chain.append(d); d = int(m.dof_parentid[d])
    h, checked = 1e-6, 0
    for k in chain:                                         # the hinges above the tarsus and the root's translations (finite
        j = int(m.dof_jntid[k])                             # differences of its quaternion rotations are not along single dofs)
        i = k - int(m.jnt_dofadr[j])
        if m.jnt_type[j] == 0 and i >= 3:
            continue
        q2 = q.copy(); q2[int(m.jnt_qposadr[j]) + i] += h
        o.reset(q2)
        p2 = o.get(fo.XPOS).reshape(-1, 3)[b] + o.get(fo.XMAT).reshape(-1, 3, 3)[b] @ local
        o.reset(q)
        p1 = o.get(fo.XPOS).reshape(-1, 3)[b] + o.get(fo.XMAT).reshape(-1, 3, 3)[b] @ local
        assert abs(f @ (p2 - p1) / h - jt[k]) < 1e-4 * np.abs(jt).max(), (k, f @ (p2 - p1) / h, jt[k])
        checked += 1
    assert checked >= 6, checked


def test_body_wrench_equals_qfrc_of_its_jacobian_transpose(emu):
    """xfrc_applied on a leg body == qfrc_applied = J^T wrench, J^T computed in fp64 (mj_applyFT restated on the oracle's kinematics)"""
    m = load_model('walk')
    b = m.body_id('walker/tarsus_T2_left')
    wrench = np.array([3.0, -2.0, 5.0, 0.02, 0.01, -0.03])
    xfrc = np.zeros((m.nbody, 6)); xfrc[b] = wrench
    o = fo.Oracle(m, tolerance=1e-12)
    q, v = random_state(m, 3, 0.1, 1.0)
    o.reset(q, v)
    qfrc = apply_ft(m, o, b, frames(m, o)[2][b], wrench[:3], wrench[3:])
    assert np.count_nonzero(qfrc) > 6                       # the root dofs and the leg chain above the tarsus
    sim_x, sim_q = st.BatchedStepper(m, 1, lib_path=emu), st.BatchedStepper(m, 1, lib_path=emu)
    e_sx, _, ref_x = applied_parity(m, sim_x, 3, xfrc=xfrc)
    e_sq, _, ref_q = applied_parity(m, sim_q, 3, qfrc=qfrc)
    assert e_sx < STAGE_TOL['smooth'] and e_sq < STAGE_TOL['smooth'], (e_sx, e_sq)
    assert rel_err(ref_x, ref_q) < 1e-12
    assert rel_err(sim_q.get(st.QFRC_SMOOTH)[0], sim_x.get(st.QFRC_SMOOTH)[0]) < STAGE_TOL['smooth']


def test_thorax_force_cancels_gravity_of_a_free_floating_fly(emu):
    """a fly held 1 cm above the floor at rest (no contacts): the acceleration of its CoM is g; with a thorax force of -M_total g it is 0.
    The CoM acceleration is (M qacc) over the root's translational dofs / M_total (internal forces cancel in those rows)."""
    m = load_model('walk')
    root = m.jnt_id('walker/')
    rq, rv, body = int(m.jnt_qposadr[root]), int(m.jnt_dofadr[root]), int(m.jnt_bodyid[root])
    mass, g = float(m.body_subtreemass[body]), np.asarray(m.opt_gravity, np.float64)
    q = m.qpos0.copy(); q[rq + 2] += 1.0
    sim = st.BatchedStepper(m, 2, lib_path=emu)
    sim.reset(q)
    xfrc = np.zeros((2, m.nbody, 6)); xfrc[1, body, :3] = -mass * g
    sim.set_applied(xfrc=xfrc)
    sim.forward()
    con = sim.get(st.CONTACT).reshape(2, st.MAXCON, 16)
    for e in range(2):                                      # self-contacts are internal forces; none touches the world body
        g12 = con[e, :int(sim.get(st.NCON)[e, 0]), 7:9].astype(np.int64)
        assert not (m.geom_bodyid[g12] == 0).any(), g12
    M = sim.get(st.QM_DENSE).reshape(2, m.nv, m.nv).astype(np.float64)
    a_com = np.einsum('eij,ej->ei', M[:, rv:rv + 3], sim.get(st.QACC).astype(np.float64)) / mass
    assert np.abs(a_com[0] - g).max() < 1e-4 * np.abs(g).max(), a_com[0]
    assert np.abs(a_com[1]).max() < 1e-4 * np.abs(g).max(), a_com[1]


def test_applied_forces_persist_reset_zeroes_only_reset_envs_and_clear_restores_the_null_path(emu):
    m = load_model('walk')
    n = 3
    q, v = random_state(m, 5, 0.05, 0.5)
    qfrc, xfrc = random_applied(m, 5)
    sim = st.BatchedStepper(m, n, lib_path=emu)
    sim.reset(q, v)
    a_q, a_x = sim.applied()
    assert not a_q.any() and not a_x.any()                  # unset reads as zero
    sim.set_applied(qfrc, xfrc)
    sim.set_control(np.zeros(m.nu))
    sim.step(3); sim.step(2)                                # persist across substeps and control steps
    a_q, a_x = sim.applied()
    assert np.array_equal(a_q, np.tile(qfrc.astype(np.float32), (n, 1))) and np.array_equal(a_x, np.tile(xfrc.astype(np.float32), (n, 1, 1)))
    sim.reset(q, v, env_ids=[1])                            # mj_resetData of env 1 only
    a_q, a_x = sim.applied()
    assert not a_q[1].any() and not a_x[1].any() and np.array_equal(a_q[[0, 2]], np.tile(qfrc.astype(np.float32), (2, 1)))
    sim.reset_hold([2], q)
    a_q, a_x = sim.applied()
    assert not a_q[2].any() and not a_x[2].any() and a_q[0].any() and a_x[0].any()
    sim.set_applied(qfrc=np.ones(m.nv), env_ids=[1])        # the listed envs only
    a_q, _ = sim.applied()
    assert np.all(a_q[1] == 1) and np.array_equal(a_q[0], qfrc.astype(np.float32)) and not a_q[2].any()
    sim.write_state(st.XFRC_APPLIED, [6 * 2 + 2, 6 * 2 + 5], np.array([[1.0, 2.0], [3.0, 4.0], [5.0, 6.0]]))   # fb_write_state columns
    _, a_x = sim.applied()
    assert a_x[2, 2, 2] == 5 and a_x[2, 2, 5] == 6 and a_x[1, 2, 2] == 3
    # clear: the step is the one of a handle that never had applied forces, bit for bit
    sim.clear_applied()
    a_q, a_x = sim.applied()
    assert not a_q.any() and not a_x.any()
    ref = st.BatchedStepper(m, n, lib_path=emu)
    ctrl = np.random.RandomState(2).uniform(-0.5, 0.5, (n, m.nu))
    for s in (sim, ref):
        s.reset(q, v); s.set_control(ctrl); s.step(4)
    assert np.array_equal(sim.get(st.QPOS), ref.get(st.QPOS)) and np.array_equal(sim.get(st.QVEL), ref.get(st.QVEL))
    with pytest.raises(st.StepperError):
        sim._check(sim._lib.fb_get(sim._h, st.QFRC_APPLIED, np.zeros(2, np.int64).ctypes.data, 1), 'fb_get')      # compact: fb_applied_ptrs


def test_zero_applied_forces_step_like_none(emu):
    """allocated but zero applied forces: the same trajectory as the null path (x + 0 = x)"""
    m = load_model('walk')
    q, v = random_state(m, 7, 0.05, 0.5)
    a, b = st.BatchedStepper(m, 2, lib_path=emu), st.BatchedStepper(m, 2, lib_path=emu)
    ctrl = np.random.RandomState(3).uniform(-0.5, 0.5, (2, m.nu))
    for s in (a, b):
        s.reset(q, v); s.set_control(ctrl)
    a.applied_ptrs()                                        # allocates, zeroed
    a.step(3); b.step(3)
    assert np.array_equal(a.get(st.QVEL), b.get(st.QVEL))


# ------------------------------------------------------------------------------------------------------------------------ GPU tier
@pytest.mark.gpu
def test_applied_forces_match_oracle_on_gpu():
    m = load_model('walk')
    for seed in (0, 1):
        qfrc, xfrc = random_applied(m, seed, bodies=8)
        for kw in (dict(qfrc=qfrc), dict(xfrc=xfrc), dict(qfrc=qfrc, xfrc=xfrc)):
            e_s, _, _ = applied_parity(m, st.BatchedStepper(m, 64), seed, env=17, **kw)
            e_sf, e_a, _ = applied_parity(m, st.BatchedStepper(m, 64), seed, env=17, free=True, **kw)
            print('applied-force parity', seed, sorted(kw), e_s, e_sf, e_a)
            assert e_s < STAGE_TOL['smooth'] and e_sf < STAGE_TOL['smooth'] and e_a < STAGE_TOL['smooth'], (seed, sorted(kw), e_s, e_sf, e_a)


@pytest.mark.gpu
def test_applied_forces_written_in_place_on_gpu():
    """fb_applied_ptrs: a policy on the GPU writes the rows in place; the step sees what fb_set would have given it, graph replay included"""
    import torch
    m = load_model('walk')
    n = 256
    q, v = random_state(m, 2, 0.05, 0.5)
    qfrc, xfrc = random_applied(m, 2)
    a, b = st.BatchedStepper(m, n), st.BatchedStepper(m, n)
    ctrl = np.random.RandomState(4).uniform(-0.5, 0.5, (n, m.nu))
    for s in (a, b):
        s.reset(q, v); s.set_control(ctrl)
    b.set_applied(qfrc, xfrc)
    qp, xp = a.applied_ptrs()

    class _V:
        def __init__(self, p, shape):
            self.__cuda_array_interface__ = {'shape': shape, 'typestr': '<f4', 'data': (int(p), False), 'version': 2}
    tq = torch.as_tensor(_V(qp, (n, m.nv)), device='cuda')
    tx = torch.as_tensor(_V(xp, (n, m.nbody, 6)), device='cuda')
    tq.copy_(torch.from_numpy(np.tile(qfrc, (n, 1)).astype(np.float32)))
    tx.copy_(torch.from_numpy(np.tile(xfrc, (n, 1, 1)).astype(np.float32)))
    torch.cuda.synchronize()
    for _ in range(3):                                      # plain launches, capture, replay
        a.step(10); b.step(10)
    assert np.array_equal(a.get(st.QPOS), b.get(st.QPOS)) and np.array_equal(a.get(st.QVEL), b.get(st.QVEL))
    a.clear_applied()
    a.reset(q, v); b.clear_applied(); b.reset(q, v)
    for s in (a, b):
        s.set_control(ctrl); s.step(10)
    assert np.array_equal(a.get(st.QPOS), b.get(st.QPOS))
