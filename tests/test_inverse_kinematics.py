"""Multi-site inverse kinematics (fb_ik_*, flybody_b200.inverse_kinematics) against the fp64 restatement of the reference's loop
(tests/ik_reference.c; targets come from the oracle's fp64 forward pass), and walking datasets written from the fits.  CPU tier: the host-emulation build of the kernel source; GPU tier
(-m gpu): the same comparisons through the CUDA library, at 4096 problems.  "Bit-identical" compares uint32 views."""
import numpy as np
import pytest

import __graft_entry__ as ge
from flybody_b200 import fly_envs, inverse_kinematics as ik, stepper as st
from flybody_b200.flymodel import load_model
from flybody_b200.synthetic import mult_quat, reciprocal_quat, rotate_vec_with_quat
from flybody_b200.trajectory_loaders import HDF5WalkingTrajectoryLoader
from oracle import fly_oracle as fo

import ik_reference as ikref

SITES = ['walker/claw_T1_left', 'walker/claw_T1_right', 'walker/claw_T2_left', 'walker/claw_T2_right', 'walker/claw_T3_left',
         'walker/claw_T3_right', 'walker/head', 'walker/thorax']
LEGS = ('T1_left', 'T3_right')


@pytest.fixture(scope='module')
def emu():
    ge.build()
    return ge.EMU


@pytest.fixture(scope='module')
def model():
    return load_model('template')


def hinges(m, legs=LEGS):
    return [j for j in m.meta['observable_joints'] if any(l in j for l in legs) and 'tarsus' not in j]


def ids(m, sites, joints):
    return [m.site_id(s) for s in sites], [m.jnt_id(j) for j in joints]


def rot(q, axis, ang):
    axis = np.asarray(axis, np.float64) / np.linalg.norm(axis)
    return mult_quat(q, np.r_[np.cos(ang / 2), np.sin(ang / 2) * axis])


def problem(m, seed, joints, amp=0.15):
    """a true pose (fitted hinges and the root moved from qpos0) and its sites as fp64 targets"""
    rs = np.random.RandomState(seed)
    q = m.qpos0.copy()
    for j in joints:
        if int(m.jnt_type[m.jnt_id(j)]) == 3:
            q[m.jnt_qposadr_of(j)] += rs.uniform(-amp, amp)
    q[0:3] += rs.uniform(-0.05, 0.05, 3)
    q[3:7] = rot(q[3:7], rs.normal(size=3), rs.uniform(0, 0.3))
    o = fo.Oracle(m)
    o.reset(q)
    o.forward()
    return q, o.get(fo.SITE_XPOS).reshape(-1, 3)[[m.site_id(s) for s in SITES]]


def reference_ik(m, q0, joints, target, **kw):
    sid, jid = ids(m, SITES, joints)
    return ikref.solve(m, q0, sid, jid, target, **kw)


def device_ik(m, lib, q0, joints, targets, n_envs=None, env_of=None, **kw):
    """problems through BatchedStepper.ik_*; env_of places problem k in env env_of[k] of a batch of n_envs (others: copies of problem 0)"""
    targets = np.asarray(targets, np.float64).reshape(-1, len(SITES), 3)
    q0 = np.broadcast_to(np.asarray(q0, np.float64).reshape(-1, m.nq), (len(targets), m.nq))
    n = n_envs or len(targets)
    env_of = np.arange(len(targets)) if env_of is None else np.asarray(env_of)
    t_all, q_all = np.repeat(targets[:1], n, 0), np.repeat(q0[:1], n, 0)
    t_all[env_of], q_all[env_of] = targets, q0
    sim = st.BatchedStepper(m, n, lib_path=lib)
    sid, jid = ids(m, SITES, joints)
    inc = kw.pop('include', None)
    sim.ik_program(sid, jid, inc, **kw)
    sim.ik_solve(t_all, q_all)
    out = sim.ik_read()
    sim.close()
    return [a[env_of] for a in out]


def bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint32) if a.dtype == np.float32 else a


# ---- 1. the fp64 reference's gradient is the derivative of its own objective --------------------------------------------------------------
def test_reference_gradient_matches_finite_differences(model):
    m = model
    joints = ['walker/'] + hinges(m)
    _, target = problem(m, 0, joints)
    q, _ = problem(m, 1, joints)
    inc = np.ones(3 * len(SITES), np.uint8)
    inc[[1, 5, 9, 22]] = 0                                     # partial mask: y of site 0, z of site 1, y of site 3, y of site 7
    sid, jid = ids(m, SITES, joints)
    f0, g = ikref.objective(m, q, sid, jid, target, inc, reg_strength=1e-3)
    assert len(g) == 6 + len(joints) - 1 and f0 > 0
    h, fd = 1e-6, []
    for i in range(len(g)):
        vals = []
        for sgn in (1, -1):
            qq = q.copy()
            if i < 3:
                qq[i] += sgn * h
            elif i < 6:
                qq[3:7] = rot(qq[3:7], np.eye(3)[i - 3], sgn * h)     # body-frame rotation: mj_integratePos of the free joint's angular dofs
            else:
                qq[m.jnt_qposadr_of(joints[i - 5])] += sgn * h
            vals.append(ikref.objective(m, qq, sid, jid, target, inc, reg_strength=1e-3)[0])
        fd.append((vals[0] - vals[1]) / (2 * h))
    # central differences in fp64 at h = 1e-6: truncation ~h^2 |f'''|, cancellation ~1e-16 f / h; both far below 1e-7 of |g|
    assert np.abs(np.asarray(fd) - g).max() <= 1e-7 * np.abs(g).max(), (np.asarray(fd), g)


# ---- 2. known answers --------------------------------------------------------------------------------------------------------------
def rigid_target(m):
    q = m.qpos0.copy()
    q[0:3] += [0.05, -0.03, 0.02]
    q[3:7] = rot(q[3:7], [0.3, 0.5, 0.8], 0.2)
    o = fo.Oracle(m)
    o.reset(q)
    o.forward()
    return q, o.get(fo.SITE_XPOS).reshape(-1, 3)[[m.site_id(s) for s in SITES]]


def test_known_answers_free_joint_and_single_hinge(model, emu):
    m = model
    q, target = rigid_target(m)
    r = reference_ik(m, m.qpos0, ['walker/'], target, max_steps=20_000)
    assert np.abs(r['qpos'][:7] - q[:7]).max() < 1e-12
    res = ik.qpos_from_site_xpos(m, SITES, target, ['walker/'], lib_path=emu)
    # fp32: site positions carry ~1e-8 cm of round-off, the root pose follows them to a few 1e-8
    assert np.abs(res.qpos[:7] - q[:7]).max() < 1e-6 and res.err_norm_first_term < 1e-12
    assert np.array_equal(res.qpos[7:], m.qpos0[7:].astype(np.float32))
    # one hinge: its angle alone moves the T1 claw
    j = 'walker/femur_T1_left'
    q = m.qpos0.copy()
    q[m.jnt_qposadr_of(j)] += 0.3
    o = fo.Oracle(m)
    o.reset(q)
    o.forward()
    target = o.get(fo.SITE_XPOS).reshape(-1, 3)[[m.site_id(s) for s in SITES]]
    r = reference_ik(m, m.qpos0, [j], target, max_steps=20_000)
    assert abs(r['qpos'][m.jnt_qposadr_of(j)] - q[m.jnt_qposadr_of(j)]) < 1e-9
    res = ik.qpos_from_site_xpos(m, SITES, target, [j], lib_path=emu)
    assert abs(res.qpos[m.jnt_qposadr_of(j)] - q[m.jnt_qposadr_of(j)]) < 1e-4


# ---- 3. the kernel source against the oracle -----------------------------------------------------------------------------------------
def fitted_qadr(m, joints):
    return np.concatenate([np.arange(7) if j == 'walker/' else [m.jnt_qposadr_of(j)] for j in joints])


# Gate of the iteration-by-iteration comparison.  The kernel's site positions carry fp32 round-off of the kinematics chain (~6e-8 relative
# to the ~0.3 cm body scale); the gradient 2 diff^T J inherits it, and the momentum sum carries it from one iteration to the next.
# Measured under emulation (problem seed 2, reg 1e-3): 2.9e-8 after 1 iteration, 1.5e-8 after 10, 7.1e-8 after 100, on qpos entries of
# order 1 (fp32 ulp 6e-8 to 1.2e-7).  Gate: 4x the measured value, at least one ulp of 1.0 (1.2e-7).
ITER_GATE = {1: 1.2e-7, 10: 1.2e-7, 100: 3e-7}


def test_kernel_source_follows_oracle_iteration_by_iteration(model, emu):
    m = model
    joints = ['walker/'] + hinges(m)
    qa = fitted_qadr(m, joints)
    _, target = problem(m, 2, joints)
    for k, gate in ITER_GATE.items():
        kw = dict(reg_strength=1e-3, progress_threshold=0.0, max_steps=k)
        r = reference_ik(m, m.qpos0, joints, target, **kw)
        q, err, err1, steps, ok = device_ik(m, emu, m.qpos0, joints, target[None], **kw)
        assert steps[0] == r['steps'] == k - 1 and not ok[0] and not r['success']
        dq = np.abs(q[0][qa] - r['qpos'][qa]).max()
        assert dq <= gate, (k, dq)
        assert np.array_equal(q[0][np.setdiff1d(np.arange(m.nq), qa)], m.qpos0[np.setdiff1d(np.arange(m.nq), qa)].astype(np.float32))


# Full solves: thousands of momentum steps amplify the fp32 differences, so qpos is compared only where reg > 0 makes the minimum
# unique.  Measured under emulation over the 8 problems, converged (3000 steps) and stopped at max_steps (150): qpos 1.0e-6 at most,
# err_norm_first_term 2.7e-5 relative at most (a site term of ~1e-6 cm^2 is a difference of squares of fp32 positions).  Gates: 5e-6 on
# qpos, 1e-4 relative (+1e-12 absolute) on the site term.  steps may differ by one check interval when the stopping ratio lands near the
# threshold at a check (seen once: 2500 against 2400).
def full_solve_problems(m, n):
    joints = ['walker/'] + hinges(m)
    out = []
    for s in range(n):
        _, t = problem(m, 100 + s, joints, amp=0.1)
        out.append(t)
    return joints, np.stack(out)


def check_full_solves(m, lib, n_check, n_batch):
    joints, targets = full_solve_problems(m, n_check)
    kws = [dict(reg_strength=1e-3, max_steps=3000), dict(reg_strength=1e-3, max_steps=150)]     # the second one stops at max_steps
    for kw in kws:
        if n_batch > n_check:
            reps = np.tile(targets, (-(-n_batch // n_check), 1, 1))[:n_batch]     # problem k sits in envs k, k + n_check, ...
            q, err, err1, steps, ok = [a[:n_check] for a in device_ik(m, lib, m.qpos0, joints, reps, **kw)]
        else:
            q, err, err1, steps, ok = device_ik(m, lib, m.qpos0, joints, targets, **kw)
        qa = fitted_qadr(m, joints)
        for k in range(n_check):
            r = reference_ik(m, m.qpos0, joints, targets[k], **kw)
            assert bool(ok[k]) == r['success'], (kw, k)
            assert abs(int(steps[k]) - r['steps']) <= 100, (kw, k, steps[k], r['steps'])
            assert abs(err1[k] - r['err_norm_first_term']) <= 1e-4 * r['err_norm_first_term'] + 1e-12, (kw, k, err1[k], r['err_norm_first_term'])
            if r['success']:
                assert np.abs(q[k][qa] - r['qpos'][qa]).max() < 5e-6, (kw, k)
    return kws


def test_full_solves_match_oracle(model, emu):
    check_full_solves(model, emu, 8, 8)


# ---- 4. masks ------------------------------------------------------------------------------------------------------------------------
def test_include_mask_and_nan_targets_drop_components(model, emu):
    m = model
    joints = ['walker/'] + hinges(m)
    _, target = problem(m, 3, joints)
    drop = [2, 4, 10, 18, 19]
    inc = np.ones(3 * len(SITES), np.uint8)
    inc[drop] = 0
    tnan = target.copy().reshape(-1)
    tnan[drop] = np.nan
    kw = dict(reg_strength=1e-3, max_steps=400, progress_threshold=0.0)
    a = device_ik(m, emu, m.qpos0, joints, target[None], include=inc, **kw)
    b = device_ik(m, emu, m.qpos0, joints, tnan.reshape(1, -1, 3), **kw)
    for x, y in zip(a, b):
        assert np.array_equal(bits(x), bits(y))
    r = reference_ik(m, m.qpos0, joints, target, include=inc, **kw)
    qa = fitted_qadr(m, joints)
    assert np.abs(a[0][0][qa] - r['qpos'][qa]).max() < 5e-6                 # the full-solve gates
    assert abs(a[2][0] - r['err_norm_first_term']) <= 1e-4 * r['err_norm_first_term'] + 1e-12
    # the reference's list form of include_inds through the public interface
    res = ik.qpos_from_site_xpos(m, SITES, target, joints, include_inds=[i for i in range(3 * len(SITES)) if inc[i]], lib_path=emu, **kw)
    assert np.array_equal(res.qpos.astype(np.float32), a[0][0])


# ---- 5. determinism ------------------------------------------------------------------------------------------------------------------
def test_result_bits_do_not_depend_on_env_slot_or_batch(model, emu):
    m = model
    joints = ['walker/'] + hinges(m)
    _, t = problem(m, 4, joints)
    _, other = problem(m, 5, joints)
    kw = dict(reg_strength=1e-3, max_steps=700)
    batch = np.repeat(other[None], 7, 0)
    batch[0] = batch[5] = t
    a = device_ik(m, emu, m.qpos0, joints, batch, **kw)
    b = device_ik(m, emu, m.qpos0, joints, t[None], **kw)
    for x, y in zip(a, b):
        assert np.array_equal(bits(x[0]), bits(x[5])) and np.array_equal(bits(x[0]), bits(y[0]))


# ---- 6. refusals ---------------------------------------------------------------------------------------------------------------------
def test_bad_programs_and_solves_are_refused(model, emu):
    m = model
    sim = st.BatchedStepper(m, 3, lib_path=emu)
    sid, jid = ids(m, SITES, ['walker/'])
    t = np.zeros((3, len(SITES), 3), np.float32)
    with pytest.raises(st.StepperError, match='no IK program'):
        sim._ik_nsite = len(SITES); sim.ik_solve(t)
    with pytest.raises(st.StepperError, match='no IK solve'):
        sim._ik_n = 1; sim.ik_read()
    for s, j, msg in (([m.nsite], jid, 'site id'), ([-1], jid, 'site id'), (sid, [m.njnt], 'joint id'), (sid, [0, 0], 'twice'),
                      (list(range(m.nsite)) * 5, jid, '64 sites')):
        with pytest.raises(st.StepperError, match=msg):
            sim.ik_program(s, j)
    with pytest.raises(st.StepperError, match='max_steps'):
        sim.ik_program(sid, jid, max_steps=0)
    sim.ik_program(sid, jid)
    with pytest.raises(st.StepperError, match='n_envs'):
        sim.ik_solve(np.zeros((4, len(SITES), 3)))
    with pytest.raises(st.StepperError, match='init_qpos'):
        q = np.tile(m.qpos0, (3, 1)); q[1, 9] = np.inf; sim.ik_solve(t, q)
    with pytest.raises(st.StepperError, match='infinite target'):
        tt = t.copy(); tt[2, 1, 0] = -np.inf; sim.ik_solve(tt)
    sim.ik_solve(t, m.qpos0)                                   # the handle still works
    sim.close()
    ball = load_model('ball')
    bj = [j for j in range(ball.njnt) if int(ball.jnt_type[j]) == 1]
    sim = st.BatchedStepper(ball, 1, lib_path=emu)
    with pytest.raises(st.StepperError, match='ball joints'):
        sim.ik_program([0], bj)
    sim.close()


# ---- 7. stepping is unchanged by a solve ------------------------------------------------------------------------------------------
def check_stepping_unchanged(m, lib, n):
    joints = ['walker/'] + hinges(m)
    _, t = problem(m, 6, joints)
    a, b = st.BatchedStepper(m, n, lib_path=lib), st.BatchedStepper(m, n, lib_path=lib)
    sig = a.state_signature()
    sid, jid = ids(m, SITES, joints)
    a.ik_program(sid, jid, reg_strength=1e-3, max_steps=300)
    assert a.state_signature() == sig == b.state_signature()
    a.ik_solve(np.repeat(t[None], n, 0))
    ctrl = np.random.RandomState(0).uniform(-0.3, 0.3, (n, m.nu))
    for s in (a, b):
        s.reset(m.qpos0)
        s.set_control(ctrl)
        s.step(3)
    for f in (st.QPOS, st.QVEL, st.ACT, st.QACC, st.SENSORDATA, st.XPOS, st.SITE_XPOS, st.NCON):
        assert np.array_equal(bits(a.get(f)), bits(b.get(f))), f
    a.close(); b.close()


def test_stepping_unchanged_by_ik(model, emu):
    check_stepping_unchanged(model, emu, 5)


# ---- 8. a walking dataset from fitted tracks ------------------------------------------------------------------------------------------
def test_dataset_round_trip(model, emu, tmp_path):
    m, T = model, 12
    sim = st.BatchedStepper(m, 1, lib_path=emu)
    sim.reset(m.qpos0)
    rs = np.random.RandomState(0)
    qs, xs = [], []
    for t in range(T):
        qs.append(sim.get(st.QPOS)[0].astype(np.float64)); xs.append(sim.get(st.SITE_XPOS)[0].reshape(-1, 3)[[m.site_id(s) for s in SITES]])
        sim.set_control(rs.uniform(-0.3, 0.3, m.nu))
        sim.step(2)
    sim.close()
    qs, xs = np.stack(qs), np.stack(xs).astype(np.float64)
    joints = hinges(m, ('T1_left', 'T1_right', 'T2_left', 'T2_right', 'T3_left', 'T3_right'))
    fit = ['walker/'] + joints
    init = qs.copy()
    init[:, [m.jnt_qposadr_of(j) for j in joints]] += 0.05              # fitted joints start off; the others stay at their recorded values
    res = ik.qpos_from_site_xpos(m, SITES, xs, fit, reg_strength=0.0, max_steps=4000, init_qpos=init, lib_path=emu)
    assert res.qpos.shape == (T, m.nq) and res.steps.shape == (T,)
    path = str(tmp_path / 'fitted.npz')
    ik.write_walking_dataset(path, m, res.qpos, 0.002, joints, SITES[:7], lib_path=emu)
    ld = HDF5WalkingTrajectoryLoader(path)
    tr = ld.full_trajectory(0)
    rq = qs[:, :7]
    rec = rotate_vec_with_quat(xs[:, :7] - rq[:, None, :3], reciprocal_quat(rq[:, None, 3:7]))
    # the fit's residual (err_norm_first_term up to ~1e-6 cm^2 over 8 sites) bounds the site error: 1e-3 cm covers it with margin
    assert np.abs(tr['root2site'] - rec).max() < 1e-3, np.abs(tr['root2site'] - rec).max()
    assert np.allclose(np.linalg.norm(tr['joint_quat'], axis=-1), 1.0, atol=1e-6)
    assert tr['qpos'].shape == (T, len(joints)) and tr['root_qvel'].shape == (T, 6)
    assert np.allclose(tr['root_qvel'][:-1, :3], np.diff(res.qpos[:, :3], axis=0) / 0.002)
    env = fly_envs.walk_imitation(ref_path=path, n_envs=1, lib_path=emu, terminal_com_dist=float('inf'))
    env.reset()
    env.close()


# ---- GPU tier ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_gpu_iterations_and_full_solves_match_oracle(model):
    ge.build()
    m = model
    joints = ['walker/'] + hinges(m)
    qa = fitted_qadr(m, joints)
    _, target = problem(m, 2, joints)
    for k, gate in ITER_GATE.items():
        kw = dict(reg_strength=1e-3, progress_threshold=0.0, max_steps=k)
        r = reference_ik(m, m.qpos0, joints, target, **kw)
        q = device_ik(m, None, m.qpos0, joints, target[None], **kw)[0]
        assert np.abs(q[0][qa] - r['qpos'][qa]).max() <= gate, k
    check_full_solves(m, None, 8, 4096)


@pytest.mark.gpu
def test_gpu_masks_determinism_and_stepping(model):
    ge.build()
    m = model
    joints = ['walker/'] + hinges(m)
    _, t = problem(m, 3, joints)
    drop = [2, 4, 10, 18, 19]
    inc = np.ones(3 * len(SITES), np.uint8)
    inc[drop] = 0
    tnan = t.copy().reshape(-1)
    tnan[drop] = np.nan
    kw = dict(reg_strength=1e-3, max_steps=400, progress_threshold=0.0)
    a = device_ik(m, None, m.qpos0, joints, t[None], **kw, include=inc)
    b = device_ik(m, None, m.qpos0, joints, tnan.reshape(1, -1, 3), **kw)
    for x, y in zip(a, b):
        assert np.array_equal(bits(x), bits(y))
    # the same problem in several slots of a 4096-problem batch, and alone
    _, other = problem(m, 5, joints)
    batch = np.repeat(other[None], 4096, 0)
    slots = [0, 5, 1000, 4095]
    batch[slots] = t
    kw = dict(reg_strength=1e-3, max_steps=700)
    big = device_ik(m, None, m.qpos0, joints, batch, **kw)
    one = device_ik(m, None, m.qpos0, joints, t[None], **kw)
    for x, y in zip(big, one):
        for s in slots:
            assert np.array_equal(bits(x[s]), bits(y[0]))
    check_stepping_unchanged(m, None, 64)
