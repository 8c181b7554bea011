"""walk_imitation with a trajectory dataset and the task hooks on the device (device_task=True): the dataset as a device bank with the
full-body reward features (fb_ref_bank_wide), per-env trajectory draws at every reset (pinned by the host through step(), drawn from the
counter hash by step_device), the full-body start pose and the DeepMimic reward in CUDA.  Held step by step against the host-side task
code ON THE SAME STEPPER, as tests/test_device_dataset_flight.py does for flight.  Host-emulation build unless marked gpu."""
import numpy as np
import pytest

import __graft_entry__ as ge
from flybody_b200 import fly_envs, rewards as rw, stepper as st
from flybody_b200.dm_env_shim import StepType
from flybody_b200.synthetic import rotate_vec_with_quat, reciprocal_quat, mult_quat
from flybody_b200.trajectory_loaders import HDF5WalkingTrajectoryLoader

FUT = 64
LENS = [80, 95, 110, 140, 72]                             # rows per trajectory: 110 and 140 exceed the slot cap of CAP rows
CAP = 100
PICK = [0, 1, 3, 1, 4]                                    # a subset with a repeat
WING = 'walker/wing_yaw_left'                             # a wing joint in the dataset's joint list: the reset puts it back at its spring
REW_RTOL, REW_ATOL = 2e-4, 1e-6                           # device fp32 reward against the host's fp64 evaluation of the same record


@pytest.fixture(scope='module')
def emu():
    ge.build()
    return ge.EMU


def record_dataset(lib, path, lens=LENS, seed=0):
    """Roll an inference-mode walk batch with random actions and store what a mocap dataset holds, trajectory k = the first lens[k]
    rows of env k (the recorder of tests/test_env_dataset.py); joint_quat is filled by a second pass through the env's own feature
    code.  The wing joint's stored angle is moved off its spring, so that a reset which left it at the dataset's value shows."""
    n, T = len(lens), max(lens)
    env = fly_envs.walk_imitation(terminal_com_dist=float('inf'), n_envs=n, lib_path=lib, reset_noise=0.03, seed=3)
    m, sim = env.model, env._sim
    jn, sn = m.meta['jnt_names'], m.meta['site_names']
    joints = [j for j in m.meta['observable_joints'] if any(k in j for k in ('coxa', 'femur', 'tibia', 'tarsus'))] + [WING]
    sites = [f'walker/claw_T{k}_{s}' for k in (1, 2, 3) for s in ('left', 'right')] + ['walker/head']
    jid = [jn.index(j) for j in joints]
    qadr, vadr, sid = m.jnt_qposadr[jid], m.jnt_dofadr[jid], [sn.index(s) for s in sites]
    actions = np.random.RandomState(seed).uniform(-0.25, 0.25, (T, n, 59)).astype(np.float32)
    env.reset()
    rec = {k: [] for k in ('root_qpos', 'qpos', 'root_qvel', 'qvel', 'root2site')}

    def grab():
        q, v = sim.get(st.QPOS).astype(np.float64), sim.get(st.QVEL).astype(np.float64)
        sx = sim.get(st.SITE_XPOS).astype(np.float64).reshape(n, -1, 3)[:, sid]
        rq = q[:, env._root_q:env._root_q + 7]
        rec['root_qpos'].append(rq); rec['qpos'].append(q[:, qadr])
        rec['root_qvel'].append(v[:, env._root_v:env._root_v + 6]); rec['qvel'].append(v[:, vadr])
        rec['root2site'].append(rotate_vec_with_quat(sx - rq[:, None, :3], reciprocal_quat(rq[:, None, 3:7])))
    grab()
    for t in range(T - 1):
        ts = env.step(actions[t])
        assert np.all(np.asarray(ts.step_type) == int(StepType.MID)), t          # one unbroken episode per env
        grab()
    env.close()
    d = {'timestep_seconds': np.float64(0.002), 'trajectory_lengths': np.asarray(lens, np.int64),
         'id2name/joints': np.array([j.split('/')[-1] for j in joints]), 'id2name/sites': np.array([s.split('/')[-1] for s in sites])}
    for k, L in enumerate(lens):
        g = f'trajectories/{k}/'
        for key in rec:
            d[g + key] = np.stack([r[k] for r in rec[key]])[:L]
        d[g + 'qpos'][:, -1] += 0.25
        d[g + 'joint_quat'] = np.tile([1.0, 0, 0, 0], (L, len(joints), 1))
    np.savez(path, **d)
    # second pass: each env replays its trajectory's actions on the host-side task code; the joint orientations it sees are the rows
    # the reward compares (rows past the episode's end are never read)
    env = fly_envs.walk_imitation(ref_path=path, terminal_com_dist=float('inf'), n_envs=n, lib_path=lib)
    for e in range(n):
        env.task.set_next_trajectory_index(e)
        env._reset_envs(np.array([e]))
    env._needs_reset[:] = False
    nj = len(env._mocap_qadr)
    jq = np.zeros((T, n, nj, 4))

    def features():
        env._sim.task_inputs(env._step_counter, np.zeros(n, np.uint8))
        r = env._sim.read_task_obs(env._rec)
        s = env._obs_slices
        return rw.joint_orientation_quat(r[:, s['_mocap_axes']].astype(np.float64).reshape(n, nj, 3), r[:, s['_mocap_qpos']].astype(np.float64))
    jq[0] = features()
    for t in range(T - FUT - 1):
        env.step(actions[t])
        jq[t + 1] = features()
    env.close()
    for k, L in enumerate(lens):
        q = jq[:L - FUT, k]
        d[f'trajectories/{k}/joint_quat'] = np.concatenate([q, np.repeat(q[-1:], FUT, 0)])
    np.savez(path, **d)
    return actions, d


@pytest.fixture(scope='module')
def dataset(emu, tmp_path_factory):
    path = str(tmp_path_factory.mktemp('walk') / 'w.npz')
    actions, d = record_dataset(emu, path)
    return path, actions, d


def check_ref_obs(env, rec, rows_of, step_now):
    """walker/ref_displacement, ref_root_quat of every env against its reference rows, from the root pose after the step"""
    q = env._sim.get(st.QPOS).astype(np.float64)[:, env._root_q:env._root_q + 7]
    obs = env._observation(rec)
    for e in range(env.n_envs):
        rows = rows_of(e)
        t = np.minimum(step_now[e] + np.arange(env._future), len(rows) - 1)
        disp = rotate_vec_with_quat(rows[t, :3] - q[e, :3], reciprocal_quat(q[e, 3:7]))
        quat = mult_quat(reciprocal_quat(q[e, 3:7])[None], rows[t, 3:7])
        assert np.allclose(obs['walker/ref_displacement'][e], disp, atol=2e-5), (e, obs['walker/ref_displacement'][e], disp)
        assert np.allclose(obs['walker/ref_root_quat'][e], quat, atol=2e-5), e


def expected_rows(d, traj, slot_len):
    """[n, 13] reference rows of an episode on `traj`, cut from the dataset in fp64 (root x, y relative to row 0)"""
    g = f'trajectories/{traj}/'
    q = np.array(d[g + 'root_qpos'], np.float64)
    q[:, :2] -= q[0, :2]
    n = min(len(q), slot_len)
    return np.concatenate([q, d[g + 'root_qvel']], 1)[:n]


def replay_picks(path, seed, resets, next_idx=None, pick=PICK):
    """the trajectory draws of a fresh loader with the same seed over a sequence of reset id lists"""
    tg = HDF5WalkingTrajectoryLoader(path, traj_indices=pick, random_state=np.random.RandomState(seed))
    out = []
    for ids, pinned in zip(resets, next_idx or [None] * len(resets)):
        for e in ids:
            out.append((e, int(pinned if pinned is not None else tg._random_state.choice(tg.traj_indices))))
    return out


def check_reset_pose(env, d, ids, traj):
    """the held envs of a reset: root on row 0 (x, y at the origin), the mocap joints at row 0, the wings at their springs"""
    q = env._sim.get(st.QPOS)
    wing = set(int(a) for a in env._wing_qadr)
    for e in ids:
        g = f'trajectories/{int(traj[e])}/'
        r0 = np.array(d[g + 'root_qpos'][0], np.float32)
        assert np.array_equal(q[e, env._root_q + 2:env._root_q + 7], r0[2:]) and np.all(q[e, env._root_q:env._root_q + 2] == 0.0), e
        j0 = np.array(d[g + 'qpos'][0], np.float32)
        for k, a in enumerate(env._mocap_qadr):
            if int(a) not in wing:
                assert q[e, a] == j0[k], (e, k)
        assert np.array_equal(q[e, env._wing_qadr], env._wing_spring.astype(np.float32)), e
        assert q[e, env._mocap_qadr[-1]] != j0[-1]                # (the dataset's wing angle is off its spring)


def drive_dataset(path, d, lib, n=5, n_steps=120, seed=7):
    """item 1: a device-task env through step(), compared with the host task code on the same stepper after every step"""
    rs = np.random.RandomState(1)
    actions = rs.uniform(-0.3, 0.3, (n_steps, n, 59)).astype(np.float32)
    actions[5, 2, 3] = np.nan                                 # NaN actions act as 0
    actions[10:, 0, :] = 1.0                                  # env 0 leaves its reference -> termination -> auto-reset
    env = fly_envs.walk_imitation(ref_path=path, traj_indices=PICK, n_envs=n, lib_path=lib, seed=4, terminal_com_dist=0.01,
                                  max_reference_steps=CAP, random_state=np.random.RandomState(seed), device_task=True)
    sim = env._sim
    ts = env.reset()
    assert np.all(np.asarray(ts.step_type) == int(StepType.FIRST)) and env._slot_len == CAP
    traj, start = env.reference_picks()
    assert np.all(start == 0)
    check_reset_pose(env, d, range(n), traj)
    resets = [list(range(n))]
    time = np.zeros(n)
    seen, terminated, rel = [np.asarray(ts.step_type, np.int64)], 0, 0.0
    for k in range(n_steps):
        resetting = env._needs_reset.copy()
        if resetting.any():
            resets.append(list(np.nonzero(resetting)[0]))
        ts = env.step(actions[k])
        step = np.where(resetting, 0, np.minimum(np.round(time / env._control_timestep).astype(np.int64), env._ref_len - 1))
        ghost = env._ref_at(step).astype(np.float32); ghost[resetting, 7:] = 0
        traj, start = env.reference_picks()
        assert np.array_equal(np.stack([traj, start], 1), env._ref_pick) and np.all(start == 0), k
        for e in np.nonzero(resetting)[0]:                    # the host mirror holds the snippet of the pick to fp32 rounding
            want = expected_rows(d, int(traj[e]), env._slot_len)
            assert env._ref_len[e] == len(want) and np.allclose(env._ref_rows[e, :len(want)], want, atol=2e-6), (k, e)
            assert np.all(env._ref_rows[e, len(want):] == env._ref_rows[e, len(want) - 1])
            assert env._episode_steps[e] == min(5001, min(LENS[traj[e]], CAP) - FUT - 1)
        if resetting.any():
            check_reset_pose(env, d, np.nonzero(resetting)[0], traj)
        # ghost: on its reference row (held envs) or coasting from it with the row's velocity
        q, v = sim.get(st.QPOS), sim.get(st.QVEL)
        want = ghost[:, :3] + np.where(resetting[:, None], 0.0, ghost[:, 7:10] * env._control_timestep)
        assert np.allclose(q[:, env._ghost_q:env._ghost_q + 3], want, atol=2e-5), k
        assert np.allclose(q[:, env._ghost_q + 3:env._ghost_q + 7], ghost[:, 3:7], atol=2e-2), k
        assert np.allclose(v[:, env._ghost_v:env._ghost_v + 6], ghost[:, 7:], atol=1e-2), k
        if resetting.any():
            assert np.array_equal(q[resetting, env._ghost_q:env._ghost_q + 7], ghost[resetting, :7]), k
        # termination / reward / discount of the host task code on the same observation record
        time = np.where(resetting, 0.0, time + env._control_timestep)
        obs = env._observation(env._rec)
        step_type, reward, discount, needs = env._task_after(env._rec, obs, resetting, time, ghost)
        assert np.array_equal(np.asarray(step_type, np.int64), np.asarray(ts.step_type, np.int64)), (k, step_type, ts.step_type)
        assert np.allclose(ts.reward, reward, rtol=REW_RTOL, atol=REW_ATOL), (k, reward, ts.reward)
        rel = max(rel, float(np.max(np.abs(ts.reward - reward) / np.maximum(np.abs(reward), 1e-30))))
        assert np.array_equal(discount, ts.discount), k
        assert np.array_equal(needs, env._needs_reset), k
        terminated += int(((np.asarray(ts.step_type) == int(StepType.LAST)) & (np.asarray(ts.discount) == 0.0)).sum())
        check_ref_obs(env, env._rec, lambda e: env._ref_rows[e, :env._ref_len[e]].astype(np.float64), np.round(time / env._control_timestep).astype(np.int64))
        seen.append(np.asarray(ts.step_type, np.int64))
    print(f'max relative reward difference device / host: {rel:.2e}')
    # the observed reset sequence replayed on a fresh loader with the same seed gives the same draws
    last = {e: j for e, j in replay_picks(path, seed, resets)}
    assert last == {e: int(traj[e]) for e in range(n)}
    env.close()
    seen = np.array(seen)
    assert (seen == int(StepType.LAST)).any() and (seen[1:] == int(StepType.FIRST)).any() and terminated > 0
    assert len(resets) >= 3
    return seen


def test_dataset_walk_device_task_matches_host_task_code(emu, dataset):
    path, _, d = dataset
    drive_dataset(path, d, emu)


def test_record_and_replay_keeps_maximal_reward(emu, dataset):
    """replaying the recorded actions on the device: the four DeepMimic factors at (20, 1, 1, 1) and the device's reward equal to the
    host's product of the factors; at step == episode_steps LAST with discount 1"""
    path, actions, d = dataset
    for k in (0, 4):
        env = fly_envs.walk_imitation(ref_path=path, terminal_com_dist=0.3, n_envs=2, lib_path=emu, device_task=True)
        env.task.set_next_trajectory_index(k)
        env.reset()
        assert list(env.reference_picks()[0]) == [k, k]
        steps = LENS[k] - FUT - 1
        for t in range(steps):
            ts = env.step(np.tile(actions[t, k], (2, 1)))
            fac = env._walk_reward_factors(env._rec, env._step_counter)
            assert np.allclose(fac[:, :4], [20.0, 1.0, 1.0, 1.0], rtol=1e-5), (t, fac[:, :4])
            assert np.all(fac[:, 4:] > 0.97) and np.all(fac[:, 4:] <= 1.0)
            assert np.allclose(ts.reward, np.prod(fac, axis=1), rtol=REW_RTOL, atol=REW_ATOL), (t, ts.reward, np.prod(fac, axis=1))
            want = int(StepType.LAST) if t + 1 == steps else int(StepType.MID)
            assert np.all(np.asarray(ts.step_type) == want) and np.all(ts.discount == 1.0), (t, ts.step_type)
        env.close()


def test_set_next_trajectory_index_through_step(emu, dataset):
    path, _, _ = dataset
    env = fly_envs.walk_imitation(ref_path=path, traj_indices=PICK, n_envs=4, lib_path=emu, device_task=True,
                                  random_state=np.random.RandomState(3))
    env.task.set_next_trajectory_index(2)                     # not in traj_indices: any index of the dataset may be named
    env.reset()
    traj, start = env.reference_picks()
    assert np.all(traj == 2) and np.all(start == 0) and env.task._next_traj_idx is None
    env.step(np.zeros((4, 59), np.float32))
    env.task.set_next_trajectory_index(4)
    with pytest.raises(RuntimeError, match='pending'):
        env.step_device(np.zeros((4, 59), np.float32))
    env.request_reset([1, 3])
    env.step(np.zeros((4, 59), np.float32))
    traj2, _ = env.reference_picks()
    assert list(traj2) == [2, 4, 2, 4] and env.task._next_traj_idx is None
    env.request_reset([0])                                    # the index was used up: a fresh draw from traj_indices
    env.step(np.zeros((4, 59), np.float32))
    traj3, _ = env.reference_picks()
    assert traj3[0] in PICK and list(traj3[1:]) == [4, 2, 4]
    flat = replay_picks(path, 3, [[0, 1, 2, 3], [1, 3], [0]], [2, 4, None])
    assert [j for _, j in flat[-3:]] == [4, 4, int(traj3[0])]
    env.close()


class _HostArray:
    """an fp32 host array exposed as __cuda_array_interface__: the emulation build's 'device' memory is host memory"""

    def __init__(self, a):
        self.a = np.ascontiguousarray(a, np.float32)
        self.__cuda_array_interface__ = {'shape': self.a.shape, 'typestr': '<f4', 'data': (self.a.ctypes.data, False), 'version': 2}


def device_draws(path, lib, n, n_steps, step):
    """item 4: counter-hash draws.  `step(env, action)` -> (observation rows, out rows [n, 4]) of one step_device call."""
    env = fly_envs.walk_imitation(ref_path=path, traj_indices=PICK, n_envs=n, lib_path=lib, seed=11, terminal_com_dist=float('inf'),
                                  device_task=True, random_state=np.random.RandomState(0))
    zero = np.zeros((n, 59), np.float32)
    count = np.zeros(n, np.int64)
    episodes = [[] for _ in range(n)]
    ends = 0
    for k in range(n_steps):
        rows, out = step(env, zero)
        st_ = out[:, 2].astype(np.int64)
        first = st_ == int(StepType.FIRST)
        count = np.where(first, 0, count + 1)
        traj, start = env.reference_picks()
        for e in np.nonzero(first)[0]:
            episodes[e].append(int(traj[e]))
            assert traj[e] in PICK and start[e] == 0, (traj[e], start[e])
        ep_steps = np.minimum(5001, np.minimum(np.asarray(LENS)[traj], env._slot_len) - (FUT + 1))
        last = st_ == int(StepType.LAST)
        assert np.array_equal(last, count == ep_steps), (k, count, ep_steps, st_)
        assert np.all(out[last, 1] == 1.0) and np.all(np.isfinite(out[:, 0])) and np.all(out[:, 0] >= 0)
        ends += int(last.sum())
        if k % 7 == 0 or last.any():
            check_ref_obs(env, rows, lambda e: expected_rows(np.load(path), int(traj[e]), env._slot_len), count)
    assert ends >= n
    firsts = [ep[0] for ep in episodes]
    assert len(set(firsts)) > 1                               # the draws differ across envs ...
    assert any(len(set(ep)) > 1 for ep in episodes)           # ... and across episodes
    env.close()
    return episodes


def _emu_step(env, a):
    env._launch_step_device(_HostArray(a))
    rows, out = np.empty((env.n_envs, env._sim._tobs_dim), np.float32), np.zeros((env.n_envs, 4), np.float32)
    env._sim.task_read(rows, out)
    return rows, out


def test_step_device_draws_on_the_device(emu, dataset):
    device_draws(dataset[0], emu, 6, 200, _emu_step)


def test_reset_noise_on_the_device(emu, dataset):
    path, _, d = dataset
    a = 0.05
    env = fly_envs.walk_imitation(ref_path=path, n_envs=6, lib_path=emu, reset_noise=a, seed=5, device_task=True,
                                  random_state=np.random.RandomState(2))
    env.reset()
    traj, _ = env.reference_picks()
    q = env._sim.get(st.QPOS).astype(np.float64)
    noisy = set(int(j) for j in env._leg_act_qadr)
    assert noisy <= set(int(j) for j in env._mocap_qadr)      # (the dataset lists every actuated leg joint)
    moved = 0
    for e in range(6):
        j0 = np.array(d[f'trajectories/{int(traj[e])}/qpos'][0], np.float32)
        for k, adr in enumerate(env._mocap_qadr[:-1]):        # (the last mocap joint is the wing: at its spring)
            if int(adr) in noisy:
                assert abs(q[e, adr] - j0[k]) <= a + 1e-6, (e, k)
                moved += q[e, adr] != j0[k]
            else:
                assert q[e, adr] == j0[k], (e, k)
    assert moved > 0.9 * 6 * len(noisy)
    env.close()


def test_refusals(emu, dataset, tmp_path):
    import test_rewards_loaders as trl
    # a trajectory of at most future_steps + 1 rows among traj_indices
    path, _, d = dataset
    short = dict(d)
    g = 'trajectories/5/'
    for key in ('root_qpos', 'qpos', 'root_qvel', 'qvel', 'root2site', 'joint_quat'):
        short[g + key] = d['trajectories/0/' + key][:FUT + 1]
    short['trajectory_lengths'] = np.concatenate([d['trajectory_lengths'], [FUT + 1]])
    sp = str(tmp_path / 'short.npz'); np.savez(sp, **short)
    with pytest.raises(NotImplementedError, match='pads with their last row'):
        fly_envs.walk_imitation(ref_path=sp, n_envs=2, lib_path=emu, device_task=True)
    fly_envs.walk_imitation(ref_path=sp, traj_indices=[0, 2], n_envs=2, lib_path=emu, device_task=True).close()     # not drawn from: accepted
    # a dataset without mocap joints
    np_ = str(tmp_path / 'nj0.npz')
    trl._write_walking_dataset(np_, np.random.RandomState(0), n_traj=2, nj=0, ns=0)
    with pytest.raises(NotImplementedError, match='mocap joints'):
        fly_envs.walk_imitation(ref_path=np_, traj_indices=[1], n_envs=2, lib_path=emu, device_task=True)
    # the C side refuses a kind 0 bank program on its own: without the feature columns, with a bank of another width, without slots or bank
    env = fly_envs.walk_imitation(ref_path=path, n_envs=2, lib_path=emu, device_task=True)
    env.reset()
    kw = {}
    upload = env._sim.task_program
    env._sim.task_program = lambda **k: kw.update(k)
    env._upload_task_program()
    env._sim.task_program = upload
    nofeat = {k: v for k, v in kw.items() if not k.startswith('obs_') or k in ('obs_refdisp_off', 'obs_refquat_off')}
    with pytest.raises(st.StepperError, match='observation columns'):
        env._sim.task_program(**nofeat)
    with pytest.raises(st.StepperError, match='15 \\+ 6 n_mocap_joints'):
        env._sim.task_program(**dict(kw, n_mocap_sites=kw['n_mocap_sites'] + 1))
    with pytest.raises(st.StepperError, match='future_steps \\+ 1'):
        env._sim.task_program(**dict(kw, future_steps=LENS[4]))
    env._sim.task_program(**kw)                               # the program as uploaded is accepted again
    env.close()
    host = fly_envs.walk_imitation(ref_path=path, n_envs=2, lib_path=emu)          # slots, no bank
    host.reset()
    with pytest.raises(st.StepperError, match='trajectory bank'):
        host._sim.task_program(**kw)
    host.close()
    inf = fly_envs.walk_imitation(n_envs=2, lib_path=emu)                          # neither slots nor bank
    inf.reset()
    with pytest.raises(st.StepperError, match='reference slots'):
        inf._sim.task_program(**kw)
    inf.close()


# ------------------------------------------------------------------------------------------------------------------- GPU
@pytest.fixture(scope='module')
def gpu_dataset(tmp_path_factory):
    path = str(tmp_path_factory.mktemp('walk_gpu') / 'w.npz')
    actions, d = record_dataset(None, path)
    return path, actions, d


@pytest.mark.gpu
def test_gpu_dataset_walk_device_task_matches_host_task_code(gpu_dataset):
    path, _, d = gpu_dataset
    drive_dataset(path, d, None)


def _torch_step(env, a):
    import torch
    rows, out = env.step_device(torch.from_numpy(a).cuda(env._device))
    torch.cuda.ExternalStream(env.physics.stepper.stream).synchronize()
    return rows.cpu().numpy(), out.cpu().numpy()


@pytest.mark.gpu
def test_gpu_step_device_draws_on_the_device(gpu_dataset):
    device_draws(gpu_dataset[0], None, 6, 200, _torch_step)


@pytest.mark.gpu
def test_gpu_4096_env_rollout_draws_every_trajectory(gpu_dataset):
    import torch
    path = gpu_dataset[0]
    n, pick = 4096, [0, 2, 3, 4, 4]
    env = fly_envs.walk_imitation(ref_path=path, traj_indices=pick, n_envs=n, seed=2, terminal_com_dist=float('inf'), device_task=True)
    stream = torch.cuda.ExternalStream(env.physics.stepper.stream)
    act = torch.zeros((n, 59), device='cuda')
    longest = max(LENS[j] for j in pick) - (FUT + 1)         # (the slot holds the longest trajectory of the dataset)
    seen = set()
    lasts = 0
    for k in range(2 * longest + 2):
        rows, out = env.step_device(act)
        if k % 25 == 0 or k > 2 * longest - 2:
            stream.synchronize()
            seen |= set(int(j) for j in env.reference_picks()[0])
            o = out.cpu().numpy()
            assert torch.isfinite(rows).all().item() and np.all(np.isfinite(o))
            lasts += int((o[:, 2] == int(StepType.LAST)).sum())
    stream.synchronize()
    assert seen == set(pick) and lasts > 0
    assert np.all(env._sim.task_episodes() >= 2)              # every env ran at least two episodes
    env.close()
