"""flight_imitation with a trajectory dataset and the task hooks on the device (device_task=True): the dataset as a device bank
(fb_ref_bank), per-env trajectory / start-step draws at every reset (pinned by the host through step(), drawn from the counter
hash by step_device) and per-env episode lengths.  Held step by step against the host-side task code ON THE SAME STEPPER, as
tests/test_device_task.py does for the shared reference.  Host-emulation build unless marked gpu."""
import numpy as np
import pytest

import __graft_entry__ as ge
from flybody_b200 import fly_envs, stepper as st
from flybody_b200.dm_env_shim import StepType
from flybody_b200.synthetic import constant_speed_trajectory, rotate_vec_with_quat, reciprocal_quat, mult_quat
from flybody_b200.trajectory_loaders import HDF5FlightTrajectoryLoader

# rows, speed (cm/s), yaw speed (rad/s), heading (rad): different lengths, speeds and headings
TRAJ = [(90, 20.0, 0.0, 0.0), (120, 32.0, 8.0, 0.5), (75, 25.0, -6.0, -1.0), (140, 15.0, 3.0, 2.0), (66, 28.0, 0.0, 3.0)]
PICK = [0, 1, 3, 1]                                       # a subset with a repeat
DT = 2e-4
FUT = 5


@pytest.fixture(scope='module')
def emu():
    ge.build()
    return ge.EMU


def write_dataset(path, spec=TRAJ):
    d = {'timestep_seconds': np.float64(DT)}
    for k, (n, sp, yaw, head) in enumerate(spec):
        q, v = constant_speed_trajectory(n_steps=n, speed=sp, yaw_speed=yaw, init_heading=head, init_pos=(0.3 * k, -0.2 * k, 1),
                                         body_rot_angle_y=-47.5, control_timestep=DT)
        d[f'trajectories/{k}/com_qpos'], d[f'trajectories/{k}/com_qvel'] = q, v
    np.savez(path, **d)
    return path


def expected_rows(env, traj, start):
    """[n, 13] reference rows of an episode at (traj, start), cut from the dataset in fp64 (root x, y relative to the start CoM)"""
    cq, cv = env.task._traj_generator.full_trajectory(traj)
    cq = np.array(cq[start:], np.float64)
    cq[:, :2] -= cq[0, :2]
    root = np.concatenate([fly_envs.com2root(cq[:, :3], cq[:, 3:7]), cq[:, 3:7]], 1)
    n = min(root.shape[0], env._slot_len)
    return np.concatenate([root, np.asarray(cv[start:], np.float64)[:, :6]], 1)[:n]


def check_ref_obs(env, rec, rows_of, step_now):
    """walker/ref_displacement, ref_root_quat of every env against its reference rows, from the root pose after the step"""
    q = env._sim.get(st.QPOS).astype(np.float64)[:, env._root_q:env._root_q + 7]
    obs = env._observation(rec)
    for e in range(env.n_envs):
        rows = rows_of(e)
        t = np.minimum(step_now[e] + np.arange(env._future), len(rows) - 1)
        disp = rotate_vec_with_quat(rows[t, :3] - q[e, :3], reciprocal_quat(q[e, 3:7]))
        quat = mult_quat(reciprocal_quat(q[e, 3:7])[None], rows[t, 3:7])
        assert np.allclose(obs['walker/ref_displacement'][e], disp, atol=1e-4), (e, obs['walker/ref_displacement'][e], disp)
        assert np.allclose(obs['walker/ref_root_quat'][e], quat, atol=2e-5), e


def replay_picks(path, seed, resets, next_idx=None):
    """the (traj, start) draws of a fresh loader with the same seed over a sequence of reset id lists"""
    tg = HDF5FlightTrajectoryLoader(path, traj_indices=PICK, random_state=np.random.RandomState(seed))
    out = []
    for ids, pinned in zip(resets, next_idx or [None] * len(resets)):
        for e in ids:
            j = pinned if pinned is not None else tg._random_state.choice(tg.traj_indices)
            out.append((e, int(j), int(tg._random_state.randint(tg.trajectory_len(j) - tg.START_MARGIN))))
    return out


def drive_dataset(path, lib, n=4, n_steps=110, seed=7):
    """part a: a device-task env through step(), compared with the host task code on the same stepper after every step"""
    rs = np.random.RandomState(1)
    actions = rs.uniform(-0.2, 0.2, (n_steps, n, 12)).astype(np.float32)
    actions[:, :, -1] = rs.uniform(-1, 1, (n_steps, n))
    actions[5, 2, 3] = np.nan                                 # NaN actions act as 0
    actions[30:, 0, :] = 1.0                                  # env 0 leaves its reference -> termination -> auto-reset
    env = fly_envs.flight_imitation(ref_path=path, traj_indices=PICK, randomize_start_step=True, n_envs=n, lib_path=lib, seed=4,
                                    terminal_com_dist=0.02, random_state=np.random.RandomState(seed), device_task=True)
    sim = env._sim
    ts = env.reset()
    assert np.all(np.asarray(ts.step_type) == int(StepType.FIRST))
    resets = [list(range(n))]
    time = np.zeros(n)
    seen = [np.asarray(ts.step_type, np.int64)]
    picks = {}
    for k in range(n_steps):
        resetting = env._needs_reset.copy()
        if resetting.any():
            resets.append(list(np.nonzero(resetting)[0]))
        ts = env.step(actions[k])
        step = np.where(resetting, 0, np.minimum(np.round(time / env._control_timestep).astype(np.int64), env._ref_len - 1))
        ghost = env._ref_at(step); ghost[:, :3] += env.task._ghost_offset; ghost = ghost.astype(np.float32); ghost[resetting, 7:] = 0
        traj, start = env.reference_picks()
        assert np.array_equal(np.stack([traj, start], 1), env._ref_pick), k
        for e in range(n):
            picks[e] = (int(traj[e]), int(start[e]))
        # the host mirror holds the dataset snippet of the pick (cut in fp64 by the loader's rule) to fp32 rounding
        for e in np.nonzero(resetting)[0]:
            want = expected_rows(env, *picks[e])
            assert env._ref_len[e] == len(want) and np.allclose(env._ref_rows[e, :len(want)], want, atol=2e-6), (k, e)
            assert np.all(env._ref_rows[e, len(want):] == env._ref_rows[e, len(want) - 1])
        # ghost: on its reference row (held envs) or coasting to the next one
        q, v = sim.get(st.QPOS), sim.get(st.QVEL)
        nxt = env._ref_at(np.minimum(step + 1, env._ref_len - 1)); nxt[:, :3] += env.task._ghost_offset
        want = np.where(resetting[:, None], ghost[:, :7], nxt[:, :7])
        assert np.allclose(q[:, env._ghost_q:env._ghost_q + 3], want[:, :3], atol=2e-4), (k, q[:, env._ghost_q:env._ghost_q + 3], want[:, :3])
        assert np.allclose(q[:, env._ghost_q + 3:env._ghost_q + 7], ghost[:, 3:7], atol=5e-4), k
        assert np.allclose(v[:, env._ghost_v:env._ghost_v + 6], ghost[:, 7:], atol=1e-2), k
        if resetting.any():                                   # a reset puts the ghost exactly on row 0 of the mirror
            assert np.array_equal(q[resetting, env._ghost_q:env._ghost_q + 7], ghost[resetting, :7]), k
            assert np.array_equal(q[resetting, env._root_q:env._root_q + 7], ghost[resetting, :7]), k
        # termination / reward / discount of the host task code on the same observation record
        time = np.where(resetting, 0.0, time + env._control_timestep)
        obs = env._observation(env._rec)
        step_type, reward, discount, needs = env._task_after(env._rec, obs, resetting, time, ghost)
        assert np.array_equal(np.asarray(step_type, np.int64), np.asarray(ts.step_type, np.int64)), (k, step_type, ts.step_type)
        assert np.allclose(reward, ts.reward, atol=2e-6), (k, reward, ts.reward)
        assert np.array_equal(discount, ts.discount), k
        assert np.array_equal(needs, env._needs_reset), k
        check_ref_obs(env, env._rec, lambda e: env._ref_rows[e, :env._ref_len[e]].astype(np.float64), np.round(time / env._control_timestep).astype(np.int64))
        seen.append(np.asarray(ts.step_type, np.int64))
    # the observed reset sequence replayed on a fresh loader with the same seed gives the same draws
    flat = replay_picks(path, seed, resets)
    last = {e: (j, s0) for e, j, s0 in flat}
    assert last == picks
    env.close()
    return np.array(seen), resets


def test_dataset_flight_device_task_matches_host_task_code(emu, tmp_path):
    seen, resets = drive_dataset(write_dataset(str(tmp_path / 'f.npz')), emu)
    assert (seen == int(StepType.LAST)).any() and (seen[1:] == int(StepType.FIRST)).any()
    assert len(resets) >= 3                                   # auto-resets after terminations and episode ends


def test_set_next_trajectory_index_through_step(emu, tmp_path):
    path = write_dataset(str(tmp_path / 'f.npz'))
    env = fly_envs.flight_imitation(ref_path=path, traj_indices=PICK, n_envs=4, lib_path=emu, device_task=True,
                                    random_state=np.random.RandomState(3))
    env.task.set_next_trajectory_index(2)                     # not in traj_indices: any index of the dataset may be named
    env.reset()
    traj, start = env.reference_picks()
    assert np.all(traj == 2) and env.task._next_traj_idx is None
    assert np.all((start >= 0) & (start < TRAJ[2][0] - 50))
    env.step(np.zeros((4, 12), np.float32))
    env.task.set_next_trajectory_index(4)
    with pytest.raises(RuntimeError, match='pending'):
        env.step_device(np.zeros((4, 12), np.float32))
    env.request_reset([1, 3])
    env.step(np.zeros((4, 12), np.float32))
    traj2, start2 = env.reference_picks()
    assert list(traj2) == [2, 4, 2, 4] and np.array_equal(start2[[0, 2]], start[[0, 2]]) and env.task._next_traj_idx is None
    env.request_reset([0])                                    # the index was used up: a fresh draw from traj_indices
    env.step(np.zeros((4, 12), np.float32))
    traj3, _ = env.reference_picks()
    assert traj3[0] in PICK and list(traj3[1:]) == [4, 2, 4]
    flat = replay_picks(path, 3, [[0, 1, 2, 3], [1, 3], [0]], [2, 4, None])
    assert [(j, s0) for _, j, s0 in flat[-3:]] == [(4, int(start2[1])), (4, int(start2[3])), (int(traj3[0]), int(env.reference_picks()[1][0]))]
    env.close()


class _HostArray:
    """an fp32 host array exposed as __cuda_array_interface__: the emulation build's 'device' memory is host memory"""

    def __init__(self, a):
        self.a = np.ascontiguousarray(a, np.float32)
        self.__cuda_array_interface__ = {'shape': self.a.shape, 'typestr': '<f4', 'data': (self.a.ctypes.data, False), 'version': 2}


def device_draws(path, lib, n, n_steps, step):
    """part c: counter-hash draws.  `step(env, action)` -> (observation rows, out rows [n, 4]) of one step_device call."""
    env = fly_envs.flight_imitation(ref_path=path, traj_indices=PICK, n_envs=n, lib_path=lib, seed=11, terminal_com_dist=float('inf'),
                                    device_task=True, random_state=np.random.RandomState(0))
    bank_len, _ = env._bank_tables()
    zero = np.zeros((n, 12), np.float32)
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
            episodes[e].append((int(traj[e]), int(start[e])))
            assert traj[e] in PICK and 0 <= start[e] < bank_len[traj[e]] - 50, (traj[e], start[e])
        ep_steps = np.minimum(np.minimum(bank_len[traj] - start, env._slot_len), round(0.6 / DT)) - (FUT + 1)
        last = st_ == int(StepType.LAST)
        assert np.array_equal(last, count == ep_steps), (k, count, ep_steps, st_)
        assert np.all(out[last, 1] == 1.0) and np.all(np.isfinite(out[:, 0]))
        ends += int(last.sum())
        if k % 7 == 0 or last.any():
            check_ref_obs(env, rows, lambda e: expected_rows(env, int(traj[e]), int(start[e])), count)
    assert ends >= n
    firsts = [p for ep in episodes for p in ep[:1]]
    assert len(set(firsts)) > 1                               # the draws differ across envs ...
    assert any(len(set(ep)) > 1 for ep in episodes)           # ... and across episodes
    env.close()
    return episodes


def test_step_device_draws_on_the_device(emu, tmp_path):
    def step(env, a):
        env._launch_step_device(_HostArray(a))
        rows, out = np.empty((env.n_envs, env._sim._tobs_dim), np.float32), np.zeros((env.n_envs, 4), np.float32)
        env._sim.task_read(rows, out)
        return rows, out
    device_draws(write_dataset(str(tmp_path / 'f.npz')), emu, 6, 200, step)


def test_short_trajectory_with_random_start_is_refused(emu, tmp_path):
    spec = TRAJ[:2] + [(50, 20.0, 0.0, 0.0)]
    path = write_dataset(str(tmp_path / 'short.npz'), spec)
    with pytest.raises(ValueError, match='longer than 50 rows'):
        fly_envs.flight_imitation(ref_path=path, n_envs=2, lib_path=emu, device_task=True)
    # not drawn from, or no random start: accepted
    fly_envs.flight_imitation(ref_path=path, traj_indices=[0, 1], n_envs=2, lib_path=emu, device_task=True).reset()
    env = fly_envs.flight_imitation(ref_path=path, randomize_start_step=False, n_envs=2, lib_path=emu, device_task=True)
    env.reset()
    # the C side refuses the same program on its own
    env.task._traj_generator._randomize_start_step = True
    with pytest.raises(st.StepperError, match='longer than start_margin'):
        env._upload_task_program()
    env.close()


# ------------------------------------------------------------------------------------------------------------------- GPU
@pytest.mark.gpu
def test_gpu_dataset_flight_device_task_matches_host_task_code(tmp_path):
    seen, _ = drive_dataset(write_dataset(str(tmp_path / 'f.npz')), None)
    assert (seen == int(StepType.LAST)).any()


def _torch_step(env, a):
    import torch
    rows, out = env.step_device(torch.from_numpy(a).cuda(env._device))
    torch.cuda.ExternalStream(env.physics.stepper.stream).synchronize()
    return rows.cpu().numpy(), out.cpu().numpy()


@pytest.mark.gpu
def test_gpu_step_device_draws_on_the_device(tmp_path):
    device_draws(write_dataset(str(tmp_path / 'f.npz')), None, 6, 200, _torch_step)


@pytest.mark.gpu
def test_gpu_4096_env_rollout_draws_every_trajectory(tmp_path):
    import torch
    spec = [(100 + 20 * k, 15.0 + 3 * k, 2.0 * (k % 3 - 1), 0.7 * k) for k in range(6)]
    path = write_dataset(str(tmp_path / 'f.npz'), spec)
    n, pick = 4096, [0, 2, 3, 5, 5]
    env = fly_envs.flight_imitation(ref_path=path, traj_indices=pick, n_envs=n, seed=2, device_task=True)
    stream = torch.cuda.ExternalStream(env.physics.stepper.stream)
    act = torch.zeros((n, 12), device='cuda')
    longest = max(r for r, *_ in spec) - (FUT + 1)
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
