"""vision_guided_flight, first cut (SURVEY.md 8(f).1), on the host-emulation build: the dm_env contract of the reference task
(`tasks/vision_flight.py`), reward factors against their definitions, fatal terrain contacts, per-episode terrains, eyes."""
import numpy as np
import pytest

import __graft_entry__ as ge
from flybody_b200 import arenas, fly_envs, stepper as st
from flybody_b200.dm_env_shim import StepType


@pytest.fixture(scope='module')
def emu():
    ge.build()
    return ge.EMU


def test_contract_and_first_steps(emu):
    env = fly_envs.vision_guided_flight(n_envs=2, lib_path=emu, seed=1)
    spec = env.observation_spec()
    assert list(spec) == ['walker/accelerometer', 'walker/actuator_activation', 'walker/gyro', 'walker/joints_pos', 'walker/joints_vel',
                          'walker/left_eye', 'walker/right_eye', 'walker/velocimeter', 'walker/world_zaxis', 'walker/task_input']
    assert spec['walker/right_eye'].shape == (2, 32, 32, 3) and spec['walker/right_eye'].dtype == np.uint8      # vision_flight.py:23-24
    assert spec['walker/joints_pos'].shape == (2, 25) and spec['walker/task_input'].shape == (2, 2)
    assert env.action_spec().shape == (12,) and env.action_spec().name.split('\t')[-1] == 'user_0'
    assert np.isclose(env.control_timestep(), 2e-4)
    ts = env.reset()
    assert np.all(ts.step_type == StepType.FIRST)
    for k, v in ts.observation.items():
        assert v.shape == spec[k].shape and v.dtype == spec[k].dtype, k
    th, tv = ts.observation['walker/task_input'][:, 0], ts.observation['walker/task_input'][:, 1]
    assert np.all((0.5 <= th) & (th <= 0.8) & (20 <= tv) & (tv <= 40))                                        # vision_flight.py:28-29
    # start: x = -5, y = 0, target height above the terrain's nearest grid point, flying at the target speed (vision_flight.py:111-139)
    q, v = env._sim.get(st.QPOS), env._sim.get(st.QVEL)
    assert np.allclose(q[:, :2], [-5.0, 0.0], atol=1e-6) and np.allclose(v[:, 0], tv, atol=1e-4)
    assert np.allclose(q[:, 2] - env.hfield_height(q[:, 0], q[:, 1]), th, atol=1e-5)
    # every env flies over its own terrain, and sees it
    assert not np.array_equal(env._terrain[0], env._terrain[1])
    assert not np.array_equal(ts.observation['walker/left_eye'][0], ts.observation['walker/left_eye'][1])
    assert ts.observation['walker/right_eye'].std() > 10
    rs = np.random.RandomState(0)
    for _ in range(15):
        ts = env.step(rs.uniform(-0.2, 0.2, (2, 12)))
        assert np.all(ts.step_type == StepType.MID) and np.all(ts.discount == 1.0)
        assert np.all((ts.reward > 0) & (ts.reward <= 1.0)) and all(np.all(np.isfinite(v)) for v in ts.observation.values())
    env.close()


def test_reward_factors_follow_their_definitions(emu):
    env = fly_envs.vision_guided_flight(n_envs=3, lib_path=emu, seed=2)
    env.reset()
    env.step(np.zeros((3, 12)))
    f = env.reward_factors(env._rec)
    assert f.shape == (3, 6) and np.all((f >= 0) & (f <= 1))
    pose = env._rec[:, env._sl['_root_pose']].astype(np.float64)
    vel = env._rec[:, env._sl['_root_qvel']].astype(np.float64)[:, :3]
    h = pose[:, 2] - env.hfield_height(pose[:, 0], pose[:, 1])
    assert np.allclose(f[:, 0], np.clip(1 - np.abs(h - env.target_height) / 0.15, 0, 1))
    ts = env.target_speed
    assert np.allclose(f[:, 1], np.where(vel[:, 0] >= ts, 1.0, np.clip(1 - (ts - vel[:, 0]) / (1.1 * ts), 0, 1)))
    assert np.allclose(f[:, 2], np.clip(1 - np.abs(np.linalg.norm(vel, axis=1) - ts) / (1.1 * ts), 0, 1))
    assert np.all(f[:, 5] == 1.0)                                      # no trench in the 'bumps' arena
    # one step after the start the fly is still close to its targets
    assert np.all(f[:, 0] > 0.9) and np.all(f[:, 2] > 0.85) and np.all(f[:, 4] > 0.9)
    env.close()


def test_terrain_contact_is_fatal_and_the_next_episode_gets_a_new_terrain(emu):
    env = fly_envs.vision_guided_flight(n_envs=2, lib_path=emu, seed=3, target_height_range=(0.5, 0.5))
    env.reset()
    terr0 = env._terrain.copy()
    # push env 1 into the ground: place it a hair above the terrain with a downward velocity
    q, v = env._sim.get(st.QPOS), env._sim.get(st.QVEL)
    q[1, 2] = env.hfield_height(q[:, 0], q[:, 1])[1] - 0.01 + 0.14
    v[1, 2] = -300.0
    env._sim.set(st.QPOS, q); env._sim.set(st.QVEL, v)
    hit = None
    for k in range(12):
        ts = env.step(np.zeros((2, 12)))
        if ts.step_type[1] == StepType.LAST:
            hit = k
            break
    assert hit is not None and ts.discount[1] == 0.0 and ts.step_type[0] == StepType.MID and ts.discount[0] == 1.0
    assert env.floor_contact()[1] and not env.floor_contact()[0]
    ts = env.step(np.zeros((2, 12)))                                   # auto-reset of env 1 only
    assert ts.step_type[1] == StepType.FIRST and ts.step_type[0] == StepType.MID
    assert np.array_equal(env._terrain[0], terr0[0]) and not np.array_equal(env._terrain[1], terr0[1])
    q = env._sim.get(st.QPOS)
    assert np.allclose(q[1, 2] - env.hfield_height(q[:, 0], q[:, 1])[1], 0.5, atol=1e-5)
    env.close()


def test_trench_arena_reward_and_time_limit(emu):
    env = fly_envs.vision_guided_flight(n_envs=1, bumps_or_trench='trench', lib_path=emu, seed=5, init_pos_x_range=(-2.5, -2.5))
    ts = env.reset()
    spec = env._arenas[0].trench_specs
    assert spec is not None and spec['x_coords'][0] <= -3.0
    env.step(np.zeros(12))
    f = env.reward_factors(env._rec)
    pose = env._rec[:, env._sl['_root_pose']]
    yc = spec['y_coords'][np.abs(spec['x_coords'] - pose[0, 0]).argmin()]
    assert np.isclose(f[0, 5], np.clip(1 - abs(pose[0, 1] - yc) / 0.15, 0, 1))
    # time limit 0.4 s = 2000 control steps is a LAST with discount 1: shorten it for the test
    env._time_limit = 5 * env.control_timestep()
    for k in range(4):
        ts = env.step(np.zeros(12))
    assert ts.step_type == StepType.LAST and ts.discount == 1.0
    env.close()


def test_terrain_bank_option(emu):
    env = fly_envs.vision_guided_flight(n_envs=4, lib_path=emu, seed=7, terrain_bank=2)
    env.reset()
    bank = [t for t, _ in env._bank]
    assert len(bank) == 2 and all(any(np.array_equal(env._terrain[e], b) for b in bank) for e in range(4))
    ts = env.step(np.zeros((4, 12)))
    assert np.all(np.isfinite(ts.reward))
    env.close()


@pytest.mark.parametrize('low_start,arena', [(True, 'bumps'), (False, 'bumps'), (False, 'trench')])
def test_device_task_matches_the_host_task_code(emu, low_start, arena):
    """fb_task_* kind 2: the vision task's hooks on the device (terrain pick from the device bank, targets, start pose, wing-beat
    generator, five reward factors, fatal world contacts, time limit) against the host-side task code of this file's env, step by step
    through terminations and auto-resets; the device is fed the host's random draws (fb_task_uniform_rows)."""
    # low start: the flies begin within contact range of the terrain -> fatal contacts (discount 0); otherwise the time limit ends episodes
    kw = dict(n_envs=3, lib_path=emu, seed=5, terrain_bank=2, time_limit=0.004, **(dict(target_height_range=(0.12, 0.2)) if low_start else {}))
    if arena == 'trench':           # start inside the corridor's x range, off its centre line: the sixth reward factor is < 1
        kw.update(bumps_or_trench='trench', init_pos_x_range=(-2.0, -1.5), init_pos_y_range=(-0.12, 0.12))
    host = fly_envs.vision_guided_flight(**kw)
    dev = fly_envs.vision_guided_flight(device_task=True, **kw)
    th = host.reset()
    dev._forced_draws = host._last_draws.copy()
    td = dev.reset()
    for k in th.observation:
        a, b = np.asarray(th.observation[k], np.float64), np.asarray(td.observation[k], np.float64)
        if a.size == 0:
            continue
        if 'eye' in k:
            assert (np.abs(a - b) <= 2).mean() > 0.99, k
        else:
            assert np.allclose(a, b, atol=1e-3 * (np.abs(a).max() + 1)), (k, np.abs(a - b).max())      # (start height: fp64 on the host, fp32 on the device)
    assert np.allclose(host._sim.get(st.QPOS), dev._sim.get(st.QPOS), atol=1e-6)
    rs = np.random.RandomState(0)
    seen_last = seen_first = False
    discounts = set()
    centre_min = 1.0
    for step in range(30):
        a = rs.uniform(-0.2, 0.2, (3, 12)).astype(np.float32)
        a[0, :] = 1.0 if step > 8 else a[0]                      # env 0 is driven off course -> terrain contact or time limit -> LAST -> auto-reset
        th = host.step(a)
        dev._forced_draws = host._last_draws.copy()
        td = dev.step(a)
        assert np.array_equal(np.asarray(th.step_type), np.asarray(td.step_type)), (step, th.step_type, td.step_type)
        # the device's reward against the host-side reward code evaluated on the device env's own state: the two envs' trajectories
        # drift apart at the fatal terrain contacts (qpos check below), which moves their rewards by up to a few 1e-3
        want = np.where(np.asarray(td.step_type) == int(StepType.FIRST), 0.0, np.prod(host.reward_factors(dev._rec), axis=1))
        assert np.allclose(want, td.reward, atol=2e-4), (step, want, td.reward)
        assert np.array_equal(th.discount, td.discount), step
        assert np.allclose(host._sim.get(st.QPOS), dev._sim.get(st.QPOS), atol=1e-2), (step, np.abs(host._sim.get(st.QPOS) - dev._sim.get(st.QPOS)).max())      # (env 0 is driven against its joint limits: the fp64-host / fp32-device wing residual difference grows chaotically)
        assert np.allclose(th.observation['walker/task_input'], td.observation['walker/task_input'], atol=1e-6)
        centre_min = min(centre_min, float(host.reward_factors(host._rec)[:, 5].min()))
        discounts |= set(np.asarray(th.discount)[np.asarray(th.step_type) == int(StepType.LAST)].tolist())
        seen_last |= bool((np.asarray(th.step_type) == int(StepType.LAST)).any())
        seen_first |= step > 0 and bool((np.asarray(th.step_type) == int(StepType.FIRST)).any())
    assert seen_last and seen_first
    assert (0.0 in discounts) if low_start else (1.0 in discounts), discounts
    if arena == 'trench':
        assert centre_min < 0.999, centre_min
    host.close(); dev.close()


def test_replacing_the_terrain_bank_invalidates_the_vision_task_program(emu):
    """fb_hfield_bank frees a replaced bank; the device task program pointed into it, so stepping needs a fresh fb_task_program"""
    env = fly_envs.vision_guided_flight(n_envs=2, lib_path=emu, seed=1, terrain_bank=2, device_task=True)
    env.reset()
    env.step(np.zeros((2, 12), np.float32))
    bank = np.stack([t for t, _ in env._bank])
    env._sim.hfield_bank(bank[::-1].copy())
    with pytest.raises(st.StepperError):
        env._sim.task_step(np.zeros((2, 12), np.float32), env._n_sub)
    env._upload_task_program(seed=1)
    ts = env.reset()
    assert np.all(np.asarray(ts.step_type) == int(StepType.FIRST))
    ts = env.step(np.zeros((2, 12), np.float32))
    assert np.all(np.isfinite(ts.reward))
    env.close()


def test_a_rejected_task_program_leaves_the_running_one_in_place(emu, monkeypatch):
    """fb_task_program checks the trench centre lines before it replaces anything: a program with a bad one is refused (-1) and
    the vision task program already on the device keeps stepping"""
    env = fly_envs.vision_guided_flight(n_envs=2, bumps_or_trench='trench', lib_path=emu, seed=1, terrain_bank=2, device_task=True)
    env.reset()
    env.step(np.zeros((2, 12), np.float32))
    sim, args = env._sim, []
    with monkeypatch.context() as mp:      # the arguments the env uploads, without replacing its bank or program
        mp.setattr(sim, 'hfield_bank', lambda heights: None)
        mp.setattr(sim, 'task_program', lambda **kw: args.append(kw))
        env._upload_task_program(seed=1)
    bad = dict(args[0], trench_len=np.ones(2, np.int32))        # a centre line of one point
    with pytest.raises(st.StepperError, match=r'\(-1\).*bad trench centre line'):
        sim.task_program(**bad)
    ts = env.step(np.zeros((2, 12), np.float32))
    assert np.all(np.isfinite(ts.reward))
    env.close()


@pytest.mark.parametrize('device_task', [False, True])
def test_capacity_overflow_is_counted_not_a_termination(emu, device_task):
    """FB_FLAGS bits 1 / 2 (contact list or constraint rows at capacity: FB_MAXCON = 64 contacts here) are not bad physics: the
    reference terminates on |qacc| only (tasks/base.py:222-225), so the episode goes on and the env counts the event"""
    env = fly_envs.vision_guided_flight(n_envs=2, lib_path=emu, seed=1, terrain_bank=2, target_height_range=(0.04, 0.05),
                                        floor_contacts_fatal=False, device_task=device_task)
    env.reset()
    ts = env.step(np.zeros((2, 12), np.float32))                      # the fly starts half inside the terrain: > 64 candidate contacts
    assert np.all(env._sim.get(st.NCON)[:, 0] == 64) and np.all(env._sim.get(st.FLAGS)[:, 0].astype(np.int64) & 6)
    assert np.all(env._sim.get(st.FLAGS)[:, 0].astype(np.int64) & 1 == 0)
    assert np.all(np.asarray(ts.step_type) == int(StepType.MID)) and np.all(np.asarray(ts.discount) == 1.0)
    assert env.n_capacity_overflows >= 2
    env.close()
