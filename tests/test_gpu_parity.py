"""Parity tests proper: the CUDA stepper on an H100, through the C ABI, against the CPU oracle."""
import numpy as np
import pytest

from flybody_b200 import stepper as st
from flybody_b200.flymodel import load_model
from oracle import fly_oracle as fo
from parity_common import compare_stage_fields, teacher_forced_errors, summarize_tf, reset_qpos

pytestmark = pytest.mark.gpu


def test_library_is_the_cuda_build():
    m = load_model('walk')
    s = st.BatchedStepper(m, 32)
    assert 'sm_90a' in s.version()
    assert s.launch_count > 0


@pytest.mark.parametrize('seed', [0, 1, 2, 3])
def test_stage_parity_walk(seed):
    m = load_model('walk')
    compare_stage_fields(m, st.BatchedStepper(m, 64), seed=seed, env=17)


@pytest.mark.parametrize('seed', [0, 1])
def test_stage_parity_flight(seed):
    m = load_model('flight')
    compare_stage_fields(m, st.BatchedStepper(m, 64), seed=seed, vel_scale=20.0, env=5)


def test_teacher_forced_200_control_steps_walk():
    """BASELINE.json config 1: 200 random-action control steps, error measured one step ahead."""
    m = load_model('walk')
    r = summarize_tf(*teacher_forced_errors(m, st.BatchedStepper(m, 32), n_steps=200, n_sub=10))
    print('teacher-forced walk:', r)
    # bulk: fp32 tolerance (gate = what is measured, x2.5); isolated contact-switch events (incl. generic convex contacts
    # whose MPR depth carries its 1e-6 support tolerance): histogram printed, at most 10 % of the steps above the bulk gate,
    # at most 2 % above 10x the gate, bounded size
    assert r['p90_q'] < 2e-6 and r['p90_v'] < 5e-4, r
    assert r['events'] <= 20 and r['hist_v']['<0.005'] >= 196 and r['max_q'] < 2e-3 and r['max_v'] < 5.0, r
    # per-substep sensor mean of every control step against the oracle's (force / touch / accelerometer / gyro / velocimeter
    # observables are this mean: reference fruitfly.py:626-665)
    assert r['p90_s'] < 2e-4 and r['sensor_events'] <= 20 and r['max_s'] < 0.5, r


def test_teacher_forced_flight():
    m = load_model('flight')
    r = summarize_tf(*teacher_forced_errors(m, st.BatchedStepper(m, 32), n_steps=50, n_sub=4, ctrl_scale=0.2), tol_v=2e-3)
    print('teacher-forced flight:', r)
    assert r['p90_q'] < 2e-6 and r['p90_v'] < 1e-3 and r['events'] <= 2, r
    assert r['p90_s'] < 2e-4 and r['max_s'] < 2e-3, r


def test_free_running_drift_walk_reported():
    """Free-running divergence over 50 control steps (chaotic contact dynamics: reported, loosely gated)."""
    m = load_model('walk')
    s = st.BatchedStepper(m, 32)
    o = fo.Oracle(m, tolerance=1e-12)
    q0 = reset_qpos(m)
    s.reset(q0)
    o.reset(q0)
    rs = np.random.RandomState(0)
    for k in range(50):
        c = rs.uniform(-0.5, 0.5, m.nu)
        s.set_control(c)
        o.set(fo.CTRL, c)
        s.step(10)
        o.control_step(10)
    e = np.abs(s.get(st.QPOS)[0][:109] - o.qpos[:109]).max()
    print(f'free-running 50 steps: max|dqpos|={e:.2e}')
    assert e < 5e-2


def test_batch_consistency_and_size_independent_properties():
    """4096 envs: identical envs give bit-identical results; padding / env index do not matter;
    quaternions stay normalised; the fly stays on the floor (no tunnelling) under random actions."""
    m = load_model('walk')
    N = 4096
    s = st.BatchedStepper(m, N)
    q0 = reset_qpos(m)
    s.reset(q0)
    rs = np.random.RandomState(0)
    for k in range(5):
        s.set_control(rs.uniform(-0.5, 0.5, m.nu))
        s.step(10)
    q = s.get(st.QPOS)
    assert np.all(q == q[0])                       # bit-exact across lanes / blocks
    assert np.all(s.get(st.FLAGS) == 0)
    # decorrelated envs
    qq = np.tile(q0, (N, 1))
    hinge = np.arange(7, 109)
    qq[:, hinge] += rs.uniform(-0.05, 0.05, (N, 102))
    s.reset(qq)
    for k in range(10):
        s.set_control(rs.uniform(-0.5, 0.5, (N, m.nu)))
        s.step(10)
    q = s.get(st.QPOS)
    assert np.all(np.isfinite(q))
    assert np.abs(np.linalg.norm(q[:, 3:7], axis=1) - 1).max() < 1e-5
    assert q[:, 2].min() > 0.02 and q[:, 2].max() < 0.3
    assert (s.get(st.FLAGS)[:, 0] != 0).mean() < 0.01
    # a shuffled copy of the batch gives the shuffled result (env order independence)
    perm = rs.permutation(N)
    s2 = st.BatchedStepper(m, N)
    s2.reset(qq[perm])
    s.reset(qq)
    c = rs.uniform(-0.5, 0.5, (N, m.nu)).astype(np.float32)
    s.set_control(c)
    s2.set_control(c[perm])
    s.step(10)
    s2.step(10)
    assert np.array_equal(s.get(st.QPOS)[perm], s2.get(st.QPOS))


def test_env_facade_on_gpu():
    from flybody_b200 import fly_envs
    env = fly_envs.walk_imitation(terminal_com_dist=float('inf'), n_envs=256)
    ts = env.reset()
    rs = np.random.RandomState(0)
    for _ in range(20):
        ts = env.step(rs.uniform(-0.5, 0.5, (256, 59)))
        assert np.all(ts.reward == 1.0)
    assert all(np.all(np.isfinite(v)) for v in ts.observation.values())


def test_flight_env_facade_on_gpu():
    from flybody_b200 import fly_envs
    env = fly_envs.flight_imitation(n_envs=128, seed=1)
    env.reset()
    rs = np.random.RandomState(0)
    for _ in range(30):
        ts = env.step(rs.uniform(-0.2, 0.2, (128, 12)))
    assert all(np.all(np.isfinite(v)) for v in ts.observation.values())
    assert np.all((ts.reward > 0.8) & (ts.reward <= 1.0))


def test_dataset_mode_envs_on_gpu(tmp_path):
    """per-env reference slots, full-body start pose, DeepMimic reward (tests/test_env_dataset.py) on the CUDA build."""
    import test_env_dataset as ds
    ds.test_dataset_mode_tracks_own_snippet_and_rewards(None, tmp_path)
    ds.test_dataset_mode_replay_keeps_maximal_reward(None, tmp_path)
    ds.test_flight_dataset_mode_per_env_trajectories(None, tmp_path)


def test_device_task_logic_on_gpu():
    """fb_task_*: the task hooks on the device against the host-side task code on the same stepper (tests/test_device_task.py)."""
    import test_device_task as dt
    dt.test_walk_device_task_matches_host_task_code(None)
    dt.test_walk_device_task_episode_end_is_a_good_termination(None)
    dt.test_walk_device_task_reset_noise_is_bounded_and_varies(None)
    dt.test_switching_the_shared_trajectory_restarts_every_env(None)      # re-uploaded programs free the replaced device buffers
    dt.test_flight_device_task_matches_host_task_code(None)


def test_vision_model_terrain_contacts_on_gpu():
    """heightfield narrowphase kernel (fb_hf_kernel) inside the step of the `vision` model: contacts, rows and forces against the
    oracle's terrain collision (tests/test_hfield.py, here on the CUDA build)."""
    import test_hfield as th
    th.check_vision_terrain_contacts(None)


def test_vision_model_stage_parity_on_gpu():
    import test_hfield as th
    th.check_vision_free_flight(None)


@pytest.mark.parametrize('low_start,arena', [(True, 'bumps'), (False, 'bumps'), (False, 'trench')])
def test_vision_device_task_logic_on_gpu(low_start, arena):
    """fb_task_* kind 2 (terrain bank pick, targets, start pose, reward factors incl. the trench centre line, fatal world contacts, time limit) on the CUDA build
    against the host-side vision task code on the same stepper, through terminations and auto-resets (tests/test_vision_env.py)."""
    import test_vision_env as tv
    tv.test_device_task_matches_the_host_task_code(None, low_start, arena)


def test_vision_device_resident_rollout_matches_host_api():
    """vision env step_device (CUDA actions in; observation rows, (reward, discount, step_type) and eye images as zero-copy views)
    against step() on a twin env."""
    import torch
    from flybody_b200 import fly_envs
    n = 32
    kw = dict(n_envs=n, seed=3, terrain_bank=4, time_limit=0.001, device_task=True)      # 5 control steps per episode
    a_env, b_env = fly_envs.vision_guided_flight(**kw), fly_envs.vision_guided_flight(**kw)
    a_env.reset(); b_env.reset()
    lay = a_env.observation_layout()
    stream = torch.cuda.ExternalStream(a_env._sim.stream)
    rs = np.random.RandomState(0)
    saw_first = False
    for k in range(12):
        act = rs.uniform(-0.3, 0.3, (n, 12)).astype(np.float32)
        ts = b_env.step(act)
        with torch.cuda.stream(stream):
            rows, out, eyes = a_env.step_device(torch.from_numpy(act).cuda(a_env._sim.device))
            stream.synchronize()
            rows_h, out_h, eyes_h = rows.cpu().numpy(), out.cpu().numpy(), eyes.cpu().numpy()
        assert np.array_equal(out_h[:, 2].astype(np.int64), np.asarray(ts.step_type, np.int64)), k
        assert np.array_equal(out_h[:, 0], np.asarray(ts.reward, np.float32)) and np.array_equal(out_h[:, 1], np.asarray(ts.discount, np.float32))
        assert np.array_equal(rows_h[:, lay['walker/gyro']].reshape(n, -1), np.asarray(ts.observation['walker/gyro']).reshape(n, -1))
        assert np.array_equal(rows_h[:, lay['walker/task_input']], np.asarray(ts.observation['walker/task_input']))
        assert np.array_equal(eyes_h[:, 1], np.asarray(ts.observation['walker/left_eye'])) and np.array_equal(eyes_h[:, 0], np.asarray(ts.observation['walker/right_eye']))
        saw_first |= bool((out_h[:, 2] == 0).any())
    assert saw_first
    a_env.close(); b_env.close()


@pytest.mark.parametrize('device_task', [False, True])
def test_sensor_observables_match_the_oracle_mean_on_gpu(device_task):
    """the buffered observables of env.reset() / env.step() against the oracle's per-substep mean, incl. the FIRST step"""
    import test_env as te
    te.check_sensor_observables_against_oracle(None, device_task)


def test_device_observation_program_matches_numpy_formulas_on_gpu():
    import test_env as te
    te.test_device_observation_program_matches_numpy_formulas(None)


def test_first_observation_is_independent_of_history_on_gpu(monkeypatch):
    import test_reset_first_obs as tr
    for dt in (False, True):
        tr.test_flight_first_observation_is_independent_of_the_previous_action(None, dt)
        tr.test_walk_first_observation_is_independent_of_the_previous_action(None, dt)
    tr.test_flight_first_accelerometer_with_a_fixed_wing_phase(None)


def test_eye_renderer_on_gpu_matches_host_emulation():
    """fb_render_eyes on the GPU against the same kernel source run by the host-emulation build (tests/test_eyes.py holds
    that one against the camera model and a brute-force ray marcher)."""
    import __graft_entry__ as ge
    from flybody_b200 import arenas, fly_envs
    ge.build()
    dim, dens = 6, 5
    nrow, ncol = arenas.grid_shape(dim, dens)
    terr = arenas.SineBumps(dim=dim, grid_density=dens, wavelength_range=(2.0, 3.0), height_range=(0.6, 0.9)).generate(np.random.RandomState(2))
    imgs = []
    for lib in (None, ge.EMU):
        env = fly_envs.flight_imitation(n_envs=3, lib_path=lib)
        env.reset()
        env.enable_eyes(size=32, fovy=150.0, terrain_shape=(nrow, ncol), half_size=float(dim), z_offset=-0.01)
        env.set_terrain(np.array([1, 2]), np.stack([terr, terr[::-1].copy()]))
        imgs.append(env.render_eyes())
        env.close()
    for name in imgs[0]:
        a, b = imgs[0][name].astype(np.int64), imgs[1][name].astype(np.int64)
        assert a.shape == (3, 32, 32, 3)
        close = np.abs(a - b).max(-1) <= 2
        assert close.mean() > 0.98, (name, close.mean())            # (fp32 contraction differs: a few horizon / checker-edge pixels may flip)
        assert a.std() > 10                                          # an image, not a constant


def test_device_resident_rollout_matches_host_api():
    """step_device (CUDA action tensor in, zero-copy observation / reward views out, no host copy) against step() on a twin env."""
    import torch
    from flybody_b200 import fly_envs
    n = 64
    a_env = fly_envs.walk_imitation(terminal_com_dist=0.05, n_envs=n, device_task=True)
    b_env = fly_envs.walk_imitation(terminal_com_dist=0.05, n_envs=n, device_task=True)
    a_env.reset(); b_env.reset()
    stream = torch.cuda.ExternalStream(a_env.physics.stepper.stream)
    rs = np.random.RandomState(0)
    lay = a_env.observation_layout()
    saw_first = False
    for k in range(20):
        act = rs.uniform(-0.5, 0.5, (n, 59)).astype(np.float32)
        ts = b_env.step(act)
        with torch.cuda.stream(stream):
            obs, out = a_env.step_device(torch.from_numpy(act).cuda())
            stream.synchronize()
            obs_h, out_h = obs.cpu().numpy(), out.cpu().numpy()
        assert np.array_equal(out_h[:, 2].astype(np.int64), np.asarray(ts.step_type, np.int64)), k
        assert np.array_equal(out_h[:, 0], np.asarray(ts.reward, np.float32)) and np.array_equal(out_h[:, 1], np.asarray(ts.discount, np.float32))
        sl, shp = lay['walker/joints_pos']
        assert np.array_equal(obs_h[:, sl].reshape((n,) + shp), ts.observation['walker/joints_pos'])   # two handles, same kernels, same inputs
        saw_first |= bool((out_h[:, 2] == 0).any())
    assert saw_first


def test_smoke_entry():
    import __graft_entry__ as ge
    ge.smoke()
