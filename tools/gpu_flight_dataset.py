"""flight_imitation with a trajectory dataset at 4096 envs: env-steps/s of the host-side task code, of the device-side task code
driven through step(), and of step_device (actions and results stay on the GPU).

    python tools/gpu_flight_dataset.py [--envs 4096] [--traj 300] [--window STEPS] [--warmup 20] [--out FILE.json]

The dataset is synthetic and seeded (constant_speed_trajectory: 400-1500 rows, random speed, yaw rate and heading), written to a
temporary directory.  Every arm is warmed up, then timed over a window that ends in a device synchronise and spans at least one
episode of the longest trajectory, so that it includes the resets of every env.  Prints one line per arm, the card and its power
limit; --out also writes them as JSON."""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from flybody_b200 import fly_envs                                    # noqa: E402
from flybody_b200.synthetic import constant_speed_trajectory, _FLY_CONTROL_TIMESTEP       # noqa: E402


def write_dataset(path, n_traj, rs):
    d = {'timestep_seconds': np.float64(_FLY_CONTROL_TIMESTEP)}
    key = lambda k: f'trajectories/{str(k).zfill(len(str(n_traj)))}/'      # the loader's zero-padded group names
    for k in range(n_traj):
        q, v = constant_speed_trajectory(n_steps=int(rs.randint(400, 1501)), speed=rs.uniform(10, 40), yaw_speed=rs.uniform(-5, 5),
                                         init_heading=rs.uniform(-np.pi, np.pi), init_pos=(0, 0, 1), body_rot_angle_y=-47.5,
                                         control_timestep=_FLY_CONTROL_TIMESTEP)
        d[key(k) + 'com_qpos'], d[key(k) + 'com_qvel'] = q, v
    np.savez(path, **d)
    return max(int(d[key(k) + 'com_qpos'].shape[0]) for k in range(n_traj))


def gpu_info():
    try:
        out = subprocess.run(['nvidia-smi', '--id=0', '--query-gpu=name,power.limit', '--format=csv,noheader,nounits'],
                             capture_output=True, text=True, timeout=20).stdout.strip().split(', ')
        return {'gpu': out[0], 'power_limit_w': float(out[1])}
    except Exception as exc:                    # the rates stand without it, but say so
        return {'gpu': None, 'power_limit_w': None, 'error': str(exc)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--envs', type=int, default=4096)
    ap.add_argument('--traj', type=int, default=300)
    ap.add_argument('--window', type=int, default=0, help='timed control steps per arm (default: one episode of the longest trajectory)')
    ap.add_argument('--warmup', type=int, default=20)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit('no CUDA device: this script measures the GPU')
    rs = np.random.RandomState(0)
    tmp = tempfile.mkdtemp(prefix='flight_ds_')
    path = os.path.join(tmp, 'flight.npz')
    try:
        longest = write_dataset(path, a.traj, rs)
        run(a, path, longest, rs)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


def run(a, path, longest, rs):
    import torch
    N = a.envs
    K = a.window or (longest - 6)                                       # future_steps + 1 = 6 rows are never an episode step
    acts = rs.uniform(-0.2, 0.2, (64, N, 12)).astype(np.float32)        # a cycle of actions: the rate does not depend on them
    make = lambda dev: fly_envs.flight_imitation(ref_path=path, n_envs=N, seed=1, device_task=dev, random_state=np.random.RandomState(2))
    res = dict(gpu_info(), envs=N, trajectories=a.traj, window_steps=K, warmup_steps=a.warmup)
    for name, dev in (('host_task', False), ('device_task_step', True)):
        env = make(dev)
        env.reset()
        for k in range(a.warmup):
            env.step(acts[k % 64])
        env._sim.sync()
        resets0 = env.device_reset_count()
        t0 = time.perf_counter()
        for k in range(K):
            ts = env.step(acts[k % 64])                                 # the host reads every step's results: synchronised
        env._sim.sync()
        dt = time.perf_counter() - t0
        res[name] = {'env_steps_per_s': N * K / dt, 'ms_per_step': 1e3 * dt / K, 'resets_in_window': env.device_reset_count() - resets0,
                     'mean_reward_last_step': float(np.mean(ts.reward))}
        print(f'{name:18s} N={N} {1e3 * dt / K:8.3f} ms/step {N * K / dt:12.0f} env-steps/s  resets in window {res[name]["resets_in_window"]}',
              flush=True)
        env.close()
    env = make(True)
    stream = torch.cuda.ExternalStream(env.physics.stepper.stream)
    with torch.cuda.stream(stream):
        tacts = torch.from_numpy(acts).cuda()
        for k in range(a.warmup):
            env.step_device(tacts[k % 64])
        stream.synchronize()
        ep0 = int(env._sim.task_episodes().sum())
        t0 = time.perf_counter()
        for k in range(K):
            obs, out = env.step_device(tacts[k % 64])
        stream.synchronize()
        dt = time.perf_counter() - t0
        ok = bool(torch.isfinite(out).all().item() and torch.isfinite(obs).all().item())
    res['step_device'] = {'env_steps_per_s': N * K / dt, 'ms_per_step': 1e3 * dt / K, 'resets_in_window': int(env._sim.task_episodes().sum()) - ep0,
                          'finite_outputs': ok}
    print(f'{"step_device":18s} N={N} {1e3 * dt / K:8.3f} ms/step {N * K / dt:12.0f} env-steps/s  resets in window '
          f'{res["step_device"]["resets_in_window"]}  finite {ok}', flush=True)
    env.close()
    print(f'card: {res["gpu"]}  power limit: {res["power_limit_w"]} W  window: {K} control steps after {a.warmup} warm-up steps', flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
