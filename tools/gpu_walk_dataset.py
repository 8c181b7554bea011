"""walk_imitation with a trajectory dataset at 4096 envs: env-steps/s of the host-side task code, of the device-side task code driven
through step(), of step_device (actions and results stay on the GPU), and of inference-mode walking through step_device for comparison.

    python tools/gpu_walk_dataset.py [--envs 4096] [--traj 300] [--window STEPS] [--warmup 20] [--repeats 2] [--out FILE.json]

The dataset is recorded from the stepper in the same call and seeded: an inference-mode walking batch of --traj envs is rolled with
small random actions, and trajectory k is the first 100-235 rows of env k: root and leg-joint qpos / qvel, claw and head sites
(the rollout stays inside one 235-step episode of the inference reference; joint_quat rows are unit quaternions: the rate does not
depend on them).  It is written to a temporary directory.  Every arm is warmed
up, then timed over a window that ends in a device synchronise and spans at least one episode of the longest trajectory, so that it
includes the resets of every env.  The two step_device arms run --repeats times, alternating, to show the run-to-run spread.  A
separate profiled pass (CUDA events per kernel kind) then gives the task kernels' time per control step of the two step_device arms.
Prints one line per arm, the card and its power limit; --out also writes them as JSON."""
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
from flybody_b200 import fly_envs, stepper as st                     # noqa: E402
from flybody_b200.synthetic import rotate_vec_with_quat, reciprocal_quat   # noqa: E402

FUT = 64


def record_dataset(path, n_traj, rs):
    """-> the longest trajectory's rows; trajectory k = the first 100-235 rows of env k of an inference-mode rollout"""
    lens = rs.randint(100, 236, n_traj)
    T = int(lens.max())
    env = fly_envs.walk_imitation(terminal_com_dist=float('inf'), n_envs=n_traj, reset_noise=0.03, seed=3, device_task=False)
    m, sim = env.model, env._sim
    jn, sn = m.meta['jnt_names'], m.meta['site_names']
    joints = [j for j in m.meta['observable_joints'] if any(k in j for k in ('coxa', 'femur', 'tibia', 'tarsus'))]
    sites = [f'walker/claw_T{k}_{s}' for k in (1, 2, 3) for s in ('left', 'right')] + ['walker/head']
    jid = [jn.index(j) for j in joints]
    qadr, vadr, sid = m.jnt_qposadr[jid], m.jnt_dofadr[jid], [sn.index(s) for s in sites]
    rec = {k: np.zeros((T, n_traj) + shp) for k, shp in (('root_qpos', (7,)), ('qpos', (len(jid),)), ('root_qvel', (6,)),
                                                         ('qvel', (len(jid),)), ('root2site', (len(sid), 3)))}
    env.reset()
    for t in range(T):
        if t:
            env.step(rs.uniform(-0.1, 0.1, (n_traj, 59)).astype(np.float32))
        q, v = sim.get(st.QPOS).astype(np.float64), sim.get(st.QVEL).astype(np.float64)
        sx = sim.get(st.SITE_XPOS).astype(np.float64).reshape(n_traj, -1, 3)[:, sid]
        rq = q[:, env._root_q:env._root_q + 7]
        rec['root_qpos'][t], rec['qpos'][t] = rq, q[:, qadr]
        rec['root_qvel'][t], rec['qvel'][t] = v[:, env._root_v:env._root_v + 6], v[:, vadr]
        rec['root2site'][t] = rotate_vec_with_quat(sx - rq[:, None, :3], reciprocal_quat(rq[:, None, 3:7]))
    env.close()
    d = {'timestep_seconds': np.float64(0.002), 'trajectory_lengths': lens.astype(np.int64),
         'id2name/joints': np.array([j.split('/')[-1] for j in joints]), 'id2name/sites': np.array([s.split('/')[-1] for s in sites])}
    key = lambda k: f'trajectories/{str(k).zfill(len(str(n_traj)))}/'      # the loader's zero-padded group names
    for k, L in enumerate(lens):
        for name, a in rec.items():
            d[key(k) + name] = a[:L, k]
        d[key(k) + 'joint_quat'] = np.tile([1.0, 0, 0, 0], (L, len(jid), 1))
    np.savez(path, **d)
    return T


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
    ap.add_argument('--repeats', type=int, default=2)
    ap.add_argument('--profile-steps', type=int, default=50)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit('no CUDA device: this script measures the GPU')
    rs = np.random.RandomState(0)
    tmp = tempfile.mkdtemp(prefix='walk_ds_')
    path = os.path.join(tmp, 'walk.npz')
    try:
        longest = record_dataset(path, a.traj, rs)
        run(a, path, longest, rs)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


def run(a, path, longest, rs):
    import torch
    N = a.envs
    K = a.window or (longest - FUT - 1)                                 # future_steps + 1 = 65 rows are never an episode step
    acts = rs.uniform(-0.1, 0.1, (64, N, 59)).astype(np.float32)        # a cycle of actions: the rate does not depend on them
    make = lambda dev: fly_envs.walk_imitation(ref_path=path, n_envs=N, seed=1, device_task=dev, random_state=np.random.RandomState(2))
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
        print(f'{name:22s} N={N} {1e3 * dt / K:8.3f} ms/step {N * K / dt:12.0f} env-steps/s  resets in window {res[name]["resets_in_window"]}',
              flush=True)
        env.close()
    tacts = torch.from_numpy(acts).cuda()
    arms = (('step_device', lambda: make(True)), ('inference_step_device', lambda: fly_envs.walk_imitation(n_envs=N, seed=1, device_task=True)))
    for rep in range(a.repeats):
        for name, new in arms:
            env = new()
            stream = torch.cuda.ExternalStream(env.physics.stepper.stream)
            with torch.cuda.stream(stream):
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
            r = {'env_steps_per_s': N * K / dt, 'ms_per_step': 1e3 * dt / K, 'resets_in_window': int(env._sim.task_episodes().sum()) - ep0,
                 'finite_outputs': ok}
            res.setdefault(name, []).append(r)
            print(f'{name:22s} N={N} {1e3 * dt / K:8.3f} ms/step {N * K / dt:12.0f} env-steps/s  resets in window {r["resets_in_window"]}  '
                  f'finite {ok}  (run {rep + 1})', flush=True)
            env.close()
    for name, new in arms:                  # profiled pass of its own: per kernel kind, ms per control step
        env = new()
        stream = torch.cuda.ExternalStream(env.physics.stepper.stream)
        with torch.cuda.stream(stream):
            for k in range(a.warmup):
                env.step_device(tacts[k % 64])
            stream.synchronize()
            env._sim.profile(True)
            for k in range(a.profile_steps):
                env.step_device(tacts[k % 64])
            stream.synchronize()
            prof = env._sim.profile_read()
            env._sim.profile(False)
        res[name + '_profile_ms_per_step'] = {k: ms / a.profile_steps for k, (ms, n) in prof.items() if n}
        print(f'{name:22s} profile, ms per control step: ' + '  '.join(f'{k} {v:.3f}' for k, v in res[name + '_profile_ms_per_step'].items()),
              flush=True)
        env.close()
    print(f'card: {res["gpu"]}  power limit: {res["power_limit_w"]} W  window: {K} control steps after {a.warmup} warm-up steps', flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
