"""template_task at 4096 envs through step_device, against inference-mode walk_imitation through step_device in the same call, and
template_task with an xfrc_applied wrench on the thorax of every env (the applied-force term of the smooth kernel switched on): one too
small to change the motion, and a push of a third of the fly's weight.

    python tools/gpu_template_task.py [--envs 4096] [--window 500] [--warmup 50] [--repeats 2] [--out FILE.json]

Every arm is warmed up, then timed over a window of control steps that ends in a device synchronise; with the default window every
template env runs a whole 500-step episode, so the resets are included.  The arms run --repeats times, alternating, to show the run-to-run
spread.  Prints one line per arm (env-steps/s, ms per control step), the card and its power limit; --out also writes them as JSON."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from flybody_b200 import fly_envs   # noqa: E402


def card():
    try:
        return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True,
                              timeout=30).stdout.strip()
    except Exception as exc:                       # the numbers below are still device-timed
        return f'unknown ({exc})'


def make(arm, n):
    if arm == 'walk_imitation':
        env = fly_envs.walk_imitation(terminal_com_dist=float('inf'), n_envs=n, device_task=True, seed=1)
    else:
        env = fly_envs.template_task(n_envs=n, device_task=True, seed=1)
        if arm != 'template':
            # 'template+xfrc': a wrench on every thorax too small to change the motion (the cost of the term alone); 'template+push': a
            # third of the fly's weight sideways on every thorax (the motion, and with it the contact work, changes)
            m = env.model
            xfrc = np.zeros((m.nbody, 6))
            xfrc[m.body_id('walker/thorax')] = (1e-7, 1e-7, 1e-7, 1e-9, 1e-9, 1e-9) if arm == 'template+xfrc' else (0.3, -0.2, 0.1, 0, 0, 0)
            env.set_applied_forces(xfrc=xfrc)
    env.reset()
    return env


def run(env, actions, steps):
    import torch
    stream = torch.cuda.ExternalStream(env._sim.stream)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    with torch.cuda.stream(stream):
        for k in range(steps):
            env.step_device(actions[k % len(actions)])
        stream.synchronize()
    return time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--envs', type=int, default=4096)
    ap.add_argument('--window', type=int, default=500)
    ap.add_argument('--warmup', type=int, default=50)
    ap.add_argument('--repeats', type=int, default=2)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit('no CUDA device: this script measures on the GPU only')
    rs = np.random.RandomState(0)
    actions = [torch.from_numpy(rs.uniform(-0.5, 0.5, (a.envs, 59)).astype(np.float32)).cuda() for _ in range(16)]
    arms = ('template', 'template+xfrc', 'template+push', 'walk_imitation')
    envs = {arm: make(arm, a.envs) for arm in arms}
    for arm in arms:
        run(envs[arm], actions, a.warmup)
    res = {arm: [] for arm in arms}
    for _ in range(a.repeats):
        for arm in arms:
            dt = run(envs[arm], actions, a.window)
            res[arm].append(dict(env_steps_per_s=a.envs * a.window / dt, ms_per_step=1e3 * dt / a.window))
    info = dict(card=card(), envs=a.envs, window=a.window, arms=res)
    print('card, power limit:', info['card'])
    for arm in arms:
        print(f'{arm:>16}: ' + '  '.join(f"{r['env_steps_per_s'] / 1e3:.1f} k env-steps/s ({r['ms_per_step']:.3f} ms/step)" for r in res[arm]))
    for env in envs.values():
        env.close()
    if a.out:
        with open(a.out, 'w') as f:
            json.dump(info, f, indent=1)


if __name__ == '__main__':
    main()
