"""Cost of per-env model parameters in the step: walking (walk_imitation, inference mode) and flight (flight_imitation) at 4096 envs
through step_device, each in three variants alternated in one call: no overlay, an overlay at the compiled values (every read site on its
per-env row), and a draw program on every parameter (every reset redraws the env's row).

    python tools/gpu_model_params.py [--envs 4096] [--window 300] [--warmup 30] [--repeats 3] [--out FILE.json]

Every arm is warmed up, then timed over a window of control steps that ends in a device synchronise; the arms run --repeats times,
alternating, to show the run-to-run spread.  Also reports the resident blocks per SM of the seven step kernels with and without the overlay
(the velocity kernel has an instance of its own for the overlay), the card and its power limit."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from flybody_b200 import fly_envs, stepper as st   # noqa: E402


def card():
    try:
        return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True,
                              timeout=30).stdout.strip()
    except Exception as exc:                       # the numbers below are still device-timed
        return f'unknown ({exc})'


def make(task, variant, n):
    if task == 'walk':
        env = fly_envs.walk_imitation(terminal_com_dist=float('inf'), n_envs=n, device_task=True, seed=1)
    else:
        env = fly_envs.flight_imitation(n_envs=n, device_task=True, seed=1)
    if variant == 'overlay':
        env.set_model_params(**{k: v[0] for k, v in env.model_params().items()})
    elif variant == 'draws':
        ranges = {}
        for k, v in env.model_params().items():
            v = v[0]
            ranges[k] = (v - 0.1 * np.abs(v), v + 0.1 * np.abs(v))
        env.randomize_model_params(seed=3, **ranges)
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
    ap.add_argument('--window', type=int, default=300)
    ap.add_argument('--warmup', type=int, default=30)
    ap.add_argument('--repeats', type=int, default=3)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit('no CUDA device: this script measures on the GPU only')
    rs = np.random.RandomState(0)
    arms = [(task, v) for task in ('walk', 'flight') for v in ('none', 'overlay', 'draws')]
    envs = {arm: make(*arm, a.envs) for arm in arms}
    actions = {}
    for arm, env in envs.items():
        dim = env.action_spec().shape[-1]
        actions.setdefault((arm[0], dim), [torch.from_numpy(rs.uniform(-0.5, 0.5, (a.envs, dim)).astype(np.float32)).cuda() for _ in range(16)])
    act = {arm: actions[(arm[0], envs[arm].action_spec().shape[-1])] for arm in arms}
    blocks = {}
    for arm in arms:
        if arm[1] != 'draws':
            blocks['/'.join(arm)] = {k: v[1] for k, v in envs[arm]._sim.step_kernel_smem().items()}
        run(envs[arm], act[arm], a.warmup)
    res = {'/'.join(arm): [] for arm in arms}
    for _ in range(a.repeats):
        for arm in arms:
            dt = run(envs[arm], act[arm], a.window)
            res['/'.join(arm)].append(dict(env_steps_per_s=a.envs * a.window / dt, ms_per_step=1e3 * dt / a.window))
    info = dict(card=card(), envs=a.envs, window=a.window, arms=res, blocks_per_sm=blocks)
    print('card, power limit:', info['card'])
    for name, b in blocks.items():
        print(f'{name:>16} blocks per SM: {b}')
    for name, r in res.items():
        print(f'{name:>16}: ' + '  '.join(f"{x['env_steps_per_s'] / 1e3:.1f} k env-steps/s ({x['ms_per_step']:.3f} ms/step)" for x in r))
    for env in envs.values():
        env.close()
    if a.out:
        with open(a.out, 'w') as f:
            json.dump(info, f, indent=1)


if __name__ == '__main__':
    main()
