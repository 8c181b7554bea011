"""walk_on_ball at 4096 envs through step_device for one whole episode (1000 control steps) after warm-up, alternated with
template_task in the same process: env-steps/s, contacts and constraint rows per env-step, and the share of envs on the generic solver
(nefc > 32).  Prints one JSON line per arm and repetition; --out FILE also writes them to FILE as a JSON list.

    python tools/gpu_walk_on_ball.py [--envs 4096] [--steps 1000] [--warmup 50] [--reps 2] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True)
    return out.stdout.strip()


def run_arm(name, n, steps, warmup):
    import torch
    from flybody_b200 import fly_envs, stepper as st
    env = fly_envs.walk_on_ball(n_envs=n, device_task=True, seed=1) if name == 'walk_on_ball' else \
        fly_envs.template_task(n_envs=n, device_task=True, seed=1, time_limit=2.0)
    env.reset()
    na = env.action_spec().shape[0]
    g = torch.Generator(device='cuda').manual_seed(0)
    acts = [torch.rand((n, na), device='cuda', generator=g) * 2 - 1 for _ in range(8)]
    stream = torch.cuda.ExternalStream(env._sim.stream)
    with torch.cuda.stream(stream):
        for k in range(warmup):
            env.step_device(acts[k % 8])
        stream.synchronize()
        t0 = time.perf_counter()
        for k in range(steps):
            env.step_device(acts[k % 8])
        stream.synchronize()
        dt = time.perf_counter() - t0
    # contact / row statistics over a separate stretch of the same rollout (reads synchronise)
    ncon, nefc = [], []
    with torch.cuda.stream(stream):
        for k in range(20):
            env.step_device(acts[k % 8])
            stream.synchronize()
            ncon.append(env._sim.get(st.NCON)[:, 0].copy())
            nefc.append(env._sim.get(st.NEFC)[:, 0].copy())
    ncon, nefc = np.array(ncon), np.array(nefc)
    env.close()
    return dict(arm=name, envs=n, steps=steps, env_steps_per_s=n * steps / dt, ms_per_control_step=1e3 * dt / steps,
                contacts_per_env_step=float(ncon.mean()), rows_per_env_step=float(nefc.mean()),
                generic_solver_share=float((nefc > 32).mean()))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--envs', type=int, default=4096)
    ap.add_argument('--steps', type=int, default=1000)
    ap.add_argument('--warmup', type=int, default=50)
    ap.add_argument('--reps', type=int, default=2)
    ap.add_argument('--out', default=None, help='also write the rows to this JSON file')
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit('no CUDA device: this tool measures on the GPU only')
    import __graft_entry__ as ge
    ge.build()
    rows = []
    gpu = card()
    for r in range(a.reps):
        for name in ('walk_on_ball', 'template_task'):
            row = run_arm(name, a.envs, a.steps, a.warmup)
            row.update(rep=r, gpu=gpu)
            print(json.dumps(row), flush=True)
            rows.append(row)
    if a.out:
        with open(a.out, 'w') as f:
            json.dump(rows, f, indent=1)


if __name__ == '__main__':
    main()
