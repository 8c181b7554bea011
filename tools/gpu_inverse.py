"""Cost of the batched inverse dynamics (fb_inverse) on walking states with ground contacts, against a control step in the same call.

    python tools/gpu_inverse.py [--envs 4096] [--rollout 50] [--reps 20] [--repeats 3] [--out FILE.json]

The states come from a `walk_imitation(device_task=True)` rollout of --rollout control steps with random actions.  The inverse is run
on each env's own FB_QACC, handed over as a device pointer (is_device = 1) and as a host array.  Every operation is warmed up, then
timed with CUDA events on the stepper's stream over --reps back-to-back calls, --repeats times: fb_inverse (the position / velocity
stage plus the inverse kernel), fb_forward (the same stage plus the forward solve) and one control step (`step_device`).  Prints the
card and its power limit beside the numbers; --out also writes them as JSON."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from flybody_b200 import fly_envs, stepper as st   # noqa: E402


def card():
    try:
        return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True,
                              timeout=30).stdout.strip()
    except Exception as exc:                       # the numbers below are still device-timed
        return f'unknown ({exc})'


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--envs', type=int, default=4096)
    ap.add_argument('--rollout', type=int, default=50)
    ap.add_argument('--reps', type=int, default=20)
    ap.add_argument('--repeats', type=int, default=3)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit('no CUDA device: this script measures on the GPU only')
    n = a.envs
    rs = np.random.RandomState(0)
    env = fly_envs.walk_imitation(terminal_com_dist=float('inf'), n_envs=n, device_task=True, seed=1)
    env.reset()
    actions = [torch.from_numpy(rs.uniform(-0.3, 0.3, (n, 59)).astype(np.float32)).cuda() for _ in range(16)]
    for k in range(a.rollout):
        env.step_device(actions[k % len(actions)])
    sim = env._sim
    stream = torch.cuda.ExternalStream(sim.stream)
    qacc_host = np.ascontiguousarray(sim.get(st.QACC))
    qacc_dev = torch.from_numpy(qacc_host).cuda()
    torch.cuda.synchronize()
    ncon, nefc = sim.get(st.NCON)[:, 0], sim.get(st.NEFC)[:, 0]
    k = [0]

    def step():
        env.step_device(actions[k[0] % len(actions)])
        k[0] += 1
    ops = {'fb_inverse (device qacc)': lambda: sim.inverse(qacc_dev.data_ptr(), n=n, is_device=True),
           'fb_inverse (host qacc)': lambda: sim.inverse(qacc_host),
           'fb_forward': lambda: sim.forward(),
           'control step (step_device)': step}

    def timed(fn, reps):
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record(stream)
        for _ in range(reps):
            fn()
        t1.record(stream)
        t1.synchronize()
        return t0.elapsed_time(t1) / reps
    res = {name: [] for name in ops}
    for name, fn in ops.items():
        timed(fn, 2)                               # warm-up
    for _ in range(a.repeats):
        for name, fn in ops.items():
            res[name].append(timed(fn, a.reps))
    info = dict(card=card(), envs=n, reps=a.reps, rollout=a.rollout, contacts_per_env=float(ncon.mean()), rows_per_env=float(nefc.mean()),
                envs_over_32_rows=float((nefc > 32).mean()), ms=res,
                inverse_problems_per_s=[n / (t / 1e3) for t in res['fb_inverse (device qacc)']])
    env.close()
    print(json.dumps(info, indent=1))
    if a.out:
        with open(a.out, 'w') as f:
            json.dump(info, f, indent=1)


if __name__ == '__main__':
    main()
