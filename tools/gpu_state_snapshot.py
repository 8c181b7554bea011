"""Cost of state rows at 4096 walking envs with the task on the device: saving every env, loading every env, loading 1 % of the envs and
fanning one slot out to every env, each against the control step measured in the same call; and `step_device` throughput with and
without an allocated bank.

    python tools/gpu_state_snapshot.py [--envs 4096] [--reps 50] [--window 200] [--warmup 30] [--repeats 3] [--out FILE.json]

Every operation is warmed up, then timed with CUDA events on the stepper's stream over --reps back-to-back calls; the operations and the
control step alternate --repeats times to show the spread.  The two throughput arms are separate envs stepped over --window control steps,
alternating as well.  Prints the card and its power limit beside the numbers; --out also writes them as JSON."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from flybody_b200 import fly_envs   # noqa: E402


def card():
    try:
        return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True,
                              timeout=30).stdout.strip()
    except Exception as exc:                       # the numbers below are still device-timed
        return f'unknown ({exc})'


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--envs', type=int, default=4096)
    ap.add_argument('--reps', type=int, default=50)
    ap.add_argument('--window', type=int, default=200)
    ap.add_argument('--warmup', type=int, default=30)
    ap.add_argument('--repeats', type=int, default=3)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit('no CUDA device: this script measures on the GPU only')
    n = a.envs
    rs = np.random.RandomState(0)
    actions = [torch.from_numpy(rs.uniform(-0.3, 0.3, (n, 59)).astype(np.float32)).cuda() for _ in range(16)]
    envs = {arm: fly_envs.walk_imitation(terminal_com_dist=float('inf'), n_envs=n, device_task=True, seed=1) for arm in ('bank', 'no bank')}
    for env in envs.values():
        env.reset()
    env = envs['bank']
    env.state_bank(n)
    stream = torch.cuda.ExternalStream(env._sim.stream)
    all_ids = np.arange(n)
    few = np.sort(rs.choice(n, max(n // 100, 1), replace=False))
    ops = {'save all': lambda: env.save_state(),
           'load all': lambda: env.load_state(all_ids, all_ids),
           'load 1 %': lambda: env.load_state(few, few),
           'fan one slot out to all': lambda: env.load_state(np.zeros(n, np.int64), all_ids)}
    k = [0]

    def step(e=env):
        e.step_device(actions[k[0] % len(actions)])
        k[0] += 1

    def timed(fn, reps, on):
        with torch.cuda.stream(on):
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0.record(on)
            for _ in range(reps):
                fn()
            t1.record(on)
            t1.synchronize()
        return t0.elapsed_time(t1) / reps

    for _ in range(a.warmup):
        step()
    env.save_state()
    for fn in ops.values():
        fn()
    res = {name: [] for name in list(ops) + ['control step']}
    for _ in range(a.repeats):
        for name, fn in ops.items():
            env.save_state()                       # (the fan-out left every env on slot 0's state)
            res[name].append(timed(fn, a.reps, stream))
            env.load_state(all_ids, all_ids)
            res['control step'].append(timed(step, a.reps, stream))
    thr = {arm: [] for arm in envs}
    streams = {arm: torch.cuda.ExternalStream(e._sim.stream) for arm, e in envs.items()}
    for arm, e in envs.items():
        timed(lambda: step(e), a.warmup, streams[arm])
    for _ in range(a.repeats):
        for arm, e in envs.items():
            ms = timed(lambda: step(e), a.window, streams[arm])
            thr[arm].append(dict(env_steps_per_s=n / ms * 1e3, ms_per_step=ms))
    info = dict(card=card(), envs=n, reps=a.reps, window=a.window, state_slots=env._sim.state_slots, row_bytes=4 * env._sim.state_slots,
                record_bytes=env._sim.record_bytes, ms=res, step_device=thr)
    print('card, power limit:', info['card'])
    print(f"state row: {info['state_slots']} slots = {info['row_bytes']} bytes per env ({info['row_bytes'] * n / 1e6:.1f} MB for {n} envs); "
          f"record: {info['record_bytes']} bytes per env")
    for name, v in res.items():
        print(f'{name:>24}: ' + '  '.join(f'{x:.3f} ms' for x in v))
    for arm, v in thr.items():
        print(f'{"step_device, " + arm:>24}: ' + '  '.join(f"{r['env_steps_per_s'] / 1e3:.1f} k env-steps/s ({r['ms_per_step']:.3f} ms)" for r in v))
    for e in envs.values():
        e.close()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, 'w') as f:
            json.dump(info, f, indent=1)


if __name__ == '__main__':
    main()
