"""H100 measurement of the batched rollouts (fb_rollout): the rollout against the hand-written host loop it replaces, the recording
cost against a plain fb_step loop, and feedback on against off.  Each pair is timed alternating, host clock around work that ends in a
device synchronise, after one warm-up of every shape.  Prints one JSON line (and writes it to --out when given).

    python tools/gpu_rollout.py [--repeats 3] [--out FILE.json]
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

from flybody_b200 import stepper as st  # noqa: E402
from flybody_b200.flymodel import load_model  # noqa: E402


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else 'unknown'


def setup(variant, n_envs, n, T, feedback=False, seed=0):
    m = load_model(variant)
    sim = st.BatchedStepper(m, n_envs)
    rs = np.random.RandomState(seed)
    q = np.repeat(m.qpos0[None], n_envs, 0)
    if m.nu != 59:
        q[:, int(m.jnt_qposadr[0]) + 2] += 2.0                      # flight: in the air
    sim.reset(q, rs.uniform(-0.1, 0.1, (n_envs, m.nv)))
    sim.forward()
    sim.state_bank(n_envs)
    sim.save_state()
    u = rs.uniform(-0.3, 0.3, (n, T, m.nu)).astype(np.float32)
    if feedback:
        nx = 2 * m.nv + m.na
        xref = np.concatenate([np.repeat(sim.get(st.QPOS)[:1], T, 0), np.zeros((T, m.nv + m.na), np.float32)], 1)
        sim.rollout_feedback(xref, (rs.uniform(-1, 1, (T, m.nu, nx)) * 1e-3).astype(np.float32))
    return m, sim, u


def rollout(sim, u, nsub):
    sim.rollout(np.arange(len(u)), u, nsub)
    return sim.rollout_read()


def host_loop(sim, u, nsub):
    """load, then per step set_control, step and the reads a hand-written loop makes"""
    n, T = u.shape[:2]
    pad = np.minimum(np.arange(sim.n_envs), n - 1)
    sim.load_state(slots=np.arange(n), env_ids=np.arange(n))
    for t in range(T):
        sim.set_control(u[pad, t])
        sim.step(nsub)
        for f in (st.QPOS, st.QVEL, st.ACT, st.CTRL, st.TIME, st.FLAGS):
            sim.get(f)


def step_loop(sim, u, nsub):
    """the same control steps without inputs or records: load, T x fb_step, synchronise"""
    sim.load_state(slots=np.arange(len(u)), env_ids=np.arange(len(u)))
    for _ in range(u.shape[1]):
        sim.step(nsub)
    sim.sync()


def timed(fn):
    t0 = time.perf_counter()
    fn()
    return time.perf_counter() - t0


def alternate(fns, repeats):
    """{name: [seconds per repeat]}: one warm-up each, then the functions in turn"""
    for fn in fns.values():
        fn()
    out = {k: [] for k in fns}
    for _ in range(repeats):
        for k, fn in fns.items():
            out[k].append(timed(fn))
    return out


def summary(times, n, T):
    return {k: {'s': [round(x, 4) for x in v], 'rollout_steps_per_s': round(n * T / min(v))} for k, v in times.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--repeats', type=int, default=3)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    res = {'card': card()}
    for name, variant, n_envs, n, T, nsub in (('walk_4096_T50', 'walk', 4096, 4096, 50, 10), ('flight_4096_T200', 'flight', 4096, 4096, 200, 4),
                                              ('flight_256_T50', 'flight', 256, 256, 50, 4)):
        m, sim, u = setup(variant, n_envs, n, T)
        times = alternate({'rollout': lambda: rollout(sim, u, nsub), 'host_loop': lambda: host_loop(sim, u, nsub),
                           'step_loop': lambda: step_loop(sim, u, nsub)}, a.repeats)
        sim.close()
        m, fsim, u = setup(variant, n_envs, n, T, feedback=True)
        _, osim, _ = setup(variant, n_envs, n, T)
        times.update(alternate({'feedback_on': lambda: rollout(fsim, u, nsub), 'feedback_off': lambda: rollout(osim, u, nsub)}, a.repeats))
        fsim.close()
        osim.close()
        res[name] = summary(times, n, T)
        print(name, json.dumps(res[name]), flush=True)
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
