"""H100 measurement of sampling-based MPC (fb_plan, flybody_b200.trajopt.sample_plan / mpc) at 4096 samples per call: seconds per
iteration (MPPI; sampling, rollouts, cost and update in one call), the device time of its kernels by fb_profile kind (the step graph's
stages against 'misc': the plan kernels, the rollout input kernel and the row loads), a plain fb_rollout of the same size, the
host-scored alternative (fb_rollout, rollout_read, numpy trajopt.cost of every sample) with the relative difference between its costs
and the device's, and the time per control step of a receding-horizon run, its set-up excluded.  Prints the card's name and power limit
with the results as one JSON line (and writes it to --out when given).

    python tools/gpu_plan.py [--iters 3] [--out FILE.json]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

from flybody_b200 import stepper as st, trajopt as tj  # noqa: E402
from flybody_b200.flymodel import load_model  # noqa: E402
from gpu_ilqr import problem  # noqa: E402
from gpu_rollout import card  # noqa: E402

CASES = (('walk', 'walk', 4, 1024, 25, 10), ('flight', 'flight', 16, 256, 50, 4))


def timed(fn):
    t0 = time.perf_counter()
    out = fn()
    return time.perf_counter() - t0, out


def profiled(sim, fn):
    sim.profile(True)
    before = sim.profile_read()
    fn()
    after = sim.profile_read()
    sim.profile(False)
    return {k: round(after[k][0] - before[k][0], 3) for k in after if after[k][1] > before[k][1]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=3)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    res = {'card': card()}
    for name, variant, L, K, T, nsub in CASES:
        m = load_model(variant)
        q, v, x_ref, Q, R = problem(m, L, T, nsub)
        sim = st.BatchedStepper(m, L * K)
        sim.state_bank(L)
        x0 = np.concatenate([q, v, np.zeros((L, m.na))], -1).astype(np.float32)
        tj._write_rows(sim, m, 0, x0, np.zeros((L, m.nu), np.float32))
        sim.plan_program(K, np.full(m.nu, 0.1, np.float32), Q, R, Q, 1.0, 1)
        slots, mean, seeds = np.arange(L), np.zeros((L, T, m.nu), np.float32), np.arange(L)
        plan = lambda n_iter: sim.plan(slots, mean, x_ref, seeds, None, nsub, n_iter)      # noqa: E731
        plan(1)                                                                           # warm-up
        sec, _ = timed(lambda: plan(a.iters))
        plan(1)
        _, cost, sc, smp, _ = sim.plan_read()
        prof_plan = profiled(sim, lambda: plan(1))
        ctrl = smp.reshape(L * K, T, m.nu)
        roll_slots = np.repeat(slots, K)
        sim.rollout(roll_slots, ctrl, nsub)                                               # warm-up
        roll_s, _ = timed(lambda: sim.rollout(roll_slots, ctrl, nsub))
        prof_roll = profiled(sim, lambda: sim.rollout(roll_slots, ctrl, nsub))
        # the host-scored alternative on the same samples
        t0 = time.perf_counter()
        sim.rollout(roll_slots, ctrl, nsub)
        t1 = time.perf_counter()
        qp, qv, ac = sim.rollout_read()[:3]
        t2 = time.perf_counter()
        xs = np.concatenate([np.repeat(x0[:, None], K, 0).reshape(L * K, 1, -1), np.concatenate([qp, qv, ac], -1)], 1)
        J = np.array([tj.cost(m, xs[i], ctrl[i], x_ref[i // K], 0, Q, R, Q) for i in range(L * K)]).reshape(L, K)
        t3 = time.perf_counter()
        sim.close()
        fin = np.isfinite(J) & np.isfinite(sc)

        # one MPC run's control steps: a run of 6 steps less a run of 1, over 5, so the handle's set-up and the first step drop out
        def mpc(n_steps):
            xr = np.concatenate([x_ref, np.repeat(x_ref[:, -1:], n_steps - 1, 1)], 1)
            return timed(lambda: tj.mpc(m, q, v, xr, n_steps, T, Q, R, n_samples=K, sigma=0.1, temperature=1.0, n_iter=1,
                                        n_substeps=nsub))[0]
        mpc_runs = [mpc(1), mpc(6)]
        mpc_s = mpc_runs[1] - mpc_runs[0]
        res[name] = {'L': L, 'n_samples': K, 'T': T, 'n_substeps': nsub,
                     'plan_s_per_iteration': round(sec / a.iters, 4),
                     'plan_profile_ms': prof_plan, 'rollout_s': round(roll_s, 4), 'rollout_profile_ms': prof_roll,
                     'host_scored_s': {'rollout': round(t1 - t0, 4), 'read': round(t2 - t1, 4), 'numpy_cost': round(t3 - t2, 4)},
                     'host_vs_device_cost_rel': float((np.abs(J - sc) / np.abs(J))[fin].max()),
                     'mpc_s_per_control_step': round(mpc_s / 5, 4), 'mpc_run_s_1_and_6_steps': [round(x, 3) for x in mpc_runs],
                     'cost_first_iteration': [float(cost[l, 0, 0]) for l in range(L)]}
        print(name, json.dumps(res[name]), flush=True)
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
