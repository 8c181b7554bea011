"""H100 measurement of batched iLQR (flybody_b200.trajopt): the time per iteration split into the finite-difference sweep, the backward
pass, the forward pass and the host work (row writes, reads and the fp64 cost) -- the solve's seconds in each phase over its accepted
iterations, the initial rollout and the final gains' pass included -- and the backward-pass kernels alone (device time from
CUDA events around each launch, fb_profile) against a numpy fp64 backward pass (tests/lqr_reference.py) on the same inputs.  The
references are rollouts of seeded controls, the initial guess zero.  Prints the card's name and power limit with the results as one
JSON line (and writes it to --out when given).

    python tools/gpu_ilqr.py [--iters 3] [--out FILE.json]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))

import lqr_reference as lr  # noqa: E402
from flybody_b200 import rollout as ro, stepper as st, trajopt as tj  # noqa: E402
from flybody_b200.flymodel import load_model  # noqa: E402
from gpu_rollout import card  # noqa: E402

CASES = (('walk', 'walk', 4, 25, 10), ('flight', 'flight', 16, 50, 4))


def problem(m, L, T, nsub, seed=0):
    rs = np.random.RandomState(seed)
    q = np.repeat(m.qpos0[None], L, 0)
    if m.nu != 59:
        q[:, int(m.jnt_qposadr[0]) + 2] += 2.0                      # flight: in the air
    v = rs.uniform(-0.1, 0.1, (L, m.nv))
    ref = ro.rollout(m, q, v, rs.uniform(-0.3, 0.3, (L, T, m.nu)), n_substeps=nsub)
    x0 = np.concatenate([q, v, np.zeros((L, m.na))], -1)
    x_ref = np.concatenate([x0[:, None], np.concatenate([ref.qpos, ref.qvel, ref.act], -1)], 1)
    Q = np.concatenate([np.ones(m.nv), np.full(m.nv, 1e-2), np.ones(m.na)])
    return q, v, x_ref, Q, 1e-3 * np.ones(m.nu)


def backward_alone(m, L, T, repeats=3):
    """device time of the backward-pass kernels against the numpy fp64 pass, on one seeded set of inputs of the case's sizes"""
    nx, nu = 2 * m.nv + m.na, m.nu
    rs = np.random.RandomState(1)
    A = (np.eye(nx) + 0.01 * rs.randn(L, T, nx, nx)).astype(np.float32)
    B = (0.1 * rs.randn(L, T, nx, nu)).astype(np.float32)
    q, r = rs.randn(L, T + 1, nx), rs.randn(L, T, nu)
    Q, R = np.ones(nx), np.ones(nu)
    sim = st.BatchedStepper(m, 1)
    sim.lqr(A, B, q, r, Q, R, Q, np.zeros(L))                       # warm-up
    ms = []
    for _ in range(repeats):
        sim.profile(True)
        before = sim.profile_read()['misc'][0]
        sim.lqr(A, B, q, r, Q, R, Q, np.zeros(L))
        ms.append(sim.profile_read()['misc'][0] - before)
        sim.profile(False)
    K = sim.lqr_read()[0]
    sim.close()
    t0 = time.perf_counter()
    Kr = [lr.backward(A[l], B[l], q[l], r[l], Q, R, Q, 0.0)[0] for l in range(L)]
    host_s = time.perf_counter() - t0
    err = max(np.abs(K[l] - Kr[l]).max() / np.abs(Kr[l]).max() for l in range(L))
    return {'kernels_ms': [round(x, 3) for x in ms], 'numpy_fp64_ms': round(1e3 * host_s, 1), 'K_rel_err': float(err)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=3)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    res = {'card': card()}
    for name, variant, L, T, nsub in CASES:
        m = load_model(variant)
        q, v, x_ref, Q, R = problem(m, L, T, nsub)
        tj.ilqr(m, q, v, np.zeros((L, T, m.nu)), x_ref, Q, R, n_substeps=nsub, max_iter=1)      # warm-up
        tim = {}
        t0 = time.perf_counter()
        out = tj.ilqr(m, q, v, np.zeros((L, T, m.nu)), x_ref, Q, R, n_substeps=nsub, max_iter=a.iters, timings=tim)
        total = time.perf_counter() - t0
        it = max(1, int(out.iterations.max()))
        res[name] = {'L': L, 'T': T, 'n_substeps': nsub, 'iterations': out.iterations.tolist(), 'total_s': round(total, 3),
                     'per_iteration_s': {k: round(v / it, 4) for k, v in tim.items()},
                     'cost_first_last': [[float(c[0]), float(c[i])] for c, i in zip(out.cost, out.iterations)],
                     'backward_alone': backward_alone(m, L, T)}
        print(name, json.dumps(res[name]), flush=True)
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
