"""H100 measurement of control-limited iLQR (box-DDP: fb_lqr_box, trajopt.ilqr(box=True)) against the unboxed pass, at tools/gpu_ilqr.py's
sizes (walk L = 4, T = 25; flight L = 16, T = 50):
  - the backward-pass kernels alone (device time from CUDA events around each launch, fb_profile's 'misc'), on the case's linearisation
    at the saturated nominal: fb_lqr, fb_lqr_box with infinite bounds, and fb_lqr_box with the bounds ilqr(box=True) sets there;
  - the QP's accepted Newton steps (median and maximum over problem steps), its stop reasons and the fraction of controls clamped;
  - ilqr with and without box on references that saturate many controls (rollouts of seeded controls drawn from twice each ctrl range,
    zero initial guess, so every adhesion control starts on its lower bound): seconds per accepted iteration by phase, accepted
    iterations, final / initial cost.
Prints the card's name and power limit with the results as one JSON line (and writes it to --out when given).

    python tools/gpu_box_ilqr.py [--iters 3] [--out FILE.json]
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

from flybody_b200 import derivatives as dv, rollout as ro, stepper as st, trajopt as tj  # noqa: E402
from flybody_b200.flymodel import load_model  # noqa: E402
from gpu_rollout import card  # noqa: E402

CASES = (('walk', 'walk', 4, 25, 10), ('flight', 'flight', 16, 50, 4))


def problem(m, L, T, nsub, seed=0):
    """standing (flight: 2 cm up) starts and references from seeded controls over twice each ctrl range; gpu_ilqr's weights"""
    rs = np.random.RandomState(seed)
    q = np.repeat(m.qpos0[None], L, 0)
    if m.nu != 59:
        q[:, int(m.jnt_qposadr[0]) + 2] += 2.0
    v = rs.uniform(-0.1, 0.1, (L, m.nv))
    lo, hi = (np.asarray(m.actuator_ctrlrange, np.float64).reshape(m.nu, 2)[:, i] for i in (0, 1))
    u = (lo + hi) / 2 + (hi - lo) * rs.uniform(-1, 1, (L, T, m.nu))
    ref = ro.rollout(m, q, v, u, n_substeps=nsub)
    x0 = np.concatenate([q, v, np.zeros((L, m.na))], -1)
    x_ref = np.concatenate([x0[:, None], np.concatenate([ref.qpos, ref.qvel, ref.act], -1)], 1)
    Q = np.concatenate([np.ones(m.nv), np.full(m.nv, 1e-2), np.ones(m.na)])
    return q, v, x_ref, Q, 1e-3 * np.ones(m.nu)


def backward_alone(m, q, v, x_ref, Q, R, nsub, repeats=3):
    """the backward-pass kernels at the zero guess's nominal (its Jacobians and gradients): plain, infinite bounds, ilqr's bounds"""
    L, T = x_ref.shape[0], x_ref.shape[1] - 1
    nx, nu = 2 * m.nv + m.na, m.nu
    limited = np.asarray(m.actuator_ctrllimited, bool)
    lo, hi = (np.asarray(m.actuator_ctrlrange, np.float32).reshape(nu, 2)[:, i].astype(np.float64) for i in (0, 1))
    u = np.zeros((L, T, nu))
    nom = ro.rollout(m, q, v, u, n_substeps=nsub)
    xbar = np.concatenate([x_ref[:, :1], np.concatenate([nom.qpos, nom.qvel, nom.act], -1)], 1)
    ubar = np.where(limited, np.clip(nom.ctrl, lo, hi), nom.ctrl).astype(np.float32).astype(np.float64)
    r = dv.transition_fd(m, xbar[:, :T, :m.nq].reshape(-1, m.nq), xbar[:, :T, m.nq:m.nq + m.nv].reshape(-1, m.nv), ubar.reshape(-1, nu),
                         n_substeps=nsub, centered=False)
    A, B = r.A.reshape(L, T, nx, nx), r.B.reshape(L, T, nx, nu)
    dx = np.stack([tj.tangent(m, xbar[l], x_ref[l]) for l in range(L)])
    qg = np.concatenate([dx[:, :T] * Q, dx[:, T:] * Q], 1)
    rg = ubar * R
    mu = np.full(L, 1e-6)
    bounds = {'plain': (None, None), 'box_infinite': (np.full((L, T, nu), -np.inf), np.full((L, T, nu), np.inf)),
              'box_ilqr': (np.where(limited, lo - ubar, -np.inf), np.where(limited, hi - ubar, np.inf))}
    sim = st.BatchedStepper(m, 1)
    out = {}
    for name, (lw, up) in bounds.items():
        sim.lqr(A, B, qg, rg, Q, R, Q, mu, lw, up)                   # warm-up
        ms = []
        for _ in range(repeats):
            sim.profile(True)
            before = sim.profile_read()['misc'][0]
            sim.lqr(A, B, qg, rg, Q, R, Q, mu, lw, up)
            ms.append(sim.profile_read()['misc'][0] - before)
            sim.profile(False)
        status = sim.lqr_read()[3]
        out[name] = {'kernels_ms': [round(x, 3) for x in ms], 'status': status.tolist()}
        if lw is not None:
            clamped, qp = sim.lqr_box_read()
            ok = (status == 0)[:, None]
            steps = qp[..., 0][np.broadcast_to(ok, qp.shape[:2])]
            reasons, counts = np.unique(qp[..., 1][np.broadcast_to(ok, qp.shape[:2])], return_counts=True)
            out[name].update({'qp_steps_median': float(np.median(steps)) if steps.size else None,
                              'qp_steps_max': int(steps.max()) if steps.size else None,
                              'qp_stop_reasons': {int(a): int(b) for a, b in zip(reasons, counts)},
                              'clamped_fraction': float((clamped != 0)[np.broadcast_to(ok[..., None], clamped.shape)].mean())})
    sim.close()
    return out


def solve(m, q, v, x_ref, Q, R, nsub, iters, box):
    L, T = x_ref.shape[0], x_ref.shape[1] - 1
    tim = {}
    t0 = time.perf_counter()
    out = tj.ilqr(m, q, v, np.zeros((L, T, m.nu)), x_ref, Q, R, n_substeps=nsub, max_iter=iters, box=box, timings=tim)
    total = time.perf_counter() - t0
    it = max(1, int(out.iterations.max()))
    res = {'iterations': out.iterations.tolist(), 'total_s': round(total, 3), 'per_iteration_s': {k: round(x / it, 4) for k, x in tim.items()},
           'final_over_initial': [float(c[i] / c[0]) for c, i in zip(out.cost, out.iterations)]}
    if box:
        res['final_clamped_fraction'] = float((out.clamped != 0).mean())
        res['K_zero_on_clamped'] = bool(not out.K[out.clamped != 0].any())
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=3)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    res = {'card': card()}
    for name, variant, L, T, nsub in CASES:
        m = load_model(variant)
        q, v, x_ref, Q, R = problem(m, L, T, nsub)
        tj.ilqr(m, q, v, np.zeros((L, T, m.nu)), x_ref, Q, R, n_substeps=nsub, max_iter=1, box=True)      # warm-up
        res[name] = {'L': L, 'T': T, 'n_substeps': nsub, 'backward_alone': backward_alone(m, q, v, x_ref, Q, R, nsub),
                     'ilqr': solve(m, q, v, x_ref, Q, R, nsub, a.iters, False), 'ilqr_box': solve(m, q, v, x_ref, Q, R, nsub, a.iters, True)}
        print(name, json.dumps(res[name]), flush=True)
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
