"""Throughput and accuracy of the batched finite-difference inverse-dynamics Jacobians (fb_fd_inverse, derivatives.inverse_fd).

    python tools/gpu_inverse_fd.py [--reps 20] [--repeats 3] [--out FILE.json]

1. Jacobians/s of the template (walking, 4096 // 649 or 4096 // 325 problems per call) and flight (4096 // 289, 4096 // 145) models,
   centred and forward, on full-size handles (derivatives.ENVS envs): --reps back-to-back fd_inverse calls with host inputs (each
   ends in a device synchronise) timed on the host, --repeats times, after a warm-up call of every configuration.
2. The per-launch split of one call of each configuration from fb_profile events (the step kinds of the position / velocity stage;
   "misc" = the fan-out / nudge, inverse and differencing kernels).
3. An eps sweep: the device's centred Jacobians at eps 3e-1 ... 1e-4 against the fp64 reference (tests/inverse_fd_reference.py) at
   eps 1e-6, on 9 constraint-free flight states (tests/smooth_states.py, without the two far from the origin) and 8 states with ground
   contacts from a rollout of the analytic-contact template model (tests/solver_states.py).  Per state the per-row errors of
   tests/test_inverse_fd.py over DfDq, DfDv, DfDa and DmDq; reported: the median and max over the states of the worst row, and the
   median over the states of the median row.
4. The fp64 reference's time per Jacobian on one CPU core of the same machine (the oracle restatement, not MuJoCo).
Prints the card and its power limit beside the numbers; --out also writes them as JSON."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
from flybody_b200 import derivatives as dv, stepper as st   # noqa: E402
from flybody_b200.flymodel import load_model   # noqa: E402
import inverse_fd_reference as ifr   # noqa: E402
import smooth_states as ss   # noqa: E402
import solver_states as sv   # noqa: E402
from gpu_fd import card   # noqa: E402
from test_inverse_fd import OUTS, errors, device, free_cases   # noqa: E402


def flight_states(n):
    """constraint-free flight states without the two far from the origin (tools/gpu_fd.py: the fp64 reference has no eps -> 0 limit
    there), with the oracle's forward qacc"""
    m = ss.free_model(load_model('flight'))
    names = [k for k in ss.state_names(m) if not k.startswith('far')][:n]
    cases = free_cases(m, names, ifr.Inverse(m))
    return m, [np.array([c[i] for c in cases]) for i in range(3)]


def template_states(n, steps=40, seed=0):
    """n envs of a rollout of the analytic-contact template model from qpos0 with random ctrl: (q, v, qacc) with ground contacts"""
    m = sv.analytic_model(load_model('template'))
    sim = st.BatchedStepper(m, n)
    sim.reset(m.qpos0)
    rs = np.random.RandomState(seed)
    for _ in range(steps):
        sim.set_control(rs.uniform(-0.3, 0.3, (n, m.nu)))
        sim.step(10)
    x = [sim.get(f).astype(np.float64) for f in (st.QPOS, st.QVEL, st.QACC)]
    ncon = sim.get(st.NCON)[:, 0]
    sim.close()
    return m, x, float(ncon.mean())


def throughput(m, x, reps, repeats):
    out = {}
    q, v, a = x
    for centered in (True, False):
        ncol = 1 + (2 if centered else 1) * 3 * m.nv
        per = max(1, dv.ENVS // ncol)
        rows = np.arange(per) % len(q)
        sim = st.BatchedStepper(m, per * ncol)
        key = 'centred' if centered else 'forward'
        call = lambda: sim.fd_inverse(q[rows], v[rows], a[rows], centered=centered)   # noqa: E731
        call()
        call()
        rates = []
        for _ in range(repeats):
            t0 = time.perf_counter()
            for _ in range(reps):
                call()
            dt = (time.perf_counter() - t0) / reps
            rates.append(per / dt)
        sim.profile(True)
        t0 = time.perf_counter()
        call()
        call_ms = (time.perf_counter() - t0) * 1e3
        split = {k: round(v[0], 4) for k, v in sim.profile_read().items() if v[1]}
        sim.profile(False)
        out[key] = dict(envs=sim.n_envs, problems=per, jacobians_per_s=[round(r, 1) for r in rates],
                        ms_per_call=[round(per / r * 1e3, 3) for r in rates], profiled_call_ms=round(call_ms, 3), event_ms=split)
        sim.close()
    return out


def sweep(m, x, epss):
    q, v, a = x
    run = ifr.Inverse(m)
    refs = [ifr.inverse_fd(m, q[p], v[p], a[p], eps=1e-6, run=run) for p in range(len(q))]
    out = {}
    for eps in epss:
        r = dv.inverse_fd(m, q, v, a, eps=eps)
        rows = [np.concatenate(list(errors(device(r, p), ref).values())) for p, ref in enumerate(refs)]
        worst = [e.max() for e in rows]
        out[f'{eps:g}'] = dict(worst_median=float(np.median(worst)), worst_max=float(np.max(worst)),
                               row_median=float(np.median([np.median(e) for e in rows])))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=20)
    ap.add_argument('--repeats', type=int, default=3)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit('no CUDA device: this script measures on the GPU only')
    mf, xf = flight_states(9)
    mt, xt, ncon = template_states(8)
    info = dict(card=card(), template_contacts_per_state=ncon, outputs=list(OUTS))
    info['throughput'] = {'template': throughput(mt, xt, a.reps, a.repeats), 'flight': throughput(mf, xf, a.reps, a.repeats)}
    epss = (3e-1, 1e-1, 3e-2, 1e-2, 3e-3, 1e-3, 3e-4, 1e-4)
    info['eps_sweep'] = {'flight (constraint-free)': sweep(mf, xf, epss), 'template (contacts)': sweep(mt, xt, epss)}
    t0 = time.perf_counter()
    ifr.inverse_fd(mt, *[c[0] for c in xt])
    info['fp64 reference (oracle restatement, not MuJoCo), one CPU core, s per centred template Jacobian'] = round(time.perf_counter() - t0, 3)
    print(json.dumps(info, indent=1))
    if a.out:
        with open(a.out, 'w') as f:
            json.dump(info, f, indent=1)


if __name__ == '__main__':
    main()
