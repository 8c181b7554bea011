"""Throughput and accuracy of the batched finite-difference transition Jacobians (fb_fd_transition, flybody_b200.derivatives).

    python tools/gpu_fd.py [--reps 20] [--repeats 3] [--out FILE.json]

1. Jacobians/s of the template (walking, 4096 // 669 or 4096 // 335 problems per call) and flight (4096 // 215, 4096 // 108) models,
   centred and forward, at n_substeps 1 and 10, on full-size handles (derivatives.ENVS envs): --reps back-to-back fd_transition calls
   (each ends in a device synchronise) timed on the host, --repeats times, after a warm-up call of every configuration.
2. The per-launch split of one call of each configuration from fb_profile events (the step kinds; "misc" = the fan-out (one
   state-copy launch), perturbation and differencing kernels).
3. An eps sweep: the device's centred A / B at eps 3e-1 ... 1e-4 against the fp64 reference (tests/fd_reference.py) at eps 1e-6, on 9
   constraint-free flight states (tests/smooth_states.py, without the two far from the origin) and 8 template states with ground contacts
   taken from a rollout.  Per state the per-column errors of tests/test_transition_fd.py; reported: the median and max over the states
   of the worst column, and the median over the states of the median column.
4. The fp64 reference's time per Jacobian on one CPU core of the same machine (the oracle restatement, not MuJoCo).
Prints the card and its power limit beside the numbers; --out also writes them as JSON."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
from flybody_b200 import derivatives as dv, stepper as st   # noqa: E402
from flybody_b200.flymodel import load_model   # noqa: E402
import fd_reference as fr   # noqa: E402
import smooth_states as ss   # noqa: E402
from test_transition_fd import col_errors   # noqa: E402


def card():
    try:
        return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True,
                              timeout=30).stdout.strip()
    except Exception as exc:                       # the numbers below are still device-timed
        return f'unknown ({exc})'


def flight_states(n):
    """constraint-free flight states of tests/smooth_states.py, without the two far from the origin (root 1e2 / 1e3 cm away): there
    the fp64 reference's own rounding grows as 1 / eps in the rotational columns (far_1e3, A[nv + 3, 5]: -0.12, -1.0, 26 at eps 1e-5,
    1e-6, 1e-7, against -4e-5 at every eps for quat_a), so it has no eps -> 0 limit to compare to"""
    m = ss.free_model(load_model('flight'))
    xs = [ss.state_inputs(m, k) for k in ss.state_names(m) if not k.startswith('far')][:n]
    return m, [np.array([x[c] for x in xs]) for c in range(4)]


def template_states(n, steps=40, seed=0):
    """n envs of a template rollout from qpos0 with random ctrl: (q, v, act, ctrl) with ground contacts"""
    m = load_model('template')
    sim = st.BatchedStepper(m, n)
    sim.reset(m.qpos0)
    rs = np.random.RandomState(seed)
    for _ in range(steps):
        sim.set_control(rs.uniform(-0.3, 0.3, (n, m.nu)))
        sim.step(10)
    x = [sim.get(f).astype(np.float64) for f in (st.QPOS, st.QVEL, st.ACT, st.CTRL)]
    ncon = sim.get(st.NCON)[:, 0]
    sim.close()
    return m, x, float(ncon.mean())


def handle(m, x, centered):
    """a full-size handle with its bank holding states x (repeated to fill the problems of one call) -> (sim, slots)"""
    ncol = 1 + (2 if centered else 1) * (2 * m.nv + m.na + m.nu)
    per = max(1, dv.ENVS // ncol)
    sim = st.BatchedStepper(m, per * ncol)
    q, v, a, u = x
    rows = np.arange(sim.n_envs) % len(q)
    sim.reset(q[rows], v[rows])
    if m.na:
        sim.set(st.ACT, a[rows])
    sim.set_control(u[rows])
    sim.forward()
    sim.state_bank(per)
    sim.save_state(slots=np.arange(per), env_ids=np.arange(per))
    return sim, np.arange(per)


def throughput(m, x, reps, repeats):
    out = {}
    for centered in (True, False):
        sim, slots = handle(m, x, centered)
        for nsub in (1, 10):
            key = f"{'centred' if centered else 'forward'} n_substeps={nsub}"
            sim.fd_transition(slots, centered=centered, n_substeps=nsub)        # warm-up (and graph capture on the second call)
            sim.fd_transition(slots, centered=centered, n_substeps=nsub)
            rates = []
            for _ in range(repeats):
                t0 = time.perf_counter()
                for _ in range(reps):
                    sim.fd_transition(slots, centered=centered, n_substeps=nsub)
                dt = (time.perf_counter() - t0) / reps
                rates.append(len(slots) / dt)
            sim.profile(True)
            t0 = time.perf_counter()
            sim.fd_transition(slots, centered=centered, n_substeps=nsub)
            call_ms = (time.perf_counter() - t0) * 1e3
            split = {k: round(v[0], 4) for k, v in sim.profile_read().items() if v[1]}
            sim.profile(False)
            out[key] = dict(envs=sim.n_envs, problems=len(slots), jacobians_per_s=[round(r, 1) for r in rates],
                            ms_per_call=[round(len(slots) / r * 1e3, 3) for r in rates], profiled_call_ms=round(call_ms, 3), event_ms=split)
        sim.close()
    return out


def sweep(m, x, epss):
    q, v, a, u = x
    refs = [fr.transition_fd(m, q[p], v[p], a[p], u[p], eps=1e-6)[:2] for p in range(len(q))]
    out = {}
    for eps in epss:
        r = dv.transition_fd(m, q, v, u, a, eps=eps)
        cols = [np.concatenate([col_errors(r.A[p], A), col_errors(r.B[p], B)]) for p, (A, B) in enumerate(refs)]
        worst = [c.max() for c in cols]
        out[f'{eps:g}'] = dict(worst_median=float(np.median(worst)), worst_max=float(np.max(worst)),
                               column_median=float(np.median([np.median(c) for c in cols])))
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
    info = dict(card=card(), template_contacts_per_state=ncon)
    info['throughput'] = {'template': throughput(mt, xt, a.reps, a.repeats), 'flight': throughput(mf, xf, a.reps, a.repeats)}
    epss = (3e-1, 1e-1, 3e-2, 1e-2, 3e-3, 1e-3, 3e-4, 1e-4)
    info['eps_sweep'] = {'flight (constraint-free)': sweep(mf, xf, epss), 'template (contacts)': sweep(mt, xt, epss)}
    t0 = time.perf_counter()
    fr.transition_fd(mt, *[c[0] for c in xt])
    info['fp64 reference (oracle restatement, not MuJoCo), one CPU core, s per centred template Jacobian'] = round(time.perf_counter() - t0, 3)
    print(json.dumps(info, indent=1))
    if a.out:
        with open(a.out, 'w') as f:
            json.dump(info, f, indent=1)


if __name__ == '__main__':
    main()
