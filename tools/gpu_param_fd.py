"""Throughput of the parameter Jacobians (fb_fd_param_*) on the H100, beside the state Jacobians for context, in one call.

    python tools/gpu_param_fd.py [--reps 10] [--out FILE.json]

On full template and flight handles (max(1, 4096 // columns) problems each), centred:
- fb_fd_param_transition at 1 and 10 substeps and fb_fd_param_inverse, with k = 4 scale directions (dof_damping, actuator_gainprm,
  body_mass, body_inertia) and with k = nv element directions of dof_damping;
- fb_fd_transition (1 and 10 substeps) and fb_fd_inverse.
The operations alternate, two repeats each; every one is warmed up, then timed with CUDA events on its handle's stream over --reps
back-to-back calls.  Reports ms per call and Jacobians (problems) per second, with the card and its power limit."""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))
from flybody_b200 import derivatives as dv, stepper as st   # noqa: E402
from flybody_b200.flymodel import load_model                # noqa: E402
from gpu_inverse import card                                 # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=10)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit('no CUDA device: this script measures on the GPU only')
    ops, sims = {}, []
    for name in ('template', 'flight'):
        m = load_model(name)
        programs = {'k=4 scales': [dv.Scale('dof_damping'), dv.Scale('actuator_gainprm'), dv.Scale('body_mass'), dv.Scale('body_inertia')],
                    f'k={m.nv} dof_damping elements': ['dof_damping']}
        ncol_t, ncol_i = 1 + 2 * (2 * m.nv + m.na + m.nu), 1 + 6 * m.nv
        for tag, params in programs.items():
            dirs, _ = dv._directions(m, params, None)
            ncol = 1 + 2 * len(dirs)
            per = max(1, 4096 // ncol)
            s = st.BatchedStepper(m, per * ncol)
            s.param_set('gravity', dv.compiled_params(m, 'gravity'))
            s.reset(m.qpos0)
            s.set_control(np.full(m.nu, 0.1))
            s.step(2)
            s.state_bank(per)
            s.save_state(slots=np.arange(per), env_ids=np.arange(per))
            q, v, qa = (s.get(f)[:per] for f in (st.QPOS, st.QVEL, st.QACC))
            s.fd_param_program(dirs)
            for nsub in (1, 10):
                ops[f'fb_fd_param_transition {name} {tag} n_substeps={nsub}'] = (
                    s, per, lambda s=s, per=per, nsub=nsub: s.fd_param_transition(np.arange(per), centered=True, n_substeps=nsub))
            ops[f'fb_fd_param_inverse {name} {tag}'] = (s, per, lambda s=s, q=q, v=v, qa=qa: s.fd_param_inverse(q, v, qa, centered=True))
            sims.append(s)
        per_t, per_i = max(1, 4096 // ncol_t), max(1, 4096 // ncol_i)
        t = st.BatchedStepper(m, per_t * ncol_t)
        t.reset(m.qpos0)
        t.set_control(np.full(m.nu, 0.1))
        t.step(2)
        t.state_bank(per_t)
        t.save_state(slots=np.arange(per_t), env_ids=np.arange(per_t))
        q, v, qa = (t.get(f)[:per_i] for f in (st.QPOS, st.QVEL, st.QACC))
        i = st.BatchedStepper(m, per_i * ncol_i)
        for nsub in (1, 10):
            ops[f'fb_fd_transition {name} n_substeps={nsub}'] = (
                t, per_t, lambda t=t, per_t=per_t, nsub=nsub: t.fd_transition(np.arange(per_t), centered=True, n_substeps=nsub))
        ops[f'fb_fd_inverse {name}'] = (i, per_i, lambda i=i, q=q, v=v, qa=qa: i.fd_inverse(q, v, qa, centered=True))
        sims += [t, i]

    def timed(sim, fn, reps):
        stream = torch.cuda.ExternalStream(sim.stream)
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record(stream)
        for _ in range(reps):
            fn()
        t1.record(stream)
        t1.synchronize()
        return t0.elapsed_time(t1) / reps
    for sim, _, fn in ops.values():
        timed(sim, fn, 2)                            # warm-up (and the first call's buffers)
    res = {name: [] for name in ops}
    for _ in range(2):
        for name, (sim, _, fn) in ops.items():
            res[name].append(timed(sim, fn, a.reps))
    info = dict(card=card(), reps=a.reps, ms=res,
                jacobians_per_s={name: [round(ops[name][1] / (ms * 1e-3)) for ms in r] for name, r in res.items()},
                problems={name: ops[name][1] for name in ops})
    for s in sims:
        s.close()
    print(json.dumps(info, indent=1))
    if a.out:
        with open(a.out, 'w') as f:
            json.dump(info, f, indent=1)


if __name__ == '__main__':
    main()
