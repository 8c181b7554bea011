"""Cost of the sensor outputs of the dynamics queries (fb_query_sensors) on the H100: each query with the switch off and on, alternating,
twice each, in one call.

    python tools/gpu_sensor_fd.py [--envs 4096] [--rollout 50] [--reps 10] [--out FILE.json]

- fb_inverse on --envs walking states with ground contacts from a `walk_imitation(device_task=True)` rollout (as tools/gpu_inverse.py),
  qacc handed over as a device pointer; and on --envs flight states (`flight_imitation`);
- fb_fd_transition on a full template handle (max(1, 4096 // columns) problems), centred, at 1 and 10 substeps, and on a full flight
  handle;
- fb_fd_inverse on a full template handle and a full flight handle, centred.
Every operation is warmed up, then timed with CUDA events on the stepper's stream over --reps back-to-back calls.  Prints the card and its
power limit beside the numbers; --out also writes them as JSON."""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))
from flybody_b200 import fly_envs, stepper as st   # noqa: E402
from flybody_b200.flymodel import load_model        # noqa: E402
from gpu_inverse import card                         # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--envs', type=int, default=4096)
    ap.add_argument('--rollout', type=int, default=50)
    ap.add_argument('--reps', type=int, default=10)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit('no CUDA device: this script measures on the GPU only')
    rs = np.random.RandomState(0)
    ops, sims = {}, []

    def rollout_env(make, nu):
        env = make(n_envs=a.envs, device_task=True, seed=1)
        env.reset()
        acts = [torch.from_numpy(rs.uniform(-0.3, 0.3, (a.envs, nu)).astype(np.float32)).cuda() for _ in range(8)]
        for k in range(a.rollout):
            env.step_device(acts[k % len(acts)])
        sim = env._sim
        qacc = torch.from_numpy(np.ascontiguousarray(sim.get(st.QACC))).cuda()
        torch.cuda.synchronize()
        return env, sim, qacc

    walk, wsim, wq = rollout_env(lambda **k: fly_envs.walk_imitation(terminal_com_dist=float('inf'), **k), 59)
    ops['fb_inverse walk'] = (wsim, lambda: wsim.inverse(wq.data_ptr(), n=a.envs, is_device=True))
    fl, fsim, fq = rollout_env(lambda **k: fly_envs.flight_imitation(terminal_com_dist=float('inf'), **k), 12)
    ops['fb_inverse flight'] = (fsim, lambda: fsim.inverse(fq.data_ptr(), n=a.envs, is_device=True))
    for name in ('template', 'flight'):
        m = load_model(name)
        ncol_t, ncol_i = 1 + 2 * (2 * m.nv + m.na + m.nu), 1 + 6 * m.nv
        per_t, per_i = max(1, 4096 // ncol_t), max(1, 4096 // ncol_i)
        t = st.BatchedStepper(m, per_t * ncol_t)
        t.reset(m.qpos0)
        t.set_control(np.full(m.nu, 0.1))
        t.step(2)
        t.state_bank(per_t)
        t.save_state(slots=np.arange(per_t), env_ids=np.arange(per_t))
        q, v, qa = (t.get(f)[:per_i] for f in (st.QPOS, st.QVEL, st.QACC))
        i = st.BatchedStepper(m, per_i * ncol_i)
        for nsub in ((1, 10) if name == 'template' else (1,)):
            ops[f'fb_fd_transition {name} centred n_substeps={nsub} ({per_t} problems)'] = (
                t, lambda t=t, per_t=per_t, nsub=nsub: t.fd_transition(np.arange(per_t), centered=True, n_substeps=nsub))
        ops[f'fb_fd_inverse {name} centred ({per_i} problems)'] = (i, lambda i=i, q=q, v=v, qa=qa: i.fd_inverse(q, v, qa, centered=True))
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
    res = {name: {'off': [], 'on': []} for name in ops}
    for sim, fn in ops.values():
        for on in (False, True):
            sim.query_sensors(on)
            timed(sim, fn, 2)                        # warm-up (and the first call's buffers)
    for _ in range(2):
        for on in (False, True):
            for name, (sim, fn) in ops.items():
                sim.query_sensors(on)
                res[name]['on' if on else 'off'].append(timed(sim, fn, a.reps))
    info = dict(card=card(), envs=a.envs, reps=a.reps, rollout=a.rollout, ms=res,
                added=[f'{name}: {np.mean(r["on"]) / np.mean(r["off"]) - 1:+.1%}' for name, r in res.items()])
    for s in sims:
        s.close()
    walk.close()
    fl.close()
    print(json.dumps(info, indent=1))
    if a.out:
        with open(a.out, 'w') as f:
            json.dump(info, f, indent=1)


if __name__ == '__main__':
    main()
