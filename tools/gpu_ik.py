"""Throughput of the batched inverse kinematics (fb_ik_*) on the template model: the root and two legs fitted to 8 sites.

    python tools/gpu_ik.py [--problems 4096] [--steps 2000] [--repeats 3] [--out FILE.json]

1. Fixed work: --problems problems with progress_threshold = 0 and max_steps = --steps, so every problem runs every iteration; device
   time (CUDA events around fb_ik_solve on the stepper's stream) -> problem-iterations / s.  One warm-up solve, then --repeats timed
   solves alternating with the default-settings arm below.
2. Default settings (reg 0, lr 0.01, beta 0.99, progress_threshold 0.01, max_steps 20000) on seeded targets: problems / s and the
   distribution of `steps`.
3. The fp64 restatement of the reference's loop the tests compare against (tests/ik_reference.c, one CPU core, not MuJoCo): time per
   iteration on a few of the same problems.
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
from flybody_b200 import stepper as st   # noqa: E402
from flybody_b200.flymodel import load_model   # noqa: E402
import ik_reference as ikref   # noqa: E402
from test_inverse_kinematics import SITES, hinges, ids, problem   # noqa: E402


def card():
    try:
        return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True,
                              timeout=30).stdout.strip()
    except Exception as exc:                       # the numbers below are still device-timed
        return f'unknown ({exc})'


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--problems', type=int, default=4096)
    ap.add_argument('--steps', type=int, default=2000)
    ap.add_argument('--repeats', type=int, default=3)
    ap.add_argument('--reference-problems', type=int, default=3)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit('no CUDA device: this script measures on the GPU only')
    m = load_model('template')
    joints = ['walker/'] + hinges(m)
    sid, jid = ids(m, SITES, joints)
    n = a.problems
    base = np.stack([problem(m, 1000 + k, joints, amp=0.1)[1] for k in range(64)])
    targets = base[np.arange(n) % len(base)] + np.random.RandomState(0).normal(0, 1e-3, (n, len(SITES), 3))
    arms = {'fixed': dict(reg_strength=1e-3, progress_threshold=0.0, max_steps=a.steps),
            'default': dict(reg_strength=0.0, lr=0.01, beta=0.99, progress_threshold=0.01, max_steps=20_000)}
    sims = {k: st.BatchedStepper(m, n) for k in arms}
    for k, kw in arms.items():
        sims[k].ik_program(sid, jid, **kw)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]

    def solve(k):
        s = sims[k]
        stream = torch.cuda.ExternalStream(s.stream)
        ev[0].record(stream)
        s.ik_solve(targets, m.qpos0)
        ev[1].record(stream)
        ev[1].synchronize()
        return ev[0].elapsed_time(ev[1]) / 1e3
    res = {'card': card(), 'problems': n, 'fitted_dofs': 6 + len(joints) - 1, 'sites': len(SITES)}
    for k in arms:
        solve(k)                                   # warm-up
    times = {k: [] for k in arms}
    for _ in range(a.repeats):
        for k in arms:
            times[k].append(solve(k))
    res['fixed_steps'] = a.steps
    res['fixed_s'] = times['fixed']
    res['problem_iterations_per_s'] = [n * a.steps / t for t in times['fixed']]
    _, _, _, steps, ok = sims['default'].ik_read()
    res['default_s'] = times['default']
    res['default_problems_per_s'] = [n / t for t in times['default']]
    res['default_success_fraction'] = float(ok.mean())
    res['default_steps_percentiles'] = {p: int(np.percentile(steps, p)) for p in (0, 10, 50, 90, 100)}
    # the fp64 reference loop on one CPU core
    ikref.lib()                                    # compiled before the clock starts
    it, tt = 0, 0.0
    for k in range(a.reference_problems):
        t0 = time.perf_counter()
        r = ikref.solve(m, m.qpos0, sid, jid, targets[k], **arms['fixed'])
        tt += time.perf_counter() - t0
        it += r['steps'] + 1
    res['fp64_reference_s_per_iteration_one_core'] = tt / it
    for s in sims.values():
        s.close()
    print(json.dumps(res, indent=1))
    if a.out:
        with open(a.out, 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
