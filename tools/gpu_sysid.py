"""H100 measurement of batched system identification (fb_sid_accumulate, flybody_b200.sysid): seconds per LM iteration (one sweep of
the parameter Jacobians of every active problem's transitions, their normal equations and the host step) split into 'fd', 'normal' and
'host', for flight (L = 16 problems of T = 64 transitions, 4 substeps, k = 3 scales), template (L = 8, T = 32, 10 substeps, k = 4 scales)
and a large-k case (every dof_damping element of the flight model); the normal-equation kernels against the host alternative on the
same chunk (fd_param_read, then numpy), times and agreement; and the flight fit with the density scale added (the known non-smooth
direction).  Prints the card's name and power limit with the results as one JSON line (and writes it to --out when given).

    python tools/gpu_sysid.py [--out FILE.json]
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

from flybody_b200 import derivatives as dv, stepper as st, sysid  # noqa: E402
from flybody_b200.flymodel import load_model  # noqa: E402
from flybody_b200.inverse_kinematics import _differentiate_pos  # noqa: E402
from gpu_rollout import card  # noqa: E402


def states(m, n, seed):
    """n start states: the reset pose with hinge angles moved by up to 0.05 rad and velocities up to 0.5 (flight: lifted 2 cm)"""
    rs = np.random.RandomState(seed)
    q = np.repeat(m.qpos0[None], n, 0).astype(np.float64)
    for j in range(m.njnt):
        if int(m.jnt_type[j]) == 3:
            q[:, int(m.jnt_qposadr[j])] += rs.uniform(-0.05, 0.05, n)
    if m.nu != 59:
        q[:, int(m.jnt_qposadr[0]) + 2] += 2.0
    return q, rs.uniform(-0.5, 0.5, (n, m.nv))


def problem(m, params, L, T, n_sub, seed=0):
    """recorded transitions of L problems whose parameter directions sit at s* in [0.85, 1.15]: -> (inputs of fit_transitions, s*)"""
    rs = np.random.RandomState(seed)
    dirs, _ = dv._directions(m, params, None)
    s_true = rs.uniform(0.85, 1.15, (L, len(dirs)))
    q, v = states(m, L * T, seed + 1)
    u = rs.uniform(-0.5, 0.5, (L * T, m.nu))
    data = st.BatchedStepper(m, L * T)
    for l in range(L):
        vals = {}
        for (kind, entries, _), s in zip(dirs, s_true[l]):
            for name, i in entries:
                row = vals.setdefault(name, dv.compiled_params(m, name).copy())
                row[i] *= s
        for name, row in vals.items():
            data.param_set(name, row, env_ids=np.arange(l * T, (l + 1) * T))
    data.reset(q, v)
    data.set_control(u)
    data.step(n_sub)
    qd, vd = data.get(st.QPOS).astype(np.float64), data.get(st.QVEL).astype(np.float64)
    data.close()
    w = np.r_[np.full(m.nv, 1e3), 1.0 / np.maximum(np.abs(vd).max(0), 1e-3), np.ones(m.na)]
    shape = lambda x: x.reshape(L, T, -1)                      # noqa: E731
    return (shape(q), shape(v), shape(u), shape(qd), shape(vd), w), s_true


def fit_case(tag, variant, params, L, T, n_sub, max_iter=20):
    m = load_model(variant)
    args, s_true = problem(m, params, L, T, n_sub)
    sweeps = [0]
    read = st.BatchedStepper.sid_read

    def counted(self, out=None):
        sweeps[0] += 1
        return read(self, out)
    st.BatchedStepper.sid_read = counted
    timings = {}
    try:
        t0 = time.perf_counter()
        fit = sysid.fit_transitions(m, *args, params=params, n_substeps=n_sub, max_iter=max_iter, timings=timings)
        wall = time.perf_counter() - t0
    finally:
        st.BatchedStepper.sid_read = read
    hist_ok = all((np.diff(h[np.isfinite(h)]) <= 0).all() for h in fit.cost)
    out = {'case': tag, 'L': L, 'T': T, 'n_substeps': n_sub, 'k': len(fit.columns), 'sweeps': sweeps[0], 'wall_s': wall,
           'per_sweep_s': {k: v / sweeps[0] for k, v in timings.items()}, 'iterations': fit.iterations.tolist(),
           'status': fit.status.tolist(), 'history_non_increasing': bool(hist_ok),
           'transitions_per_s': sweeps[0] and L * T * sweeps[0] / max(timings.get('fd', 0.0), 1e-12)}
    return out, m, fit, s_true


def scale_error(m, fit, params, s_true):
    err = []
    for j, p in enumerate(params):
        name = p.fields[0]
        base = dv.compiled_params(m, name)
        i = int(np.argmax(np.abs(base)))
        err.append(np.abs(fit.values[name][:, i] / base[i] / s_true[:, j] - 1).max())
    return err


def device_vs_host(variant, params, n_envs=4096, n_sub=4):
    """one chunk of a 4096-env handle: fb_sid_accumulate + fb_sid_read against fd_param_read + numpy, times and agreement"""
    m = load_model(variant)
    dirs, _ = dv._directions(m, params, None)
    n = n_envs // (1 + 2 * len(dirs))
    q, v = states(m, n, 5)
    u = np.random.RandomState(6).uniform(-0.5, 0.5, (n, m.nu))
    sim = st.BatchedStepper(m, n_envs)
    dv._param_setup(sim, m, dirs, False, n)
    dv._bank_rows(sim, m, (q, v, u, np.zeros((n, m.na))), n)
    nx, L = 2 * m.nv + m.na, 16
    W = np.ones(nx)
    problem_id = np.arange(n) % L
    sim.fd_param_transition(np.arange(n), n_substeps=n_sub)
    _, qn, vn, an = sim.fd_param_read()
    obs = np.concatenate([qn, vn, an], 1) + np.float32(1e-3)
    best_dev, best_host = np.inf, np.inf
    for _ in range(3):
        sim.fd_param_transition(np.arange(n), n_substeps=n_sub)
        sim.sync()
        t0 = time.perf_counter()
        sim.sid_accumulate(st.SID_TRANSITION, L, problem_id, W, target=obs)
        H, g, cost, _, _ = sim.sid_read()
        best_dev = min(best_dev, time.perf_counter() - t0)
        t0 = time.perf_counter()
        dxdp, qn, vn, an = sim.fd_param_read()
        J = dxdp.astype(np.float64)
        r = np.concatenate([_differentiate_pos(m, obs[:, :m.nq].astype(np.float64), qn.astype(np.float64), 1.0),
                            (np.concatenate([vn, an], 1) - obs[:, m.nq:]).astype(np.float64)], 1)
        Hh = np.zeros((L, len(dirs), len(dirs)))
        gh = np.zeros((L, len(dirs)))
        np.add.at(Hh, problem_id, np.einsum('nri,r,nrj->nij', J, W, J))
        np.add.at(gh, problem_id, np.einsum('nri,r,nr->ni', J, W, r))
        best_host = min(best_host, time.perf_counter() - t0)
    sim.close()
    return {'model': variant, 'k': len(dirs), 'transitions': n, 'device_s': best_dev, 'host_s': best_host,
            'H_rel_diff': float(np.abs(H - Hh).max() / np.abs(Hh).max()), 'g_rel_diff': float(np.abs(g - gh).max() / np.abs(gh).max())}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    res = {'card': card()}
    print('card:', res['card'], flush=True)
    flight = [dv.Scale('dof_damping'), dv.Scale('actuator_gainprm'), dv.Scale('body_mass')]
    template = [dv.Scale('dof_damping'), dv.Scale('body_mass', 'body_inertia'), dv.Scale('actuator_gainprm'), dv.Scale('dof_armature')]
    fm = load_model('flight')
    cases = [('flight k=3', 'flight', flight, 16, 64, 4), ('template k=4', 'template', template, 8, 32, 10),
             ('flight every dof_damping element', 'flight', [('dof_damping', np.flatnonzero(dv.compiled_params(fm, 'dof_damping') > 0))], 4, 16, 4)]
    res['fits'] = []
    for tag, variant, params, L, T, n_sub in cases:
        out, m, fit, s_true = fit_case(tag, variant, params, L, T, n_sub, max_iter=20 if len(params) < 8 else 5)
        if all(isinstance(p, dv.Scale) for p in params):
            out['worst_scale_error'] = [float(e) for e in scale_error(m, fit, params, s_true)]
        print(json.dumps(out), flush=True)
        res['fits'].append(out)
    res['normal_equations'] = [device_vs_host('flight', flight), device_vs_host('template', template, n_sub=10)]
    print(json.dumps(res['normal_equations']), flush=True)
    dens = flight + [dv.Scale('density')]
    out, m, fit, s_true = fit_case('flight with density', 'flight', dens, 4, 64, 4)
    out['scale_error'] = [float(e) for e in scale_error(m, fit, dens, s_true)]
    out['density_fit_over_true'] = (fit.values['density'][:, 0] / float(m.opt_density) / s_true[:, 3]).tolist()
    print(json.dumps(out), flush=True)
    res['density'] = out
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
