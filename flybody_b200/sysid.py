"""Batched system identification on the device: fit each problem's model parameters to recorded motion or to inverse dynamics.

`fit_transitions` fits one-step predictions: problem l has T recorded transitions (qpos, qvel, ctrl, act) -> (qpos_next, qvel_next,
act_next) of n_substeps substeps with ctrl held, e.g. consecutive rows of a recorded or `rollout.rollout` trajectory, and the residual
of a transition is the predicted next state minus the recorded one in transition_fd's tangent.  `fit_inverse` fits inverse dynamics:
the residual is qfrc_inverse - target at recorded (qpos, qvel, qacc); a weight on the six root dofs alone asks for no ghost force at the
root.  Problems are flies, trials or bootstrap draws, L of them at once, each with its own parameter values.

Both run Levenberg-Marquardt over the parameter directions of `derivatives.parameter_fd` (element and `Scale` directions).  One
iteration for the active problems writes the rows at the trial values, runs the parameter-Jacobian sweep a handle at a time and, after
each chunk, `fb_sid_accumulate`, which forms the weighted normal equations H = sum c J^T W J, g = sum c J^T W r and the cost
sum c r^T W r / 2 on the device from the Jacobians the sweep left there; one `fb_sid_read` then returns the k x k system of each
problem, and the step is solved on the host in fp64:
  (H + lambda diag H) delta = -g;  a trial is accepted when its cost is strictly lower (its H and g are then in hand; lambda /= 10),
  otherwise lambda *= 10 and the next trial is solved from the kept H and g.  A trial that would make a non-negative field negative, or
  give a scale delta <= -1, is rejected without a sweep.  A direction whose diagonal is exactly 0 (the data do not reach it, e.g. an
  actuator gain at zero ctrl) is held.
An element direction adds delta_j to its element; a scale direction multiplies its entries by (1 + delta_j), and the next column is again
d / ds at s = 1.  A problem stops converged (status 0) when an accepted step lowers the cost by at most tol (relative), when the solved
step is at most tol (relative to the values: a scale delta, or an element delta over max(|theta|, floor)) or at cost 0; at max_iter
accepted steps (1); when lambda passes LAMBDA_MAX (2); or with a non-finite cost at the start (3).  The sums are fixed-order on the
device and the host step is per problem, so a problem's result depends on neither L, nor its position, nor ENVS.
"""
from collections import namedtuple

import numpy as np

from . import derivatives as dv
from . import stepper as st
from .trajopt import _Clock

ENVS = 4096                      # envs of the handle: max(1, ENVS // columns) transitions per sweep launch
LAMBDA0, LAMBDA_MAX = 1e-3, 1e10
CONVERGED, ITER_CAP, LAMBDA_CAP, NONFINITE = 0, 1, 2, 3

Fit = namedtuple('Fit', ['values', 'cost', 'iterations', 'status', 'H', 'g', 'count', 'columns'])

_SIGNED = {'actuator_gainprm', 'actuator_biasprm', 'gravity', 'wind'}    # the fields fb_param_set does not keep >= 0
_ACTUATION = {'actuator_gainprm', 'actuator_biasprm'}


def _rows(name, x, L, T, width):
    x = np.asarray(x, np.float64)
    if x.shape != (L, T, width):
        raise ValueError(f'{name} {x.shape} against {(L, T, width)}')
    if not np.isfinite(x).all():
        raise ValueError(f'{name} is not finite')
    return x


def _prepare(m, params, floors, values, L, inverse):
    """-> (directions, labels, {name: [L, size] fp64} start values of every parameter)"""
    dirs, labels = dv._directions(m, params, floors)
    seen = set()
    for _, entries, _ in dirs:
        for e in entries:
            if e in seen:
                raise ValueError(f'directions share the element {e[0]}[{e[1]}]: the fit would move it twice')
            seen.add(e)
    act = sorted({n for _, ent, _ in dirs for n, _ in ent} & _ACTUATION)
    if inverse and act:
        raise ValueError(f'{act}: qfrc_inverse excludes actuation, so their columns are 0')
    vals = {}
    for name, v, size in dv._value_inputs(m, values):
        x = dv.compiled_params(m, name) if v is None else np.asarray(v, np.float64)
        if x.ndim == 2 and x.shape[0] != L:
            raise ValueError(f'values[{name!r}] has {x.shape[0]} rows for {L} problems')
        vals[name] = np.array(np.broadcast_to(x.reshape(-1, size), (L, size)))
    return dirs, labels, vals


def _step(H, g, lam):
    """the LM step of one problem, directions with a zero diagonal held (None: the system is singular)"""
    dg = np.diag(H)
    free = dg > 0
    delta = np.zeros(len(g))
    if free.any():
        A = H[np.ix_(free, free)] + lam * np.diag(dg[free])
        try:
            delta[free] = np.linalg.solve(A, -g[free])
        except np.linalg.LinAlgError:
            return None
    return delta if np.isfinite(delta).all() else None


def _trial(dirs, vals, l, delta):
    """problem l's values moved by delta ({name: row}), or None when a non-negative field would go negative or a scale to <= 0"""
    out = {}
    for (kind, entries, _), d in zip(dirs, delta):
        if kind == st.FD_SCALE and d <= -1:
            return None
        for name, i in entries:
            row = out.setdefault(name, vals[name][l].copy())
            row[i] = row[i] * (1 + d) if kind == st.FD_SCALE else row[i] + d
            if name not in _SIGNED and row[i] < 0:
                return None
    return out


def _size(dirs, vals, l, delta):
    """the step relative to the values: a scale delta as it is, an element delta over max(|theta|, floor)"""
    rel = [abs(d) if kind == st.FD_SCALE else abs(d) / max(abs(vals[ent[0][0]][l][ent[0][1]]), fl[0])
           for (kind, ent, fl), d in zip(dirs, delta)]
    return max(rel)


def _lm(dirs, vals, L, sweep, max_iter, tol, clock):
    """Levenberg-Marquardt for L problems; sweep(idx, {name: [len(idx), size]}) -> (cost, H, g, count) of problems idx at those values"""
    if max_iter < 0 or not tol >= 0:
        raise ValueError('max_iter >= 0 and tol >= 0')
    J, H, g, count = sweep(np.arange(L), vals)
    hist = np.full((L, max_iter + 1), np.nan)
    hist[:, 0] = J
    iters, lam = np.zeros(L, np.int64), np.full(L, LAMBDA0)
    status = np.where(np.isfinite(J), -1, NONFINITE)
    if max_iter == 0:
        status[status < 0] = ITER_CAP
    while (status < 0).any():
        trials = {}
        for l in np.flatnonzero(status < 0):
            while True:                                # trials rejected without a sweep
                delta = _step(H[l], g[l], lam[l])
                if delta is not None and (J[l] == 0 or _size(dirs, vals, l, delta) <= tol):
                    status[l] = CONVERGED
                    break
                t = None if delta is None else _trial(dirs, vals, l, delta)
                if t is not None:
                    trials[l] = t
                    break
                lam[l] *= 10
                if lam[l] > LAMBDA_MAX:
                    status[l] = LAMBDA_CAP
                    break
        if not trials:
            continue
        idx = np.array(sorted(trials))
        tv = {name: v[idx].copy() for name, v in vals.items()}
        for p, l in enumerate(idx):
            for name, row in trials[l].items():
                tv[name][p] = row
        clock.lap('host')
        Jt, Ht, gt, ct = sweep(idx, tv)
        for p, l in enumerate(idx):
            if Jt[p] < J[l]:
                gain = (J[l] - Jt[p]) / J[l]
                for name, row in trials[l].items():
                    vals[name][l] = row
                J[l], H[l], g[l], count[l] = Jt[p], Ht[p], gt[p], ct[p]
                lam[l] /= 10
                iters[l] += 1
                hist[l, iters[l]] = J[l]
                if gain <= tol:
                    status[l] = CONVERGED
                elif iters[l] >= max_iter:
                    status[l] = ITER_CAP
            else:
                lam[l] *= 10
                if lam[l] > LAMBDA_MAX:
                    status[l] = LAMBDA_CAP
        clock.lap('host')
    return J, H, g, count, hist[:, :int(iters.max()) + 1], iters, status


def _fit(m, dirs, labels, vals, L, T, write, query, weights, target, sample_weight, ncol, max_iter, tol, device, lib_path, timings,
         slots):
    """the shell of both fits: one handle, the sweep (write(sim, flat transition ids, problem of each, values rows, k) writes a chunk
    and runs its parameter-Jacobian query), the LM loop and the result"""
    per = max(1, ENVS // ncol)
    clock = _Clock(timings)
    fitted = sorted({n for _, ent, _ in dirs for n, _ in ent}, key=st.PARAMS.index)
    sim = st.BatchedStepper(m, min(per, L * T) * ncol, device=device, lib_path=lib_path)
    try:
        dv._param_setup(sim, m, dirs, False, min(per, L * T) if slots else None)

        def sweep(idx, tv):
            n = len(idx) * T
            for c0 in range(0, n, per):
                k = min(per, n - c0)
                f = c0 + np.arange(k)
                p, t = f // T, f % T
                l = idx[p]
                write(sim, l, t, [(name, tv[name][p]) for name in st.PARAMS], k)
                clock.lap('fd')
                sim.sid_accumulate(query, len(idx), p, weights, None if target is None else target[l, t],
                                   None if sample_weight is None else sample_weight[l, t], reset=c0 == 0)
                clock.lap('normal')
            H, g, cost, count, _ = sim.sid_read()
            clock.lap('normal')
            return cost, H, g, count

        J, H, g, count, hist, iters, status = _lm(dirs, vals, L, sweep, max_iter, tol, clock)
    finally:
        sim.close()
    return Fit({name: vals[name] for name in fitted}, hist, iters, status, H, g, count, list(labels))


def _weights(name, w, n):
    w = np.asarray(w, np.float64).reshape(-1)
    if w.shape != (n,) or not np.isfinite(w).all() or (w < 0).any():
        raise ValueError(f'{name}: {n} weights >= 0 and finite')
    return w


def _sample_weight(sample_weight, L, T):
    if sample_weight is None:
        return None
    c = np.asarray(sample_weight, np.float32)
    if c.shape != (L, T) or not np.isfinite(c).all() or (c < 0).any():
        raise ValueError(f'sample_weight: [{L}, {T}] weights >= 0 and finite')
    return c


def fit_transitions(model, qpos, qvel, ctrl, qpos_next, qvel_next, weights, *, params, act=None, act_next=None, values=None,
                    sample_weight=None, floors=None, n_substeps=1, max_iter=20, tol=1e-6, eps=1e-2, centered=True, device=0,
                    lib_path=None, timings=None):
    """Fit L problems' parameters to their one-step predictions: qpos [L, T, nq], qvel [L, T, nv], ctrl [L, T, nu], act [L, T, na]
    (zeros when None) and the recorded next states qpos_next, qvel_next, act_next (zeros when None) after n_substeps substeps with
    ctrl held.  weights [nx] (nx = 2 nv + na) weigh the residual rows (dq, qvel, act); sample_weight [L, T] (None: 1) weighs the
    transitions.  params, values (the start: {name: [L, size] or [size]}, compiled when not given), floors, eps and centered are
    derivatives.parameter_fd's.  timings: a dict that gets the seconds spent in 'fd' (row writes and the parameter-Jacobian sweeps),
    'normal' (the normal equations on the device and their read) and 'host' (the LM steps).

    Returns Fit(values {field: [L, size]} of the fitted fields, cost [L, iters + 1] (the start and each accepted step; nan after the
    problem stopped), iterations [L] (accepted steps), status [L] (CONVERGED, ITER_CAP, LAMBDA_CAP, NONFINITE), H [L, k, k], g [L, k] and
    count [L] (transitions summed) at the returned values, columns: one label per direction).  sigma^2 H^-1 is the covariance of the
    estimate under residuals of variance sigma^2 / weight; a direction with a near-singular H is one the data do not pin down."""
    m = model
    q = np.asarray(qpos, np.float64)
    if q.ndim != 3:
        raise ValueError(f'qpos {q.shape} against [L, T, {m.nq}]')
    L, T = q.shape[:2]
    nx = 2 * m.nv + m.na
    q = _rows('qpos', q, L, T, m.nq)
    v, u = _rows('qvel', qvel, L, T, m.nv), _rows('ctrl', ctrl, L, T, m.nu)
    a = _rows('act', np.zeros((L, T, m.na)) if act is None else act, L, T, m.na)
    obs = np.concatenate([_rows('qpos_next', qpos_next, L, T, m.nq), _rows('qvel_next', qvel_next, L, T, m.nv),
                          _rows('act_next', np.zeros((L, T, m.na)) if act_next is None else act_next, L, T, m.na)], -1).astype(np.float32)
    w = _weights('weights', weights, nx)
    c = _sample_weight(sample_weight, L, T)
    dirs, labels, vals = _prepare(m, params, floors, values, L, False)

    def write(sim, l, t, rows, k):
        dv._bank_rows(sim, m, (q[l, t], v[l, t], u[l, t], a[l, t]), k, rows)
        sim.fd_param_transition(np.arange(k), eps=eps, centered=centered, n_substeps=n_substeps)

    ncol = 1 + (2 if centered else 1) * len(dirs)
    return _fit(m, dirs, labels, vals, L, T, write, st.SID_TRANSITION, w, obs, c, ncol, max_iter, tol, device, lib_path, timings, True)


def fit_inverse(model, qpos, qvel, qacc, weights, *, params, target=None, values=None, sample_weight=None, floors=None, max_iter=20,
                tol=1e-6, eps=1e-2, centered=True, device=0, lib_path=None, timings=None):
    """Fit L problems' parameters to inverse dynamics: qfrc_inverse (inverse_dynamics.inverse's: M qacc + qfrc_bias - qfrc_passive -
    qfrc_constraint) at qpos [L, T, nq], qvel [L, T, nv], qacc [L, T, nv] against target [L, T, nv] (zeros when None), residual rows
    weighed by weights [nv] (e.g. 1 on the root's six dofs and 0 elsewhere: no ghost force at the root).  Actuator gain and bias
    directions are refused: qfrc_inverse excludes actuation.  The rest as fit_transitions."""
    m = model
    q = np.asarray(qpos, np.float64)
    if q.ndim != 3:
        raise ValueError(f'qpos {q.shape} against [L, T, {m.nq}]')
    L, T = q.shape[:2]
    q = _rows('qpos', q, L, T, m.nq)
    v, qa = _rows('qvel', qvel, L, T, m.nv), _rows('qacc', qacc, L, T, m.nv)
    tgt = None if target is None else _rows('target', target, L, T, m.nv).astype(np.float32)
    w = _weights('weights', weights, m.nv)
    c = _sample_weight(sample_weight, L, T)
    dirs, labels, vals = _prepare(m, params, floors, values, L, True)

    def write(sim, l, t, rows, k):
        dv._write_values(sim, m, rows, k)                         # FD problem i takes env i's parameters
        sim.fd_param_inverse(q[l, t], v[l, t], qa[l, t], eps=eps, centered=centered)

    ncol = 1 + (2 if centered else 1) * len(dirs)
    return _fit(m, dirs, labels, vals, L, T, write, st.SID_INVERSE, w, tgt, c, ncol, max_iter, tol, device, lib_path, timings, False)
