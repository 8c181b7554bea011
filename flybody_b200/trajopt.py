"""Trajectory optimisation on the device: batched iLQR (Tassa, Erez & Todorov 2012) over the stepper's finite-difference Jacobians.

`ilqr` finds controls that track a reference snippet (like the ones `walk_imitation` / `flight_imitation` track) on the physics this
stepper runs, for L problems at once.  Each iteration linearises the nominal trajectory with `fb_fd_transition` (A and B of every
control step), runs the Riccati backward pass on the device (`fb_lqr`, fp64), and runs the forward pass as one rollout call over
L x len(alphas) line-search rollouts, rollout (l, alpha) applying problem l's law from a bank (`fb_rollout_feedback_bank`):
ctrl = u_t + alpha k_t + K_t (x_t - xbar_t).  The returned gains K are a TVLQR law around the returned trajectory that
`rollout.rollout` applies as it is.  `lqr_backward` is the backward pass alone, e.g. for a TVLQR stabiliser (q = r = 0).

`sample_plan` is sampling-based trajectory optimisation on the same cost, MPPI or predictive sampling, with every iteration (noise,
rollouts, cost and update) on the device in one `fb_plan` call; `mpc` runs it in a receding-horizon loop for L plants.

The cost is sum_t |x_t - xref_t|^2_Q / 2 + |u_t - uref_t|^2_R / 2 + |x_T - xref_T|^2_Qf / 2 with diagonal weights, the state difference
in transition_fd's tangent (mj_differentiatePos for qpos), evaluated in fp64 on the host.  The nominal ctrl is the recorded ctrl clamped
to actuator_ctrlrange where the actuator is ctrl-limited (what the step applied), so an open-loop `rollout.rollout` of the returned ctrl
reproduces the returned trajectory bit for bit.

The actuators' ctrl ranges can enter the backward pass too: `ilqr(box=True)` runs control-limited DDP (Tassa, Mansard & Todorov 2014,
`fb_lqr_box`).  At each step k solves the box-constrained QP min 1/2 k'Quu k + Qu'k over lo - ubar <= k <= hi - ubar on the ctrl-limited
actuators by projected Newton, and K has zero rows on the controls clamped at a bound, so the expected decrease dV describes the step
the clamping plant takes and the returned TVLQR gains do not push on saturated controls.  `lqr_backward(lower=, upper=)` is that pass
alone.

As in `derivatives` and `rollout`, every Jacobian and every rollout starts from a cold solver warm start (its state is written and
`forward` run), and no heightfield program is set up, so the vision model runs without terrain contacts.  There is no CPU fallback:
without the CUDA library the calls raise `StepperError`.
"""
import time
from collections import namedtuple

import numpy as np

from . import stepper as st
from .inverse_kinematics import _differentiate_pos

ENVS = 4096          # envs of the handle a solve runs on (rounded down to whole Jacobian problems)

LQR = namedtuple('LQR', ['K', 'k', 'dV', 'status'])
BoxLQR = namedtuple('BoxLQR', ['K', 'k', 'dV', 'status', 'clamped', 'qp'])
ILQR = namedtuple('ILQR', ['qpos', 'qvel', 'act', 'ctrl', 'K', 'cost', 'iterations', 'converged'])
BoxILQR = namedtuple('BoxILQR', ILQR._fields + ('clamped',))

# regularisation schedule (Tassa et al. 2012, section II-F): mu is added to Quu
MU_MIN, MU_MAX, MU_FACTOR = 1e-6, 1e10, 2.0
ACCEPT = 1e-4        # a step is accepted when actual / expected decrease exceeds this


def lqr_backward(model, A, B, q, r, Q, R, Qf, mu=0.0, lower=None, upper=None, device=0, lib_path=None):
    """The iLQR backward pass of L problems on the device (`fb_lqr`, fp64): A [L, T, nx, nx] and B [L, T, nx, nu] (as transition_fd
    returns them, used in fp32), gradients q [L, T + 1, nx] and r [L, T, nu], diagonal weights Q [nx], R [nu], Qf [nx] and mu (scalar or
    [L]) added to Quu.  With q = r = 0, K is the TVLQR law of the weights.

    Returns LQR(K [L, T, nu, nx], k [L, T, nu], dV [L, 2], status [L]): dV = (sum k'Qu, sum k'Quu k / 2), the expected change of the
    cost for a step alpha being alpha dV1 + alpha^2 dV2; status t + 1 when Quu is not positive definite at step t (0: solved).

    With bounds lower and / or upper [L, T, nu] on du = u - ubar (+-inf allowed; the other one unbounded when None) it is the
    control-limited pass (`fb_lqr_box`): k_t minimises the step's QP inside the bounds, K_t has zero rows on the controls clamped at
    k_t, and status is t + 1 when the free block of Quu is not positive definite.  Returns BoxLQR(K, k, dV, status, clamped [L, T, nu]
    (-1 at lower, +1 at upper, 0 free), qp [L, T, 2] (the QP's accepted Newton steps and stop reason, see the header))."""
    L = np.shape(A)[0]
    sim = st.BatchedStepper(model, 1, device=device, lib_path=lib_path)
    try:
        sim.lqr(A, B, q, r, Q, R, Qf, np.broadcast_to(np.asarray(mu, np.float64), (L,)), lower, upper)
        if lower is None and upper is None:
            return LQR(*sim.lqr_read())
        return BoxLQR(*sim.lqr_read(), *sim.lqr_box_read())
    finally:
        sim.close()


def tangent(model, x, xref):
    """x - xref [.., nx] in transition_fd's tangent, fp64: mj_differentiatePos(xref qpos, x qpos), then the qvel and act differences;
    x, xref [.., nq + nv + na]"""
    nq, nv = model.nq, model.nv
    x = np.asarray(x, np.float64)
    shape = x.shape
    x, xref = x.reshape(-1, shape[-1]), np.broadcast_to(np.asarray(xref, np.float64), shape).reshape(-1, shape[-1])
    dq = _differentiate_pos(model, xref[:, :nq], x[:, :nq], 1.0)
    return np.concatenate([dq, x[:, nq:] - xref[:, nq:]], -1).reshape(shape[:-1] + (2 * nv + model.na,))


def cost(model, x, u, x_ref, u_ref, Q, R, Qf):
    """the tracking cost of one trajectory x [T + 1, nq + nv + na], u [T, nu] (fp64)"""
    dx, du = tangent(model, x, x_ref), np.asarray(u, np.float64) - u_ref
    T = du.shape[0]
    return 0.5 * (float((dx[:T] ** 2 * Q).sum()) + float((du ** 2 * R).sum()) + float((dx[T] ** 2 * Qf).sum()))


class _Clock:
    """seconds spent per phase, into a caller's dict"""

    def __init__(self, out):
        self.out, self.t = out, time.perf_counter()

    def lap(self, phase):
        t = time.perf_counter()
        if self.out is not None:
            self.out[phase] = self.out.get(phase, 0.0) + t - self.t
        self.t = t


def _write_rows(sim, m, slot0, x, u):
    """states x [n, nq + nv + na] with ctrl u [n, nu] into bank slots slot0 .. slot0 + n - 1, a handle of envs at a time (a cold warm
    start: written, then forward) -> the states as the envs hold them"""
    nq, nv, N = m.nq, m.nv, sim.n_envs
    held = []
    for c0 in range(0, len(x), N):
        k = min(N, len(x) - c0)
        pad = c0 + np.minimum(np.arange(N), k - 1)
        sim.reset(x[pad, :nq], x[pad, nq:nq + nv])
        if m.na:
            sim.set(st.ACT, x[pad, nq + nv:])
        sim.set_control(u[pad])
        sim.forward()
        sim.save_state(slots=slot0 + np.arange(k), env_ids=np.arange(k))
        held.append(np.concatenate([sim.get(st.QPOS)[:k], sim.get(st.QVEL)[:k], sim.get(st.ACT)[:k]], -1))
    return np.concatenate(held)


def _rollouts(sim, m, x0, ctrl, n_substeps, clock, law=None, xbar=None, K=None):
    """rollouts from x0 [n, nr] (fp32 values) through ctrl [n, T, nu] (fp32), a handle of envs at a time; with law [n], rollout i applies
    the law (xbar [L, T, nr], K [L, T, nu, nx]) law[i] -> (the states after each step [n, T, nr], the recorded ctrl [n, T, nu])"""
    N, xs, us = sim.n_envs, [], []
    for c0 in range(0, len(x0), N):
        k = min(N, len(x0) - c0)
        _write_rows(sim, m, 0, x0[c0:c0 + k], ctrl[c0:c0 + k, 0])
        if law is None:
            sim.rollout_feedback()
        else:
            sim.rollout_feedback_bank(xbar, K, law[c0:c0 + k])
        clock.lap('host')
        sim.rollout(np.arange(k), ctrl[c0:c0 + k], n_substeps)
        clock.lap('forward')
        q, v, a, u = sim.rollout_read()[:4]
        xs.append(np.concatenate([q, v, a], -1))
        us.append(u)
    return np.concatenate(xs), np.concatenate(us)


def _check(name, x, shape, nonneg=False):
    x = np.asarray(x, np.float64)
    if x.shape != shape:
        raise ValueError(f'{name} {x.shape} against {shape}')
    if not np.isfinite(x).all():
        raise ValueError(f'{name} is not finite')
    if nonneg and (x < 0).any():
        raise ValueError(f'{name} has negative weights')
    return x


def ilqr(model, qpos, qvel, ctrl, x_ref, Q, R, Qf=None, act=None, u_ref=None, n_substeps=1, max_iter=50, tol=1e-6,
         alphas=2.0 ** -np.arange(8), eps=1e-2, centered=True, box=False, device=0, lib_path=None, timings=None):
    """iLQR for L problems: initial states qpos [L, nq], qvel [L, nv], act [L, na] (zeros when None), initial controls ctrl [L, T, nu],
    reference states x_ref [L, T + 1, nq + nv + na] and controls u_ref [L, T, nu] (zeros when None), diagonal weights Q [nx], R [nu],
    Qf [nx] (Q when None), nx = 2 nv + na; each control step is n_substeps substeps with ctrl held.  eps and centered are
    transition_fd's.  A problem stops when an accepted step lowers its cost by less than tol (relative) or the expected decrease of a
    full step is below tol (converged), after max_iter accepted steps, or when its regularisation passes MU_MAX.  timings: a dict that
    gets the seconds spent in 'fd' (Jacobians), 'backward', 'forward' (rollouts) and 'host' (row writes, reads and the fp64 cost).
    box: every backward pass is the control-limited one (`lqr_backward` with bounds): du_t is bounded by lo - ubar_t and hi - ubar_t on
    the ctrl-limited actuators (fp64 from the fp32 applied ubar, so lower <= 0 <= upper exactly) and unbounded on the others.  The
    forward pass, the acceptance test and the regularisation schedule are unchanged.

    Returns ILQR(qpos, qvel, act [L, T + 1, .], ctrl [L, T, nu], K [L, T, nu, nx], cost [L, iters + 1], iterations [L], converged [L]):
    the trajectory as the device ran it (fp64 arrays of fp32 values), the TVLQR gains of a backward pass at it, the cost before the first
    step and after each accepted one (nan after the problem stopped), and the accepted steps.  With box, BoxILQR: the same fields and
    clamped [L, T, nu], the clamped sets of the final gains' pass (their rows of K are zero)."""
    m = model
    nq, nv, na, nu = m.nq, m.nv, m.na, m.nu
    nx, nr = 2 * nv + na, nq + nv + na
    u0 = np.asarray(ctrl, np.float64)
    if u0.ndim != 3 or u0.shape[2] != nu or u0.shape[1] < 1:
        raise ValueError(f'ctrl {u0.shape} against [L, T, {nu}]')
    L, T = u0.shape[:2]
    u0 = _check('ctrl', u0, (L, T, nu))
    q0, v0 = _check('qpos', qpos, (L, nq)), _check('qvel', qvel, (L, nv))
    a0 = _check('act', np.zeros((L, na)) if act is None else act, (L, na))
    x_ref = _check('x_ref', x_ref, (L, T + 1, nr))
    u_ref = _check('u_ref', np.zeros((L, T, nu)) if u_ref is None else u_ref, (L, T, nu))
    Q, R = _check('Q', Q, (nx,), True), _check('R', R, (nu,), True)
    Qf = Q if Qf is None else _check('Qf', Qf, (nx,), True)
    alphas = np.asarray(alphas, np.float64).reshape(-1)
    if not len(alphas) or not (np.isfinite(alphas) & (alphas > 0)).all():
        raise ValueError('alphas must be positive and finite')
    if max_iter < 0 or not tol >= 0:
        raise ValueError('max_iter >= 0 and tol >= 0')
    limited = np.asarray(m.actuator_ctrllimited, bool)
    lo, hi = (np.asarray(m.actuator_ctrlrange, np.float32).reshape(nu, 2)[:, i] for i in (0, 1))

    def applied(u):                                            # what the step applies: ctrl-limited actuators clamped (fp32)
        return np.where(limited, np.minimum(np.maximum(u, lo), hi), u).astype(np.float32)

    ncol = 1 + (2 if centered else 1) * (nx + nu)
    per = max(1, ENVS // ncol)
    clock = _Clock(timings)
    sim = st.BatchedStepper(m, per * ncol, device=device, lib_path=lib_path)
    try:
        sim.state_bank(max(L * T, sim.n_envs))
        x0 = _write_rows(sim, m, 0, np.concatenate([q0, v0, a0], -1).astype(np.float32), u0[:, 0].astype(np.float32))
        xs, us = _rollouts(sim, m, x0, u0.astype(np.float32), n_substeps, clock)
        xbar = np.concatenate([x0[:, None], xs], 1).astype(np.float64)      # [L, T + 1, nr]
        ubar = applied(us).astype(np.float64)
        J = np.array([cost(m, xbar[l], ubar[l], x_ref[l], u_ref[l], Q, R, Qf) for l in range(L)])
        hist = np.full((L, max_iter + 1), np.nan)
        hist[:, 0] = J
        mu, delta = np.zeros(L), np.ones(L)
        iters, converged = np.zeros(L, np.int64), np.zeros(L, bool)
        active = np.full(L, max_iter > 0)
        A, B = np.zeros((L, T, nx, nx), np.float32), np.zeros((L, T, nx, nu), np.float32)
        stale = np.ones(L, bool)                               # the nominal changed since its Jacobians
        clock.lap('host')

        def jacobians(idx):
            _write_rows(sim, m, 0, xbar[idx, :T].reshape(-1, nr).astype(np.float32), ubar[idx].reshape(-1, nu).astype(np.float32))
            out_a, out_b = [], []
            clock.lap('host')
            for c0 in range(0, len(idx) * T, per):
                k = min(per, len(idx) * T - c0)
                sim.fd_transition(c0 + np.arange(k), eps=eps, centered=centered, n_substeps=n_substeps)
                clock.lap('fd')
                a, b = sim.fd_read()[:2]
                out_a.append(a)
                out_b.append(b)
            A[idx], B[idx] = np.concatenate(out_a).reshape(len(idx), T, nx, nx), np.concatenate(out_b).reshape(len(idx), T, nx, nu)
            stale[idx] = False
            clock.lap('host')

        def backward(idx):
            dx = np.stack([tangent(m, xbar[l], x_ref[l]) for l in idx])
            q = np.concatenate([dx[:, :T] * Q, dx[:, T:] * Qf], 1)
            r = (ubar[idx] - u_ref[idx]) * R
            bounds = (np.where(limited, lo - ubar[idx], -np.inf), np.where(limited, hi - ubar[idx], np.inf)) if box else ()
            clock.lap('host')
            sim.lqr(A[idx], B[idx], q, r, Q, R, Qf, mu[idx], *bounds)
            clock.lap('backward')
            return sim.lqr_read() + (sim.lqr_box_read()[:1] if box else ())

        def raise_mu(l):
            delta[l] = max(MU_FACTOR, delta[l] * MU_FACTOR)
            mu[l] = max(MU_MIN, mu[l] * delta[l])
            return mu[l] <= MU_MAX

        while active.any():
            idx = np.flatnonzero(active)
            if stale[idx].any():
                jacobians(idx[stale[idx]])
            K, k, dV, status = backward(idx)[:4]
            go = []
            for i, l in enumerate(idx):
                if status[i]:
                    active[l] = raise_mu(l)
                elif -(dV[i, 0] + dV[i, 1]) <= tol * J[l]:     # nothing left to gain
                    converged[l], active[l] = True, False
                else:
                    go.append(i)
            if not go:
                continue
            go = np.array(go)
            nal = len(alphas)
            law = np.repeat(np.arange(len(go)), nal)
            u_try = np.concatenate([(ubar[idx[i]][None] + alphas[:, None, None] * k[i][None]) for i in go]).astype(np.float32)
            x_start = np.repeat(xbar[idx[go], 0], nal, 0).astype(np.float32)
            xs, us = _rollouts(sim, m, x_start, u_try, n_substeps, clock, law, xbar[idx[go], :T].astype(np.float32),
                               K[go].astype(np.float32))
            for j, i in enumerate(go):
                l = idx[i]
                best, best_J = None, J[l]
                for a, alpha in enumerate(alphas):
                    r = j * nal + a
                    xa = np.concatenate([xbar[l, :1], xs[r]], 0)
                    ua = applied(us[r]).astype(np.float64)
                    Ja = cost(m, xa, ua, x_ref[l], u_ref[l], Q, R, Qf)
                    expected = -(alpha * dV[i, 0] + alpha ** 2 * dV[i, 1])
                    if expected > 0 and (J[l] - Ja) / expected > ACCEPT and Ja < best_J:
                        best, best_J = (xa, ua), Ja
                if best is None:
                    active[l] = raise_mu(l)
                    continue
                gain = (J[l] - best_J) / J[l]
                xbar[l], ubar[l], J[l] = best[0], best[1], best_J
                iters[l] += 1
                hist[l, iters[l]] = J[l]
                stale[l] = True
                delta[l] = min(1 / MU_FACTOR, delta[l] / MU_FACTOR)
                mu[l] = mu[l] * delta[l] if mu[l] * delta[l] > MU_MIN else 0.0
                if gain < tol:
                    converged[l], active[l] = True, False
                elif iters[l] >= max_iter:
                    active[l] = False
            clock.lap('host')

        # the TVLQR gains at the returned trajectory (each problem's last regularisation)
        idx = np.arange(L)
        if stale.any():
            jacobians(idx[stale])
        K = np.zeros((L, T, nu, nx))
        clamped = np.zeros((L, T, nu), np.int32)
        todo = idx
        while len(todo):
            out = backward(todo)
            done = out[3] == 0
            K[todo[done]] = out[0][done]
            if box:
                clamped[todo[done]] = out[4][done]
            todo = np.array([l for l in todo[~done] if raise_mu(l)], np.int64)
        clock.lap('host')
    finally:
        sim.close()
    n = int(iters.max()) + 1
    res = ILQR(xbar[..., :nq], xbar[..., nq:nq + nv], xbar[..., nq + nv:], ubar, K, hist[:, :n], iters, converged)
    return BoxILQR(*res, clamped) if box else res


SamplePlan = namedtuple('SamplePlan', ['qpos', 'qvel', 'act', 'ctrl', 'cost', 'status'])
MPC = namedtuple('MPC', ['qpos', 'qvel', 'act', 'ctrl', 'cost', 'status'])


def _plan_inputs(m, qpos, qvel, act, x_ref, u_ref, Q, R, Qf, L, T, sigma, temperature, n_samples, hold, n_iter, n_substeps):
    """the checked inputs of sample_plan / mpc: x0 [L, nr], x_ref [L, T', nr], u_ref [L, T' - 1, nu], Q, R, Qf, sigma [nu]"""
    nq, nv, na, nu = m.nq, m.nv, m.na, m.nu
    nx, nr = 2 * nv + na, nq + nv + na
    q0, v0 = _check('qpos', qpos, (L, nq)), _check('qvel', qvel, (L, nv))
    a0 = _check('act', np.zeros((L, na)) if act is None else act, (L, na))
    x_ref = _check('x_ref', x_ref, (L, T + 1, nr))
    u_ref = _check('u_ref', np.zeros((L, T, nu)) if u_ref is None else u_ref, (L, T, nu))
    Q, R = _check('Q', Q, (nx,), True), _check('R', R, (nu,), True)
    Qf = Q if Qf is None else _check('Qf', Qf, (nx,), True)
    sigma = _check('sigma', np.broadcast_to(np.asarray(sigma, np.float64), (nu,)), (nu,), True)
    if not (np.isfinite(temperature) and temperature >= 0):
        raise ValueError('temperature must be >= 0 and finite')
    if n_samples < 2 or hold < 1 or n_iter < 1 or n_substeps < 1:
        raise ValueError('n_samples >= 2, hold >= 1, n_iter >= 1 and n_substeps >= 1')
    return np.concatenate([q0, v0, a0], -1), x_ref, u_ref, Q, R, Qf, sigma


def _seeds(seed, L):
    """one seed per problem: seed + l for a scalar, else the given [L]"""
    s = np.asarray(seed, np.int64)
    return (s + np.arange(L)) if s.ndim == 0 else s.reshape(L)


def sample_plan(model, qpos, qvel, ctrl0, x_ref, Q, R, Qf=None, act=None, u_ref=None, n_samples=256, sigma=0.1, temperature=0.0,
                hold=1, n_iter=10, n_substeps=1, seed=0, device=0, lib_path=None):
    """Sampling-based trajectory optimisation of L tracking problems on the device (`fb_plan`): initial states qpos [L, nq], qvel [L, nv],
    act [L, na] (zeros when None), the initial nominal controls ctrl0 [L, T, nu], reference states x_ref [L, T + 1, nq + nv + na] and
    controls u_ref [L, T, nu] (zeros when None), diagonal weights Q [nx], R [nu], Qf [nx] (Q when None) of `cost`.  Each of n_iter
    iterations rolls out n_samples samples per problem, mean + sigma (scalar or [nu]) times standard normal noise held over `hold`
    control steps (sample 0 the mean itself), clamped to the ctrl range of ctrl-limited actuators, and moves the mean: temperature > 0,
    MPPI's exp(-(J - J_min) / temperature)-weighted average; temperature = 0, predictive sampling's lowest-cost sample.  seed: a scalar
    (problem l takes seed + l) or [L] seeds; a problem's result depends on its seed and inputs alone.  Problems run 4096 // n_samples at
    a time on one handle, each from a cold warm start (its state written and `forward` run), as `ilqr`'s.

    Returns SamplePlan(qpos, qvel, act [L, T + 1, .], ctrl [L, T, nu], cost [L, n_iter, 2], status [L]): the final mean and its
    trajectory from one rollout on the device (bit for bit what `rollout.rollout` gives for it), each iteration's nominal (the mean's
    clamped sequence, before that iteration's update) and best cost, and per problem 0 or 1 + the first iteration whose samples all
    scored +inf (a bad state: the mean was kept)."""
    m = model
    nq, nv, nu = m.nq, m.nv, m.nu
    u0 = np.asarray(ctrl0, np.float64)
    if u0.ndim != 3 or u0.shape[2] != nu or u0.shape[1] < 1:
        raise ValueError(f'ctrl0 {u0.shape} against [L, T, {nu}]')
    L, T = u0.shape[:2]
    u0 = _check('ctrl0', u0, (L, T, nu))
    x0, x_ref, u_ref, Q, R, Qf, sigma = _plan_inputs(m, qpos, qvel, act, x_ref, u_ref, Q, R, Qf, L, T, sigma, temperature, n_samples,
                                                     hold, n_iter, n_substeps)
    seeds = _seeds(seed, L)
    per = max(1, ENVS // n_samples)
    sim = st.BatchedStepper(m, min(L, per) * n_samples, device=device, lib_path=lib_path)
    means, costs, status, xs = [], [], [], []
    try:
        sim.state_bank(min(L, per))
        sim.plan_program(n_samples, sigma, Q, R, Qf, temperature, hold)
        for c0 in range(0, L, per):
            k, sl = min(per, L - c0), slice(c0, c0 + min(per, L - c0))
            _write_rows(sim, m, 0, x0[sl].astype(np.float32), u0[sl, 0].astype(np.float32))
            sim.plan(np.arange(k), u0[sl], x_ref[sl], seeds[sl], u_ref[sl], n_substeps, n_iter)
            mean, cost_k, _, _, status_k = sim.plan_read(samples=False)
            x_held = _write_rows(sim, m, 0, x0[sl].astype(np.float32), mean[:, 0])      # rollout.rollout's rows for the mean
            sim.rollout(np.arange(k), mean, n_substeps)
            q, v, a = sim.rollout_read()[:3]
            xs.append(np.concatenate([x_held[:, None], np.concatenate([q, v, a], -1)], 1))
            means.append(mean)
            costs.append(cost_k)
            status.append(status_k)
    finally:
        sim.close()
    x = np.concatenate(xs).astype(np.float64)
    return SamplePlan(x[..., :nq], x[..., nq:nq + nv], x[..., nq + nv:], np.concatenate(means).astype(np.float64), np.concatenate(costs),
                      np.concatenate(status))


def mpc(model, qpos, qvel, x_ref, n_steps, horizon, Q, R, Qf=None, act=None, u_ref=None, ctrl0=None, n_samples=256, sigma=0.1,
        temperature=0.0, hold=1, n_iter=1, n_substeps=1, seed=0, device=0, lib_path=None):
    """Receding-horizon sampling MPC of L plants: initial states qpos [L, nq], qvel [L, nv], act [L, na] (zeros when None), reference
    states x_ref [L, n_steps + horizon, nq + nv + na] and controls u_ref [L, n_steps + horizon - 1, nu] (zeros when None), the
    planner's arguments as `sample_plan`'s, ctrl0 [L, horizon, nu] the first warm start (zeros when None).  At control step s each plant
    plans n_iter iterations from its state against x_ref[:, s : s + horizon + 1], warm-started from the previous plan shifted by one step
    (its last step repeated), applies the plan's first control for one control step (a T = 1 rollout from the plant's state row) and
    saves the env back into that row, so the solver warm start carries over as in one continuous rollout.  The plant's first row is
    written with the first applied control (as `rollout.rollout` writes it), so the plant trajectory is bit for bit `rollout.rollout`
    of the applied controls.  The plan of step s uses problem seeds of (seed, plant, s).  Plants run 4096 // n_samples at a time.

    Returns MPC(qpos, qvel, act [L, n_steps + 1, .], ctrl [L, n_steps, nu], cost [L, n_steps, n_iter, 2], status [L, n_steps]): the
    plant trajectory, the applied controls, and each step's plan record (nominal and best cost per iteration, status)."""
    m = model
    nq, nv, nu = m.nq, m.nv, m.nu
    L = np.shape(qpos)[0]
    H, S = int(horizon), int(n_steps)
    if H < 1 or S < 1:
        raise ValueError('horizon >= 1 and n_steps >= 1')
    x0, x_ref, u_ref, Q, R, Qf, sigma = _plan_inputs(m, qpos, qvel, act, x_ref, u_ref, Q, R, Qf, L, S + H - 1, sigma, temperature,
                                                     n_samples, hold, n_iter, n_substeps)
    u0 = _check('ctrl0', np.zeros((L, H, nu)) if ctrl0 is None else ctrl0, (L, H, nu)).astype(np.float32)
    seeds = _seeds(seed, L)
    per = max(1, ENVS // n_samples)
    sim = st.BatchedStepper(m, min(L, per) * n_samples, device=device, lib_path=lib_path)
    xs, us, costs, stats = [], [], [], []
    try:
        sim.state_bank(min(L, per))
        sim.plan_program(n_samples, sigma, Q, R, Qf, temperature, hold)
        for c0 in range(0, L, per):
            k, sl = min(per, L - c0), slice(c0, c0 + min(per, L - c0))
            rows = np.arange(k)
            mean = u0[sl]
            _write_rows(sim, m, 0, x0[sl].astype(np.float32), mean[:, 0])
            x, u, cost, status = [], [], [], []
            for s in range(S):
                sim.plan(rows, mean, x_ref[sl, s:s + H + 1], (seeds[sl] * 1000003 + s) & 0xffffffff, u_ref[sl, s:s + H], n_substeps, n_iter)
                mean, cost_s, _, _, status_s = sim.plan_read(samples=False)
                if s == 0:
                    x.append(_write_rows(sim, m, 0, x0[sl].astype(np.float32), mean[:, 0]))
                sim.rollout(rows, mean[:, :1], n_substeps)
                q, v, a, uc = sim.rollout_read()[:4]
                sim.save_state(slots=rows, env_ids=rows)
                x.append(np.concatenate([q[:, 0], v[:, 0], a[:, 0]], -1))
                u.append(uc[:, 0])
                cost.append(cost_s)
                status.append(status_s)
                mean = np.concatenate([mean[:, 1:], mean[:, -1:]], 1)
            xs.append(np.stack(x, 1))
            us.append(np.stack(u, 1))
            costs.append(np.stack(cost, 1))
            stats.append(np.stack(status, 1))
    finally:
        sim.close()
    x = np.concatenate(xs).astype(np.float64)
    return MPC(x[..., :nq], x[..., nq:nq + nv], x[..., nq + nv:], np.concatenate(us).astype(np.float64), np.concatenate(costs),
               np.concatenate(stats))
