"""Sampling-based MPC on the device (fb_plan, flybody_b200.trajopt.sample_plan / mpc): the noise against a numpy restatement of its
hash and Box-Muller (plan_reference), each sample's cost against trajopt.cost of a rollout of that sample from the same row, the MPPI
mean against an fp64 weighted average, predictive sampling's argmin and its exact invariants, the bad-state score, independence of
position, batch and run, descent on reachable references, the receding-horizon loop, refusals.  CPU tier: the host-emulation build on
small handles (the constraint-free flight model, and walk / ball with contacts); GPU tier (-m gpu): the same through the CUDA library on
4096-env handles for walk, template, ball and flight at their tasks' substep counts, with torch CUDA tensors in and out.

Gates are 2.5 x the larger of the host-emulation and H100 measurements (both named beside each constant)."""
import numpy as np
import pytest

import __graft_entry__ as ge
import plan_reference as pr
import smooth_states as ss
from flybody_b200 import rollout as ro, stepper as st, trajopt as tj
from flybody_b200.flymodel import load_model
from test_ilqr import reachable, weights
from test_model_params import start_state
from test_rollout import SUBSTEPS, bits, fill_bank, inputs

# ---- gates (measured: host emulation / H100 80GB HBM3 at a 700 W power limit; worst case) -------------------------------------------
NOISE_TOL = 1.0e-6         # samples against the restatement, in units of sigma: measured 0 emu / 0 H100 (every sample equal bit for bit;
                           # the gate leaves room for one fp32 rounding of the fp64 noise, |u| / sigma < 8)
COST_TOL = 6.9e-8          # sample_cost against trajopt.cost of the sample's rollout, relative: measured 2.7e-8 emu (walk) / 2.5e-8 H100
                           # (flight)
MPPI_TOL = 1.2e-7          # the MPPI mean against the fp64 weighted average, relative to max |u|: measured 4.6e-8 emu (flight) /
                           # 3.2e-8 H100 (flight)
DESCENT = 0.42             # final / first nominal cost on reachable flight references (T = 3, zero guess, 15 iterations): measured
                           # 0.166 emu (32 samples) / 0.079 H100 (1024 samples), the worse of MPPI and predictive sampling

GPU_ENVS = 4096


@pytest.fixture(scope='module')
def emu():
    ge.build()
    return ge.EMU


def gpu_lib():
    ge.build()
    return None


def model(variant):
    return ss.free_model(load_model('flight')) if variant == 'flight' else load_model(variant)


def problems(sim, m, L, T, nsub, seed=0):
    """bank rows 0 .. L-1 of seeded start states and references x_ref [L, T + 1, nr]: rollouts of seeded controls from them"""
    q0, v0, a0 = fill_bank(sim, m, [start_state(m, seed + s) for s in range(L)], sensors=False)
    x0 = np.concatenate([q0, v0, a0], -1)
    sim.rollout(np.arange(L), inputs(m, L, T, seed + 7)[0], nsub)
    q, v, a = sim.rollout_read()[:3]
    return x0, np.concatenate([x0[:, None], np.concatenate([q, v, a], -1)], 1).astype(np.float64)


def program(m, v):
    nx = 2 * m.nv + m.na
    Q, R = weights(m, np.reshape(v, (-1, m.nv)))
    return dict(sigma=np.full(m.nu, 0.4, np.float32), Q=Q[:nx], R=R)


def guess(m, L, T, hold, seed=8):
    """a nominal sequence constant over each noise knot (so a sample's knots are exactly constant too)"""
    u = inputs(m, L, T, seed)[0]
    return u[:, np.arange(T) // hold * hold]


def sample_costs(sim, m, x0, x_ref, smp, nsub, Q, R):
    """trajopt.cost of each sample's rollout from its problem's row (fb_rollout, the plan's envs) -> [L, K]"""
    L, K, T = smp.shape[:3]
    sim.rollout(np.repeat(np.arange(L), K), smp.reshape(L * K, T, -1), nsub)
    q, v, a = sim.rollout_read()[:3]
    x = np.concatenate([np.repeat(x0[:, None], K, 0).reshape(L * K, 1, -1), np.concatenate([q, v, a], -1)], 1)
    l = np.repeat(np.arange(L), K)
    return np.array([tj.cost(m, x[i], smp.reshape(L * K, T, -1)[i], x_ref[l[i]], 0, Q, R, Q) for i in range(L * K)]).reshape(L, K)


# ---- 1. noise, cost and the MPPI update -----------------------------------------------------------------------------------------------
def check_sample_cost_update(lib, variant, envs, L, K, T, torch_io=False, measure=None):
    m, nsub, hold = model(variant), SUBSTEPS[variant], 2
    sim = st.BatchedStepper(m, envs, lib_path=lib)
    x0, x_ref = problems(sim, m, L, T, nsub)
    p = program(m, x_ref[..., m.nq:m.nq + m.nv])
    mean0, seeds = guess(m, L, T, hold), 11 + np.arange(L)
    # the temperature at the median cost gap of this iteration's samples (they do not depend on it), so several carry weight
    sim.plan_program(K, p['sigma'], p['Q'], p['R'], p['Q'], 1.0, hold)
    sim.plan(np.arange(L), mean0, x_ref, seeds, None, nsub, 1)
    sc = sim.plan_read()[2]
    temp = float(np.median(sc - sc.min(1, keepdims=True)))
    sim.plan_program(K, p['sigma'], p['Q'], p['R'], p['Q'], temp, hold)
    if torch_io:
        import torch
        dev = [torch.as_tensor(np.ascontiguousarray(x, np.float32), device='cuda') for x in (mean0, x_ref)]
        sim.plan(np.arange(L), dev[0].data_ptr(), dev[1].data_ptr(), seeds, None, nsub, 1, T=T, is_device=True)
        out = [torch.zeros(sh, dtype=dt, device='cuda') for sh, dt in (((L, T, m.nu), torch.float32), ((L, 1, 2), torch.float64),
                                                                      ((L, K), torch.float64), ((L, K, T, m.nu), torch.float32),
                                                                      ((L,), torch.int32))]
        sim.plan_read(out)
        mean1, cost, sc, smp, status = (x.cpu().numpy() for x in out)
    else:
        sim.plan(np.arange(L), mean0, x_ref, seeds, None, nsub, 1)
        mean1, cost, sc, smp, status = sim.plan_read()
    assert (status == 0).all()
    sig = p['sigma'].astype(np.float64)
    lim = np.asarray(m.actuator_ctrllimited, bool)
    lo, hi = (np.asarray(m.actuator_ctrlrange, np.float32).reshape(m.nu, 2)[:, i] for i in (0, 1))
    errs = {'noise': 0.0, 'cost': 0.0, 'mppi': 0.0}
    for l in range(L):
        ref = pr.samples(m, mean0[l], p['sigma'], seeds[l], 0, K, hold)
        errs['noise'] = max(errs['noise'], float((np.abs(smp[l].astype(np.float64) - ref) / sig).max()))
        assert np.array_equal(bits(smp[l, 0]), bits(ref[0]))                         # sample 0: the clamped mean, exactly
        assert np.array_equal(bits(smp[l, :, 0:T - 1:hold]), bits(smp[l, :, 1:T:hold]))   # knots constant within hold
        assert not np.array_equal(smp[l, 1], smp[l, 2])
        if lim.any():
            assert ((smp[l][..., lim] >= lo[lim]) & (smp[l][..., lim] <= hi[lim])).all()
            assert ((smp[l][..., lim] == lo[lim]) | (smp[l][..., lim] == hi[lim])).any()    # the clamp was exercised
    J = sample_costs(sim, m, x0, x_ref, smp, nsub, p['Q'], p['R'])
    errs['cost'] = float((np.abs(sc - J) / J).max())
    assert np.array_equal(cost[:, 0, 0], sc[:, 0]) and np.array_equal(cost[:, 0, 1], sc.min(1))
    for l in range(L):
        want = pr.mppi(smp[l], sc[l], temp)
        errs['mppi'] = max(errs['mppi'], float(np.abs(mean1[l] - want).max() / np.abs(want).max()))
        w = np.exp(-(sc[l] - sc[l].min()) / temp)
        assert (w > 1e-3).sum() >= 2, w                                              # more than one sample carries weight
    if measure is not None:
        measure.append(errs)
    assert errs['noise'] < NOISE_TOL and errs['cost'] < COST_TOL and errs['mppi'] < MPPI_TOL, errs
    sim.close()


@pytest.mark.parametrize('variant,L,K', [('flight', 2, 6), ('walk', 1, 4), ('ball', 1, 4)])
def test_sample_cost_update_under_emulation(emu, variant, L, K):
    check_sample_cost_update(emu, variant, L * K, L, K, 3 if variant == 'flight' else 2)


@pytest.mark.gpu
@pytest.mark.parametrize('variant', ['walk', 'flight', 'template', 'ball'])
def test_gpu_sample_cost_update(variant):
    check_sample_cost_update(gpu_lib(), variant, GPU_ENVS, 4, 1024, 6, torch_io=True)


# ---- 1b. the noise is standard normal --------------------------------------------------------------------------------------------------
def check_noise_moments(lib, envs, L, K, T):
    """eps = (u - mean) / sigma over every sample k > 0, step and actuator of L problems (mean 0 and sigma 1e-3, so no clamp is reached):
    its mean and variance within 5 standard errors of N(0, 1)'s"""
    m = model('flight')
    sim = st.BatchedStepper(m, envs, lib_path=lib)
    x0, x_ref = problems(sim, m, L, 1, 1)
    x_ref = np.repeat(x_ref[:, :1], T + 1, 1)
    nx = 2 * m.nv + m.na
    sigma = np.full(m.nu, 1e-3, np.float32)
    sim.plan_program(K, sigma, np.ones(nx), np.ones(m.nu), np.ones(nx), 0.0, 1)
    sim.plan(np.arange(L), np.zeros((L, T, m.nu)), x_ref, 100 + np.arange(L), None, 1, 1)
    smp = sim.plan_read()[3]
    lo, hi = (np.asarray(m.actuator_ctrlrange, np.float32).reshape(m.nu, 2)[:, i] for i in (0, 1))
    assert ((smp > lo) & (smp < hi)).all()
    eps = smp[:, 1:].astype(np.float64).ravel() / sigma[0]
    n = eps.size
    assert abs(eps.mean()) < 5 / np.sqrt(n), (eps.mean(), n)
    assert abs(eps.var() - 1) < 5 * np.sqrt(2 / n), (eps.var(), n)
    sim.close()


def test_noise_moments_under_emulation(emu):
    check_noise_moments(emu, 64, 2, 32, 50)


@pytest.mark.gpu
def test_gpu_noise_moments():
    check_noise_moments(gpu_lib(), GPU_ENVS, 4, 1024, 25)


# ---- 2. predictive sampling: the argmin, bit for bit, and its exact invariants ---------------------------------------------------------
def check_predictive(lib, variant, envs, L, K, T, n_iter):
    m, nsub = model(variant), SUBSTEPS[variant]
    sim = st.BatchedStepper(m, envs, lib_path=lib)
    x0, x_ref = problems(sim, m, L, T, nsub)
    p = program(m, x_ref[..., m.nq:m.nq + m.nv])
    sim.plan_program(K, p['sigma'], p['Q'], p['R'], p['Q'], 0.0, 1)
    mean0, seeds = guess(m, L, T, 1), 3 + np.arange(L)
    sim.plan(np.arange(L), mean0, x_ref, seeds, None, nsub, 1)
    mean1, _, sc, smp, _ = sim.plan_read()
    for l in range(L):
        assert np.array_equal(bits(mean1[l]), bits(smp[l, pr.argmin(sc[l])]))
    sim.plan(np.arange(L), mean0, x_ref, seeds, None, nsub, n_iter)
    mean, cost, sc, smp, status = sim.plan_read()
    assert (status == 0).all()
    assert (np.diff(cost[:, :, 0], axis=1) <= 0).all(), cost[:, :, 0]            # the nominal's cost never increases
    assert np.array_equal(cost[:, 1:, 0], cost[:, :-1, 1])                       # nominal at i + 1 = best at i, bit for bit
    for l in range(L):
        assert np.array_equal(bits(mean[l]), bits(smp[l, pr.argmin(sc[l])]))
    sim.close()


def test_predictive_under_emulation(emu):
    check_predictive(emu, 'flight', 12, 2, 6, 3, 3)


@pytest.mark.gpu
@pytest.mark.parametrize('variant', ['walk', 'flight', 'template', 'ball'])
def test_gpu_predictive(variant):
    check_predictive(gpu_lib(), variant, GPU_ENVS, 4, 1024, 6, 3)


# ---- 3. a bad state scores +inf; its problem keeps its mean and reports it ------------------------------------------------------------
def check_bad_state(lib, envs, K):
    m, nsub, T = model('flight'), SUBSTEPS['flight'], 2
    sim = st.BatchedStepper(m, envs, lib_path=lib)
    (q, v), (qb, vb) = start_state(m, 0), start_state(m, 1)
    fill_bank(sim, m, [(q, v), (qb, vb * 1e30)], sensors=False)
    nr = m.nq + m.nv + m.na
    x_ref = np.zeros((2, T + 1, nr))
    x_ref[:, :, :m.nq] = q
    p = program(m, v[None])
    sim.plan_program(K, p['sigma'], p['Q'], p['R'], p['Q'], 1.0, 1)
    mean0 = guess(m, 2, T, 1)
    sim.plan([0, 1], mean0, x_ref, [1, 2], None, nsub, 2)
    mean, cost, sc, smp, status = sim.plan_read()
    assert np.isfinite(sc[0]).all() and np.isinf(sc[1]).all() and (sc[1] > 0).all()
    assert status.tolist() == [0, 1]
    assert np.isinf(cost[1]).all() and np.isfinite(cost[0]).all()
    assert np.array_equal(bits(mean[1]), bits(mean0[1]))                          # every weight 0: the mean stays
    sim.rollout([1], smp[1, :1], nsub)
    assert sim.rollout_read()[5][0, 0] & 1                                       # the env's bad-state flag
    # problem 0 alone: the same bits (the bad problem does not leak into it)
    sim.plan([0], mean0[:1], x_ref[:1], [1], None, nsub, 2)
    one = sim.plan_read()
    assert all(np.array_equal(a[0], b[0]) for a, b in zip(one, (mean, cost, sc, smp, status)))
    sim.close()
    # good and bad samples in one problem: actuator 3 without its ctrl limit and with sigma 300 (a ctrl of 1e3 on it sets the flag, 1e2
    # does not), so the +inf samples get weight 0 beside finite ones and the MPPI mean is the finite samples' average
    a = m.copy()
    lim = a.actuator_ctrllimited.copy()
    lim[3] = 0
    a.a['actuator_ctrllimited'] = lim
    a.rebuild()
    sim = st.BatchedStepper(a, envs, lib_path=lib)
    fill_bank(sim, a, [(q, v)], sensors=False)
    sig = np.full(a.nu, 0.01, np.float32)
    sig[3] = 300.0
    temp = 1e3
    sim.plan_program(K, sig, p['Q'], p['R'], p['Q'], temp, 1)
    sim.plan([0], mean0[:1], x_ref[:1], [3], None, nsub, 1)
    mean, cost, sc, smp, status = sim.plan_read()
    bad = np.isinf(sc[0])
    assert bad.any() and (~bad[1:]).any() and not bad[0] and status[0] == 0, sc
    sim.rollout(np.zeros(K, np.int32), smp[0], nsub)
    assert np.array_equal(sim.rollout_read()[5][:, -1] & 1 != 0, bad)             # +inf exactly where the env's flag is set
    want = pr.mppi(smp[0], sc[0], temp)
    assert np.isfinite(mean).all() and np.abs(mean[0] - want).max() / np.abs(want).max() < MPPI_TOL
    sim.close()


def test_bad_state_under_emulation(emu):
    check_bad_state(emu, 8, 4)


@pytest.mark.gpu
def test_gpu_bad_state():
    check_bad_state(gpu_lib(), GPU_ENVS, 1024)


# ---- 4. independence of position, batch and run; the seed ---------------------------------------------------------------------------
def check_independence(lib, envs, K, T):
    m, nsub = model('flight'), SUBSTEPS['flight']
    sim = st.BatchedStepper(m, envs, lib_path=lib)
    x0, x_ref = problems(sim, m, 3, T, nsub)
    p = program(m, x_ref[..., m.nq:m.nq + m.nv])
    sim.plan_program(K, p['sigma'], p['Q'], p['R'], p['Q'], 5.0, 2)
    mean0, seeds = guess(m, 3, T, 2), np.array([5, 6, 7])

    def run(idx, sd=None):
        idx = np.asarray(idx)
        sim.plan(idx, mean0[idx], x_ref[idx], seeds[idx] if sd is None else sd, None, nsub, 2)
        return sim.plan_read()

    full = run([0, 1, 2])
    for i, l in enumerate([2, 0, 1, 2]):
        for got in (run([l]), run([2, 0, 1, 2])):
            j = 0 if len(got[0]) == 1 else i
            assert all(np.array_equal(a[j], b[l]) for a, b in zip(got, full)), (i, l)
    assert all(np.array_equal(a, b) for a, b in zip(run([0, 1, 2]), full))
    short = sim.plan_read(samples=False)                                           # samples left on the device
    assert short[2] is None and short[3] is None
    assert all(np.array_equal(short[i], full[i]) for i in (0, 1, 4))
    other = run([0], [99])
    assert not np.array_equal(other[3][0, 1:], full[3][0, 1:])
    assert other[1][0, 0, 0] == full[1][0, 0, 0]                                 # the first nominal is the input's either way
    sim.close()


def test_independence_under_emulation(emu):
    check_independence(emu, 16, 4, 3)


@pytest.mark.gpu
def test_gpu_independence():
    check_independence(gpu_lib(), GPU_ENVS, 1024, 6)


# ---- 5. descent on reachable references ----------------------------------------------------------------------------------------------
def check_descent(lib, L, T, K, n_iter, measure=None):
    m, nsub = model('flight'), SUBSTEPS['flight']
    q, v, ustar, x_ref = reachable(m, L, T, nsub, lib, scale=0.3)
    Q, R = weights(m, x_ref[..., m.nq:m.nq + m.nv].reshape(-1, m.nv))
    frac = {}
    for name, temp in (('mppi', 0.3), ('predictive', 0.0)):
        res = tj.sample_plan(m, q, v, np.zeros((L, T, m.nu)), x_ref, Q, R, n_samples=K, sigma=0.05, temperature=temp, n_iter=n_iter,
                             n_substeps=nsub, seed=1, lib_path=lib)
        assert (res.status == 0).all()
        frac[name] = float((res.cost[:, -1, 0] / res.cost[:, 0, 0]).max())       # the nominal's cost, last iteration over first
        # the returned trajectory is rollout.rollout's of the returned ctrl, bit for bit
        ol = ro.rollout(m, q, v, res.ctrl, n_substeps=nsub, lib_path=lib)
        for a, b in ((ol.qpos, res.qpos[:, 1:]), (ol.qvel, res.qvel[:, 1:]), (ol.act, res.act[:, 1:])):
            assert np.array_equal(bits(a), bits(b))
        if temp == 0.0:                                                          # the returned mean is the last iteration's best
            for l in range(L):
                x = np.concatenate([res.qpos[l], res.qvel[l], res.act[l]], -1)
                assert tj.cost(m, x, res.ctrl[l], x_ref[l], 0, Q, R, Q) == pytest.approx(res.cost[l, -1, 1], rel=COST_TOL)
    if measure is not None:
        measure.append(frac)
    assert max(frac.values()) < DESCENT, frac


def test_descent_under_emulation(emu):
    check_descent(emu, 2, 3, 32, 15)


@pytest.mark.gpu
def test_gpu_descent():
    check_descent(gpu_lib(), 4, 3, 1024, 15)


# ---- 6. the receding-horizon loop ----------------------------------------------------------------------------------------------------
def check_mpc(lib, L, n_steps, horizon, K, n_iter):
    m, nsub = model('flight'), SUBSTEPS['flight']
    q, v, ustar, x_ref = reachable(m, L, n_steps + horizon - 1, nsub, lib, scale=0.3)
    Q, R = weights(m, x_ref[..., m.nq:m.nq + m.nv].reshape(-1, m.nv))
    q1 = q.copy()                                                                # a perturbed start: every hinge angle off by 0.1 rad
    q1[:, np.asarray(m.jnt_qposadr)[np.asarray(m.jnt_type) == 3]] += 0.1
    res = tj.mpc(m, q1, v, x_ref, n_steps, horizon, Q, R, u_ref=ustar, ctrl0=ustar[:, :horizon], n_samples=K, sigma=0.1,
                 temperature=0.0, n_iter=n_iter, n_substeps=nsub, seed=4, lib_path=lib)
    assert res.ctrl.shape == (L, n_steps, m.nu) and res.cost.shape == (L, n_steps, n_iter, 2) and (res.status == 0).all()
    # the plant trajectory is one continuous rollout.rollout of the applied controls, bit for bit
    ol = ro.rollout(m, q1, v, res.ctrl, n_substeps=nsub, lib_path=lib)
    for a, b in ((ol.qpos, res.qpos[:, 1:]), (ol.qvel, res.qvel[:, 1:]), (ol.act, res.act[:, 1:]), (ol.ctrl, res.ctrl)):
        assert np.array_equal(bits(a), bits(b))
    # it tracks the reference better than replaying the reference's own controls open loop from the perturbed start
    rep = ro.rollout(m, q1, v, ustar[:, :n_steps], n_substeps=nsub, lib_path=lib)

    def track(qp, qv, ac):
        x = np.concatenate([qp, qv, ac], -1)
        return (tj.tangent(m, x, x_ref[:, 1:n_steps + 1]) ** 2 * Q).sum((1, 2))

    assert (track(res.qpos[:, 1:], res.qvel[:, 1:], res.act[:, 1:]) < track(rep.qpos, rep.qvel, rep.act)).all()


def test_mpc_under_emulation(emu):
    check_mpc(emu, 2, 8, 4, 64, 3)


@pytest.mark.gpu
def test_gpu_mpc():
    check_mpc(gpu_lib(), 16, 8, 4, 256, 3)


# ---- 7. refusals -----------------------------------------------------------------------------------------------------------------------
def test_refusals(emu):
    m = model('flight')
    nx, nr, T, nsub = 2 * m.nv + m.na, m.nq + m.nv + m.na, 2, 1
    sim = st.BatchedStepper(m, 6, lib_path=emu)
    mean, x_ref = np.zeros((2, T, m.nu)), np.zeros((2, T + 1, nr))
    x_ref[:, :, :m.nq] = m.qpos0
    args = dict(sigma=np.ones(m.nu), Q=np.ones(nx), R=np.ones(m.nu))
    with pytest.raises(st.StepperError, match='no plan to read'):
        sim.plan_read()
    with pytest.raises(st.StepperError, match='no state bank'):
        sim.plan([0, 0], mean, x_ref, [0, 1])
    fill_bank(sim, m, [start_state(m, 0)], sensors=False)
    with pytest.raises(st.StepperError, match='no plan program'):
        sim.plan([0, 0], mean, x_ref, [0, 1])
    for kw, what in ((dict(n_samples=1), 'n_samples >= 2'), (dict(hold=0), 'hold >= 1'), (dict(temperature=-1.0), 'temperature'),
                     (dict(temperature=np.inf), 'temperature'), (dict(sigma=-np.ones(m.nu)), 'sigma'),
                     (dict(sigma=np.full(m.nu, np.nan)), 'sigma'), (dict(Q=-np.ones(nx)), 'Q must'), (dict(R=np.full(m.nu, np.inf)), 'R must'),
                     (dict(Qf=-np.ones(nx)), 'Qf must')):
        with pytest.raises(st.StepperError, match=what):
            sim.plan_program(**{**dict(n_samples=3), **args, **kw})
    sim.plan_program(3, **args)
    with pytest.raises(st.StepperError, match='L \\* n_samples'):
        sim.plan([0, 0, 0], np.zeros((3, T, m.nu)), np.repeat(x_ref[:1], 3, 0), [0, 1, 2])
    for kw, what in ((dict(mean=mean[:, :0], x_ref=x_ref[:, :1]), 'T >= 1'), (dict(n_substeps=0), 'n_substeps'), (dict(n_iter=0), 'n_iter'),
                     (dict(slots=[0, 5]), 'out of range'), (dict(slots=[0, 1]), 'never written'),
                     (dict(mean=np.full_like(mean, np.nan)), 'non-finite'), (dict(x_ref=np.full_like(x_ref, np.inf)), 'non-finite'),
                     (dict(u_ref=np.full_like(mean, np.nan)), 'non-finite')):
        with pytest.raises(st.StepperError, match=what):
            sim.plan(**{**dict(slots=[0, 0], mean=mean, x_ref=x_ref, seeds=[0, 1], n_substeps=nsub), **kw})
    with pytest.raises(ValueError, match='seeds'):
        sim.plan([0, 0], mean, x_ref, [0])
    sim.plan([0, 0], mean, x_ref, [0, 1])
    sim.plan_read()
    sim.plan_program(0)                                                           # cleared: nothing to plan or read
    with pytest.raises(st.StepperError, match='no plan to read'):
        sim.plan_read()
    with pytest.raises(st.StepperError, match='no plan program'):
        sim.plan([0, 0], mean, x_ref, [0, 1])
    sim.close()
    # a model without actuators
    a = m.copy()
    for k, x in a.a.items():
        if k.startswith('actuator_') and isinstance(x, np.ndarray):
            a.a[k] = x[:0]
    a.a['nu'] = a.meta['nu'] = 0
    sim = st.BatchedStepper(a.rebuild(), 4, lib_path=emu)
    with pytest.raises(st.StepperError, match='no actuators'):
        sim.plan_program(3, np.ones(0), np.ones(nx), np.ones(0))
    sim.close()
    # the front ends
    q, v = (np.stack([x] * 2) for x in start_state(m, 0))
    call = lambda **kw: tj.sample_plan(m, **{**dict(qpos=q, qvel=v, ctrl0=mean, x_ref=x_ref, Q=np.ones(nx), R=np.ones(m.nu),   # noqa: E731
                                                    n_samples=3, n_iter=1, lib_path=emu), **kw})
    for kw, what in ((dict(x_ref=x_ref[:, :T]), 'x_ref'), (dict(ctrl0=mean[0]), 'ctrl0'), (dict(sigma=-1.0), 'negative'),
                     (dict(temperature=-1.0), 'temperature'), (dict(n_samples=1), 'n_samples'), (dict(R=-np.ones(m.nu)), 'negative')):
        with pytest.raises(ValueError, match=what):
            call(**kw)
    with pytest.raises(ValueError, match='x_ref'):
        tj.mpc(m, q, v, x_ref, 3, 2, np.ones(nx), np.ones(m.nu), n_samples=3, lib_path=emu)
