"""Batched iLQR (fb_lqr, fb_rollout_feedback_bank, flybody_b200.trajopt): the backward-pass kernel against an fp64 restatement
(lqr_reference) and against the infinite-horizon gain of scipy's discrete Riccati solver, its known answers and its independence of
position and batch; the law bank of the rollouts bit for bit against shared-law calls and against an fp64 restatement of the law; the
conventions of the forward pass to first order; the optimiser (descent, bit-for-bit replay of its result, independence of the batch,
its TVLQR gains); refusals.  CPU tier: the host-emulation build on small handles (the constraint-free flight model, T <= 6, L <= 3);
GPU tier (-m gpu): the same through the CUDA library on 4096-env handles, plus the walk, template and ball models at 10 substeps.

Gates are 2.5 x the larger of the host-emulation and H100 measurements (both named beside each constant)."""
import numpy as np
import pytest
import scipy.linalg

import __graft_entry__ as ge
import lqr_reference as lr
import smooth_states as ss
from flybody_b200 import rollout as ro, stepper as st, trajopt as tj
from flybody_b200 import derivatives as dv
from flybody_b200.flymodel import load_model
from test_model_params import start_state
from test_rollout import SUBSTEPS, bits, fill_bank, inputs, read_all, state_rows, tangent

# ---- gates (measured: host emulation / H100 80GB HBM3 at a 700 W power limit; worst case) -------------------------------------------
LQR_TOL = 5.0e-15          # K, k and dV against the restatement, relative to the largest entry: measured 2.0e-15 emu / 2.0e-15 H100
DARE_TOL = 3.3e-14         # K_0 of a long horizon against the infinite-horizon gain, relative: measured 1.3e-14 emu / 1.3e-14 H100
FIRST_ORDER = 3.5e-5       # |actual / expected decrease - 1| at alpha = 1e-3 (flight): measured 1.4e-5 emu / 1.1e-5 H100
REACH = 2.0e-8             # final / initial cost on reachable flight references: measured 6.0e-9 emu (T = 5) / 7.8e-9 H100 (T = 6)
BANK_CTRL_GATE = 1.35e-6   # recorded ctrl against u + K_law (x - xref_law) in fp64, relative as CTRL_GATE: measured 2.7e-7 emu (walk) /
                           # 5.4e-7 H100 (walk and template on 4096 rollouts; test_rollout's CTRL_GATE is flight's)

GPU_ENVS = 4096


def flight():
    return ss.free_model(load_model('flight'))


def random_problem(m, L, T, seed):
    nx, nu = 2 * m.nv + m.na, m.nu
    rs = np.random.RandomState(seed)
    A = (np.eye(nx) + 0.1 * rs.randn(L, T, nx, nx)).astype(np.float32)
    B = (0.3 * rs.randn(L, T, nx, nu)).astype(np.float32)
    q, r = rs.randn(L, T + 1, nx), rs.randn(L, T, nu)
    Q, R, Qf = rs.uniform(0.1, 1, nx), rs.uniform(0.1, 1, nu), rs.uniform(0.1, 1, nx)
    return A, B, q, r, Q, R, Qf


def rel(a, b):
    return np.abs(a - b).max() / max(np.abs(b).max(), 1e-300)


# ---- 1-3. the backward pass -----------------------------------------------------------------------------------------------------------
def check_backward(lib, measure=None):
    m = flight()
    L, T = 3, 5
    A, B, q, r, Q, R, Qf = random_problem(m, L, T, 0)
    mu = np.array([0.0, 0.5, 3.0])
    out = tj.lqr_backward(m, A, B, q, r, Q, R, Qf, mu, lib_path=lib)
    assert (out.status == 0).all()
    err = 0.0
    for l in range(L):
        K, k, dV, status = lr.backward(A[l], B[l], q[l], r[l], Q, R, Qf, mu[l])
        assert status == 0
        err = max(err, rel(out.K[l], K), rel(out.k[l], k), rel(out.dV[l], dV))
    if measure is not None:
        measure.append(err)
    assert err < LQR_TOL, err
    # alone and at another position in a larger batch: the same bits
    for l in range(L):
        one = tj.lqr_backward(m, A[l:l + 1], B[l:l + 1], q[l:l + 1], r[l:l + 1], Q, R, Qf, mu[l], lib_path=lib)
        assert all(np.array_equal(x[0], y[l]) for x, y in zip(one[:3], out[:3])), l
    perm = [2, 0, 1, 2]
    big = tj.lqr_backward(m, A[perm], B[perm], q[perm], r[perm], Q, R, Qf, mu[perm], lib_path=lib)
    for i, l in enumerate(perm):
        assert all(np.array_equal(x[i], y[l]) for x, y in zip(big[:3], out[:3])), (i, l)


def test_backward_under_emulation(emu):
    check_backward(emu)


@pytest.mark.gpu
def test_gpu_backward():
    check_backward(gpu_lib())


def check_dare(lib, measure=None):
    m = flight()
    nx, nu, T = 2 * m.nv + m.na, m.nu, 300
    rs = np.random.RandomState(1)
    A = 0.95 * scipy.linalg.qr(rs.randn(nx, nx))[0]
    B = 0.3 * rs.randn(nx, nu)
    A, B = A.astype(np.float32).astype(np.float64), B.astype(np.float32).astype(np.float64)
    Q, R = rs.uniform(0.1, 1, nx), rs.uniform(0.1, 1, nu)
    P = scipy.linalg.solve_discrete_are(A, B, np.diag(Q), np.diag(R))
    Kinf = -np.linalg.solve(np.diag(R) + B.T @ P @ B, B.T @ P @ A)
    out = tj.lqr_backward(m, np.broadcast_to(A, (1, T, nx, nx)), np.broadcast_to(B, (1, T, nx, nu)), np.zeros((1, T + 1, nx)),
                          np.zeros((1, T, nu)), Q, R, Q, lib_path=lib)
    err = rel(out.K[0, 0], Kinf)
    if measure is not None:
        measure.append(err)
    assert err < DARE_TOL, err


def test_dare_under_emulation(emu):
    check_dare(emu)


@pytest.mark.gpu
def test_gpu_dare():
    check_dare(gpu_lib())


def check_known_answers(lib):
    m = flight()
    nx, nu, L, T = 2 * m.nv + m.na, m.nu, 2, 4
    A, B, q, r, Q, R, Qf = random_problem(m, L, T, 2)
    # no state cost and no control gradient: nothing to gain, exactly
    out = tj.lqr_backward(m, A, B, np.zeros_like(q), np.zeros_like(r), np.zeros(nx), R, np.zeros(nx), lib_path=lib)
    assert (out.status == 0).all() and not out.K.any() and not out.k.any() and not out.dV.any()
    # an indefinite Quu at step t0: R < 0 where B_t0 = 0, Quu positive definite at the later steps
    t0 = 1
    B2 = np.zeros((L, T, nx, nu), np.float32)
    B2[:, t0 + 1:, :nu] = 10 * np.eye(nu, dtype=np.float32)
    out = tj.lqr_backward(m, A, B2, q, r, Q, -np.ones(nu), Qf, lib_path=lib)
    assert (out.status == t0 + 1).all(), out.status
    assert lr.backward(A[0], B2[0], q[0], r[0], Q, -np.ones(nu), Qf, 0.0)[3] == t0 + 1


def test_known_answers_under_emulation(emu):
    check_known_answers(emu)


@pytest.mark.gpu
def test_gpu_known_answers():
    check_known_answers(gpu_lib())


# ---- 4. the law bank ------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope='module')
def emu():
    ge.build()
    return ge.EMU


def gpu_lib():
    ge.build()
    return None


def check_law_bank(lib, variant, n_envs, n, measure=None):
    m = load_model(variant)
    nsub, T, nx, nr = SUBSTEPS[variant], 3, 2 * m.nv + m.na, m.nq + m.nv + m.na
    sim = st.BatchedStepper(m, n_envs, lib_path=lib)
    q0, v0, a0 = fill_bank(sim, m, [start_state(m, s) for s in range(2)], sensors=False)
    u, _, _ = inputs(m, n, T, 3)
    slots = np.arange(n) % 2
    rs = np.random.RandomState(4)
    L = 3
    xref = np.repeat(np.concatenate([q0, v0, a0], -1)[[0, 1, 0]][:, None], T, 1).astype(np.float32)
    xref[..., m.nq:] += rs.uniform(-0.05, 0.05, (L, T, m.nv + m.na)).astype(np.float32)
    K = (rs.uniform(-1, 1, (L, T, m.nu, nx)) / nx).astype(np.float32)
    law = rs.randint(0, L, n)
    # L = 1 without a list is the shared law, bit for bit
    sim.rollout_feedback(xref[0], K[0])
    sim.rollout(slots, u, nsub)
    shared = read_all(sim, False)
    sim.rollout_feedback_bank(xref[:1], K[:1], np.zeros(n, np.int32))
    sim.rollout(slots, u, nsub)
    assert all(np.array_equal(bits(a), bits(b)) for a, b in zip(read_all(sim, False)[:5], shared[:5]))
    sim._check(sim._lib.fb_rollout_feedback_bank(sim._h, 1, T, xref[0].ctypes.data, K[0].ctypes.data, None, 0, 0), 'bank')
    sim.rollout(slots, u, nsub)
    assert all(np.array_equal(bits(a), bits(b)) for a, b in zip(read_all(sim, False)[:5], shared[:5]))
    # rollouts of different laws: each equals a shared-law call with its law
    sim.rollout_feedback_bank(xref, K, law)
    sim.rollout(slots, u, nsub)
    got = read_all(sim, False)
    for j in range(L):
        sim.rollout_feedback(xref[j], K[j])
        sim.rollout(slots, u, nsub)
        want = read_all(sim, False)
        sel = law == j
        assert all(np.array_equal(bits(a[sel]), bits(b[sel])) for a, b in zip(got[:5], want[:5])), j
    # the recorded ctrl against u + K_law (x - xref_law) in fp64
    x = state_rows(m, q0[slots], v0[slots], a0[slots], got[:3])
    dx = tangent(m, x, xref[law]).reshape(n, T, nx)
    Kl = K[law].astype(np.float64)
    want = u + np.einsum('ntux,ntx->ntu', Kl, dx)
    scale = np.abs(u) + np.einsum('ntux,ntx->ntu', np.abs(Kl), np.abs(dx))
    assert np.abs(dx).max() > 1e-3
    err = (np.abs(got[3] - want) / scale).max()
    if measure is not None:
        measure.append(err)
    assert err < BANK_CTRL_GATE, err
    sim.close()


@pytest.mark.parametrize('variant', ['flight', 'walk'])
def test_law_bank_under_emulation(emu, variant):
    check_law_bank(emu, variant, 5, 5)


@pytest.mark.gpu
@pytest.mark.parametrize('variant', ['walk', 'flight', 'template', 'ball'])
def test_gpu_law_bank(variant):
    check_law_bank(gpu_lib(), variant, GPU_ENVS, GPU_ENVS)


def test_law_bank_refusals(emu):
    m = load_model('flight')
    nx, nr, T = 2 * m.nv + m.na, m.nq + m.nv + m.na, 2
    sim = st.BatchedStepper(m, 3, lib_path=emu)
    fill_bank(sim, m, [start_state(m, 0)], sensors=False)
    x, K = np.zeros((2, T, nr), np.float32), np.zeros((2, T, m.nu, nx), np.float32)
    u = np.zeros((2, T, m.nu), np.float32)
    with pytest.raises(st.StepperError, match='outside'):
        sim.rollout_feedback_bank(x, K, [0, 2])
    with pytest.raises(st.StepperError, match='outside'):
        sim.rollout_feedback_bank(x, K, [-1, 0])
    with pytest.raises(st.StepperError, match='needs a law list'):
        sim._check(sim._lib.fb_rollout_feedback_bank(sim._h, 2, T, x.ctypes.data, K.ctypes.data, None, 0, 0), 'bank')
    with pytest.raises(st.StepperError, match='non-finite'):
        sim.rollout_feedback_bank(np.full_like(x, np.nan), K, [0, 1])
    sim.rollout_feedback_bank(x, K, [0, 1])
    with pytest.raises(st.StepperError, match='law list has 2 rollouts'):
        sim.rollout([0, 0, 0], np.zeros((3, T, m.nu)))
    with pytest.raises(st.StepperError, match='feedback law has 2 steps'):
        sim.rollout([0, 0], np.zeros((2, 3, m.nu)))
    sim.rollout([0, 0], u)
    sim.rollout_feedback()
    sim.rollout([0, 0, 0], np.zeros((3, T, m.nu)))
    # the backward pass
    A, B = np.zeros((1, T, nx, nx), np.float32), np.zeros((1, T, nx, m.nu), np.float32)
    args = [np.zeros((1, T + 1, nx)), np.zeros((1, T, m.nu)), np.ones(nx), np.ones(m.nu), np.ones(nx), np.zeros(1)]
    with pytest.raises(st.StepperError, match='no backward pass'):
        sim.lqr_read()
    with pytest.raises(st.StepperError, match='non-finite A'):
        sim.lqr(np.full_like(A, np.inf), B, *args)
    with pytest.raises(st.StepperError, match='non-finite mu'):
        sim.lqr(A, B, *args[:5], np.full(1, np.nan))
    with pytest.raises(ValueError):
        sim.lqr(A, B[:, :1], *args)
    sim.close()
    # the front end
    q, v = start_state(m, 0)
    with pytest.raises(ValueError, match='needs law'):
        ro.rollout(m, np.stack([q] * 3), np.stack([v] * 3), np.zeros((3, T, m.nu)), x_ref=x, K=K, lib_path=emu)
    with pytest.raises(ValueError, match='ints in'):
        ro.rollout(m, np.stack([q] * 3), np.stack([v] * 3), np.zeros((3, T, m.nu)), x_ref=x, K=K, law=[0, 1, 2], lib_path=emu)
    with pytest.raises(ValueError, match='bank'):
        ro.rollout(m, q, v, np.zeros((T, m.nu)), x_ref=x[0], K=K[0], law=[0], lib_path=emu)


# ---- 5-6. the forward pass and the optimiser ------------------------------------------------------------------------------------------
def reachable(m, L, T, nsub, lib, seed=0, scale=0.3):
    """L reference trajectories that are rollouts of seeded controls u*, from seeded start states"""
    st0 = [start_state(m, seed + s) for s in range(L)]
    q, v = np.array([s[0] for s in st0]), np.array([s[1] for s in st0])
    ustar = np.random.RandomState(seed).uniform(-scale, scale, (L, T, m.nu))
    ref = ro.rollout(m, q, v, ustar, n_substeps=nsub, lib_path=lib)
    x0 = np.concatenate([q, v, np.zeros((L, m.na))], -1)
    x_ref = np.concatenate([x0[:, None], np.concatenate([ref.qpos, ref.qvel, ref.act], -1)], 1)
    return q, v, ustar, x_ref


def weights(m, v):
    nx = 2 * m.nv + m.na
    Q = np.concatenate([np.ones(m.nv), 1 / np.maximum(1, np.abs(v).max(0)) ** 2, np.ones(m.na)])
    return Q[:nx], 1e-3 * np.ones(m.nu)


def check_first_order(lib, measure=None):
    m = flight()
    nsub, T, nx, nr = SUBSTEPS['flight'], 4, 2 * m.nv + m.na, m.nq + m.nv + m.na
    q, v, ustar, x_ref = reachable(m, 1, T, nsub, lib)
    Q, R = weights(m, v)
    u = np.zeros((1, T, m.nu))
    nom = ro.rollout(m, q, v, u, n_substeps=nsub, lib_path=lib)
    xbar = np.concatenate([np.concatenate([q, v], -1)[:, None], np.concatenate([nom.qpos, nom.qvel, nom.act], -1)], 1)
    ubar = nom.ctrl
    J = tj.cost(m, xbar[0], ubar[0], x_ref[0], 0, Q, R, Q)
    r = dv.transition_fd(m, xbar[0, :T, :m.nq], xbar[0, :T, m.nq:m.nq + m.nv], ubar[0], n_substeps=nsub, lib_path=lib)
    dx = tj.tangent(m, xbar[0], x_ref[0])
    out = tj.lqr_backward(m, r.A[None], r.B[None], np.concatenate([dx[:T] * Q, dx[T:] * Q])[None], (ubar * R), Q, R, Q, lib_path=lib)
    alpha = 1e-3
    ua = ubar + alpha * out.k
    roll = ro.rollout(m, q, v, ua, n_substeps=nsub, x_ref=xbar[:, :T].astype(np.float32), K=out.K.astype(np.float32), law=[0],
                      lib_path=lib)
    xa = np.concatenate([xbar[0, :1], np.concatenate([roll.qpos[0], roll.qvel[0], roll.act[0]], -1)], 0)
    Ja = tj.cost(m, xa, roll.ctrl[0], x_ref[0], 0, Q, R, Q)
    ratio = (J - Ja) / -(alpha * out.dV[0, 0] + alpha ** 2 * out.dV[0, 1])
    if measure is not None:
        measure.append(abs(ratio - 1))
    assert abs(ratio - 1) < FIRST_ORDER, ratio


def test_first_order_under_emulation(emu):
    check_first_order(emu)


@pytest.mark.gpu
def test_gpu_first_order():
    check_first_order(gpu_lib())


def check_optimiser(lib, variant, L, T, envs, monkeypatch, measure=None):
    m = flight() if variant == 'flight' else load_model(variant)
    nsub = SUBSTEPS[variant]
    monkeypatch.setattr(tj, 'ENVS', envs)
    q, v, ustar, x_ref = reachable(m, L, T, nsub, lib)
    Q, R = weights(m, v)
    guess = np.zeros((L, T, m.nu))
    guess[-1] = ustar[-1] + np.random.RandomState(3).uniform(-0.1, 0.1, (T, m.nu))      # a perturbed guess for the last problem
    res = tj.ilqr(m, q, v, guess, x_ref, Q, R, n_substeps=nsub, max_iter=6, centered=False, lib_path=lib)
    c = res.cost
    for l in range(L):
        seq = c[l][~np.isnan(c[l])]
        assert len(seq) == res.iterations[l] + 1
        assert (np.diff(seq) <= 0).all(), seq                  # accepted costs never increase
        assert seq[-1] < seq[0]
    frac = max(c[l][res.iterations[l]] / c[l, 0] for l in range(L))
    if measure is not None:
        measure.append(frac)
    if variant == 'flight':
        assert frac < REACH, frac
    # an open-loop rollout of the returned ctrl reproduces the trajectory, and its fp64 cost is the reported one
    ol = ro.rollout(m, res.qpos[:, 0], res.qvel[:, 0], res.ctrl, act=res.act[:, 0], n_substeps=nsub, lib_path=lib)
    for a, b in ((ol.qpos, res.qpos[:, 1:]), (ol.qvel, res.qvel[:, 1:]), (ol.act, res.act[:, 1:]), (ol.ctrl, res.ctrl)):
        assert np.array_equal(bits(a), bits(b))
    for l in range(L):
        x = np.concatenate([res.qpos[l], res.qvel[l], res.act[l]], -1)
        assert tj.cost(m, x, ol.ctrl[l], x_ref[l], 0, Q, R, Q) == c[l][res.iterations[l]]
    # problem 0 alone: the same bits
    one = tj.ilqr(m, q[:1], v[:1], guess[:1], x_ref[:1], Q, R, n_substeps=nsub, max_iter=6, centered=False, lib_path=lib)
    assert one.iterations[0] == res.iterations[0]
    for a, b in zip(one[:5], res[:5]):
        assert np.array_equal(a[0], b[0])
    if variant != 'flight':
        return
    # the returned gains stabilise (on the constraint-free model, as test_rollout's TVLQR check): perturbed starts end closer to the
    # trajectory than the open loop
    seeds = 4
    rs = np.random.RandomState(5)
    l = 0
    q0 = np.repeat(res.qpos[l, :1], seeds, 0)
    v0 = res.qvel[l, :1] + 1e-2 * rs.uniform(-1, 1, (seeds, m.nv)) * np.maximum(1, np.abs(res.qvel[l, 0]))
    xs = np.concatenate([res.qpos[l], res.qvel[l], res.act[l]], -1)
    end = {}
    for name, fb in (('open', {}), ('closed', dict(x_ref=xs[:T].astype(np.float32), K=res.K[l].astype(np.float32)))):
        r = ro.rollout(m, q0, v0, np.repeat(res.ctrl[l:l + 1], seeds, 0), n_substeps=nsub, lib_path=lib, **fb)
        d = tj.tangent(m, np.concatenate([r.qpos[:, -1], r.qvel[:, -1], r.act[:, -1]], -1), xs[T])
        end[name] = np.sqrt((d ** 2 * Q).sum(-1))
    assert (end['closed'] < end['open']).all(), end


def test_optimiser_under_emulation(emu, monkeypatch):
    check_optimiser(emu, 'flight', 3, 5, 120, monkeypatch)


@pytest.mark.gpu
@pytest.mark.parametrize('variant,L,T', [('flight', 3, 6), ('walk', 2, 3), ('template', 2, 3), ('ball', 2, 3)])
def test_gpu_optimiser(variant, L, T, monkeypatch):
    check_optimiser(gpu_lib(), variant, L, T, GPU_ENVS, monkeypatch)


def test_front_end_refusals(emu):
    m = flight()
    nx, nr, T, L = 2 * m.nv + m.na, m.nq + m.nv + m.na, 2, 2
    q, v = (np.stack([x] * L) for x in start_state(m, 0))
    u, x_ref, Q, R = np.zeros((L, T, m.nu)), np.zeros((L, T + 1, nr)), np.ones(nx), np.ones(m.nu)
    call = lambda **kw: tj.ilqr(m, **{**dict(qpos=q, qvel=v, ctrl=u, x_ref=x_ref, Q=Q, R=R, lib_path=emu), **kw})   # noqa: E731
    with pytest.raises(ValueError, match='x_ref'):
        call(x_ref=x_ref[:, :T])
    with pytest.raises(ValueError, match='ctrl'):
        call(ctrl=u[0])
    with pytest.raises(ValueError, match='qpos'):
        call(qpos=q[:1])
    with pytest.raises(ValueError, match='not finite'):
        call(ctrl=np.full_like(u, np.nan))
    with pytest.raises(ValueError, match='negative'):
        call(R=-R)
    with pytest.raises(ValueError, match='negative'):
        call(Qf=-Q)
    with pytest.raises(ValueError, match='alphas'):
        call(alphas=[1.0, 0.0])
