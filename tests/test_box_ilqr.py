"""Control-limited iLQR (box-DDP; fb_lqr_box, trajopt.lqr_backward(lower=, upper=), trajopt.ilqr(box=True)): the box backward pass
against an fp64 restatement (boxqp_reference), each step's k against scipy's bounded least squares and the KKT conditions, its known
answers and its independence of position and batch; the forward pass to first order at a nominal with saturated controls; the optimiser
on references that saturate many controls (descent, bit-for-bit replay, independence of the batch, zero gain rows on clamped controls);
refusals; and a fixed heap over repeated calls.  CPU tier: the host-emulation build on small handles (the constraint-free flight model);
GPU tier (-m gpu): the same through the CUDA library on 4096-env handles, plus the walk, template and ball models at 10 substeps.

Gates are 2.5 x the larger of the host-emulation and H100 measurements (both named beside each constant)."""
import numpy as np
import pytest
import scipy.optimize

import __graft_entry__ as ge
import boxqp_reference as br
from flybody_b200 import rollout as ro, stepper as st, trajopt as tj
from flybody_b200 import derivatives as dv
from flybody_b200.flymodel import load_model
from test_device_buffers import _heap_in_use
from test_ilqr import LQR_TOL, flight, random_problem, rel, weights
from test_model_params import start_state
from test_rollout import SUBSTEPS, bits

# ---- gates (measured: host emulation / H100 80GB HBM3 at a 700 W power limit; worst case) -------------------------------------------
BOX_TOL = 5.5e-15          # K, k and dV against the restatement, relative to the largest entry: measured 2.1e-15 emu / 2.1e-15 H100
BVLS_TOL = 8.5e-15         # k against scipy's BVLS on the same QP, relative: measured 3.4e-15 emu / 3.4e-15 H100
KKT_TOL = 2.3e-15          # free gradient of the QP at k, relative to |Qu| + |Quu| |k|: measured 9.2e-16 emu / 9.2e-16 H100
BOX_FIRST_ORDER = 3.1e-4   # |actual / expected decrease - 1| at alpha = 1e-3, saturated flight nominal: measured 1.2e-4 emu / 1.8e-5 H100
                           # (the unboxed pass's ratio there, not gated: 0.99966 on both)
BOX_REACH = 2.2e-6         # final / initial cost on saturating flight references: measured 7.0e-10 emu (T = 5) / 8.8e-7 H100 (T = 6)

GPU_ENVS = 4096


@pytest.fixture(scope='module')
def emu():
    ge.build()
    return ge.EMU


def gpu_lib():
    ge.build()
    return None


def random_bounds(L, T, nu, seed):
    """bounds around 0 of mixed widths: narrow, wide, one-sided and infinite, lower < upper"""
    rs = np.random.RandomState(seed)
    lo, hi = -rs.uniform(0.01, 1.0, (L, T, nu)), rs.uniform(0.01, 1.0, (L, T, nu))
    lo[rs.rand(L, T, nu) < 0.15] = 0.0
    hi[(rs.rand(L, T, nu) < 0.15) & (lo < 0)] = 0.0
    lo[rs.rand(L, T, nu) < 0.1] = -np.inf
    hi[rs.rand(L, T, nu) < 0.1] = np.inf
    return lo, hi


def _record(measure, name, value):
    if measure is not None:
        measure[name] = max(measure.get(name, 0.0), float(value))


# ---- the backward pass against the restatement and an independent optimum ------------------------------------------------------------
def check_reference(lib, measure=None):
    m = flight()
    nu, L, T = m.nu, 4, 5
    A, B, q, r, Q, R, Qf = random_problem(m, L, T, 0)
    lo, hi = random_bounds(L, T, nu, 1)
    mu = np.array([0.0, 0.5, 3.0, 0.0])
    out = tj.lqr_backward(m, A, B, q, r, Q, R, Qf, mu, lower=lo, upper=hi, lib_path=lib)
    assert isinstance(out, tj.BoxLQR) and (out.status == 0).all()
    assert (out.clamped != 0).sum() > L * T                      # the bounds bind
    err = bv = kkt = 0.0
    for l in range(L):
        qps = {}
        K, k, dV, status, clamped, qp = br.backward(A[l], B[l], q[l], r[l], Q, R, Qf, mu[l], lo[l], hi[l], record=qps)
        assert status == 0
        err = max(err, rel(out.K[l], K), rel(out.k[l], k), rel(out.dV[l], dV))
        assert np.array_equal(out.clamped[l], clamped), l
        assert np.array_equal(out.qp[l], qp), (l, out.qp[l], qp)
        for t in range(T):
            H, g0 = qps[t]
            x = out.k[l, t]
            assert (lo[l, t] <= x).all() and (x <= hi[l, t]).all()
            # the same QP as a bounded least-squares problem: 1/2 x'Hx + g0'x = 1/2 |C'x + C^-1 g0|^2 + const, H = C C'
            c = np.linalg.cholesky(H)
            ls = scipy.optimize.lsq_linear(c.T, -np.linalg.solve(c, g0), bounds=(lo[l, t], hi[l, t]), method='bvls', tol=1e-15)
            bv = max(bv, rel(x, ls.x))
            # KKT: a free control's gradient vanishes, a clamped one points out of the box
            g = g0 + H @ x
            cl = out.clamped[l, t]
            assert (g[cl == -1] > 0).all() and (g[cl == 1] < 0).all()
            assert (x[cl == -1] == lo[l, t][cl == -1]).all() and (x[cl == 1] == hi[l, t][cl == 1]).all()
            scale = np.abs(g0).max() + np.abs(H).max() * np.abs(x).max()
            kkt = max(kkt, np.abs(g[cl == 0]).max(initial=0.0) / scale)
    _record(measure, 'reference', err)
    _record(measure, 'bvls', bv)
    _record(measure, 'kkt', kkt)
    assert err < BOX_TOL, err
    assert bv < BVLS_TOL, bv
    assert kkt < KKT_TOL, kkt
    # alone and at another position in a larger batch: the same bits
    for l in range(L):
        one = tj.lqr_backward(m, A[l:l + 1], B[l:l + 1], q[l:l + 1], r[l:l + 1], Q, R, Qf, mu[l], lower=lo[l:l + 1], upper=hi[l:l + 1],
                              lib_path=lib)
        assert all(np.array_equal(x[0], y[l]) for x, y in zip(one, out)), l
    perm = [3, 1, 0, 2, 3]
    big = tj.lqr_backward(m, A[perm], B[perm], q[perm], r[perm], Q, R, Qf, mu[perm], lower=lo[perm], upper=hi[perm], lib_path=lib)
    for i, l in enumerate(perm):
        assert all(np.array_equal(x[i], y[l]) for x, y in zip(big, out)), (i, l)


def test_reference_under_emulation(emu):
    check_reference(emu)


@pytest.mark.gpu
def test_gpu_reference():
    check_reference(gpu_lib())


def check_known_answers(lib, measure=None):
    m = flight()
    nx, nu, L, T = 2 * m.nv + m.na, m.nu, 2, 4
    A, B, q, r, Q, R, Qf = random_problem(m, L, T, 2)
    mu = np.array([0.0, 0.7])
    # infinite bounds: fb_lqr's answer
    plain = tj.lqr_backward(m, A, B, q, r, Q, R, Qf, mu, lib_path=lib)
    inf = tj.lqr_backward(m, A, B, q, r, Q, R, Qf, mu, lower=np.full((L, T, nu), -np.inf), upper=np.full((L, T, nu), np.inf), lib_path=lib)
    assert np.array_equal(inf.status, plain.status) and not inf.clamped.any()
    same = all(np.array_equal(a, b) for a, b in zip(inf[:3], plain[:3]))
    _record(measure, 'infinite_bounds_bit_identical', same)
    assert max(rel(inf.K, plain.K), rel(inf.k, plain.k), rel(inf.dV, plain.dV)) < LQR_TOL
    # B = 0: K = 0 and k = clamp(-r / (R + mu))
    lo, hi = random_bounds(L, T, nu, 3)
    out = tj.lqr_backward(m, A, np.zeros_like(B), q, r, Q, R, Qf, mu, lower=lo, upper=hi, lib_path=lib)
    want = np.clip(-r / (R + mu[:, None, None]), lo, hi)
    assert (out.status == 0).all() and not out.K.any()
    assert rel(out.k, want) < LQR_TOL
    at = (want == lo) | (want == hi)
    assert at.any() and np.array_equal(out.k[at], want[at])
    # lower = upper = 0 and R < 0: every control clamped, nothing factored, and nothing to gain, exactly
    zero, Bs = np.zeros((L, T, nu)), 0.01 * B
    assert (tj.lqr_backward(m, A, Bs, q, r, Q, -np.ones(nu), Qf, lib_path=lib).status > 0).all()     # Quu is indefinite
    out = tj.lqr_backward(m, A, Bs, q, r, Q, -np.ones(nu), Qf, lower=zero, upper=zero, lib_path=lib)
    assert (out.status == 0).all() and not out.K.any() and not out.k.any() and not out.dV.any()
    assert (out.qp[..., 1] == 6).all() and (out.clamped != 0).all()
    # an indefinite free block at step t0 (R < 0 where B_t0 = 0), positive definite at the later steps: status t0 + 1, as the reference
    t0 = 1
    B2 = np.zeros((L, T, nx, nu), np.float32)
    B2[:, t0 + 1:, :nu] = 10 * np.eye(nu, dtype=np.float32)
    lo, hi = -np.ones((L, T, nu)), np.ones((L, T, nu))
    out = tj.lqr_backward(m, A, B2, q, r, Q, -np.ones(nu), Qf, lower=lo, upper=hi, lib_path=lib)
    assert (out.status == t0 + 1).all(), out.status
    assert (out.qp[:, t0, 1] == -1).all()
    assert br.backward(A[0], B2[0], q[0], r[0], Q, -np.ones(nu), Qf, 0.0, lo[0], hi[0])[3] == t0 + 1


def test_known_answers_under_emulation(emu):
    check_known_answers(emu)


@pytest.mark.gpu
def test_gpu_known_answers():
    check_known_answers(gpu_lib())


# ---- the forward pass at a saturated nominal and the optimiser ------------------------------------------------------------------------
def ranges(m):
    limited = np.asarray(m.actuator_ctrllimited, bool)
    lo, hi = (np.asarray(m.actuator_ctrlrange, np.float32).reshape(m.nu, 2)[:, i].astype(np.float64) for i in (0, 1))
    return limited, lo, hi


def saturating(m, L, T, nsub, lib, seed=0):
    """L reference trajectories that are rollouts of seeded controls drawn from twice each ctrl range (so about half of them clamp)"""
    _, lo, hi = ranges(m)
    st0 = [start_state(m, seed + s) for s in range(L)]
    q, v = np.array([s[0] for s in st0]), np.array([s[1] for s in st0])
    mid, half = (lo + hi) / 2, (hi - lo) / 2
    ustar = mid + 2 * half * np.random.RandomState(seed).uniform(-1, 1, (L, T, m.nu))
    ref = ro.rollout(m, q, v, ustar, n_substeps=nsub, lib_path=lib)
    x0 = np.concatenate([q, v, np.zeros((L, m.na))], -1)
    x_ref = np.concatenate([x0[:, None], np.concatenate([ref.qpos, ref.qvel, ref.act], -1)], 1)
    return q, v, ustar, x_ref


def check_first_order(lib, measure=None):
    """The nominal is the reference's seeded controls, perturbed by 30 % of each half-range and clamped by the plant; the control cost pulls
    towards the unclamped seeded controls u*, so on the controls u* puts beyond a bound the optimal step points out of the box.  The box
    QP clamps exactly those (k_c = 0), and its dV predicts the closed-loop decrease to first order; the unboxed k pushes on them and the
    plant clamps it."""
    m = flight()
    nsub, T = SUBSTEPS['flight'], 4
    limited, lo, hi = ranges(m)
    q, v, ustar, x_ref = saturating(m, 1, T, nsub, lib)
    Q, R = weights(m, v)[0], np.full(m.nu, 0.1)
    applied = lambda u: np.where(limited, np.clip(u, lo, hi), u).astype(np.float32).astype(np.float64)      # noqa: E731
    u0 = ustar + 0.3 * (hi - lo) / 2 * np.random.RandomState(7).uniform(-1, 1, ustar.shape)
    nom = ro.rollout(m, q, v, u0, n_substeps=nsub, lib_path=lib)
    xbar = np.concatenate([np.concatenate([q, v], -1)[:, None], np.concatenate([nom.qpos, nom.qvel, nom.act], -1)], 1)
    ubar = applied(nom.ctrl)
    at = (ubar == lo) | (ubar == hi)
    assert at.sum() >= T * m.nu // 4
    J = tj.cost(m, xbar[0], ubar[0], x_ref[0], ustar[0], Q, R, Q)
    r = dv.transition_fd(m, xbar[0, :T, :m.nq], xbar[0, :T, m.nq:m.nq + m.nv], ubar[0], n_substeps=nsub, lib_path=lib)
    dx = tj.tangent(m, xbar[0], x_ref[0])
    args = (m, r.A[None], r.B[None], np.concatenate([dx[:T] * Q, dx[T:] * Q])[None], (ubar - ustar) * R, Q, R, Q)
    bounds = dict(lower=np.where(limited, lo - ubar, -np.inf), upper=np.where(limited, hi - ubar, np.inf))
    box = tj.lqr_backward(*args, **bounds, lib_path=lib)
    assert box.clamped.any() and not (box.clamped != 0)[~at].any() and not box.k[box.clamped != 0].any()
    alpha, ratio = 1e-3, {}
    for name, out in (('box', box), ('plain', tj.lqr_backward(*args, lib_path=lib))):
        roll = ro.rollout(m, q, v, ubar + alpha * out.k, n_substeps=nsub, x_ref=xbar[:, :T].astype(np.float32),
                          K=out.K.astype(np.float32), law=[0], lib_path=lib)
        xa = np.concatenate([xbar[0, :1], np.concatenate([roll.qpos[0], roll.qvel[0], roll.act[0]], -1)], 0)
        Ja = tj.cost(m, xa, applied(roll.ctrl[0]), x_ref[0], ustar[0], Q, R, Q)
        ratio[name] = (J - Ja) / -(alpha * out.dV[0, 0] + alpha ** 2 * out.dV[0, 1])
    _record(measure, 'first_order', abs(ratio['box'] - 1))
    if measure is not None:
        measure['first_order_unboxed_ratio'] = float(ratio['plain'])
    assert abs(ratio['box'] - 1) < BOX_FIRST_ORDER, ratio


def test_first_order_under_emulation(emu):
    check_first_order(emu)


@pytest.mark.gpu
def test_gpu_first_order():
    check_first_order(gpu_lib())


def check_optimiser(lib, variant, L, T, envs, monkeypatch, measure=None):
    m = flight() if variant == 'flight' else load_model(variant)
    nsub = SUBSTEPS[variant]
    monkeypatch.setattr(tj, 'ENVS', envs)
    q, v, ustar, x_ref = saturating(m, L, T, nsub, lib)
    Q, R = weights(m, v)
    guess = np.zeros((L, T, m.nu))
    kw = dict(n_substeps=nsub, max_iter=6, centered=False, lib_path=lib)
    res = tj.ilqr(m, q, v, guess, x_ref, Q, R, box=True, **kw)
    assert isinstance(res, tj.BoxILQR)
    c = res.cost
    for l in range(L):
        seq = c[l][~np.isnan(c[l])]
        assert len(seq) == res.iterations[l] + 1
        assert (np.diff(seq) <= 0).all(), seq                  # accepted costs never increase
        assert seq[-1] < seq[0]
    frac = max(c[l][res.iterations[l]] / c[l, 0] for l in range(L))
    _record(measure, f'reach_{variant}', frac)
    if variant == 'flight':
        assert frac < BOX_REACH, frac
    # the final gains: zero rows exactly where a control is clamped, and some clamp
    assert res.clamped.any()
    assert not res.K[res.clamped != 0].any()
    # an open-loop rollout of the returned ctrl reproduces the trajectory, and its fp64 cost is the reported one
    ol = ro.rollout(m, res.qpos[:, 0], res.qvel[:, 0], res.ctrl, act=res.act[:, 0], n_substeps=nsub, lib_path=lib)
    for a, b in ((ol.qpos, res.qpos[:, 1:]), (ol.qvel, res.qvel[:, 1:]), (ol.act, res.act[:, 1:]), (ol.ctrl, res.ctrl)):
        assert np.array_equal(bits(a), bits(b))
    for l in range(L):
        x = np.concatenate([res.qpos[l], res.qvel[l], res.act[l]], -1)
        assert tj.cost(m, x, ol.ctrl[l], x_ref[l], 0, Q, R, Q) == c[l][res.iterations[l]]
    # problem 0 alone: the same bits
    one = tj.ilqr(m, q[:1], v[:1], guess[:1], x_ref[:1], Q, R, box=True, **kw)
    assert one.iterations[0] == res.iterations[0]
    for a, b in zip(one, res):
        assert np.array_equal(a[0], b[0])
    # the unboxed solver on the same problems, reported
    if measure is not None:
        plain = tj.ilqr(m, q, v, guess, x_ref, Q, R, **kw)
        measure[f'unboxed_{variant}'] = {'iterations': plain.iterations.tolist(), 'boxed_iterations': res.iterations.tolist(),
                                         'final_over_initial': [float(p[i] / p[0]) for p, i in zip(plain.cost, plain.iterations)],
                                         'boxed_final_over_initial': [float(p[i] / p[0]) for p, i in zip(c, res.iterations)]}


def test_optimiser_under_emulation(emu, monkeypatch):
    check_optimiser(emu, 'flight', 3, 5, 120, monkeypatch)


@pytest.mark.gpu
@pytest.mark.parametrize('variant,L,T', [('flight', 3, 6), ('walk', 2, 3), ('template', 2, 3), ('ball', 2, 3)])
def test_gpu_optimiser(variant, L, T, monkeypatch):
    check_optimiser(gpu_lib(), variant, L, T, GPU_ENVS, monkeypatch)


# ---- refusals and buffers -------------------------------------------------------------------------------------------------------------
def test_refusals(emu):
    m = flight()
    nx, nu, T = 2 * m.nv + m.na, m.nu, 2
    sim = st.BatchedStepper(m, 1, lib_path=emu)
    A, B = np.zeros((1, T, nx, nx), np.float32), np.zeros((1, T, nx, nu), np.float32)
    args = [A, B, np.zeros((1, T + 1, nx)), np.zeros((1, T, nu)), np.ones(nx), np.ones(nu), np.ones(nx), np.zeros(1)]
    lo, hi = -np.ones((1, T, nu)), np.ones((1, T, nu))
    with pytest.raises(st.StepperError, match='no backward pass'):
        sim.lqr_box_read()
    with pytest.raises(ValueError, match='lower'):
        sim.lqr(*args, lo[:, :1], hi)
    with pytest.raises(ValueError, match='upper'):
        sim.lqr(*args, lo, hi[..., :1])
    bad = lo.copy()
    bad[0, 1, 3] = np.nan
    with pytest.raises(st.StepperError, match=r'NaN bound at \[0\]\[1\]\[3\]'):
        sim.lqr(*args, bad, hi)
    with pytest.raises(st.StepperError, match='NaN bound'):
        sim.lqr(*args, lo, np.where(bad != bad, np.nan, hi))
    bad = lo.copy()
    bad[0, 0, 2] = 2.0
    with pytest.raises(st.StepperError, match=r'lower > upper at \[0\]\[0\]\[2\]'):
        sim.lqr(*args, bad, hi)
    with pytest.raises(st.StepperError, match='excludes every finite'):
        sim.lqr(*args, np.full_like(lo, np.inf), np.full_like(hi, np.inf))
    with pytest.raises(st.StepperError, match='non-finite A'):
        sim.lqr(np.full_like(A, np.inf), *args[1:], lo, hi)
    ptrs = [x.ctypes.data for x in args]
    with pytest.raises(st.StepperError, match='must not be NULL'):
        sim._check(sim._lib.fb_lqr_box(sim._h, 1, T, *ptrs, None, hi.ctypes.data, 0), 'fb_lqr_box')
    sim.lqr(*args, lo, hi)
    clamped, qp = sim.lqr_box_read()
    assert clamped.shape == (1, T, nu) and qp.shape == (1, T, 2)
    sim.lqr(*args)
    with pytest.raises(st.StepperError, match='was fb_lqr, without bounds'):
        sim.lqr_box_read()
    sim.lqr(*args, None, hi)                                   # one bound: the other unbounded
    sim.lqr_box_read()
    sim.close()


def test_repeated_passes_keep_the_heap(emu):
    m = flight()
    nu, L, T = m.nu, 3, 5
    A, B, q, r, Q, R, Qf = random_problem(m, L, T, 0)
    lo, hi = random_bounds(L, T, nu, 1)
    sim = st.BatchedStepper(m, 1, lib_path=emu)
    run = lambda: sim.lqr(A, B, q, r, Q, R, Qf, np.zeros(L), lo, hi)      # noqa: E731
    run()
    before = _heap_in_use()
    for _ in range(20):
        run()
        sim.lqr_box_read()
    grown = _heap_in_use() - before
    sim.close()
    assert grown < 8 * L * T * nu, grown                       # less than one call's bounds
