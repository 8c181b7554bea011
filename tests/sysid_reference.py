"""fp64 restatement of fb_sid_accumulate (flybody_b200/csrc/fb_sid.h): the weighted normal equations of fit problems from the outputs of
the same parameter-Jacobian query, read back with fd_param_read / fd_param_inverse_read"""
import numpy as np

from flybody_b200.inverse_kinematics import _differentiate_pos


def transition_residual(m, pred, obs):
    """x'_pred (-) x'_obs [n, nx] of next states [n, nq + nv + na]: mj_differentiatePos(obs qpos, pred qpos), then the qvel and act
    differences"""
    nq = m.nq
    pred, obs = np.asarray(pred, np.float64), np.asarray(obs, np.float64)
    return np.concatenate([_differentiate_pos(m, obs[:, :nq], pred[:, :nq], 1.0), pred[:, nq:] - obs[:, nq:]], 1)


def normal_equations(J, r, W, problem, L, sample_weight=None, bad=None):
    """J [n, rows, k], r [n, rows], W [rows], problem [n] (-1: skipped) -> H [L, k, k], g [L, k], cost [L], count [L], bad [L]; a transition
    with weight 0 is skipped, a bad one (bad[i], or non-finite r or J) adds +inf to the cost and nothing to H or g"""
    n, _, k = J.shape
    J, r, W = np.asarray(J, np.float64), np.asarray(r, np.float64), np.asarray(W, np.float64)
    c = np.ones(n) if sample_weight is None else np.asarray(sample_weight, np.float64)
    H, g, cost = np.zeros((L, k, k)), np.zeros((L, k)), np.zeros(L)
    count, nbad = np.zeros(L, np.int64), np.zeros(L, np.int64)
    for i in range(n):
        l = int(problem[i])
        if l < 0 or not c[i] > 0:
            continue
        count[l] += 1
        if (bad is not None and bad[i]) or not (np.isfinite(r[i]).all() and np.isfinite(J[i]).all()):
            cost[l], nbad[l] = np.inf, nbad[l] + 1
            continue
        H[l] += c[i] * J[i].T @ (W[:, None] * J[i])
        g[l] += c[i] * J[i].T @ (W * r[i])
        cost[l] += c[i] * 0.5 * r[i] @ (W * r[i])
    return H, g, cost, count, nbad
