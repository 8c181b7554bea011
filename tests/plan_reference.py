"""fp64 restatement of the sampling planner (fb_plan, csrc/fb_plan.h) for the tests: the noise (the counter hash and Box-Muller), the
samples, the cost (trajopt.cost), the MPPI average and the predictive-sampling argmin."""
import numpy as np

from flybody_b200.trajopt import cost  # noqa: F401  (the cost the kernels restate)

M32 = np.uint64(0xffffffff)


def tk_mix(x):
    x = np.asarray(x, np.uint64) & M32
    x ^= x >> np.uint64(16)
    x = (x * np.uint64(0x7feb352d)) & M32
    x ^= x >> np.uint64(15)
    x = (x * np.uint64(0x846ca68b)) & M32
    x ^= x >> np.uint64(16)
    return x


def plan_hash(seed, it, k, knot, a, which):
    u = lambda x: np.asarray(x, np.uint64) & M32                    # noqa: E731
    inner = tk_mix((u(knot) * np.uint64(0xc2b2ae35) + ((u(a) << np.uint64(1)) | u(which))) & M32)
    inner = tk_mix((u(k) * np.uint64(0x85ebca6b) + inner) & M32)
    inner = tk_mix((u(it) * np.uint64(0x9e3779b9) + inner) & M32)
    return tk_mix(u(seed) ^ np.uint64(0x3c6ef372) ^ inner)


def normal(seed, it, k, knot, a):
    """the standard normal of (seed, iteration, sample, knot, actuator), fp64"""
    u1 = (plan_hash(seed, it, k, knot, a, 0).astype(np.float64) + 1.0) * 2.0 ** -32
    u2 = plan_hash(seed, it, k, knot, a, 1).astype(np.float64) * 2.0 ** -32
    return np.sqrt(-2.0 * np.log(u1)) * np.cos(2 * np.pi * u2)


def samples(m, mean, sigma, seed, it, K, hold):
    """the K samples [K, T, nu] (fp32) of one problem's iteration `it` from its mean [T, nu]"""
    T, nu = mean.shape
    k, t, a = np.meshgrid(np.arange(K), np.arange(T), np.arange(nu), indexing='ij')
    eps = np.where(k > 0, normal(seed, it, k, t // hold, a), 0.0)
    u = (mean.astype(np.float32).astype(np.float64)[None] + np.asarray(sigma, np.float32).astype(np.float64) * eps).astype(np.float32)
    lim = np.asarray(m.actuator_ctrllimited, bool)
    lo, hi = (np.asarray(m.actuator_ctrlrange, np.float32).reshape(nu, 2)[:, i] for i in (0, 1))
    return np.where(lim, np.minimum(np.maximum(u, lo), hi), u).astype(np.float32)


def mppi(u, J, temperature):
    """the fp64 weighted average of samples u [K, T, nu] with costs J [K]"""
    w = np.where(np.isfinite(J), np.exp(-(J - J.min()) / temperature), 0.0)
    return np.einsum('k,ktu->tu', w, u.astype(np.float64)) / w.sum()


def argmin(J):
    return int(np.argmin(J))                                           # (the first of equal costs)
