// fb_plan.h -- sampling-based MPC on the device (fb_plan): MPPI (Williams et al. 2017, the information-theoretic update without the
// control cross term) and predictive sampling (Howell et al. 2022, MuJoCo MPC), batched over L tracking problems of K samples each.
// One iteration of problem l, from state-bank row slots[l] and its nominal control sequence mean [T][nu]:
//   sample   u_k,t = clamp(mean_t + sigma * eps_k,floor(t / hold)) (clamp: ctrl-limited actuators only, as the actuation stage), eps a
//            standard normal by Box-Muller from a counter hash of (seed_l, iteration, k, knot, actuator) in an index space of its own;
//            sample 0 has eps = 0 (the clamped mean)                                                         (kplan_sample)
//   roll out all L K samples open loop through the rollout input kernel (a DevRoll of the plan's ctrl, K = nullptr) and the step graph
//   score    J_k = 1/2 sum_{t<T} (|x_t (-) xref_t|^2_Q + |u_k,t - uref_t|^2_R) + 1/2 |x_T (-) xref_T|^2_Qf in fp64 from the fp32 state,
//            (-) roll_tangent (transition_fd's tangent); +inf once the env sets the bad-state flag (bit value 1 of d.flags)   (kplan_cost)
//   update   temperature > 0: w_k = exp(-(J_k - J_min) / temperature), mean_t = sum_k w_k u_k,t / sum_k w_k (fp64, stored fp32);
//            temperature = 0: mean = the lowest-cost sample, bit for bit (ties: the lowest index); every J_k = +inf: mean unchanged and
//            the problem's status set                                                                        (kplan_weights, kplan_update)
// One warp per work unit, no atomics, no shared memory; every sum is one fixed-order sum of the problem's own data (lane partials added
// in lane order), so a problem's bits depend on neither its index, nor L, nor the other problems.
#pragma once
#include "fb_task.h"
#include "fb_rollout.h"

#define PLAN_STEPS 4             // control steps of one update warp

struct DevPlan {
  int L, K, T, hold, n_iter, iter, t;       // problems, samples per problem, steps, knot spacing, iterations, the iteration and the step
                                            // a launch serves (t = -1: the initial state)
  double temperature;
  const float* sigma;                       // [nu]
  const double *Q, *R, *Qf;                 // [nx], [nu], [nx]
  const unsigned* seed;                     // [L]
  const float *xref, *uref;                 // [L][T + 1][nq + nv + na], [L][T][nu] (uref nullptr: 0)
  float *mean, *ctrl;                       // [L][T][nu]; the samples [L K][T][nu] (what the rollout input kernel reads)
  double *J, *w;                            // [L K] the samples' costs and weights
  double* wsum;                             // [L]
  int* sel;                                 // [L] the lowest-cost sample (-1: every sample scored +inf)
  double* hist;                             // [L][n_iter][2] the nominal's (sample 0's) cost and the best cost of each iteration
  int* status;                              // [L] 0, or 1 + the first iteration whose samples all scored +inf
};

// the counter hash of one uniform word of the plan's noise: (seed, iteration, sample, knot, actuator, which of the two words)
FB_DEV unsigned plan_hash(unsigned seed, int iter, int k, int knot, int a, unsigned which) {
  return tk_mix(seed ^ 0x3c6ef372u ^ tk_mix((unsigned)iter * 0x9e3779b9u +
                tk_mix((unsigned)k * 0x85ebca6bu + tk_mix((unsigned)knot * 0xc2b2ae35u + ((unsigned)a << 1 | which)))));
}
// a standard normal (Box-Muller, fp64) from two 32-bit words: u1 in (0, 1], u2 in [0, 1).  On the device cospi(2 u2): its argument
// needs no large-angle reduction, which keeps the sample kernel off a stack frame.
FB_DEV double plan_normal(unsigned seed, int iter, int k, int knot, int a) {
  const double u1 = ((double)plan_hash(seed, iter, k, knot, a, 0) + 1.0) * 2.3283064365386963e-10;
  const double u2 = (double)plan_hash(seed, iter, k, knot, a, 1) * 2.3283064365386963e-10;
#ifdef __CUDACC__
  return sqrt(-2.0 * log(u1)) * cospi(2.0 * u2);
#else
  return sqrt(-2.0 * log(u1)) * cos(6.283185307179586 * u2);
#endif
}

// all T rows of sample i into the plan's ctrl
FB_WARPFN void kplan_sample(const DevModel& m, const DevPlan& p, int i) {
  const int nu = m.nu, l = i / p.K, k = i - l * p.K, n = p.T * nu;
  const float* mean = p.mean + (size_t)l * n;
  float* u = p.ctrl + (size_t)i * n;
  const unsigned seed = p.seed[l];
  WPAR_BEGIN
    for (int j = lane; j < n; j += FB_NY) {
      const int t = j / nu, a = j - t * nu;
      float v = mean[j];
      if (k > 0) v = (float)((double)v + (double)p.sigma[a] * plan_normal(seed, p.iter, k, t / p.hold, a));
      if (MLD(m.actuator_ctrllimited[a])) v = clampf(v, MLD(m.actuator_ctrlrange[2 * a]), MLD(m.actuator_ctrlrange[2 * a + 1]));
      u[j] = v;
    }
  WPAR_END
}

// env i's cost terms: t = -1, the initial state's (Q); t >= 0, after step t, the new state's (Q, Qf after the last step) and the R term
// of the step's control.  Lanes sum their components, lane 0 adds the lane partials in lane order.
FB_WARPFN void kplan_cost(const DevModel& m, const DevData& d, const DevPlan& p, int e) {
  const int nx = 2 * m.nv + m.na, nu = m.nu, nr = m.nq + m.nv + m.na, l = e / p.K, t = p.t;
  const float* xr = p.xref + ((size_t)l * (p.T + 1) + (t + 1)) * nr;
  const double* W = t == p.T - 1 ? p.Qf : p.Q;
  LREG(double, part);
  WPAR_BEGIN
    double a = 0.0;
    for (int c = lane; c < nx; c += FB_NY) { const double dx = roll_tangent(m, d, e, xr, c); a = fma(W[c] * dx, dx, a); }
    if (t >= 0) {
      const float* u = p.ctrl + ((size_t)e * p.T + t) * nu;
      const float* ur = p.uref ? p.uref + ((size_t)l * p.T + t) * nu : nullptr;
      for (int r = lane; r < nu; r += FB_NY) { const double du = (double)u[r] - (ur ? (double)ur[r] : 0.0); a = fma(p.R[r] * du, du, a); }
    }
    L(part) = a;
  WPAR_END
  WPAR_BEGIN
    double sum = 0.0;
    for (int y = 0; y < FB_NY; y++) sum += SHF(part, y);
    if (lane == 0) {
      const double J = (AT(d.flags, 0) & 1) ? HUGE_VAL : (t < 0 ? 0.0 : p.J[e]) + 0.5 * sum;
      p.J[e] = J < HUGE_VAL ? J : HUGE_VAL;      // (a NaN scores +inf too)
    }
  WPAR_END
}

// problem l: the lowest cost and its sample, the weights and their sum, the iteration's record and status
FB_WARPFN void kplan_weights(const DevPlan& p, int l) {
  const int K = p.K;
  const double* J = p.J + (size_t)l * K;
  double* w = p.w + (size_t)l * K;
  LREG(double, jb); LREG(int, kb); LREG(double, ws);
  WPAR_BEGIN
    double b = HUGE_VAL; int bk = K;
    for (int k = lane; k < K; k += FB_NY) if (J[k] < b) { b = J[k]; bk = k; }
    L(jb) = b; L(kb) = bk;
  WPAR_END
  double jmin = HUGE_VAL; int kmin = K;      // every lane reduces the lanes' minima in lane order, so every lane holds the result
  WPAR_BEGIN
    double b = HUGE_VAL; int bk = K;
    for (int y = 0; y < FB_NY; y++) {
      const double v = SHF(jb, y); const int k = SHF(kb, y);
      if (v < b || (v == b && k < bk)) { b = v; bk = k; }
    }
    jmin = b; kmin = bk;
  WPAR_END
  const bool none = kmin >= K;
  WPAR_BEGIN
    double a = 0.0;
    if (p.temperature > 0.0 && !none)
      for (int k = lane; k < K; k += FB_NY) { const double v = J[k] < HUGE_VAL ? exp(-(J[k] - jmin) / p.temperature) : 0.0; w[k] = v; a += v; }
    L(ws) = a;
  WPAR_END
  WPAR_BEGIN
    double sum = 0.0;
    for (int y = 0; y < FB_NY; y++) sum += SHF(ws, y);
    if (lane == 0) {
      p.wsum[l] = sum; p.sel[l] = none ? -1 : kmin;
      double* h = p.hist + ((size_t)l * p.n_iter + p.iter) * 2;
      h[0] = J[0]; h[1] = jmin;
      if (p.iter == 0) p.status[l] = 0;
      if (none && p.status[l] == 0) p.status[l] = p.iter + 1;
    }
  WPAR_END
}

// problem l's mean over steps [t0, t0 + PLAN_STEPS): the weighted average of its samples (k in order), or a copy of the best one
FB_WARPFN void kplan_update(const DevModel& m, const DevPlan& p, int w) {
  const int nu = m.nu, nb = (p.T + PLAN_STEPS - 1) / PLAN_STEPS, l = w / nb, t0 = (w - l * nb) * PLAN_STEPS;
  const int t1 = t0 + PLAN_STEPS < p.T ? t0 + PLAN_STEPS : p.T, K = p.K, sel = p.sel[l];
  if (sel < 0) return;
  const size_t row = (size_t)p.T * nu;
  const float* U = p.ctrl + (size_t)l * K * row;
  const double* wk = p.w + (size_t)l * K;
  float* mean = p.mean + (size_t)l * row;
  WPAR_BEGIN
    for (int j = t0 * nu + lane; j < t1 * nu; j += FB_NY) {
      if (p.temperature > 0.0) {
        double a = 0.0;
        for (int k = 0; k < K; k++) a = fma(wk[k], (double)U[(size_t)k * row + j], a);
        mean[j] = (float)(a / p.wsum[l]);
      } else {
        mean[j] = U[(size_t)sel * row + j];
      }
    }
  WPAR_END
}
