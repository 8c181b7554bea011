// fb_sid.h -- batched system identification (fb_sid_accumulate): the weighted normal equations of L fit problems, accumulated on the
// device from what the last parameter-Jacobian query left there, so nothing of the Jacobians is read back to the host.
//   transition  (after fb_fd_param_transition) FD problem i: r = x'_pred (-) x'_obs, nx = 2 nv + na rows, x'_pred the nominal column's
//               next state (FdNom), (-) transition_fd's tangent (fd_dof / fd_subquat per dof: mj_differentiatePos(x'_obs qpos,
//               x'_pred qpos), then the qvel and act differences: roll_tangent's, for two rows); J = dxdp [nx][k] of the query's block
//   inverse     (after fb_fd_param_inverse) r = qfrc_inverse - target, nv rows; J = DfDp^T, read in place from its [k][nv] block
// Per fit problem l, over the FD problems mapped to it, in fp64 from the fp32 inputs (W a diagonal weight [rows], c_i > 0 a per-transition
// weight; c_i <= 0 or NaN: the transition is left out):
//   H_l += c_i J^T W J,  g_l += c_i J^T W r,  cost_l += c_i r^T W r / 2,  count_l += 1
// A transition whose residual or Jacobian is not finite, or (transition) whose nominal env set the bad-state flag (bit value 1 of d.flags,
// as kplan_cost reads it), adds +inf to cost_l and 1 to bad_l, and nothing to H_l or g_l.
// Determinism: no atomics; each transition's term is computed alone (lane partials, summed in lane order) and added to the running fp64
// sums in transition order (ksid_sum walks a fit problem's transitions serially), so a problem's bits depend on neither its index, nor L,
// nor the other problems' transitions, nor on how its transitions are split across calls.
#pragma once
#include "fb_fd.h"

struct DevSid {
  int L, k, rows, nr;                       // fit problems, directions, residual rows (nx or nv), row width of x'_pred and x'_obs
  int ncol;                                 // envs per FD problem (the nominal env of problem i: i ncol)
  bool inverse, reset;                      // the query; start the sums from 0
  const float *J, *pred, *target;           // the query's block and nominal outputs; the targets [n][nr] (nullptr: 0, an inverse)
  const float* sw;                          // [n] c_i (nullptr: 1)
  const double* W;                          // [rows]
  double *res, *tcost;                      // [n][rows] the residuals, [n] each transition's c_i r^T W r / 2 (+inf: bad)
  int* tbad;                                // [n]
  const int *order, *ptr;                   // fit problem l's FD problems: order[ptr[l] .. ptr[l + 1]), in transition order
  double *H, *g, *cost;                     // [L][k][k] (both triangles), [L][k], [L]
  int *count, *bad;                         // [L]
};

FB_DEV bool sid_finite(double v) { return v - v == 0.0; }
// entry (r, a) of FD problem i's J
FB_DEV float sid_J(const DevSid& p, int i, int r, int a) {
  return p.inverse ? p.J[((size_t)i * p.k + a) * p.rows + r] : p.J[((size_t)i * p.rows + r) * p.k + a];
}
// residual row c of a transition: x (x'_pred) minus y (x'_obs), rows [nr] in qpos, qvel, act order
FB_DEV double sid_tangent(const DevModel& m, const float* x, const float* y, int c) {
  const int nq = m.nq, nv = m.nv;
  if (c < nv) {
    int qa, axis; fd_dof(m, c, &qa, &axis);
    if (axis >= 0) return comp(fd_subquat(q4(y[qa], y[qa + 1], y[qa + 2], y[qa + 3]), q4(x[qa], x[qa + 1], x[qa + 2], x[qa + 3])), axis);
    return (double)x[qa] - (double)y[qa];
  }
  return (double)x[nq + c - nv] - (double)y[nq + c - nv];
}

// the residual, cost term and bad mark of FD problem i = order[t]
FB_WARPFN void ksid_resid(const DevModel& m, const DevData& d, const DevSid& p, int t) {
  const int i = p.order[t], k = p.k;
  const float* x = p.pred + (size_t)i * p.nr;
  const float* y = p.target ? p.target + (size_t)i * p.nr : nullptr;
  double* r = p.res + (size_t)i * p.rows;
  LREG(double, part); LREG(int, nf);
  WPAR_BEGIN
    double a = 0.0; int bad = 0;
    for (int c = lane; c < p.rows; c += FB_NY) {
      const double v = p.inverse ? (double)x[c] - (y ? (double)y[c] : 0.0) : sid_tangent(m, x, y, c);
      r[c] = v;
      bad |= !sid_finite(v);
      for (int j = 0; j < k; j++) bad |= !sid_finite((double)sid_J(p, i, c, j));
      a = fma(p.W[c] * v, v, a);
    }
    L(part) = a; L(nf) = bad;
  WPAR_END
  WPAR_BEGIN
    double sum = 0.0; int bad = 0;
    for (int l = 0; l < FB_NY; l++) { sum += SHF(part, l); bad |= SHF(nf, l); }
    if (lane == 0) {
      if (!p.inverse) bad |= d.flags[(unsigned)(i * p.ncol) * d.rec] & 1;
      const double c = p.sw ? (double)p.sw[i] : 1.0;
      p.tbad[i] = bad != 0;
      p.tcost[i] = bad ? HUGE_VAL : c * (0.5 * sum);
    }
  WPAR_END
}

// entry o of fit problem l (w = l E + o, E = k (k + 1) / 2 + k + 1): H(a, b) for a <= b (row-major upper triangle, written to both
// triangles), then g(a), then cost, count and bad
FB_WARPFN void ksid_sum(const DevSid& p, int w) {
  const int k = p.k, nh = k * (k + 1) / 2, E = nh + k + 1, l = w / E, o = w - l * E;
  int a = 0, b = 0;
  if (o < nh) { int t = o; while (t >= k - a) { t -= k - a; a++; } b = a + t; }
  else if (o < nh + k) a = o - nh;
  const int kind = o < nh ? 0 : o < nh + k ? 1 : 2;
  double* out = kind == 0 ? p.H + ((size_t)l * k + a) * k + b : kind == 1 ? p.g + (size_t)l * k + a : p.cost + l;
  double acc = p.reset ? 0.0 : *out;        // (lane 0's is the sum; the others only follow the loop)
  int cnt = p.reset ? 0 : p.count[l], nbad = p.reset ? 0 : p.bad[l];
  // column a of J: entry (row, a) of FD problem i at J + i rows k + a sa + row sr (inverse: DfDp [k][nv]; transition: dxdp [nx][k])
  const size_t sa = p.inverse ? p.rows : 1, sr = p.inverse ? 1 : p.k;
  LREG(double, part);
  for (int t = p.ptr[l]; t < p.ptr[l + 1]; t++) {
    const int i = p.order[t];
    const float c = p.sw ? p.sw[i] : 1.0f;
    if (!(c > 0.0f)) continue;
    if (kind == 2) { acc += p.tcost[i]; cnt++; nbad += p.tbad[i]; continue; }
    if (p.tbad[i]) continue;
    const float* J = p.J + (size_t)i * p.rows * k;
    const float *ja = J + a * sa, *jb = J + b * sa;
    const double* r = p.res + (size_t)i * p.rows;
    WPAR_BEGIN
      double s = 0.0;
      if (kind == 0) for (int row = lane; row < p.rows; row += FB_NY) s = fma((double)ja[row * sr] * p.W[row], (double)jb[row * sr], s);
      else for (int row = lane; row < p.rows; row += FB_NY) s = fma((double)ja[row * sr] * p.W[row], r[row], s);
      L(part) = s;
    WPAR_END
    WPAR_BEGIN
      double sum = 0.0;
      for (int y = 0; y < FB_NY; y++) sum += SHF(part, y);
      if (lane == 0) acc += (double)c * sum;
    WPAR_END
  }
  WPAR_BEGIN
    if (lane == 0) {
      *out = acc;
      if (kind == 0 && a != b) p.H[((size_t)l * k + b) * k + a] = acc;
      if (kind == 2) { p.count[l] = cnt; p.bad[l] = nbad; }
    }
  WPAR_END
}
