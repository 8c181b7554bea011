// fb_fd.h -- batched finite-difference Jacobians: of the stepper's transition (MuJoCo mjd_transitionFD / mjd_stepFD; DevFd) and of
// the inverse dynamics (mjd_inverseFD with flg_actuation = 0; DevFdInv), and of both with respect to the per-env model parameters
// (DevFdPrm, DevFdPrmInv; below).  All use one column scheme (FdCols):
//
// One problem occupies ncol consecutive envs.  Column 0 is the nominal; column c > 0 nudges one input j: centred, columns 1 + 2j / 2 + 2j
// by +delta / -delta; forward, column 1 + j by +delta.  delta_j = eps max(1, |x_j|), with x_j the hinge angle, the free joint's
// translation component, qvel, act, ctrl or qacc (rotational tangent coordinates: x_j = 0).  The stepper is fp32: a relative step keeps
// fast coordinates (the wings' qvel of ~1e3 rad/s) resolved, where an absolute one would drown in their rounding.  A perturb kernel (one
// warp per env) nudges the env's input in place (mj_integratePos for dq) and records the signed step in delta (0: the nominal, an env
// past the problems, or a ctrl nudge its range rules out); a diff kernel (one warp per (problem, input)) divides the outputs' difference
// between the plus and the minus env (the nominal where that side was not nudged) by the difference of their steps.
//   transition: x = (dq [nv], qvel [nv], act [na]), u = ctrl [nu]; the envs are copies of the problem's state row (the state bank's
//               fan-out), stepped n_substeps substeps.  The ctrl rule is MuJoCo's, evaluated in kfd_perturb only: forward if the
//               actuator is not ctrl-limited or ctrl and ctrl + delta both lie in its range; backward if (centred or no forward nudge)
//               and the same holds for ctrl - delta.  kfd_diff writes column j of row-major A [nx][nx] or B [nx][nu], mj_differentiatePos
//               per joint for the dq rows; column 0's warp copies out the nominal next state.
//   inverse:    inputs (dq [nv], qvel [nv], qacc [nv]); kfdi_perturb writes the problem's qpos, qvel and qacc rows (the envs past the
//               problems take the last one's), launch_step1 and kinv_run (on DevFdInv::inv) follow, and kfdi_diff writes row i (MuJoCo's
//               transposed layout: the derivative with respect to input i) of DfDq, DfDv or DfDa, and of DmDq (the sparse qM order) for
//               a dq input; input 0's warp copies out the nominal qfrc_inverse.
// Fixed-order arithmetic and no atomics: a problem's bits do not depend on its position in the batch or the batch size.  The parameters
// and buffers are the kernels' own, so DevModel / DevData, the record and the step kernels are untouched.
#pragma once
#include "fb_ik.h"
#include "fb_inverse.h"

struct FdCols {
  int n, ncol, nin, centered;             // problems, envs per problem, inputs, centred
  float eps;
  float* delta;                           // [Np] the signed step of the env's column
};
struct DevFd : FdCols {
  int nx;                                 // state size 2 nv + na (inputs nx + nu)
  float *A, *B;                           // [n][nx][nx], [n][nx][nu]
  float* next;                            // [n][nq + nv + na] the nominal column's next qpos, qvel, act
};

// the input column c nudges (-1: the nominal) and the direction it tries
FB_DEV int fd_input(const FdCols& p, int c, int* dir) {
  if (c == 0) { *dir = 0; return -1; }
  if (p.centered) { *dir = ((c - 1) & 1) ? -1 : 1; return (c - 1) >> 1; }
  *dir = 1; return c - 1;
}
// the signed step of a ranged input (MuJoCo's ctrl rule): fwd / back tell whether x + delta / x - delta (with x) lie in the range
FB_DEV float fd_ranged_step(const FdCols& p, int dir, float delta, bool fwd, bool back) {
  return p.centered ? (dir > 0 ? (fwd ? delta : 0.0f) : (back ? -delta : 0.0f)) : (fwd ? delta : (back ? -delta : 0.0f));
}
FB_DEV bool fd_ctrl_in_range(const DevModel& m, int i, float a, float b) {
  if (!MLD(m.actuator_ctrllimited[i])) return true;
  const float lo = MLD(m.actuator_ctrlrange[2 * i]), hi = MLD(m.actuator_ctrlrange[2 * i + 1]);
  return a >= lo && a <= hi && b >= lo && b <= hi;
}
// dof k's joint: its type, the qpos address of the coordinate (hinge, translation) or of the quaternion (rotation), and the rotation axis
// (-1: not a rotational coordinate)
FB_DEV void fd_dof(const DevModel& m, int k, int* qa, int* axis) {
  const int j = MLD(m.dof_jntid[k]), t = MLD(m.jnt_type[j]), c = k - MLD(m.jnt_dofadr[j]);
  *qa = MLD(m.jnt_qposadr[j]); *axis = -1;
  if (t == FB_JNT_FREE) { if (c < 3) *qa += c; else { *qa += 3; *axis = c - 3; } }
  else if (t == FB_JNT_BALL) *axis = c;
}
// nudge input j of env e in place: dq (j < nv), qvel (j < 2 nv) or the caller's coordinate xhi (inputs past 2 nv).  step(x, delta_j)
// gives the signed step (0: no nudge; x nullptr for a rotation).  -> that step
template <typename S> FB_DEV float fd_nudge(const DevModel& m, const DevData& d, const FdCols& p, int e, int j, float* xhi, S step) {
  const int nv = m.nv;
  int qa = 0, axis = -1;
  float* x = xhi;                                 // the coordinate (nullptr: a rotation)
  if (j < nv) { fd_dof(m, j, &qa, &axis); x = axis < 0 ? &AT(d.qpos, qa) : nullptr; }
  else if (j < 2 * nv) x = &AT(d.qvel, j - nv);
  const float s = step(x, p.eps * fmaxf(1.0f, x ? fabsf(*x) : 0.0f));
  if (s != 0.0f) {
    if (x) *x += s;
    else integrate_quat(d, e, qa, v3(axis == 0 ? s : 0.0f, axis == 1 ? s : 0.0f, axis == 2 ? s : 0.0f));
  }
  return s;
}
// the envs input j of problem pr differences: b / a the plus / minus env, the nominal where that side was not nudged
FB_DEV void fd_pair(const FdCols& p, int pr, int j, int* a, int* b) {
  const int e0 = pr * p.ncol;
  *a = *b = e0;
  if (p.centered) {
    const int ep = e0 + 1 + 2 * j, em = ep + 1;
    if (p.delta[ep] != 0.0f) *b = ep;
    if (p.delta[em] != 0.0f) *a = em;
  } else {
    const int ec = e0 + 1 + j;
    if (p.delta[ec] > 0.0f) *b = ec;
    if (p.delta[ec] < 0.0f) *a = ec;
  }
}

FB_WARPFN void kfd_perturb(const DevModel& m, const DevData& d, const DevFd& p, int e) {
  WPAR_BEGIN
    if (lane == 0) {
      int dir = 0;
      const int j = e < p.n * p.ncol ? fd_input(p, e % p.ncol, &dir) : -1, nv = m.nv;
      float step = 0.0f;
      if (j >= 0) {
        float* xhi = j < 2 * nv ? nullptr : j < p.nx ? &AT(d.act, j - 2 * nv) : &AT(d.ctrl, j - p.nx);
        step = fd_nudge(m, d, p, e, j, xhi, [&](const float* x, float delta) {
          if (j < p.nx) return dir * delta;
          const int i = j - p.nx;
          const bool fwd = fd_ctrl_in_range(m, i, *x, *x + delta);
          const bool back = (p.centered || !fwd) && fd_ctrl_in_range(m, i, *x - delta, *x);
          return fd_ranged_step(p, dir, delta, fwd, back);
        });
      }
      p.delta[e] = step;
    }
  WPAR_END
}

// MuJoCo mju_subQuat(q2, q1): the body-frame rotation vector v with q1 exp(v) = q2.  Equal quaternions give exactly 0: in fp32 the
// vector part of conj(q) q is rounding noise of ~1e-8, which over a step of 1e-3 would put ~1e-5 into columns that do not reach q.
FB_DEV V3 fd_subquat(Q4 q1, Q4 q2) {
  if (q1.w == q2.w && q1.x == q2.x && q1.y == q2.y && q1.z == q2.z) return v3(0, 0, 0);
  const Q4 dq = qmul(q4(q1.w, -q1.x, -q1.y, -q1.z), q2);
  const V3 ax = v3(dq.x, dq.y, dq.z);
  const float s = norm(ax);
  if (!(s > 0.0f)) return v3(0, 0, 0);
  float ang = 2.0f * atan2f(s, dq.w);
  if (ang > 3.14159265358979f) ang -= 2.0f * 3.14159265358979f;
  return ax * (ang / s);
}
FB_DEV Q4 fd_quat(const DevData& d, int e, int qa) { return q4(AT(d.qpos, qa), AT(d.qpos, qa + 1), AT(d.qpos, qa + 2), AT(d.qpos, qa + 3)); }
// state row i: env b's next state minus env a's (mj_differentiatePos for the dq rows)
FB_DEV float fd_state_diff(const DevModel& m, const DevData& d, int b, int a, int i) {
  const int nv = m.nv;
  if (i < nv) {
    int qa, axis; fd_dof(m, i, &qa, &axis);
    if (axis >= 0) return comp(fd_subquat(fd_quat(d, a, qa), fd_quat(d, b, qa)), axis);
    return d.qpos[(unsigned)b * d.rec + qa] - d.qpos[(unsigned)a * d.rec + qa];
  }
  const float* f = i < 2 * nv ? d.qvel + (i - nv) : d.act + (i - 2 * nv);
  return f[(unsigned)b * d.rec] - f[(unsigned)a * d.rec];
}
FB_WARPFN void kfd_diff(const DevModel& m, const DevData& d, const DevFd& p, int w) {
  const int pr = w / p.nin, j = w % p.nin, e0 = pr * p.ncol;
  int a, b; fd_pair(p, pr, j, &a, &b);
  const float den = p.delta[b] - p.delta[a];
  float* out = j < p.nx ? p.A + (size_t)pr * p.nx * p.nx + j : p.B + (size_t)pr * p.nx * (p.nin - p.nx) + (j - p.nx);
  const int stride = j < p.nx ? p.nx : p.nin - p.nx;
  const int nq = m.nq, nv = m.nv, nnext = nq + nv + m.na;
  WPAR_BEGIN
    for (int i = lane; i < p.nx; i += FB_NY) out[(size_t)i * stride] = a == b ? 0.0f : fd_state_diff(m, d, b, a, i) / den;
    if (j == 0) {
      float* nx = p.next + (size_t)pr * nnext;
      const int e = e0;
      for (int i = lane; i < nnext; i += FB_NY) nx[i] = i < nq ? AT(d.qpos, i) : (i < nq + nv ? AT(d.qvel, i - nq) : AT(d.act, i - nq - nv));
    }
  WPAR_END
}

// ---- inverse-dynamics Jacobians: of qfrc_inverse = M qacc + qfrc_bias - qfrc_passive - qfrc_constraint (fb_inverse.h) and of qM
struct DevFdInv : FdCols {
  float *qpos, *qvel, *qacc;              // [cap][nq], [cap][nv], [cap][nv] the problems
  DevInv inv;                             // the inverse kernel's parameter: inv.qacc holds every env's (nudged) qacc
  float *DfDq, *DfDv, *DfDa;              // [n][nv][nv]: DfDq[i][j] = d qfrc_inverse_j / d dq_i
  float* DmDq;                            // [n][nv][nM]: d qM / d dq_i in the sparse qM order
  float* qfrc;                            // [n][nv] the nominal column's qfrc_inverse
};

FB_WARPFN void kfdi_perturb(const DevModel& m, const DevData& d, const DevFdInv& p, int e) {
  const int nq = m.nq, nv = m.nv, pr = e / p.ncol < p.n ? e / p.ncol : p.n - 1;
  float* qa_e = p.inv.qacc + (size_t)e * nv;
  WPAR_BEGIN
    for (int i = lane; i < nq; i += FB_NY) AT(d.qpos, i) = p.qpos[(size_t)pr * nq + i];
    for (int i = lane; i < nv; i += FB_NY) { AT(d.qvel, i) = p.qvel[(size_t)pr * nv + i]; qa_e[i] = p.qacc[(size_t)pr * nv + i]; }
  WPAR_END
  WPAR_BEGIN
    if (lane == 0) {
      int dir = 0;
      const int j = e < p.n * p.ncol ? fd_input(p, e % p.ncol, &dir) : -1;
      p.delta[e] = j < 0 ? 0.0f : fd_nudge(m, d, p, e, j, j < 2 * nv ? nullptr : qa_e + (j - 2 * nv), [&](const float*, float delta) { return dir * delta; });
    }
  WPAR_END
}

FB_WARPFN void kfdi_diff(const DevModel& m, const DevData& d, const DevFdInv& p, int w) {
  const int nv = m.nv, nM = m.nM, pr = w / p.nin, i = w % p.nin, e0 = pr * p.ncol;
  int a, b; fd_pair(p, pr, i, &a, &b);
  const float den = p.delta[b] - p.delta[a];
  const int blk = i / nv, r = i % nv;
  float* out = (blk == 0 ? p.DfDq : blk == 1 ? p.DfDv : p.DfDa) + ((size_t)pr * nv + r) * nv;
  const float *fb = p.inv.qfrc_inverse + (size_t)b * nv, *fa = p.inv.qfrc_inverse + (size_t)a * nv;
  WPAR_BEGIN
    for (int k = lane; k < nv; k += FB_NY) out[k] = (fb[k] - fa[k]) / den;
    if (blk == 0) {
      float* dm = p.DmDq + ((size_t)pr * nv + r) * nM;
      const float *mb = d.qM + (size_t)b * d.rec, *ma = d.qM + (size_t)a * d.rec;
      for (int t = lane; t < nM; t += FB_NY) dm[t] = (mb[t] - ma[t]) / den;
    }
    if (i == 0) {
      const float* f0 = p.inv.qfrc_inverse + (size_t)e0 * nv;
      for (int k = lane; k < nv; k += FB_NY) p.qfrc[(size_t)pr * nv + k] = f0[k];
    }
  WPAR_END
}

// ---- sensor Jacobians (fb_query_sensors on).  Their own parameters beside DevFd / DevFdInv, whose kernels keep their layout.
//   transition: C = ds/dx [n][nsd][nx] and D = ds/du [n][nsd][nu] (row-major, as A and B), s the sensors of x, the state before the
//               step (MuJoCo's definition).  kfd_snap copies an env's sensors of one stage into snap: the velocity stage after the
//               launch_step1 of the nudged x, the acceleration stage after the first substep's step2 (which the step1 of x' leaves).
//               kfd_sdiff writes column j of C or D and, for j = 0, the nominal sensordata.
//   inverse:    DsDq, DsDv, DsDa [n][nv][nsd] (MuJoCo's transposed layout); kinv_sensors writes every env's sensordata after the
//               inverse, kfdi_sdiff writes row i of one block and, for i = 0, the nominal sensordata.
struct DevFdSens {
  DevFd fd;
  float* snap;                            // [Np][nsd] the sensors of each env's x
  float *C, *D;                           // [n][nsd][nx], [n][nsd][nu]
  float* sensordata;                      // [n][nsd] the nominal column's
};
FB_WARPFN void kfd_snap(const DevModel& m, const DevData& d, const DevFdSens& p, int e, bool acc) {
  float* out = p.snap + (size_t)e * m.nsensordata;
  WPAR_BEGIN
    for (int s = lane; s < m.nsensor; s += FB_NY)
      if (sens_acc_stage(m.sensor_type[s]) == acc) for (int k = 0; k < m.sensor_dim[s]; k++) out[m.sensor_adr[s] + k] = AT(d.sensordata, m.sensor_adr[s] + k);
  WPAR_END
}
FB_WARPFN void kfd_sdiff(const DevModel& m, const DevFdSens& p, int w) {
  const FdCols& c = p.fd;
  const int pr = w / c.nin, j = w % c.nin, nsd = m.nsensordata, nx = p.fd.nx, nu = c.nin - nx;
  int a, b; fd_pair(c, pr, j, &a, &b);
  const float den = c.delta[b] - c.delta[a];
  float* out = j < nx ? p.C + (size_t)pr * nsd * nx + j : p.D + (size_t)pr * nsd * nu + (j - nx);
  const int stride = j < nx ? nx : nu;
  const float *sb = p.snap + (size_t)b * nsd, *sa = p.snap + (size_t)a * nsd;
  WPAR_BEGIN
    for (int i = lane; i < nsd; i += FB_NY) out[(size_t)i * stride] = a == b ? 0.0f : (sb[i] - sa[i]) / den;
    if (j == 0) for (int i = lane; i < nsd; i += FB_NY) p.sensordata[(size_t)pr * nsd + i] = p.snap[(size_t)pr * c.ncol * nsd + i];
  WPAR_END
}
struct DevFdInvSens {
  DevFdInv fdi;
  const float* sens;                      // [Np][nsd] every env's sensordata (kinv_sensors on fdi.inv)
  float *DsDq, *DsDv, *DsDa;              // [n][nv][nsd]: DsDq[i][k] = d sensordata_k / d dq_i
  float* sensordata;                      // [n][nsd] the nominal column's
};
FB_WARPFN void kfdi_sdiff(const DevModel& m, const DevFdInvSens& p, int w) {
  const FdCols& c = p.fdi;
  const int nv = m.nv, nsd = m.nsensordata, pr = w / c.nin, i = w % c.nin;
  int a, b; fd_pair(c, pr, i, &a, &b);
  const float den = c.delta[b] - c.delta[a];
  const int blk = i / nv, r = i % nv;
  float* out = (blk == 0 ? p.DsDq : blk == 1 ? p.DsDv : p.DsDa) + ((size_t)pr * nv + r) * nsd;
  const float *sb = p.sens + (size_t)b * nsd, *sa = p.sens + (size_t)a * nsd;
  WPAR_BEGIN
    for (int k = lane; k < nsd; k += FB_NY) out[k] = (sb[k] - sa[k]) / den;
    if (i == 0) for (int k = lane; k < nsd; k += FB_NY) p.sensordata[(size_t)pr * nsd + k] = p.sens[(size_t)pr * c.ncol * nsd + k];
  WPAR_END
}

// ---- parameter Jacobians (fb_fd_param_*): the inputs are directions in the model-parameter overlay (DevData::prm) instead of the
// state.  The host resolves a direction program (fb_fd_param_program) to overlay slots once, so the kernels know nothing of the field
// layout.  An element direction nudges one slot by delta = eps max(|theta|, floor) (the column: d / d theta); a scale direction
// multiplies each of its slots by (1 +- eps) (the column: d / ds at s = 1 of theta <- s theta).  A dof_damping entry also writes the
// row's derived M_damp slot (as kprm_draw).  The range rule is the ctrl rule (fd_ranged_step) on [0, inf) for the non-negative fields;
// a scale direction (0 < eps < 1) never leaves it.  The columns (FdCols, nin = k directions) and fd_pair are the state columns'.
//   transition: kfdp_perturb nudges the fanned-out rows' overlay in place; kfdp_diff writes column j of dxdp [n][nx][k] (row-major as
//               B, fd_state_diff) and, for j = 0, the nominal next state; the sensors reuse kfd_snap and kfd_sdiff (DevFdSens with
//               nx = 0: dsdp [n][nsd][k] in the D slot).
//   inverse:    kfdpi_rows saves env pr's overlay row for problem pr (the fan-out overwrites it); kfdpi_perturb writes an env's
//               qpos, qvel, qacc and row and nudges it; kfdpi_diff writes row j of DfDp [n][k][nv] (transposed as DfDq) and of DsDp
//               [n][k][nsd], and for j = 0 the nominal qfrc_inverse and sensordata.
enum { FB_FD_ELEMENT = 0, FB_FD_SCALE = 1 };
struct DevFdPrmProg {
  const int* kind;                        // [k] FB_FD_ELEMENT / FB_FD_SCALE
  const int* ptr;                         // [k + 1] direction j's entries ptr[j] .. ptr[j + 1] - 1 (an element direction has one)
  const int *slot, *mslot, *nonneg;       // per entry: the overlay slot, the derived M_damp slot (-1: none), a non-negative field
  const float* floor;                     // per entry: the floor of an element direction's step
};
struct DevFdPrm : FdCols {
  DevFdPrmProg g;
  int nx;                                 // 2 nv + na
  float* dxdp;                            // [n][nx][k]
  float* next;                            // [n][nq + nv + na] the nominal column's next qpos, qvel, act
};
// the signed step of direction j of an env whose overlay row is `row` (every lane computes the same)
FB_DEV float fdp_step(const FdCols& p, const DevFdPrmProg& g, const float* row, int j, int dir) {
  if (g.kind[j] == FB_FD_SCALE) return dir * p.eps;
  const int t = g.ptr[j];
  const float x = row[g.slot[t]], delta = p.eps * fmaxf(fabsf(x), g.floor[t]);
  const bool nn = g.nonneg[t] != 0, fwd = !nn || x + delta >= 0.0f;
  const bool back = (p.centered || !fwd) && (!nn || x - delta >= 0.0f);
  return fd_ranged_step(p, dir, delta, fwd, back);
}
// lane's share of moving direction j of `row` by the step s
FB_DEV void fdp_apply(const DevFdPrmProg& g, float* row, int j, float s, int lane) {
  const bool scale = g.kind[j] == FB_FD_SCALE;
  for (int t = g.ptr[j] + lane; t < g.ptr[j + 1]; t += FB_NY) {
    const float v = row[g.slot[t]], w = scale ? fmaf(v, s, v) : v + s;
    row[g.slot[t]] = w;
    if (g.mslot[t] >= 0) row[g.mslot[t]] = w;
  }
}
// nudge env e's overlay row for its column and record the step in delta
FB_WARPFN void fdp_nudge_row(const DevData& d, const FdCols& p, const DevFdPrmProg& g, int e) {
  float* row = d.prm + (size_t)e * d.prm_stride;
  int dir = 0;
  const int j = e < p.n * p.ncol ? fd_input(p, e % p.ncol, &dir) : -1;
  float s = 0.0f;
  WPAR_BEGIN s = j < 0 ? 0.0f : fdp_step(p, g, row, j, dir); WPAR_END      // (every lane reads the row before any writes it)
  WPAR_BEGIN
    if (s != 0.0f) fdp_apply(g, row, j, s, lane);
    if (lane == 0) p.delta[e] = s;
  WPAR_END
}
FB_WARPFN void kfdp_perturb(const DevData& d, const DevFdPrm& p, int e) { fdp_nudge_row(d, p, p.g, e); }
FB_WARPFN void kfdp_diff(const DevModel& m, const DevData& d, const DevFdPrm& p, int w) {
  const int pr = w / p.nin, j = w % p.nin, e0 = pr * p.ncol;
  int a, b; fd_pair(p, pr, j, &a, &b);
  const float den = p.delta[b] - p.delta[a];
  float* out = p.dxdp + (size_t)pr * p.nx * p.nin + j;
  const int nq = m.nq, nv = m.nv, nnext = nq + nv + m.na;
  WPAR_BEGIN
    for (int i = lane; i < p.nx; i += FB_NY) out[(size_t)i * p.nin] = a == b ? 0.0f : fd_state_diff(m, d, b, a, i) / den;
    if (j == 0) {
      float* nx = p.next + (size_t)pr * nnext;
      const int e = e0;
      for (int i = lane; i < nnext; i += FB_NY) nx[i] = i < nq ? AT(d.qpos, i) : (i < nq + nv ? AT(d.qvel, i - nq) : AT(d.act, i - nq - nv));
    }
  WPAR_END
}

struct DevFdPrmInv : FdCols {
  DevFdPrmProg g;
  const float *qpos, *qvel, *qacc;        // [cap][nq], [cap][nv], [cap][nv] the problems
  float* rows;                            // [cap][prm_stride] problem pr's overlay row: env pr's at call time
  DevInv inv;                             // the inverse kernel's parameter (inv.qacc: every env's qacc)
  float* DfDp;                            // [n][k][nv]: DfDp[j][i] = d qfrc_inverse_i / d direction j
  float* qfrc;                            // [n][nv] the nominal column's qfrc_inverse
  const float* sens;                      // [Np][nsd] every env's sensordata (kinv_sensors), nullptr: sensors off
  float *DsDp, *sensordata;               // [n][k][nsd], [n][nsd]
};
FB_WARPFN void kfdpi_rows(const DevData& d, const DevFdPrmInv& p, int pr) {
  const unsigned P = d.prm_stride;
  WPAR_BEGIN for (unsigned t = lane; t < P; t += FB_NY) p.rows[(size_t)pr * P + t] = d.prm[(size_t)pr * P + t]; WPAR_END
}
FB_WARPFN void kfdpi_perturb(const DevModel& m, const DevData& d, const DevFdPrmInv& p, int e) {
  const int nq = m.nq, nv = m.nv, pr = e / p.ncol < p.n ? e / p.ncol : p.n - 1;
  const unsigned P = d.prm_stride;
  WPAR_BEGIN
    for (int i = lane; i < nq; i += FB_NY) AT(d.qpos, i) = p.qpos[(size_t)pr * nq + i];
    for (int i = lane; i < nv; i += FB_NY) { AT(d.qvel, i) = p.qvel[(size_t)pr * nv + i]; p.inv.qacc[(size_t)e * nv + i] = p.qacc[(size_t)pr * nv + i]; }
    for (unsigned t = lane; t < P; t += FB_NY) d.prm[(size_t)e * P + t] = p.rows[(size_t)pr * P + t];
  WPAR_END
  fdp_nudge_row(d, p, p.g, e);
}
FB_WARPFN void kfdpi_diff(const DevModel& m, const DevFdPrmInv& p, int w) {
  const int nv = m.nv, nsd = m.nsensordata, pr = w / p.nin, j = w % p.nin, e0 = pr * p.ncol;
  int a, b; fd_pair(p, pr, j, &a, &b);
  const float den = p.delta[b] - p.delta[a];
  float* out = p.DfDp + ((size_t)pr * p.nin + j) * nv;
  const float *fb = p.inv.qfrc_inverse + (size_t)b * nv, *fa = p.inv.qfrc_inverse + (size_t)a * nv;
  WPAR_BEGIN
    for (int k = lane; k < nv; k += FB_NY) out[k] = a == b ? 0.0f : (fb[k] - fa[k]) / den;
    if (j == 0) for (int k = lane; k < nv; k += FB_NY) p.qfrc[(size_t)pr * nv + k] = p.inv.qfrc_inverse[(size_t)e0 * nv + k];
    if (p.sens) {
      float* so = p.DsDp + ((size_t)pr * p.nin + j) * nsd;
      const float *sb = p.sens + (size_t)b * nsd, *sa = p.sens + (size_t)a * nsd;
      for (int k = lane; k < nsd; k += FB_NY) so[k] = a == b ? 0.0f : (sb[k] - sa[k]) / den;
      if (j == 0) for (int k = lane; k < nsd; k += FB_NY) p.sensordata[(size_t)pr * nsd + k] = p.sens[(size_t)e0 * nsd + k];
    }
  WPAR_END
}
