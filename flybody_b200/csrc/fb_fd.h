// fb_fd.h -- batched finite-difference Jacobians: of the stepper's transition (MuJoCo mjd_transitionFD / mjd_stepFD), of the inverse
// dynamics (mjd_inverseFD with flg_actuation = 0), and of both with respect to the per-env model parameters.  All four queries run one
// column scheme: kfd_perturb, the evaluation, kfd_diff (kfd_rows and kfd_snap beside them).
//
// One problem occupies ncol consecutive envs.  Column 0 is the nominal; column c > 0 nudges one input j: centred, columns 1 + 2j / 2 + 2j
// by +delta / -delta; forward, column 1 + j by +delta.  kfd_perturb (one warp per env) nudges the env's input in place and records the
// signed step in delta (0: the nominal, an env past the problems, or a nudge a range rules out); kfd_diff (one warp per (problem,
// input)) divides the outputs' difference between the plus and the minus env (the nominal where that side was not nudged) by the
// difference of their steps.  The two axes:
//   inputs      the state: dq [nv] (mj_integratePos), qvel [nv], then act [na] and ctrl [nu] (transition) or qacc [nv] (inverse), by
//               delta_j = eps max(1, |x_j|) (x_j the hinge angle, the free joint's translation component, qvel, act, ctrl or qacc;
//               rotational tangent coordinates: x_j = 0).  The stepper is fp32: a relative step keeps fast coordinates (the wings'
//               qvel of ~1e3 rad/s) resolved, where an absolute one would drown in their rounding.  ctrl follows MuJoCo's rule: forward
//               if the actuator is not ctrl-limited or ctrl and ctrl + delta lie in its range; backward if (centred or no forward
//               nudge) and the same holds for ctrl - delta (fd_ranged_step).
//               Or the directions of a parameter program (DevFdPrmProg, below) in the overlay row of the env.
//   evaluation  transition: the envs are copies of the problem's state-bank row (the state bank's fan-out), stepped by launch_step1 and
//               n_substeps substeps; the outputs are fd_state_diff's (mj_differentiatePos per joint for the dq rows), stored as
//               column j of row-major blocks (A [nx][nx], B [nx][nu], dxdp [nx][k]).  Sensors: kfd_snap copies each env's sensors
//               of x, the state before the step, into a per-env buffer (the velocity stage after launch_step1, the acceleration
//               stage after the first substep's step2), differenced as C, D and dsdp.
//               inverse: kfd_perturb also writes the problem's qpos, qvel and qacc rows (and, for the parameter Jacobians, its overlay
//               row, which kfd_rows saved before the fan-out overwrote it); launch_step1 and kinv_run follow; the outputs are
//               qfrc_inverse's, stored as row j of blocks in MuJoCo's transposed layout (DfDq, DfDv, DfDa [nv][nv], DfDp [k][nv]),
//               and for a state dq input the qM difference (DmDq [nv][nM]).  Sensors: kinv_sensors' per-env sensordata, differenced
//               as DsDq, DsDv, DsDa, DsDp.
// kfd_diff's outputs are data (FdBlock): inputs [j0, j0 + w) -> L values each, the difference of a per-env buffer or of the state; and
// for j = 0 the nominal column's outputs (FdNom).  Fixed-order arithmetic and no atomics: a problem's bits do not depend on its
// position in the batch or the batch size.  The parameters and buffers are the kernels' own, so DevModel / DevData, the record and the
// step kernels are untouched.
#pragma once
#include "fb_ik.h"
#include "fb_inverse.h"

// parameter directions: the host resolves a direction program (fb_fd_param_program) to overlay slots once, so the kernels know nothing
// of the field layout.  An element direction nudges one slot by delta = eps max(|theta|, floor) (the column: d / d theta); a scale
// direction multiplies each of its slots by (1 +- eps) (the column: d / ds at s = 1 of theta <- s theta).  A dof_damping entry also
// writes the row's derived M_damp slot (as kprm_draw).  The range rule is the ctrl rule on [0, inf) for the non-negative fields; a scale
// direction (0 < eps < 1) never leaves it.
enum { FB_FD_ELEMENT = 0, FB_FD_SCALE = 1 };
struct DevFdPrmProg {
  const int* kind;                        // [k] FB_FD_ELEMENT / FB_FD_SCALE (nullptr: the inputs are the state)
  const int* ptr;                         // [k + 1] direction j's entries ptr[j] .. ptr[j + 1] - 1 (an element direction has one)
  const int *slot, *mslot, *nonneg;       // per entry: the overlay slot, the derived M_damp slot (-1: none), a non-negative field
  const float* floor;                     // per entry: the floor of an element direction's step
};
// an output of kfd_diff: inputs [j0, j0 + w) -> L values each, the difference of env rows of src (stride floats apart; nullptr: the
// state, fd_state_diff); problem pr's [w][L] block (rows: input j0 + r is row r) or [L][w] block (input j0 + r is column r) at
// out + pr L w
struct FdBlock {
  const float* src; unsigned stride; int L, j0, w; bool rows, sensor;
  float* out;
};
// the nominal column's output: L values of env row pr ncol of src into out + pr L (src nullptr: the next qpos, qvel, act)
struct FdNom {
  const float* src; unsigned stride; int L;
  float* out;
};
enum { FB_FD_NBLK = 7 };                  // the inverse: DfDq, DfDv, DfDa, DmDq, DsDq, DsDv, DsDa
struct DevFdQ {
  int n, ncol, nin, centered;             // problems, envs per problem, inputs, centred
  float eps;
  float* delta;                           // [Np] the signed step of the env's column
  int ju;                                 // the first ctrl input (nin: none)
  DevFdPrmProg g;                         // the parameter directions (g.kind nullptr: the state)
  const float *qpos, *qvel, *qacc;        // [n][nq], [n][nv], [n][nv] an inverse's problems (qpos nullptr: a transition)
  float* rows;                            // [n][prm_stride] problem pr's overlay row, env pr's at call time (nullptr: none)
  DevInv inv;                             // an inverse's kernel parameter: inv.qacc holds every env's (nudged) qacc
  int nblk;
  FdBlock blk[FB_FD_NBLK];                // the first nblk are written
  FdNom nom[2];                           // the outputs, the sensor outputs
};

// the input column c nudges (-1: the nominal) and the direction it tries
FB_DEV int fd_input(const DevFdQ& p, int c, int* dir) {
  if (c == 0) { *dir = 0; return -1; }
  if (p.centered) { *dir = ((c - 1) & 1) ? -1 : 1; return (c - 1) >> 1; }
  *dir = 1; return c - 1;
}
// the signed step of a ranged input (MuJoCo's ctrl rule): fwd / back tell whether x + delta / x - delta (with x) lie in the range
FB_DEV float fd_ranged_step(const DevFdQ& p, int dir, float delta, bool fwd, bool back) {
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
// the signed step of direction j of an env whose overlay row is `row` (every lane computes the same)
FB_DEV float fdp_step(const DevFdQ& p, const DevFdPrmProg& g, const float* row, int j, int dir) {
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
// the envs input j of problem pr differences: b / a the plus / minus env, the nominal where that side was not nudged
FB_DEV void fd_pair(const DevFdQ& p, int pr, int j, int* a, int* b) {
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

// problem pr's overlay row: env pr's, saved before the fan-out overwrites it
FB_WARPFN void kfd_rows(const DevData& d, const DevFdQ& p, int pr) {
  const unsigned P = d.prm_stride;
  WPAR_BEGIN for (unsigned t = lane; t < P; t += FB_NY) p.rows[(size_t)pr * P + t] = d.prm[(size_t)pr * P + t]; WPAR_END
}
FB_WARPFN void kfd_perturb(const DevModel& m, const DevData& d, const DevFdQ& p, int e) {
  const int nq = m.nq, nv = m.nv;
  if (p.qpos) {                                   // an inverse: the problem's rows (the envs past the problems take the last one's)
    const int pr = e / p.ncol < p.n ? e / p.ncol : p.n - 1;
    const unsigned P = d.prm_stride;
    WPAR_BEGIN
      for (int i = lane; i < nq; i += FB_NY) AT(d.qpos, i) = p.qpos[(size_t)pr * nq + i];
      for (int i = lane; i < nv; i += FB_NY) { AT(d.qvel, i) = p.qvel[(size_t)pr * nv + i]; p.inv.qacc[(size_t)e * nv + i] = p.qacc[(size_t)pr * nv + i]; }
      if (p.rows) for (unsigned t = lane; t < P; t += FB_NY) d.prm[(size_t)e * P + t] = p.rows[(size_t)pr * P + t];
    WPAR_END
  }
  int dir = 0;
  const int j = e < p.n * p.ncol ? fd_input(p, e % p.ncol, &dir) : -1;
  if (p.g.kind) {                                 // a parameter direction in the env's overlay row
    float* row = d.prm + (size_t)e * d.prm_stride;
    float s = 0.0f;
    WPAR_BEGIN s = j < 0 ? 0.0f : fdp_step(p, p.g, row, j, dir); WPAR_END      // (every lane reads the row before any writes it)
    WPAR_BEGIN
      if (s != 0.0f) fdp_apply(p.g, row, j, s, lane);
      if (lane == 0) p.delta[e] = s;
    WPAR_END
    return;
  }
  WPAR_BEGIN                                      // a state input: dq (mj_integratePos), qvel, act or qacc, ctrl
    if (lane == 0) {
      float s = 0.0f;
      if (j >= 0) {
        int qa = 0, axis = -1;
        float* x;                                   // the coordinate (nullptr: a rotation)
        if (j < nv) { fd_dof(m, j, &qa, &axis); x = axis < 0 ? &AT(d.qpos, qa) : nullptr; }
        else if (j < 2 * nv) x = &AT(d.qvel, j - nv);
        else if (j < p.ju) x = (p.qpos ? p.inv.qacc + (size_t)e * nv : &AT(d.act, 0)) + (j - 2 * nv);
        else x = &AT(d.ctrl, j - p.ju);
        const float delta = p.eps * fmaxf(1.0f, x ? fabsf(*x) : 0.0f);
        if (j < p.ju) s = dir * delta;
        else {
          const int i = j - p.ju;
          const bool fwd = fd_ctrl_in_range(m, i, *x, *x + delta);
          const bool back = (p.centered || !fwd) && fd_ctrl_in_range(m, i, *x - delta, *x);
          s = fd_ranged_step(p, dir, delta, fwd, back);
        }
        if (s != 0.0f) {
          if (x) *x += s;
          else integrate_quat(d, e, qa, v3(axis == 0 ? s : 0.0f, axis == 1 ? s : 0.0f, axis == 2 ? s : 0.0f));
        }
      }
      p.delta[e] = s;
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
FB_WARPFN void kfd_diff(const DevModel& m, const DevData& d, const DevFdQ& p, int w) {
  const int pr = w / p.nin, j = w % p.nin, e0 = pr * p.ncol;
  int a, b; fd_pair(p, pr, j, &a, &b);
  const float den = p.delta[b] - p.delta[a];
  WPAR_BEGIN
#pragma unroll
    for (int o = 0; o < FB_FD_NBLK; o++) {
      const FdBlock& k = p.blk[o];
      if (o >= p.nblk || j < k.j0 || j >= k.j0 + k.w) continue;
      const int r = j - k.j0;
      float* out = k.out + (size_t)pr * k.L * k.w + (k.rows ? (size_t)r * k.L : (size_t)r);
      const size_t step = k.rows ? 1 : k.w;
      for (int i = lane; i < k.L; i += FB_NY)
        out[i * step] = a == b ? 0.0f : (k.src ? k.src[(size_t)b * k.stride + i] - k.src[(size_t)a * k.stride + i] : fd_state_diff(m, d, b, a, i)) / den;
    }
    if (j == 0) {
      const int e = e0, nq = m.nq, nv = m.nv;
#pragma unroll
      for (int o = 0; o < 2; o++) {
        const FdNom& c = p.nom[o];
        for (int i = lane; i < c.L; i += FB_NY)
          c.out[(size_t)pr * c.L + i] = c.src ? c.src[(size_t)e0 * c.stride + i] : i < nq ? AT(d.qpos, i) : (i < nq + nv ? AT(d.qvel, i - nq) : AT(d.act, i - nq - nv));
      }
    }
  WPAR_END
}

// the sensors of one stage (acc: the acceleration stage) of env e into its row of snap [Np][nsd]
FB_WARPFN void kfd_snap(const DevModel& m, const DevData& d, float* snap, int e, bool acc) {
  float* out = snap + (size_t)e * m.nsensordata;
  WPAR_BEGIN
    for (int s = lane; s < m.nsensor; s += FB_NY)
      if (sens_acc_stage(m.sensor_type[s]) == acc) for (int k = 0; k < m.sensor_dim[s]; k++) out[m.sensor_adr[s] + k] = AT(d.sensordata, m.sensor_adr[s] + k);
  WPAR_END
}
