// fb_rollout.h -- batched rollouts (MuJoCo mujoco.rollout.rollout; fb_rollout): n rollouts of T control steps, rollout i in env i from a
// state-bank row, driven by its own control sequence and, optionally, a time-varying linear feedback law from a bank of L laws.
// A control step is three launches: kroll_input (one warp per env) writes the step's inputs into the env's record, step_run replays the
// step graph (n_substeps x [step2 ; step1], ctrl held), kroll_record (one warp per rollout) copies the state after the step into the
// rollout's row t.  DevRoll is the kernels' own parameter: DevData and the step kernels are untouched, so the step graph is captured
// once and replayed for every control step.  Fixed-order arithmetic and no atomics: a rollout's bits do not depend on its slot, its
// position in the batch or the batch size.
//   inputs:   ctrl [n][T][nu] (written as given: the actuation stage clamps ctrl-limited actuators, as for d->ctrl); optional
//             qfrc_applied [n][T][nv] and xfrc_applied [n][T][nbody][6] (nullptr: the row's applied forces persist, as in mjData).
//             Envs past n take the last rollout's sequence (the state bank's fan-out).
//   feedback: ctrl = u_t + K_t (x_t (-) xref_t), x_t the env's state before step t, xref and K the rows of law[i] (law 0 without
//             a law list) in the bank xref [L][T][nq + nv + na], K [L][T][nu][nx] with nx = 2 nv + na; (-) is transition_fd's tangent
//             (fd_dof / fd_subquat per dof, mj_differentiatePos(xref qpos, qpos), then the qvel and act differences), so gains from a
//             Riccati recursion on its A and B apply as they are.  The tangent goes to the warp's shared slice; lane r sums row r of K_t
//             in column order (the rollouts of one law read the same K_t, which stays in L2).
//   records:  after step t, row [i][t] of qpos, qvel, act, ctrl as written, time and the env's flags; with sensors, sensordata and
//             sensor_mean = sensor_sum / n_substeps (fb_get's FB_SENSOR_MEAN, the same division).
#pragma once
#include "fb_fd.h"

struct DevRoll {
  int n, T, t, nsub;                      // rollouts, control steps, the step a launch serves, substeps per control step
  const float *ctrl, *qfrc, *xfrc;        // [n][T][nu], [n][T][nv], [n][T][6 nbody] (qfrc / xfrc nullptr: not written)
  const float *xref, *K;                  // [L][T][nq + nv + na], [L][T][nu][nx] (nullptr: open loop)
  float *qpos, *qvel, *act, *ctrl_out, *time;   // [n][T][nq], [nv], [na], [nu], [1]
  int* flags;                             // [n][T]
  float *sensordata, *sensor_mean;        // [n][T][nsd] (nullptr: not recorded)
};

// component i of env e's state minus the nominal row xr, in the tangent space of transition_fd's A and B
FB_DEV float roll_tangent(const DevModel& m, const DevData& d, int e, const float* xr, int i) {
  const int nq = m.nq, nv = m.nv;
  if (i < nv) {
    int qa, axis; fd_dof(m, i, &qa, &axis);
    if (axis >= 0) return comp(fd_subquat(q4(xr[qa], xr[qa + 1], xr[qa + 2], xr[qa + 3]), fd_quat(d, e, qa)), axis);
    return AT(d.qpos, qa) - xr[qa];
  }
  if (i < 2 * nv) return AT(d.qvel, i - nv) - xr[nq + i - nv];
  return AT(d.act, i - 2 * nv) - xr[nq + i - nv];
}

// law [n]: the law of each rollout (nullptr: law 0).  It is the input kernel's own parameter, so the record kernel's is unchanged.
FB_WARPFN void kroll_input(const DevModel& m, const DevData& d, const DevRoll& p, const int* law, float* dx, int e) {
  const int nu = m.nu, nv = m.nv, nxf = 6 * m.nbody;
  const int i = e < p.n ? e : p.n - 1;
  const size_t row = (size_t)i * p.T + p.t;
  const float* u = p.ctrl + row * nu;
  if (p.K) {
    const int nx = 2 * nv + m.na;
    const size_t lt = (size_t)(law ? law[i] : 0) * p.T + p.t;
    const float* xr = p.xref + lt * (m.nq + nv + m.na);
    const float* K = p.K + lt * nu * nx;
    WPAR_BEGIN for (int c = lane; c < nx; c += FB_NY) dx[c] = roll_tangent(m, d, e, xr, c); WPAR_END
    WPAR_BEGIN
      for (int r = lane; r < nu; r += FB_NY) {
        const float* k = K + (size_t)r * nx;
        float acc = 0.0f;
        for (int c = 0; c < nx; c++) acc = fmaf(k[c], dx[c], acc);
        AT(d.ctrl, r) = u[r] + acc;
      }
    WPAR_END
  } else {
    WPAR_BEGIN for (int r = lane; r < nu; r += FB_NY) AT(d.ctrl, r) = u[r]; WPAR_END
  }
  WPAR_BEGIN
    if (p.qfrc) for (int k = lane; k < nv; k += FB_NY) d.qfrc_applied[(size_t)e * nv + k] = p.qfrc[row * nv + k];
    if (p.xfrc) for (int k = lane; k < nxf; k += FB_NY) d.xfrc_applied[(size_t)e * nxf + k] = p.xfrc[row * nxf + k];
  WPAR_END
}

FB_WARPFN void kroll_record(const DevModel& m, const DevData& d, const DevRoll& p, int e) {
  const int nq = m.nq, nv = m.nv, na = m.na, nu = m.nu, nsd = m.nsensordata;
  const size_t row = (size_t)e * p.T + p.t;
  WPAR_BEGIN
    for (int k = lane; k < nq; k += FB_NY) p.qpos[row * nq + k] = AT(d.qpos, k);
    for (int k = lane; k < nv; k += FB_NY) p.qvel[row * nv + k] = AT(d.qvel, k);
    for (int k = lane; k < na; k += FB_NY) p.act[row * na + k] = AT(d.act, k);
    for (int k = lane; k < nu; k += FB_NY) p.ctrl_out[row * nu + k] = AT(d.ctrl, k);
    if (lane == 0) { p.time[row] = AT(d.time, 0); p.flags[row] = AT(d.flags, 0); }
    if (p.sensordata) {
      const float ns = (float)p.nsub;
      for (int k = lane; k < nsd; k += FB_NY) { p.sensordata[row * nsd + k] = AT(d.sensordata, k); p.sensor_mean[row * nsd + k] = AT(d.sensor_sum, k) / ns; }
    }
  WPAR_END
}
