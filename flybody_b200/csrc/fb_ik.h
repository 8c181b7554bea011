// fb_ik.h -- batched multi-site inverse kinematics (reference flybody/inverse_kinematics.py: qpos_from_site_xpos).
//
// One IK problem per env, one warp per problem.  An iteration is the reference's (inverse_kinematics.py:101-130):
//   gradient of ||s(q) - s*||^2 + reg ||q_hinge||^2 over the fitted dofs -> momentum u <- beta u + g -> mj_integratePos(qpos, -lr u)
//   -> kinematics (kpos_p0 / kpos_p1 of the position kernel, then the program's sites only) -> every FB_IK_CHECK iterations the
//   objective and the stopping test lr |u| / err < progress_threshold.
// The env's record holds qpos and the kinematics outputs (ref, xpos, xquat, Sang, Slin); everything else of the solve (targets,
// momentum, loop index, results) lives in the program's own buffers (DevIk), so DevModel / DevData and the step kernels are untouched.
// A launch runs at most DevIk::iters iterations; the host relaunches while problems are live.  Every sum has a fixed order, so a
// problem's result does not depend on its env slot, the batch size or where the launches split the loop.
#pragma once
#include "fb_tree.h"

#define FB_IK_MAXSITE 64
#define FB_IK_CHECK 100            // iterations between objective checks (the reference's `step % 100 == 0`)

struct DevIk {
  int n, n_site, n_fdof, n_fjnt, iters, max_steps;
  float reg, lr, beta, thr;
  const int* site_id;                     // [n_site] model site ids
  const unsigned char* include;           // [3 n_site] components in the objective (reference include_inds)
  const int* fdof;                        // [n_fdof] model dof of each fitted dof (joint order, then dof order within the joint)
  const int* fdof_hqadr;                  // [n_fdof] qpos address of a fitted hinge (regularised), -1 for free-joint dofs
  const unsigned long long* below;        // [n_fdof] bit s: site s is on the dof's body or below it
  const int *fjnt_type, *fjnt_qadr, *fjnt_fd0;   // [n_fjnt] fitted joints: type, qpos address, first fitted dof
  const float* target;                    // [Np][n_site][3] world-frame targets; NaN: the component is excluded for that problem
  float* u;                               // [Np][n_fdof] momentum, carried across launches
  int *step, *done;                       // [Np] next loop index; 1 once the problem has stopped
  float *err, *err_first; int* steps; unsigned char* success;   // [Np] results
  int* live;                              // problems that did not stop in the last launch
};
// per-warp scratch (floats): residual r_s = 2 (x_s - t_s) and moment x_s x r_s per site, the site's squared error, momentum, step
#define FB_IK_SH(nfd) (7 * FB_IK_MAXSITE + 2 * (((nfd) + 3) & ~3))

// kinematics of the position kernel's first two phases: root on lane 0, one branch list per lane
FB_WARPFN void ik_kinematics(const DevModel& m, const DevData& d, ShTree& sh, int e) {
  WPAR_BEGIN kpos_p0(m, d, sh, e, lane); WPAR_END
  WPAR_BEGIN kpos_p1(m, d, sh, e, lane); WPAR_END
}
// site phase: positions of the program's sites only (relative to ref, as kpos_p1b computes them) against the targets moved into the
// record's frame; excluded components contribute nothing
FB_WARPFN void ik_sites(const DevModel& m, const DevData& d, const DevIk& p, float* sh, int e) {
  float *R = sh, *M = sh + 3 * FB_IK_MAXSITE, *D2 = sh + 6 * FB_IK_MAXSITE;
  WPAR_BEGIN
    const V3 ref = v3(AT(d.ref, 0), AT(d.ref, 1), AT(d.ref, 2));
    for (int s = lane; s < p.n_site; s += FB_NY) {
      const int t = p.site_id[s], b = MLD(m.site_bodyid[t]);
      const V3 x = ld3(d.xpos, b, d, e) + mul(q2m(ld4(d.xquat, b, d, e)), mld3(m.site_pos, t));
      const float* tg = p.target + ((size_t)e * p.n_site + s) * 3;
      float df[3] = {x.x - (tg[0] - ref.x), x.y - (tg[1] - ref.y), x.z - (tg[2] - ref.z)};
      float d2 = 0;
#pragma unroll
      for (int c = 0; c < 3; c++) {
        if (!p.include[3 * s + c] || tg[c] != tg[c]) df[c] = 0;
        d2 += df[c] * df[c];
      }
      const V3 r = v3(2 * df[0], 2 * df[1], 2 * df[2]), mo = cross(x, r);
      R[3 * s] = r.x; R[3 * s + 1] = r.y; R[3 * s + 2] = r.z;
      M[3 * s] = mo.x; M[3 * s + 1] = mo.y; M[3 * s + 2] = mo.z;
      D2[s] = d2;
    }
  WPAR_END
}
// mj_integratePos of a free or ball joint's rotation (MuJoCo mju_quatIntegrate): the quaternion qpos[qa .. qa + 3], normalised, turned
// by the body-frame rotation vector w.  The IK step and the finite-difference perturbation (fb_fd.h) share it.
FB_DEV void integrate_quat(const DevData& d, int e, int qa, V3 w) {
  const float ang = norm(w);
  Q4 q = qnormalize(q4(AT(d.qpos, qa), AT(d.qpos, qa + 1), AT(d.qpos, qa + 2), AT(d.qpos, qa + 3)));
  q = qnormalize(qmul(q, axisangle(normalized(w), ang)));
  AT(d.qpos, qa) = q.w; AT(d.qpos, qa + 1) = q.x; AT(d.qpos, qa + 2) = q.y; AT(d.qpos, qa + 3) = q.z;
}
// warp-uniform sums in index order (every lane reads the same shared values)
FB_DEV float ik_sum(const float* a, int n) { float s = 0; for (int i = 0; i < n; i++) s += a[i]; return s; }
FB_DEV float ik_sumsq(const float* a, int n) { float s = 0; for (int i = 0; i < n; i++) s += a[i] * a[i]; return s; }

// run up to p.iters iterations of problem e (one warp)
FB_WARPFN void kik_run(const DevModel& m, const DevData& d, const DevIk& p, float* sh, int e) {
  if (p.done[e]) return;
  float *R = sh, *M = sh + 3 * FB_IK_MAXSITE, *D2 = sh + 6 * FB_IK_MAXSITE;
  float *U = sh + 7 * FB_IK_MAXSITE, *STP = U + ((p.n_fdof + 3) & ~3);
  ShTree tree;                  // the slice argument of kpos_p0 / kpos_p1 (neither touches it)
  const int nfd = p.n_fdof;
  WPAR_BEGIN for (int i = lane; i < nfd; i += FB_NY) U[i] = p.u[(size_t)e * nfd + i]; WPAR_END
  ik_kinematics(m, d, tree, e);
  ik_sites(m, d, p, sh, e);
  int step = p.step[e];
  const int end = step + p.iters < p.max_steps ? step + p.iters : p.max_steps;
  float err = p.err[e];
  int stop = 0, ok = 0;
  for (; step < end; step++) {
    // gradient over the fitted dofs (sites below the dof, in site order), momentum, step
    WPAR_BEGIN
      for (int i = lane; i < nfd; i += FB_NY) {
        const int k = p.fdof[i];
        V3 sr = v3(0, 0, 0), sm = v3(0, 0, 0);
        for (unsigned long long bits = p.below[i]; bits; bits &= bits - 1) {
#ifdef __CUDACC__
          const int s = __ffsll((long long)bits) - 1;
#else
          const int s = __builtin_ctzll(bits);
#endif
          sr = sr + v3(R[3 * s], R[3 * s + 1], R[3 * s + 2]); sm = sm + v3(M[3 * s], M[3 * s + 1], M[3 * s + 2]);
        }
        float g = dot(ld3(d.Sang, k, d, e), sm) + dot(ld3(d.Slin, k, d, e), sr);
        if (p.fdof_hqadr[i] >= 0) g += 2 * p.reg * AT(d.qpos, p.fdof_hqadr[i]);
        const float u = p.beta * U[i] + g;
        U[i] = u; STP[i] = -p.lr * u;
      }
    WPAR_END
    // mj_integratePos: hinge += step; free joint: position += linear step, quaternion turned by the body-frame angular step
    WPAR_BEGIN
      for (int j = lane; j < p.n_fjnt; j += FB_NY) {
        const int qa = p.fjnt_qadr[j], f = p.fjnt_fd0[j];
        if (p.fjnt_type[j] == FB_JNT_HINGE) { AT(d.qpos, qa) += STP[f]; continue; }
        for (int c = 0; c < 3; c++) AT(d.qpos, qa + c) += STP[f + c];
        integrate_quat(d, e, qa + 3, v3(STP[f + 3], STP[f + 4], STP[f + 5]));
      }
    WPAR_END
    ik_kinematics(m, d, tree, e);
    ik_sites(m, d, p, sh, e);
    if (step % FB_IK_CHECK == 0) {
      float hq = 0;
      for (int i = 0; i < nfd; i++) if (p.fdof_hqadr[i] >= 0) { const float q = AT(d.qpos, p.fdof_hqadr[i]); hq += q * q; }
      err = ik_sum(D2, p.n_site) + p.reg * hq;
      // err == 0: converged (the reference divides by it)
      if (err == 0.0f || p.lr * sqrtf(ik_sumsq(U, nfd)) / err < p.thr) { stop = 1; ok = 1; break; }
    }
    if (step == p.max_steps - 1) { stop = 1; break; }
  }
  WPAR_BEGIN
    for (int i = lane; i < nfd; i += FB_NY) p.u[(size_t)e * nfd + i] = U[i];
    if (lane == 0) {
      p.err[e] = err;
      if (stop) { p.done[e] = 1; p.success[e] = (unsigned char)ok; p.steps[e] = step; p.err_first[e] = ik_sum(D2, p.n_site); p.step[e] = step; }
      else {
        p.step[e] = step;
#ifdef __CUDACC__
        atomicAdd(p.live, 1);
#else
        *p.live += 1;
#endif
      }
    }
  WPAR_END
}
