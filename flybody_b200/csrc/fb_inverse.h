// fb_inverse.h -- batched inverse dynamics (MuJoCo mj_inverse, continuous time): the forces that produce a given acceleration.
//
// One problem per env, one warp per problem.  The env's record holds the position / velocity stage of its state (launch_step1:
// kinematics, qM with armature, the chain-sparse constraint rows with D, K, B, imp, pos, margin, qfrc_bias, qfrc_passive); qacc comes
// in and the results go out through the kernel's own parameter (DevInv), so the kernel writes nothing into the record and DevModel /
// DevData and the step kernels are untouched.
//   per row:  aref = -B (J qvel) - K imp (pos - margin),  jar = J qacc - aref,  efc_force from reg_head (MuJoCo mj_constraintUpdate:
//             limits and frictionless rows, the three cone zones of an elliptic contact; the head row of a contact evaluates its
//             three rows)
//   per dof:  qfrc_constraint = J^T efc_force (rows in order),  M qacc over the tree-sparse qM (mj_mulM),
//             qfrc_inverse = M qacc + qfrc_bias - qfrc_passive - qfrc_constraint
// Noslip is not inverted (as in MuJoCo): on a model with noslip iterations the forces are those of the soft model.  Every sum has a
// fixed order and there are no atomics, so a problem's bits do not depend on its env slot or the batch size.
#pragma once
#include "fb_solver_reg.h"

struct DevInv {
  int n;                                  // problems (envs 0 .. n-1)
  float* qacc;                            // [Np][nv] input accelerations
  float *qfrc_inverse, *qfrc_constraint;  // [Np][nv]
  float* efc_force;                       // [Np][FB_MAXEFC] rows >= nefc hold 0
};
#define FB_INV_SH (4 * FB_SOLVE_NCAP)     // per-warp floats: the J^T f accumulators (nv <= 4 * FB_SOLVE_NCAP, build_model)

// jar of row r: J qacc - aref, both products over chain a, then chain b below its join with chain a (the order of kref)
FB_DEV float inv_jar(const DevModel& m, const DevData& d, const float* qa, int e, int r) {
  const int la = AT(d.efc_la, r), lb = AT(d.efc_lb, r);
  float vel = 0, acc = 0;
  if (la >= 0) {
    const int adr = m.dof_Madr[la], len = m.dof_chainlen[la];
    for (int t = 0; t < len; t++) { const int k = m.dof_anc[adr + t]; const float j = EJC(d.efc_J, r, t); vel += j * AT(d.qvel, k); acc += j * qa[k]; }
  }
  if (lb >= 0) {
    const int adr = m.dof_Madr[lb], len = m.dof_chainlen[lb] - (la >= 0 ? m.dof_lca[lb * m.nv + la] : 0);
    for (int t = 0; t < len; t++) { const int k = m.dof_anc[adr + t]; const float j = EJC(d.efc_J, r, FB_ZCAP + t); vel += j * AT(d.qvel, k); acc += j * qa[k]; }
  }
  const float aref = -EFC(d.efc_B, r) * vel - EFC(d.efc_K, r) * EFC(d.efc_imp, r) * (EFC(d.efc_pos, r) - EFC(d.efc_margin, r));
  return acc - aref;
}

FB_WARPFN void kinv_run(const DevModel& m, const DevData& d, const DevInv& p, float* sh, int e) {
  const int nv = m.nv, n = AT(d.nefc, 0);
  const float* qa = p.qacc + (size_t)e * nv;
  float* fo = p.efc_force + (size_t)e * FB_MAXEFC;
  // ---- forces: one lane per head row (a plain row, or the normal row of an elliptic contact, which writes its two friction rows too)
  WPAR_BEGIN
    for (int r = lane; r < FB_MAXEFC; r += FB_NY) {
      if (r >= n) { fo[r] = 0.0f; continue; }
      int kind = 0; float mu = 0, c1 = 0, c2 = 0;
      if (EFC(d.efc_type, r) == FB_CT_ELLIPTIC) {
        const int ci = EFC(d.efc_id, r);
        kind = 1 + (r - AT(d.con_efcadr, ci));
        mu = AT(d.con_mu, ci); c1 = CON_F(d.con_fric, ci, 0, 2); c2 = CON_F(d.con_fric, ci, 1, 2);
      }
      if (kind >= 2) continue;                                  // friction rows: written by their head
      RegHead o;
      if (kind == 0) {
        reg_head(0, inv_jar(m, d, qa, e, r), 0, 0, EFC(d.efc_D, r), 0, 0, 0, 0, 0, o);
        fo[r] = o.f0;
      } else {
        reg_head(1, inv_jar(m, d, qa, e, r), inv_jar(m, d, qa, e, r + 1), inv_jar(m, d, qa, e, r + 2),
                 EFC(d.efc_D, r), EFC(d.efc_D, r + 1), EFC(d.efc_D, r + 2), mu, c1, c2, o);
        fo[r] = o.f0; fo[r + 1] = o.f1; fo[r + 2] = o.f2;
      }
    }
    for (int i = 0; i < FB_INV_SH / FB_NY; i++) sh[lane + FB_NY * i] = 0.0f;
  WPAR_END
  // ---- qfrc_constraint = J^T f: row after row (a warp barrier orders them), lanes over the row's chain slots, whose dofs are distinct
  // (chain b only below its join with chain a), so every dof sums its rows in row order
  for (int r = 0; r < n; r++) {
    WPAR_BEGIN
      const int la = AT(d.efc_la, r), lb = AT(d.efc_lb, r);
      const int La = la >= 0 ? m.dof_chainlen[la] : 0, Jb = lb >= 0 ? m.dof_chainlen[lb] - (la >= 0 ? m.dof_lca[lb * nv + la] : 0) : 0;
      const float f = fo[r];
      for (int s = lane; s < La + Jb; s += FB_NY) {
        if (s < La) sh[m.dof_anc[m.dof_Madr[la] + s]] += EJC(d.efc_J, r, s) * f;
        else sh[m.dof_anc[m.dof_Madr[lb] + s - La]] += EJC(d.efc_J, r, FB_ZCAP + s - La) * f;
      }
    WPAR_END
  }
  // ---- per dof: M qacc (diagonal, the row's ancestors, then the dofs below it: descendant c holds M[c][k] at chain offset
  // chainlen[c] - chainlen[k]), then the inverse force
  WPAR_BEGIN
    for (int k = lane; k < nv; k += FB_NY) {
      const int adr = m.dof_Madr[k], len = m.dof_chainlen[k], se = m.dof_subend[k];
      float mq = AT(d.qM, adr) * qa[k];
      for (int t = 1; t < len; t++) mq += AT(d.qM, adr + t) * qa[m.dof_anc[adr + t]];
      for (int c = k + 1; c <= se; c++) mq += AT(d.qM, m.dof_Madr[c] + m.dof_chainlen[c] - len) * qa[c];
      const float qc = sh[k];
      p.qfrc_constraint[(size_t)e * nv + k] = qc;
      p.qfrc_inverse[(size_t)e * nv + k] = mq + AT(d.qfrc_bias, k) - AT(d.qfrc_passive, k) - qc;
    }
  WPAR_END
}
