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

// ---- sensordata under the inverse (fb_query_sensors on).  Its own parameter beside DevInv, so the inverse kernels keep their layout.
// Velocity-stage sensors (gyro, velocimeter) are copied from what launch_step1 left in the record; the acceleration-stage ones restate
// the finish kernel's F5 - F9 (mj_rnePostConstraint + mj_sensorAcc) at the problem's qacc and the inverse's efc_force instead of the
// solver's.  The scratch (contact wrench, delta acceleration and force per body) lives in the warp's shared-memory slice, so the record
// is only read.  As in the step, xfrc_applied does not enter the force sensors (MuJoCo's cfrc_ext has it).
struct DevInvSens {
  DevInv inv;                             // the inverse: its qacc and efc_force
  float* sensordata;                      // [Np][nsensordata]
};
#define FB_INVS_SH(nbody) (18 * (nbody))  // per-warp floats: contact wrench, delta acceleration and force of every body, 6 each
FB_DEV bool sens_acc_stage(int type) { return type != FB_SENS_GYRO && type != FB_SENS_VELOCIMETER; }
FB_DEV S6 sh_ld6(const float* a, int b) { S6 s; s.a = v3(a[6 * b], a[6 * b + 1], a[6 * b + 2]); s.l = v3(a[6 * b + 3], a[6 * b + 4], a[6 * b + 5]); return s; }
FB_DEV void sh_st6(float* a, int b, const S6& s) {
  a[6 * b] = s.a.x; a[6 * b + 1] = s.a.y; a[6 * b + 2] = s.a.z; a[6 * b + 3] = s.l.x; a[6 * b + 4] = s.l.y; a[6 * b + 5] = s.l.z; }
// delta_from_parent (fb_constraint.h) with the accelerations qa of the caller
FB_DEV void inv_delta_from_parent(const DevModel& m, const DevData& d, int e, const float* qa, int b, S6& dl) {
  for (int kk = 0; kk < m.body_dofnum[b]; kk++) {
    const int k = m.body_dofadr[b] + kk; const float a = qa[k];
    dl.a = dl.a + ld3(d.Sang, k, d, e) * a; dl.l = dl.l + ld3(d.Slin, k, d, e) * a;
  }
}
FB_WARPFN void kinv_sensors(const DevModel& m, const DevData& d, const DevInvSens& p, float* sh, int e) {
  const int nb = m.nbody, ncon = AT(d.ncon, 0);
  const float* qa = p.inv.qacc + (size_t)e * m.nv;
  const float* fo = p.inv.efc_force + (size_t)e * FB_MAXEFC;
  float* out = p.sensordata + (size_t)e * m.nsensordata;
  float *xw = sh, *bdel = sh + 6 * nb, *bfrc = sh + 12 * nb;
  // velocity stage; the contact wrenches (F5: lane 0, contacts in order) and the roots' deltas (F6)
  WPAR_BEGIN
    for (int s = lane; s < m.nsensor; s += FB_NY)
      if (!sens_acc_stage(m.sensor_type[s])) for (int k = 0; k < m.sensor_dim[s]; k++) out[m.sensor_adr[s] + k] = AT(d.sensordata, m.sensor_adr[s] + k);
    for (int k = lane; k < 6 * nb; k += FB_NY) xw[k] = 0.0f;
  WPAR_END
  WPAR_BEGIN
    if (lane == 0) {
      for (int ci = 0; ci < ncon; ci++) {
        const int adr = AT(d.con_efcadr, ci); if (adr < 0) continue;
        const int dim = AT(d.con_dim, ci);
        V3 F = v3(0, 0, 0);
        for (int r = 0; r < dim; r++) F = F + v3(CON_F(d.con_frame, ci, 3 * r, 9), CON_F(d.con_frame, ci, 3 * r + 1, 9), CON_F(d.con_frame, ci, 3 * r + 2, 9)) * fo[adr + r];
        const V3 pos = v3(CON_F(d.con_pos, ci, 0, 3), CON_F(d.con_pos, ci, 1, 3), CON_F(d.con_pos, ci, 2, 3));
        const V3 tq = cross(pos, F);
        const int b1 = m.geom_bodyid[AT(d.con_geom1, ci)], b2 = m.geom_bodyid[AT(d.con_geom2, ci)];
        S6 w2 = sh_ld6(xw, b2); w2.a = w2.a + tq; w2.l = w2.l + F; sh_st6(xw, b2, w2);
        S6 w1 = sh_ld6(xw, b1); w1.a = w1.a - tq; w1.l = w1.l - F; sh_st6(xw, b1, w1);
      }
    }
    if (lane == 1) for (int r = 0; r < m.nroot; r++) { const int b = m.root_body[r]; S6 dl; dl.a = dl.l = v3(0, 0, 0); inv_delta_from_parent(m, d, e, qa, b, dl); sh_st6(bdel, b, dl); }
  WPAR_END
  // F7: the delta-acceleration chains and body forces f_b = f0_b + I_b delta_b - ext_b, one lane per list
  WPAR_BEGIN
    const int y = lane;
    if (y < m.nlist) {
      int prev = -1; S6 cd; cd.a = cd.l = v3(0, 0, 0);
      FB_LIST_LOOP_FWD {
        if (!m.body_sensacc[b]) { prev = -1; continue; }
        const int pa = m.body_parentid[b];
        if (pa != prev) cd = sh_ld6(bdel, pa);
        inv_delta_from_parent(m, d, e, qa, b, cd);
        sh_st6(bdel, b, cd);
        prev = b;
        if (m.body_sensfrc[b]) {
          I10 I = ld10(d.inert10, b, d, e); V3 L, pm; inert_mul(I, cd.a, cd.l, L, pm);
          S6 f = ld6(d.bfrc0, b, d, e), x = sh_ld6(xw, b);
          f.a = f.a + L - x.a; f.l = f.l + pm - x.l;
          sh_st6(bfrc, b, f);
        }
      }
    }
  WPAR_END
  // F8: subtree sums of the force-sensor bodies
  WPAR_BEGIN
    const int y = lane;
    if (y < m.nlist) {
      FB_LIST_LOOP_REV {
        if (!m.body_sensfrc[b]) continue;
        const int pa = m.body_parentid[b];
        if (!m.body_sensfrc[pa]) continue;
        S6 f = sh_ld6(bfrc, b), pf = sh_ld6(bfrc, pa);
        pf.a = pf.a + f.a; pf.l = pf.l + f.l; sh_st6(bfrc, pa, pf);
      }
    }
  WPAR_END
  // F9: accelerometer, force, touch
  WPAR_BEGIN
    for (int s = lane; s < m.nsensor; s += FB_NY) {
      const int tp = m.sensor_type[s], site = m.sensor_objid[s], adr = m.sensor_adr[s], b = m.site_bodyid[site];
      if (tp == FB_SENS_ACCELEROMETER) {
        S6 a = ld6(d.bacc, b, d, e), v = ld6(d.bvel, b, d, e); const S6 dl = sh_ld6(bdel, b);
        a.a = a.a + dl.a; a.l = a.l + dl.l;
        const V3 ps = ld3(d.site_xpos, site, d, e);
        const V3 vp = v.l + cross(v.a, ps);
        const V3 acc = a.l + cross(a.a, ps) + cross(v.a, vp);
        const V3 o = mulT(ld9(d.site_xmat, site, d, e), acc);
        out[adr] = o.x; out[adr + 1] = o.y; out[adr + 2] = o.z;
      } else if (tp == FB_SENS_FORCE) {
        const V3 o = mulT(ld9(d.site_xmat, site, d, e), sh_ld6(bfrc, b).l);
        out[adr] = o.x; out[adr + 1] = o.y; out[adr + 2] = o.z;
      } else if (tp == FB_SENS_TOUCH) {
        float sum = 0;
        for (int ci = 0; ci < ncon; ci++) {
          const int ea = AT(d.con_efcadr, ci); if (ea < 0) continue;
          const int b1 = m.geom_bodyid[AT(d.con_geom1, ci)], b2 = m.geom_bodyid[AT(d.con_geom2, ci)];
          if (b != b1 && b != b2) continue;
          const float fn = fo[ea]; if (fn <= 0) continue;
          V3 ray = v3(CON_F(d.con_frame, ci, 0, 9), CON_F(d.con_frame, ci, 1, 9), CON_F(d.con_frame, ci, 2, 9));
          if (b == b2) ray = ray * -1.0f;
          const V3 pos = v3(CON_F(d.con_pos, ci, 0, 3), CON_F(d.con_pos, ci, 1, 3), CON_F(d.con_pos, ci, 2, 3));
          const V3 ssz = mld3(m.site_size, site);
          float hit;
          if (m.site_type[site] == FB_GEOM_CAPSULE) hit = ray_capsule(ld3(d.site_xpos, site, d, e), ld9(d.site_xmat, site, d, e), ssz, pos, ray);
          else { float xx[2]; const V3 dif = pos - ld3(d.site_xpos, site, d, e); hit = ray_quad(dot(ray, ray), dot(ray, dif), dot(dif, dif) - ssz.x * ssz.x, xx); }
          if (hit >= 0) sum += fn;
        }
        out[adr] = sum;
      }
    }
  WPAR_END
}
