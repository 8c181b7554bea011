// fb_tree.h -- tree-structured stages: kinematics, composite inertia, sparse L^T D L factorisation
// and solve, body velocities, RNE bias, passive (spring/damper/fluid) forces.
//
// Thread mapping of every "tree kernel": one warp per env; lane y < nlist walks one branch list of the
// kinematic tree (a leg, the abdomen chain, the head sub-tree ...) in topological order.  The root
// bodies (free joints) are handled by y == 0; the lists exchange their contributions to the root through
// the env's shared-memory slice.  Each kernel is a sequence of *phases* separated by warp barriers (see
// fb_run in flybody_b200.cu).
#pragma once
#include "fb_math.h"

// Shared memory of one warp (= one env) in the tree kernels.  Fixed part: one float per lane for small reductions.
// Dynamic part (sized per launch), in this order where present:
//   PART  [FB_PARTR][FB_PARTK]  partial sums towards the root: per branch list (crb: 10, rne: 12, packed), or the
//                            factorisation's root-block partials (21) of FB_PARTR lanes at a time              -- pos, vel
//   LS    [nM]               the joint-space inertia / its factor                                     -- pos
//   XS    [nv + FB_ROOTD*nlist], LDS [nM]   right-hand side and staged factor of the triangular solves -- smooth, finish
struct ShTree { float red[FB_NY]; const unsigned* prog; const unsigned* pad_; };   // prog: the CTA's copy of the sweep program (smooth / finish kernels)
#define FB_PARTK 21
#define FB_PARTR 8             // 8 rows instead of one per lane: the position kernel's CTA then fits 8 per SM (and the larger L1 carveout)
#define FB_PARTF (FB_PARTR * FB_PARTK)
#define PART(yy, k) part_[(yy) * FB_PARTK + (k)]
#define PARTL(l, k, K) part_[(l) * (K) + (k)]     // K entries per branch list l
static_assert(FB_NLMAX * 12 <= FB_PARTR * FB_PARTK, "the per-list partial sums must fit PART");

// dynamic shared memory that follows the fixed struct (per-kernel scratch: the L^T D L rows during the
// factorisation, the right-hand side during tree solves)
template <typename Sh> FB_DEV float* sh_dyn(Sh& sh) { return reinterpret_cast<float*>(reinterpret_cast<unsigned char*>(&sh) + ((sizeof(Sh) + 15) & ~(size_t)15)); }
#define LS(k) ldsh[k]
#define XS(k) xs[k]

#define FB_PHASE_ARGS const DevModel& m, const DevData& d, ShTree& sh, int e, int y
#define FB_LIST_LOOP_FWD for (int li_ = 0, b = 0; li_ < m.list_num[y] && ((b = m.list_body[m.list_adr[y] + li_]), true); li_++)
#define FB_LIST_LOOP_REV for (int li_ = m.list_num[y] - 1, b = 0; li_ >= 0 && ((b = m.list_body[m.list_adr[y] + li_]), true); li_--)

// ---------------------------------------------------------------------------------------------
// K1 kinematics (MuJoCo mj_kinematics + mj_comPos; reference model fruitfly.xml:307-731)
// Ball joints (MuJoCo's BALL cases; the free joint's branches restate them for its rotational half), called between FB_NO_MERGE barriers.
// Pose: the normalised quaternion from qpos turns the body about the anchor (mj_kinematics); the dof axes are the columns of the
// body frame (mj_comPos)
FB_DEV void ball_pose(const DevModel& m, const DevData& d, int e, int j, int qa, int da, V3& pos, Q4& quat) {
  V3 jp = mld3(m.jnt_pos, j);
  V3 anchor = pos + mul(q2m(quat), jp);
  quat = qmul(quat, qnormalize(q4(AT(d.qpos, qa), AT(d.qpos, qa + 1), AT(d.qpos, qa + 2), AT(d.qpos, qa + 3))));
  M3 R = q2m(quat);
  pos = anchor - mul(R, jp);
  for (int i = 0; i < 3; i++) {
    V3 ax = col(R, i);
    st3(d.Sang, da + i, d, e, ax);
    st3(d.Slin, da + i, d, e, cross(anchor, ax));
  }
}
// chain part: pose of body b from its parent's pose (pp, pq) and the joint coordinates; writes xpos, xquat
// and the motion subspaces of the body's dofs.  Returns the body's pose for the next link of the chain.
FB_DEV void body_pose(const DevModel& m, const DevData& d, int e, int b, V3 ppos, Q4 pq, V3 ref, V3& pos, Q4& quat) {
  M3 pR = q2m(pq);
  pos = ppos + mul(pR, mld3(m.body_pos, b));
  quat = qmul(pq, mld4(m.body_quat, b));
  int jn = MLD(m.body_jntnum[b]);
  for (int k = 0; k < jn; k++) {
    int j = MLD(m.body_jntadr[b]) + k, qa = MLD(m.jnt_qposadr[j]), da = MLD(m.jnt_dofadr[j]);
    const int jt = MLD(m.jnt_type[j]);
    if (jt == FB_JNT_FREE) {
      pos = v3(AT(d.qpos, qa), AT(d.qpos, qa + 1), AT(d.qpos, qa + 2)) - ref;
      quat = qnormalize(q4(AT(d.qpos, qa + 3), AT(d.qpos, qa + 4), AT(d.qpos, qa + 5), AT(d.qpos, qa + 6)));
      M3 R = q2m(quat);
      for (int i = 0; i < 3; i++) {
        V3 ei = v3(i == 0, i == 1, i == 2);
        st3(d.Sang, da + i, d, e, v3(0, 0, 0));
        st3(d.Slin, da + i, d, e, ei);
        V3 ax = col(R, i);
        st3(d.Sang, da + 3 + i, d, e, ax);
        st3(d.Slin, da + 3 + i, d, e, cross(pos, ax));
      }
    } else if (jt == FB_JNT_BALL) {
      FB_NO_MERGE(); ball_pose(m, d, e, j, qa, da, pos, quat); FB_NO_MERGE();
    } else {
      M3 R = q2m(quat);
      V3 jp = mld3(m.jnt_pos, j), ja = mld3(m.jnt_axis, j);
      V3 anchor = pos + mul(R, jp);
      V3 axis = mul(R, ja);
      quat = qmul(quat, axisangle(ja, AT(d.qpos, qa) - MLD(m.qpos0[qa])));
      R = q2m(quat);
      pos = anchor - mul(R, jp);
      st3(d.Sang, da, d, e, axis);
      st3(d.Slin, da, d, e, cross(anchor, axis));
    }
  }
  quat = qnormalize(quat);
  st3(d.xpos, b, d, e, pos); st4(d.xquat, b, d, e, quat);
}
// per-body part (no dependence between bodies): rotation matrix, inertial frame, spatial inertia about ref
// CRBS(b, k): the composite inertias while they are being accumulated (kpos_p1b .. kpos_p3b) live in the shared-memory region that
// later holds the inertia matrix rows (LS): the backward accumulation along the lists is a chain of read-modify-writes, which as
// global-memory traffic costs an L2 round trip per body (12.8 % of the position kernel's stall samples, profiles/README.md)
#define CRBS(b, k) ldsh[(b) * 10 + (k)]
FB_DEV void body_derived(const DevModel& m, const DevData& d, int e, int b, float* ldsh) {
  V3 pos = ld3(d.xpos, b, d, e); Q4 quat = ld4(d.xquat, b, d, e);
  M3 R = q2m(quat);
  st9(d.xmat, b, d, e, R);
  V3 ipos = pos + mul(R, mld3(m.body_ipos, b));
  M3 iR = q2m(qmul(quat, mld4(m.body_iquat, b)));
  st3(d.xipos, b, d, e, ipos); st9(d.ximat, b, d, e, iR);
  float mass = PRM(FB_P_BODY_MASS, m.body_mass)[b];
  V3 di = mld3(PRM(FB_P_BODY_INERTIA, m.body_inertia), b);
  float Ic[6];   // xx yy zz xy xz yz of R diag(di) R^T
  Ic[0] = iR.m[0] * iR.m[0] * di.x + iR.m[1] * iR.m[1] * di.y + iR.m[2] * iR.m[2] * di.z;
  Ic[1] = iR.m[3] * iR.m[3] * di.x + iR.m[4] * iR.m[4] * di.y + iR.m[5] * iR.m[5] * di.z;
  Ic[2] = iR.m[6] * iR.m[6] * di.x + iR.m[7] * iR.m[7] * di.y + iR.m[8] * iR.m[8] * di.z;
  Ic[3] = iR.m[0] * iR.m[3] * di.x + iR.m[1] * iR.m[4] * di.y + iR.m[2] * iR.m[5] * di.z;
  Ic[4] = iR.m[0] * iR.m[6] * di.x + iR.m[1] * iR.m[7] * di.y + iR.m[2] * iR.m[8] * di.z;
  Ic[5] = iR.m[3] * iR.m[6] * di.x + iR.m[4] * iR.m[7] * di.y + iR.m[5] * iR.m[8] * di.z;
  float cc = dot(ipos, ipos);
  float I[10];
  I[0] = mass; I[1] = mass * ipos.x; I[2] = mass * ipos.y; I[3] = mass * ipos.z;
  I[4] = Ic[0] + mass * (cc - ipos.x * ipos.x); I[5] = Ic[1] + mass * (cc - ipos.y * ipos.y); I[6] = Ic[2] + mass * (cc - ipos.z * ipos.z);
  I[7] = Ic[3] - mass * ipos.x * ipos.y; I[8] = Ic[4] - mass * ipos.x * ipos.z; I[9] = Ic[5] - mass * ipos.y * ipos.z;
  st10(d.inert10, b, d, e, I);
  for (int k = 0; k < 10; k++) CRBS(b, k) = I[k];
}

FB_DEV void kpos_p0(FB_PHASE_ARGS) {
  if (y != 0) return;
  // reference point = position of the first root's free joint, one for all trees (MuJoCo takes each tree's own subtree CoM).  fp32
  // positions stay resolved for bodies near that root; a second tree far from it (a ghost 1e3 cm away) loses about 100x of its
  // inertia's accuracy (tests/smooth_states.py moves the whole scene in its far states, as the tasks keep the ghost on the walker)
  int rb = m.root_body[0];
  V3 ref = v3(0, 0, 0);
  if (m.body_jntnum[rb] > 0 && m.jnt_type[m.body_jntadr[rb]] == FB_JNT_FREE) {
    int qa = m.jnt_qposadr[m.body_jntadr[rb]];
    ref = v3(AT(d.qpos, qa), AT(d.qpos, qa + 1), AT(d.qpos, qa + 2));
  }
  AT(d.ref, 0) = ref.x; AT(d.ref, 1) = ref.y; AT(d.ref, 2) = ref.z;
  // world body
  st3(d.xpos, 0, d, e, v3(0, 0, 0) - ref); st4(d.xquat, 0, d, e, q4(1, 0, 0, 0));
  for (int r = 0; r < m.nroot; r++) { V3 pos; Q4 q; body_pose(m, d, e, m.root_body[r], v3(0, 0, 0) - ref, q4(1, 0, 0, 0), ref, pos, q); }
}
// chains: a list is walked in topological order; the parent pose is carried in registers when the parent is the
// body visited just before (the usual case along a leg / the abdomen), otherwise re-read from the record
FB_DEV void kpos_p1(FB_PHASE_ARGS) {
  if (y >= m.nlist) return;
  V3 ref = v3(AT(d.ref, 0), AT(d.ref, 1), AT(d.ref, 2));
  int prev = -1; V3 cpos = v3(0, 0, 0); Q4 cq = q4(1, 0, 0, 0);
  FB_LIST_LOOP_FWD {
    int p = MLD(m.body_parentid[b]);
    V3 ppos; Q4 pq;
    if (p == prev) { ppos = cpos; pq = cq; } else { ppos = ld3(d.xpos, p, d, e); pq = ld4(d.xquat, p, d, e); }
    body_pose(m, d, e, b, ppos, pq, ref, cpos, cq);
    prev = b;
  }
}
// all 32 lanes: per-body derived quantities, geom and site frames
FB_DEV void kpos_p1b(FB_PHASE_ARGS) {
  float* part_ = sh_dyn(sh); float* ldsh = part_ + FB_PARTF; (void)part_;
  for (int b = y; b < m.nbody; b += FB_NY) {
    if (b == 0) { M3 I; for (int k = 0; k < 9; k++) I.m[k] = (k % 4 == 0) ? 1.f : 0.f;
      st9(d.xmat, 0, d, e, I); st3(d.xipos, 0, d, e, ld3(d.xpos, 0, d, e)); st9(d.ximat, 0, d, e, I);
      { float z10[10] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0}; st10(d.inert10, 0, d, e, z10); for (int k = 0; k < 10; k++) CRBS(0, k) = 0; }
    } else body_derived(m, d, e, b, ldsh);
  }
  for (int g = y; g < m.ngeom; g += FB_NY) {
    int b = m.geom_bodyid[g]; V3 pos = ld3(d.xpos, b, d, e); Q4 quat = ld4(d.xquat, b, d, e);
    st3(d.geom_xpos, g, d, e, pos + mul(q2m(quat), mld3(m.geom_pos, g)));
    st9(d.geom_xmat, g, d, e, q2m(qmul(quat, mld4(m.geom_quat, g))));
  }
  for (int t = y; t < m.nsite; t += FB_NY) {
    int b = m.site_bodyid[t]; V3 pos = ld3(d.xpos, b, d, e); Q4 quat = ld4(d.xquat, b, d, e);
    st3(d.site_xpos, t, d, e, pos + mul(q2m(quat), mld3(m.site_pos, t)));
    st9(d.site_xmat, t, d, e, q2m(qmul(quat, mld4(m.site_quat, t))));
  }
}
// K2 composite inertia, backward accumulation (MuJoCo mj_crb); the running sum of a chain stays in registers
FB_DEV void kpos_p2(FB_PHASE_ARGS) {
  float* part_ = sh_dyn(sh); float* ldsh = part_ + FB_PARTF;
  if (y >= m.nlist) return;
  float acc[10], carry[10]; int carry_to = -1;
  for (int k = 0; k < 10; k++) { acc[k] = 0; carry[k] = 0; }
  FB_LIST_LOOP_REV {
    float cur[10];
    for (int k = 0; k < 10; k++) cur[k] = CRBS(b, k);
    if (carry_to == b) { for (int k = 0; k < 10; k++) { cur[k] += carry[k]; CRBS(b, k) = cur[k]; } }
    else if (carry_to >= 0) { for (int k = 0; k < 10; k++) CRBS(carry_to, k) += carry[k]; }   // branch point: flush
    int p = m.body_parentid[b];
    if (m.body_isroot[p]) { for (int k = 0; k < 10; k++) acc[k] += cur[k]; carry_to = -1; }
    else { for (int k = 0; k < 10; k++) carry[k] = cur[k]; carry_to = p; }
  }
  if (carry_to >= 0) for (int k = 0; k < 10; k++) CRBS(carry_to, k) += carry[k];
  for (int k = 0; k < 10; k++) PARTL(y, k, 10) = acc[k];
}
FB_DEV void kpos_p3(FB_PHASE_ARGS) {       // composite inertia of the root bodies: lanes over (root, component)
  float* part_ = sh_dyn(sh); float* ldsh = part_ + FB_PARTF;
  for (int t = y; t < 10 * m.nroot; t += FB_NY) {
    int r = t / 10, k = t - 10 * r, b = m.root_body[r];
    float s = CRBS(b, k);
    for (int l = 0; l < m.nlist; l++) if (m.list_root[l] == r) s += PARTL(l, k, 10);
    CRBS(b, k) = s;
  }
}
// the finished composite inertias go to the record (mass_row, the subtree-CoM observable and the task hooks read them there;
// the shared region is overwritten by the inertia matrix next)
FB_DEV void kpos_p3b(FB_PHASE_ARGS) {
  float* part_ = sh_dyn(sh); float* ldsh = part_ + FB_PARTF; (void)part_;
  for (int b = y; b < m.nbody; b += FB_NY) { float v[10]; for (int k = 0; k < 10; k++) v[k] = CRBS(b, k); st10(d.crb10, b, d, e, v); }
}
// joint-space inertia entries of dof i (row of the sparse lower triangle along the ancestor chain)
FB_DEV void mass_row(const DevModel& m, const DevData& d, int e, float* ldsh, int i) {
  int b = m.dof_bodyid[i];
  I10 I = ld10(d.crb10, b, d, e);
  V3 L, p;
  inert_mul(I, ld3(d.Sang, i, d, e), ld3(d.Slin, i, d, e), L, p);
  const int adr = m.dof_Madr[i], len = m.dof_chainlen[i];
  const float* arm = PRM(FB_P_DOF_ARMATURE, m.dof_armature);
  int t = 0;
  for (; t + 4 <= len; t += 4) {       // four ancestors at a time: their motion-axis loads are in flight together (a store to qM between
    // two loads would otherwise order them: the compiler cannot rule out that the arrays overlap)
    const int j0 = m.dof_anc[adr + t], j1 = m.dof_anc[adr + t + 1], j2 = m.dof_anc[adr + t + 2], j3 = m.dof_anc[adr + t + 3];
    const V3 a0 = ld3(d.Sang, j0, d, e), l0 = ld3(d.Slin, j0, d, e), a1 = ld3(d.Sang, j1, d, e), l1 = ld3(d.Slin, j1, d, e);
    const V3 a2 = ld3(d.Sang, j2, d, e), l2 = ld3(d.Slin, j2, d, e), a3 = ld3(d.Sang, j3, d, e), l3 = ld3(d.Slin, j3, d, e);
    float v0 = dot(a0, L) + dot(l0, p), v1 = dot(a1, L) + dot(l1, p), v2 = dot(a2, L) + dot(l2, p), v3_ = dot(a3, L) + dot(l3, p);
    if (t == 0) v0 += arm[i];
    AT(d.qM, adr + t) = v0; LS(adr + t) = v0; AT(d.qM, adr + t + 1) = v1; LS(adr + t + 1) = v1;
    AT(d.qM, adr + t + 2) = v2; LS(adr + t + 2) = v2; AT(d.qM, adr + t + 3) = v3_; LS(adr + t + 3) = v3_;
  }
  for (; t < len; t++) {
    const int j = m.dof_anc[adr + t];
    float v = dot(ld3(d.Sang, j, d, e), L) + dot(ld3(d.Slin, j, d, e), p);
    if (t == 0) v += arm[i];
    AT(d.qM, adr + t) = v; LS(adr + t) = v;
  }
}
FB_DEV void kpos_p4(FB_PHASE_ARGS) {      // all 32 lanes over the dofs
  float* part_ = sh_dyn(sh); float* ldsh = part_ + FB_PARTF; (void)part_;
  for (int i = y; i < m.nv; i += FB_NY) mass_row(m, d, e, ldsh, i);
}
// Copy the factor held in shared memory out to `dst`.  Convention of qLD / qLDe: the diagonal holds D[k], the off-diagonal
// entries stay UNSCALED, M'[k][anc] = D[k] L[k][anc] -- every consumer multiplies a whole row by one 1/D[k] instead of
// scaling each entry here.
FB_DEV void ld_writeout(const DevModel& m, const DevData& d, ShTree& sh, int e, int y, float* dst) {
  float* part_ = sh_dyn(sh); float* ldsh = part_ + FB_PARTF; (void)part_;
  for (int k = y; k < m.nM; k += FB_NY) AT(dst, k) = LS(k);
}
// re-initialise the shared rows with M + h*diag(damping) for the second factorisation (Euler with implicit damping); with a parameter
// overlay the env's own M_damp, which follows its dof_damping (fb_param_set, kprm_draw)
FB_DEV void ld_reinit_damped(const DevModel& m, const DevData& d, ShTree& sh, int e, int y) {
  float* part_ = sh_dyn(sh); float* ldsh = part_ + FB_PARTF; (void)part_;
  const float* md = d.prm ? (const float*)d.prm + (unsigned)e * d.prm_stride + (unsigned)d.prm_mdamp : m.M_damp;
  for (int k = y; k < m.nM; k += FB_NY) LS(k) = AT(d.qM, k) + m.timestep * md[k];
}

// sparse L^T D L factorisation (Featherstone; MuJoCo mj_factorM).  Row k of LD holds (k,k), (k,parent(k)), ...
// at dof_Madr[k] + t.  The lists advance in lock-step, one dof per step (deepest first); the rank-1 updates of the
// ancestor rows of the step's dofs are dealt to all 32 lanes (factor_step_sched).  Updates that land in the root block are
// summed into sh.part (21 entries per lane) and applied by the root lane afterwards.
#define FB_FSUB 3
// packed per-(step, lane) header of the lock-step sweeps (tsolve_blob), one word instead of the dependent chain list dof ->
// dof_Madr / dof_chainlen / dof_depth.  adr | len << 12 | depth << 18 | dof << 24, ~0 = idle
#define FB_HDR_IDLE 0xffffffffu
#define HDR_ADR(h) ((int)((h) & 4095u))
#define HDR_LEN(h) ((int)(((h) >> 12) & 63u))
#define HDR_DOF(h) ((int)((h) >> 24))
#define FB_ROOTD6 6            // dofs of a root body (free joint)
// One step of the sweep: the dofs k of this step (one per list) subtract their rank-1 term from the rows of their non-root ancestors,
// row(anc_t)[s] -= (r_k[t] / D_k) r_k[t + s]  (the item carries the row address of the t-th ancestor; the root's dofs are the tail of every chain
// and are handled by factor_root_accum).  The (k, t) pairs of a step touch different rows, so they are independent work items; the
// host deals them to the 32 lanes longest-first onto the least loaded lane (DevModel::fs_rng / fs_items, built in fb_create) --
// round 1 gave every list 3 fixed lanes, which kept 12 of 32 busy.  The item after the current one is loaded while this one runs.
FB_DEV void factor_step_sched(const DevModel& m, const DevData& d, ShTree& sh, int e, int y, unsigned rng) {
  float* part_ = sh_dyn(sh); float* ldsh = part_ + FB_PARTF; (void)part_;
  const int cnt = (int)(rng >> 16);
  if (cnt == 0) return;
  const FsItem* ip = m.fs_items + (rng & 0xffffu);
  FsItem it = ip[0];
  for (int q = 0; q < cnt; q++) {
    const FsItem nx = q + 1 < cnt ? ip[q + 1] : it;
    const int adrk = (int)(it.x & 4095u), t = (int)((it.x >> 12) & 63u), li = (int)(it.x >> 18), adri = (int)it.y;
    const float a = LS(adrk + t) * (1.0f / LS(adrk));
    int s2 = 0;
    for (; s2 + 4 <= li; s2 += 4) {                          // batched so that the loads are in flight together
      float r0 = LS(adrk + t + s2), r1 = LS(adrk + t + s2 + 1), r2 = LS(adrk + t + s2 + 2), r3 = LS(adrk + t + s2 + 3);
      float x0 = LS(adri + s2), x1 = LS(adri + s2 + 1), x2 = LS(adri + s2 + 2), x3 = LS(adri + s2 + 3);
      LS(adri + s2) = x0 - a * r0; LS(adri + s2 + 1) = x1 - a * r1; LS(adri + s2 + 2) = x2 - a * r2; LS(adri + s2 + 3) = x3 - a * r3;
    }
    for (; s2 < li; s2++) LS(adri + s2) -= a * LS(adrk + t + s2);
    it = nx;
  }
}
// Root blocks.  Once the lists are eliminated, row k of a non-root dof holds its final (unscaled) coupling r_k to the
// root's dofs and D_k; the Schur update of the root block is sum_k r_k r_k^T / D_k.  32 lanes split the dofs, each
// accumulates the 21 packed lower-triangle entries in registers ...
FB_DEV void factor_root_accum(const DevModel& m, const DevData& d, ShTree& sh, int e, int y, int r, float acc[21]) {
  float* part_ = sh_dyn(sh); float* ldsh = part_ + FB_PARTF; (void)part_;
#pragma unroll
  for (int j = 0; j < 21; j++) acc[j] = 0;
  for (int k = y; k < m.nv; k += FB_NY) {
    if (m.dof_rootidx[k] != r) continue;
    int adrk = m.dof_Madr[k], len = m.dof_chainlen[k], nr = len - 1 - m.dof_depth[k];
    float invD = 1.0f / LS(adrk), rr[FB_ROOTD6];
#pragma unroll
    for (int il = 0; il < FB_ROOTD6; il++) rr[il] = il < nr ? LS(adrk + len - 1 - il) : 0.0f;     // coupling to root dof il
#pragma unroll
    for (int i = 0; i < FB_ROOTD6; i++) {
      float a = rr[i] * invD;
#pragma unroll
      for (int j = 0; j <= i; j++) acc[i * (i + 1) / 2 + (i - j)] += a * rr[j];                   // row i, (i-j)-th ancestor
    }
  }
}
// ... 21 lanes add the partials up (one packed entry each), in lane order: lanes y0 .. y0 + FB_PARTR - 1 put theirs into PART,
// then the summing lanes add them on; a sum over all 32 lanes takes FB_NY / FB_PARTR such rounds ...
FB_DEV void factor_root_put(ShTree& sh, int y, int y0, const float acc[21]) {
  float* part_ = sh_dyn(sh);
  if (y < y0 || y >= y0 + FB_PARTR) return;
#pragma unroll
  for (int j = 0; j < 21; j++) PART(y - y0, j) = acc[j];
}
FB_DEV void factor_root_sum(ShTree& sh, int y, float& acc) {
  float* part_ = sh_dyn(sh);
  if (y >= 21) return;
#pragma unroll
  for (int l = 0; l < FB_PARTR; l++) acc += PART(l, y);
}
FB_DEV void factor_root_gather(const DevModel& m, const DevData& d, ShTree& sh, int e, int y, int r, float acc) {
  float* part_ = sh_dyn(sh); float* ldsh = part_ + FB_PARTF;
  if (y >= 21) return;
  int il = 0; while ((il + 1) * (il + 2) / 2 <= y) il++;
  int s = y - il * (il + 1) / 2;
  int b = m.root_body[r], nd = m.body_dofnum[b], d0 = m.body_dofadr[b];
  if (il >= nd) return;
  LS(m.dof_Madr[d0 + il] + s) -= acc;
}
// ... then one lane per root body factors its dense (<= 6x6) block
FB_DEV void factor_root(const DevModel& m, const DevData& d, ShTree& sh, int e, int y) {
  float* part_ = sh_dyn(sh); float* ldsh = part_ + FB_PARTF; (void)part_;
  if (y >= m.nroot) return;
  int b = m.root_body[y], nd = m.body_dofnum[b], d0 = m.body_dofadr[b];
  for (int kl = nd - 1; kl >= 0; kl--) {
    int adrk = m.dof_Madr[d0 + kl];
    float invD = 1.0f / LS(adrk);
    for (int t = 1; t <= kl; t++) {
      int il = kl - t, adri = m.dof_Madr[d0 + il];
      float a = LS(adrk + t) * invD;
      for (int s = 0; s <= il; s++) LS(adri + s) -= a * LS(adrk + t + s);
    }
  }
}
// warp function: the whole factorisation of the rows currently held in shared memory
FB_WARPFN void kpos_factor(const DevModel& m, const DevData& d, ShTree& sh, int e) {
#ifdef __CUDACC__
  {   // the schedule entry of the NEXT step is loaded while this step's rank-1 updates run (one dependent global load less per step)
    const int lane = threadIdx.x; const unsigned* hp = m.fs_rng + lane;
    unsigned hd = m.max_list_ndof > 0 ? hp[0] : 0u;
    for (int step = 0; step < m.max_list_ndof; step++) {
      const unsigned nxt = step + 1 < m.max_list_ndof ? hp[(step + 1) * FB_NY] : 0u;
      factor_step_sched(m, d, sh, e, lane, hd); __syncwarp();
      hd = nxt;
    }
  }
#else
  for (int step = 0; step < m.max_list_ndof; step++) {
    WPAR_BEGIN factor_step_sched(m, d, sh, e, lane, m.fs_rng[step * FB_NY + lane]); WPAR_END
  }
#endif
  for (int r = 0; r < m.nroot; r++) {
    if (!m.root_haslists[r]) continue;
    LREGA(float, acc, 21); LREG(float, tot);
    WPAR_BEGIN { float a[21]; factor_root_accum(m, d, sh, e, lane, r, a);
#pragma unroll
      for (int j = 0; j < 21; j++) LA(acc, j) = a[j];
      L(tot) = 0.0f; } WPAR_END
    for (int y0 = 0; y0 < FB_NY; y0 += FB_PARTR) {
      WPAR_BEGIN { float a[21];
#pragma unroll
        for (int j = 0; j < 21; j++) a[j] = LA(acc, j);
        factor_root_put(sh, lane, y0, a); } WPAR_END
      WPAR_BEGIN factor_root_sum(sh, lane, L(tot)); WPAR_END
    }
    WPAR_BEGIN factor_root_gather(m, d, sh, e, lane, r, L(tot)); WPAR_END
  }
  WPAR_BEGIN factor_root(m, d, sh, e, lane); WPAR_END
}
FB_DEV void kpos_p6w(FB_PHASE_ARGS) { ld_writeout(m, d, sh, e, y, d.qLD); }
FB_DEV void kpos_p6d(FB_PHASE_ARGS) { ld_reinit_damped(m, d, sh, e, y); }
FB_DEV void kpos_p9(FB_PHASE_ARGS) { ld_writeout(m, d, sh, e, y, d.qLDe); }

// ---------------------------------------------------------------------------------------------
// x <- (L^T D L)^-1 x (MuJoCo mj_solveLD).  x lives in shared memory: XS(0..nv) plus FB_ROOTD private accumulators per
// list at XS(nv + FB_ROOTD*l + il) for the updates that land on the root's dofs.  The lists advance in lock-step, one
// dof per step; the FB_FSUB lanes of a list split that dof's ancestor chain (the sweep program below gives the shared slot
// of the t-th ancestor without pointer chasing).
#define FB_ROOTD 6
// Sweep program of the triangular solves, copied once per CTA into shared memory (DevModel::tsolve_blob): the packed step
// headers of both directions and, per entry of the packed factor, the shared slot of its ancestor (L^-T sweep: the lists'
// private root accumulators; L^-1 sweep: the dof itself) as bytes.  The sweeps then touch no global table at all.
#define TS_HDR_A(sh, m) ((sh).prog)
#define TS_HDR_C(sh, m) ((sh).prog + (m).ts_hdr_words)
#define TS_SLOT8(sh, m) (reinterpret_cast<const unsigned char*>((sh).prog + 2 * (m).ts_hdr_words))
#define TS_ANC8(sh, m) (TS_SLOT8(sh, m) + (m).ts_nm_pad)
#define FB_NXS(m) (((m).nv + FB_ROOTD * (m).nlist + 3) & ~3)      // multiple of 4: the staged factor behind it stays 16-byte aligned
#define LDS(k) lds[k]
// Stage a factor into the warp's shared slice with asynchronous 16-byte copies (cp.async): issued early (first phase
// of the kernel / right after the previous solve), waited for at the start of tri_solve, so the DRAM latency overlaps
// the phases in between and the sweeps only touch shared memory.  Record arrays start on 16-byte boundaries.
FB_DEV void tsolve_stage_issue(const DevModel& m, const DevData& d, ShTree& sh, int e, int y, const float* LD) {
  float* xs = sh_dyn(sh); float* lds = xs + FB_NXS(m);
#ifdef __CUDACC__
  unsigned sa = (unsigned)__cvta_generic_to_shared(lds);
  for (int k = 4 * y; k < m.nM; k += 4 * FB_NY) asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(sa + 4u * k), "l"(&AT(LD, k)) : "memory");
  asm volatile("cp.async.commit_group;" ::: "memory");
#else
  for (int k = y; k < m.nM; k += FB_NY) LDS(k) = AT(LD, k);
#endif
}
FB_DEV void tsolve_stage_wait(FB_PHASE_ARGS) {
  float* xs = sh_dyn(sh);
#ifdef __CUDACC__
  asm volatile("cp.async.wait_all;" ::: "memory");
#endif
  for (int k = y; k < FB_ROOTD * m.nlist; k += FB_NY) XS(m.nv + k) = 0;      // the lists' private root accumulators
}
// x <- L^-T x restricted to the list dofs, deepest first: x[anc] -= L[k][anc] x[k]
FB_DEV void tsolve_a_step_h(const DevModel& m, const DevData& d, ShTree& sh, int e, int y, unsigned hd) {
  float* xs = sh_dyn(sh); const float* lds = xs + FB_NXS(m);
  if (hd == FB_HDR_IDLE) return;
  const int sub = y % FB_FSUB, k = HDR_DOF(hd), adrk = HDR_ADR(hd), len = HDR_LEN(hd);
  const unsigned char* slot8 = TS_SLOT8(sh, m);
  float xk = XS(k) / LDS(adrk);                    // rows are stored unscaled: L[k][anc] x[k] = M'[k][anc] (x[k] / D[k])
  for (int t = 1 + sub; t < len; t += FB_FSUB) XS(slot8[adrk + t]) -= LDS(adrk + t) * xk;
}
FB_DEV void tsolve_a_step(const DevModel& m, const DevData& d, ShTree& sh, int e, int y, int step) {
  tsolve_a_step_h(m, d, sh, e, y, TS_HDR_A(sh, m)[step * FB_NY + y]);
}
// root blocks: collect the lists' contributions, then the dense (<= 6x6) back / scale / forward substitution
FB_DEV void tsolve_b_gather(FB_PHASE_ARGS) {
  float* xs = sh_dyn(sh);
  for (int r = 0; r < m.nroot; r++) {
    int b = m.root_body[r], nd = m.body_dofnum[b], d0 = m.body_dofadr[b];
    if (y >= nd) continue;
    float acc = 0;
    for (int l = 0; l < m.nlist; l++) if (m.list_root[l] == r) acc += XS(m.nv + FB_ROOTD * l + y);
    XS(d0 + y) += acc;
  }
}
FB_DEV void tsolve_root_a(FB_PHASE_ARGS) {       // x <- L^-T x inside the root block, one lane per root body
  float* xs = sh_dyn(sh); const float* lds = xs + FB_NXS(m);
  if (y >= m.nroot) return;
  int b = m.root_body[y], nd = m.body_dofnum[b], d0 = m.body_dofadr[b];
  for (int kl = nd - 1; kl >= 0; kl--) {
    int adrk = m.dof_Madr[d0 + kl]; float xk = XS(d0 + kl) / LDS(adrk);
    for (int t = 1; t <= kl; t++) XS(d0 + kl - t) -= LDS(adrk + t) * xk;
  }
}
FB_DEV void tsolve_root_c(FB_PHASE_ARGS) {       // x <- L^-1 x inside the root block
  float* xs = sh_dyn(sh); const float* lds = xs + FB_NXS(m);
  if (y >= m.nroot) return;
  int b = m.root_body[y], nd = m.body_dofnum[b], d0 = m.body_dofadr[b];
  for (int kl = 0; kl < nd; kl++) {
    int adrk = m.dof_Madr[d0 + kl];
    float p = 0;
    for (int t = 1; t <= kl; t++) p += LDS(adrk + t) * XS(d0 + kl - t);
    XS(d0 + kl) -= p / LDS(adrk);
  }
}
FB_DEV void tsolve_scale(FB_PHASE_ARGS) {        // x <- D^-1 x
  float* xs = sh_dyn(sh); const float* lds = xs + FB_NXS(m);
  for (int k = y; k < m.nv; k += FB_NY) XS(k) /= LDS(m.dof_Madr[k]);
}
// x <- L^-1 x on the list dofs, shallowest first: x[k] -= sum_t L[k][anc_t] x[anc_t]
FB_DEV void tsolve_c_step(const DevModel& m, const DevData& d, ShTree& sh, int e, int y, int step) {
  float* xs = sh_dyn(sh); const float* lds = xs + FB_NXS(m);
  const unsigned hd = TS_HDR_C(sh, m)[step * FB_NY + y];
  if (hd == FB_HDR_IDLE) return;
  const int sub = y % FB_FSUB, adrk = HDR_ADR(hd), len = HDR_LEN(hd);
  const unsigned char* anc8 = TS_ANC8(sh, m);
  float p = 0;
  for (int t = 1 + sub; t < len; t += FB_FSUB) p += LDS(adrk + t) * XS(anc8[adrk + t]);
  sh.red[y] = p;
}
FB_DEV void tsolve_c_fin(const DevModel& m, const DevData& d, ShTree& sh, int e, int y, int step) {
  float* xs = sh_dyn(sh); const float* lds = xs + FB_NXS(m);
  const unsigned hd = TS_HDR_C(sh, m)[step * FB_NY + y];
  if (hd == FB_HDR_IDLE || y % FB_FSUB != 0) return;
  float p = 0;
  for (int u = 0; u < FB_FSUB; u++) p += sh.red[y + u];
  XS(HDR_DOF(hd)) -= p / LDS(HDR_ADR(hd));
}
// M^-1 = L^-1 D^-1 L^-T is applied in halves so that callers can work between them (the factor must have been issued
// with tsolve_stage_issue by this warp):
//   tsolve_a : wait for the staged factor, x <- L^-T x
//   tsolve_c : x <- L^-1 x
FB_WARPFN void tsolve_a(const DevModel& m, const DevData& d, ShTree& sh, int e) {
  WPAR_BEGIN tsolve_stage_wait(m, d, sh, e, lane); WPAR_END
#ifdef __CUDACC__
  { const int lane = threadIdx.x; const unsigned* hp = TS_HDR_A(sh, m) + lane;
    unsigned hd = m.max_list_ndof > 0 ? hp[0] : FB_HDR_IDLE;
    for (int step = 0; step < m.max_list_ndof; step++) {
      const unsigned nxt = step + 1 < m.max_list_ndof ? hp[(step + 1) * FB_NY] : FB_HDR_IDLE;      // next step's header in flight during this step
      tsolve_a_step_h(m, d, sh, e, lane, hd); __syncwarp();
      hd = nxt;
    } }
#else
  for (int step = 0; step < m.max_list_ndof; step++) { WPAR_BEGIN tsolve_a_step(m, d, sh, e, lane, step); WPAR_END }
#endif
  WPAR_BEGIN tsolve_b_gather(m, d, sh, e, lane); WPAR_END
  WPAR_BEGIN tsolve_root_a(m, d, sh, e, lane); WPAR_END
}
#ifdef __CUDACC__
// GPU: the three partial dot products of a list are combined with two shuffles instead of a trip through shared memory
// and a second barrier (the host emulation runs the lanes one after the other and keeps the two-section form)
FB_DEV void tsolve_c_step_shfl(const DevModel& m, const DevData& d, ShTree& sh, int e, int y, unsigned hd) {
  float* xs = sh_dyn(sh); const float* lds = xs + FB_NXS(m);
  const bool active = hd != FB_HDR_IDLE;
  const int sub = y % FB_FSUB, k = HDR_DOF(hd), adrk = HDR_ADR(hd);
  const unsigned char* anc8 = TS_ANC8(sh, m);
  float p = 0;
  if (active) {
    const int len = HDR_LEN(hd);
    for (int t = 1 + sub; t < len; t += FB_FSUB) p += LDS(adrk + t) * XS(anc8[adrk + t]);
  }
  float p1 = __shfl_down_sync(0xffffffffu, p, 1), p2 = __shfl_down_sync(0xffffffffu, p, 2);
  if (active && sub == 0) XS(k) -= (p + p1 + p2) / LDS(adrk);
}
#endif
FB_WARPFN void tsolve_c(const DevModel& m, const DevData& d, ShTree& sh, int e) {
  WPAR_BEGIN tsolve_root_c(m, d, sh, e, lane); WPAR_END
#ifdef __CUDACC__
  { const int lane = threadIdx.x; const unsigned* hp = TS_HDR_C(sh, m) + lane;
    unsigned hd = m.max_list_ndof > 0 ? hp[0] : FB_HDR_IDLE;
    for (int step = 0; step < m.max_list_ndof; step++) {
      const unsigned nxt = step + 1 < m.max_list_ndof ? hp[(step + 1) * FB_NY] : FB_HDR_IDLE;
      tsolve_c_step_shfl(m, d, sh, e, lane, hd); __syncwarp();
      hd = nxt;
    } }
#else
  for (int step = 0; step < m.max_list_ndof; step++) {
    WPAR_BEGIN tsolve_c_step(m, d, sh, e, lane, step); WPAR_END
    WPAR_BEGIN tsolve_c_fin(m, d, sh, e, lane, step); WPAR_END
  }
#endif
}
FB_WARPFN void tri_solve(const DevModel& m, const DevData& d, ShTree& sh, int e) {
  tsolve_a(m, d, sh, e);
  WPAR_BEGIN tsolve_scale(m, d, sh, e, lane); WPAR_END
  tsolve_c(m, d, sh, e);
}

// ---------------------------------------------------------------------------------------------
// K4 velocities + RNE bias, K5-K7 passive forces (MuJoCo mj_comVel, mj_rne, mj_passive)
FB_DEV S6 motion_cross(const S6& v, V3 Sa, V3 Sl) { S6 r; r.a = cross(v.a, Sa); r.l = cross(v.a, Sl) + cross(v.l, Sa); return r; }

// The three dofs da .. da + 2 of a ball joint (MuJoCo mj_comVel's BALL case, which FREE falls through to):
// v += S qd (qacc != nullptr: a += S qacc) and the cdof_dot term.  Ball joints sit on root bodies (fb_create), so the velocity before
// them is (0, vlin) and sum_i cdof_dot_i qd_i = (0, vlin x w).
FB_DEV void rot3_vel_acc(const DevData& d, int e, int da, V3 vlin, const float* qacc, S6& v, S6& a) {
  V3 w = v3(0, 0, 0);
  for (int i = 0; i < 3; i++) {
    float qd = AT(d.qvel, da + i);
    V3 Sa = ld3(d.Sang, da + i, d, e), Sl = ld3(d.Slin, da + i, d, e);
    v.a = v.a + Sa * qd; v.l = v.l + Sl * qd;
    w = w + Sa * qd;
    if (qacc) { float qa = AT(qacc, da + i); a.a = a.a + Sa * qa; a.l = a.l + Sl * qa; }
  }
  a.l = a.l + cross(vlin, w);
}
// inertial force of body b: I a + v x* (I v), [torque about ref; force]
FB_DEV S6 body_inertial_force(const DevModel& m, const DevData& d, int e, int b, const float* bvel, const float* bacc) {
  I10 I = ld10(d.inert10, b, d, e);
  S6 v = ld6(bvel, b, d, e), a = ld6(bacc, b, d, e);
  V3 L, p, La, pa;
  inert_mul(I, v.a, v.l, L, p); inert_mul(I, a.a, a.l, La, pa);
  S6 f;
  f.a = La + cross(v.a, L) + cross(v.l, p);
  f.l = pa + cross(v.a, p);
  return f;
}
FB_DEV float pow4(float x) { float y = x * x; return y * y; }
// fluid wrench on body b about ref (inertia-box model, or ellipsoid model for flagged bodies).  OVL: density, viscosity, wind, mass
// and inertia of the env's overlay row.  The velocity kernel runs at its register limit, so the overlay gets a kernel instance of its
// own (launch_step1) instead of a test in this one: the instance without it is the code of a handle that never set parameters.
template <bool OVL> FB_DEV S6 body_fluid_wrench(const DevModel& m, const DevData& d, int e, int b) {
  S6 out; out.a = v3(0, 0, 0); out.l = v3(0, 0, 0);
  const float* prm = d.prm + (unsigned)e * d.prm_stride;
  float rho = OVL ? prm[d.prm_off[FB_P_DENSITY]] : m.density, eta = OVL ? prm[d.prm_off[FB_P_VISCOSITY]] : m.viscosity;
  float mass = OVL ? prm[d.prm_off[FB_P_BODY_MASS] + b] : m.body_mass[b];
  if ((rho <= 0 && eta <= 0) || mass < FB_MINVAL) return out;
  S6 bv = ld6(d.bvel, b, d, e);
  const float* wp = prm + d.prm_off[FB_P_WIND];
  V3 wind = OVL ? v3(wp[0], wp[1], wp[2]) : v3(m.wind[0], m.wind[1], m.wind[2]);
  const float PI = 3.14159265358979f;
  if (!m.body_fluid_ellipsoid[b]) {
    V3 I = mld3(OVL ? prm + d.prm_off[FB_P_BODY_INERTIA] : m.body_inertia, b);
    float bx = sqrtf(fmaxf(FB_MINVAL, I.y + I.z - I.x) / mass * 6.0f);
    float by = sqrtf(fmaxf(FB_MINVAL, I.x + I.z - I.y) / mass * 6.0f);
    float bz = sqrtf(fmaxf(FB_MINVAL, I.x + I.y - I.z) / mass * 6.0f);
    V3 c = ld3(d.xipos, b, d, e);
    M3 R = ld9(d.ximat, b, d, e);
    V3 lw = mulT(R, bv.a), lv = mulT(R, bv.l + cross(bv.a, c) - wind);
    V3 tq = v3(0, 0, 0), fr = v3(0, 0, 0);
    if (eta > 0) {
      float diam = (bx + by + bz) / 3.0f;
      tq = lw * (-PI * diam * diam * diam * eta);
      fr = lv * (-3.0f * PI * diam * eta);
    }
    if (rho > 0) {
      fr.x -= 0.5f * rho * by * bz * fabsf(lv.x) * lv.x;
      fr.y -= 0.5f * rho * bx * bz * fabsf(lv.y) * lv.y;
      fr.z -= 0.5f * rho * bx * by * fabsf(lv.z) * lv.z;
      tq.x -= rho * bx * (pow4(by) + pow4(bz)) * fabsf(lw.x) * lw.x / 64.0f;
      tq.y -= rho * by * (pow4(bx) + pow4(bz)) * fabsf(lw.y) * lw.y / 64.0f;
      tq.z -= rho * bz * (pow4(bx) + pow4(by)) * fabsf(lw.z) * lw.z / 64.0f;
    }
    V3 F = mul(R, fr), T = mul(R, tq);
    out.l = F; out.a = T + cross(c, F);
    return out;
  }
  // ellipsoid model (reference flybody/ellipsoid_fluid_model.py:88-310) for every fluid geom of this body
  for (int g = 0; g < m.nfluid; g++) {
    if (m.fluid_bodyid[g] != b) continue;
    const float* coef = m.fluid_coef + 12 * g;
    if (coef[0] == 0.0f) continue;
    V3 size = mld3(m.fluid_size, g);
    V3 bpos = ld3(d.xpos, b, d, e); Q4 bq = ld4(d.xquat, b, d, e);
    M3 bR = q2m(bq);
    V3 gpos = bpos + mul(bR, mld3(m.fluid_pos, g));
    M3 gR = q2m(qmul(bq, mld4(m.fluid_quat, g)));
    V3 lw = mulT(gR, bv.a), lv = mulT(gR, bv.l + cross(bv.a, gpos) - wind);
    float blunt = coef[1], slender = coef[2], angc = coef[3], kutta = coef[4], magnus = coef[5];
    V3 vmass = v3(coef[6], coef[7], coef[8]), vin = v3(coef[9], coef[10], coef[11]);
    V3 vlm = v3(rho * vmass.x * lv.x, rho * vmass.y * lv.y, rho * vmass.z * lv.z);
    V3 vam = v3(rho * vin.x * lw.x, rho * vin.y * lw.y, rho * vin.z * lw.z);
    V3 tq = cross(vlm, lv) + cross(vam, lw);
    V3 fr = cross(vlm, lw);
    float volume = 4.0f / 3.0f * PI * size.x * size.y * size.z;
    float dmax = fmaxf(size.x, fmaxf(size.y, size.z)), dmin = fminf(size.x, fminf(size.y, size.z));
    float dmid = size.x + size.y + size.z - dmax - dmin;
    float A_max = PI * dmax * dmid;
    V3 magf = cross(lw, lv) * (magnus * rho * volume);
    float s12 = size.y * size.z, s20 = size.z * size.x, s01 = size.x * size.y;
    float proj_denom = pow4(s12) * lv.x * lv.x + pow4(s20) * lv.y * lv.y + pow4(s01) * lv.z * lv.z;
    float proj_num = (s12 * lv.x) * (s12 * lv.x) + (s20 * lv.y) * (s20 * lv.y) + (s01 * lv.z) * (s01 * lv.z);
    // the products of 1e-3 .. 1e-1 cm semi-axes underflow fp32 MINVAL=1e-15; use a scaled guard
    float A_proj = PI * sqrtf(proj_denom / fmaxf(1e-37f, proj_num));
    V3 nrm = v3(s12 * s12 * lv.x, s20 * s20 * lv.y, s01 * s01 * lv.z);
    float speed = norm(lv);
    float cos_alpha = proj_num / fmaxf(1e-37f, speed * proj_denom);
    V3 kc = cross(nrm, lv) * (kutta * rho * cos_alpha * A_proj);
    V3 kf = cross(kc, lv);
    float eqD = 2.0f / 3.0f * (size.x + size.y + size.z);
    float lin_coef = 3.0f * PI * eqD, ang_coef = PI * eqD * eqD * eqD;
    float I_max = 8.0f / 15.0f * PI * dmid * pow4(dmax);
    float II0 = 8.0f / 15.0f * PI * size.x * pow4(fmaxf(size.y, size.z));
    float II1 = 8.0f / 15.0f * PI * size.y * pow4(fmaxf(size.z, size.x));
    float II2 = 8.0f / 15.0f * PI * size.z * pow4(fmaxf(size.x, size.y));
    V3 mom = v3(lw.x * (angc * II0 + slender * (I_max - II0)), lw.y * (angc * II1 + slender * (I_max - II1)),
                lw.z * (angc * II2 + slender * (I_max - II2)));
    float drag_lin = eta * lin_coef + rho * speed * (A_proj * blunt + slender * (A_max - A_proj));
    float drag_ang = eta * ang_coef + rho * norm(mom);
    tq = tq - lw * drag_ang;
    fr = fr + magf + kf - lv * drag_lin;
    tq = tq * coef[0]; fr = fr * coef[0];
    V3 F = mul(gR, fr), T = mul(gR, tq);
    out.l = out.l + F; out.a = out.a + T + cross(gpos, F);
  }
  return out;
}

// velocity stage.  Chain part (lists): body velocities and bias accelerations, the parent's values carried in
// registers along a chain.  Per-body part (all lanes): inertial bias force and fluid wrench.  Backward part
// (lists): subtree sums, carried in registers.  Per-dof part (all lanes): projections onto the dofs.
FB_DEV void vel_acc_from_parent(const DevModel& m, const DevData& d, int e, int b, S6& v, S6& a) {
  int jn = m.body_jntnum[b];
  for (int k = 0; k < jn; k++) {
    int j = m.body_jntadr[b] + k, da = m.jnt_dofadr[j];
    if (m.jnt_type[j] == FB_JNT_FREE) {
      V3 vlin = v3(AT(d.qvel, da), AT(d.qvel, da + 1), AT(d.qvel, da + 2)), w = v3(0, 0, 0);
      for (int i = 0; i < 6; i++) {
        float qd = AT(d.qvel, da + i);
        V3 Sa = ld3(d.Sang, da + i, d, e), Sl = ld3(d.Slin, da + i, d, e);
        v.a = v.a + Sa * qd; v.l = v.l + Sl * qd;
        if (i >= 3) w = w + Sa * qd;
      }
      a.l = a.l + cross(vlin, w);
    } else if (m.jnt_type[j] == FB_JNT_BALL) { FB_NO_MERGE(); rot3_vel_acc(d, e, da, v.l, nullptr, v, a); FB_NO_MERGE(); }
    else {
      float qd = AT(d.qvel, da);
      V3 Sa = ld3(d.Sang, da, d, e), Sl = ld3(d.Slin, da, d, e);
      S6 r = motion_cross(v, Sa, Sl);
      a.a = a.a + r.a * qd; a.l = a.l + r.l * qd;
      v.a = v.a + Sa * qd; v.l = v.l + Sl * qd;
    }
  }
  st6(d.bvel, b, d, e, v); st6(d.bacc, b, d, e, a);
}
FB_DEV void st6v(float* arr, int b, const DevData& d, int e, const float* v) { st3(arr, 2 * b, d, e, v3(v[0], v[1], v[2])); st3(arr, 2 * b + 1, d, e, v3(v[3], v[4], v[5])); }
FB_DEV void add6v(float* arr, int b, const DevData& d, int e, const float* v) {
  S6 s = ld6(arr, b, d, e); s.a = s.a + v3(v[0], v[1], v[2]); s.l = s.l + v3(v[3], v[4], v[5]); st6(arr, b, d, e, s);
}
FB_DEV void kvel_p0(FB_PHASE_ARGS) {
  // inputs written by the position kernel three launches ago: ask for them now, all lines at once
  prefetch_rec(d.Sang, FB_V3S * m.nv, d, e, y); prefetch_rec(d.Slin, FB_V3S * m.nv, d, e, y); prefetch_rec(d.inert10, FB_I10S * m.nbody, d, e, y);
  prefetch_rec(d.xipos, FB_V3S * m.nbody, d, e, y); prefetch_rec(d.ximat, FB_M3S * m.nbody, d, e, y);
  if (y != 0) return;
  S6 z; z.a = v3(0, 0, 0); z.l = v3(0, 0, 0);
  st6(d.bvel, 0, d, e, z);
  S6 g = z; g.l = v3(-PRMS(FB_P_GRAVITY, 0, m.gravity[0]), -PRMS(FB_P_GRAVITY, 1, m.gravity[1]), -PRMS(FB_P_GRAVITY, 2, m.gravity[2]));
  st6(d.bacc, 0, d, e, g);
  for (int r = 0; r < m.nroot; r++) { S6 v = z, a = g; vel_acc_from_parent(m, d, e, m.root_body[r], v, a); }
}
FB_DEV void kvel_p1(FB_PHASE_ARGS) {
  if (y >= m.nlist) return;
  int prev = -1; S6 cv, ca; cv.a = cv.l = ca.a = ca.l = v3(0, 0, 0);
  FB_LIST_LOOP_FWD {
    int p = m.body_parentid[b];
    if (p != prev) { cv = ld6(d.bvel, p, d, e); ca = ld6(d.bacc, p, d, e); }
    vel_acc_from_parent(m, d, e, b, cv, ca);
    prev = b;
  }
}
// (Subtree sums of the velocity stage stay in the record: moving them to shared memory as in the position kernel costs 3.3 KB more
// shared memory per warp, which shrinks the L1 the scattered record loads live in.)
// all lanes over bodies: bias force (kept un-accumulated in bfrc0 for the sensor pass) and fluid wrench
template <bool OVL> FB_DEV void kvel_p1b(FB_PHASE_ARGS) {
  for (int b = y; b < m.nbody; b += FB_NY) {
    S6 f; f.a = f.l = v3(0, 0, 0); S6 fl = f;
    if (b > 0) { f = body_inertial_force(m, d, e, b, d.bvel, d.bacc); fl = body_fluid_wrench<OVL>(m, d, e, b); }
    st6(d.bfrc, b, d, e, f); st6(d.bfrc0, b, d, e, f); st6(d.bfl, b, d, e, fl);
  }
}
// subtree sums of (bias force, fluid wrench): child -> parent along the lists
FB_DEV void kvel_p2(FB_PHASE_ARGS) {
  float* part_ = sh_dyn(sh);
  if (y >= m.nlist) return;
  float acc[12], carry[12]; int carry_to = -1;
  for (int k = 0; k < 12; k++) { acc[k] = 0; carry[k] = 0; }
  FB_LIST_LOOP_REV {
    float cur[12];
    { S6 f_ = ld6(d.bfrc, b, d, e), g_ = ld6(d.bfl, b, d, e);
      cur[0] = f_.a.x; cur[1] = f_.a.y; cur[2] = f_.a.z; cur[3] = f_.l.x; cur[4] = f_.l.y; cur[5] = f_.l.z;
      cur[6] = g_.a.x; cur[7] = g_.a.y; cur[8] = g_.a.z; cur[9] = g_.l.x; cur[10] = g_.l.y; cur[11] = g_.l.z; }
    if (carry_to == b) { for (int k = 0; k < 12; k++) cur[k] += carry[k]; st6v(d.bfrc, b, d, e, cur); st6v(d.bfl, b, d, e, cur + 6); }
    else if (carry_to >= 0) { add6v(d.bfrc, carry_to, d, e, carry); add6v(d.bfl, carry_to, d, e, carry + 6); }
    int p = m.body_parentid[b];
    if (m.body_isroot[p]) { for (int k = 0; k < 12; k++) acc[k] += cur[k]; carry_to = -1; }
    else { for (int k = 0; k < 12; k++) carry[k] = cur[k]; carry_to = p; }
  }
  if (carry_to >= 0) { add6v(d.bfrc, carry_to, d, e, carry); add6v(d.bfl, carry_to, d, e, carry + 6); }
  for (int k = 0; k < 12; k++) PARTL(y, k, 12) = acc[k];
}
FB_DEV void sensors_vel(const DevModel& m, const DevData& d, int e, int y);
FB_DEV void kvel_p3(FB_PHASE_ARGS) {
  float* part_ = sh_dyn(sh);
  for (int t = y; t < 12 * m.nroot; t += FB_NY) {      // lanes over (root, component): the lists' partial sums onto the root bodies
    const int r = t / 12, k = t - 12 * r, b = m.root_body[r];
    float a = 0;
    for (int l = 0; l < m.nlist; l++) if (m.list_root[l] == r) a += PARTL(l, k, 12);
    if (k < 6) AT(d.bfrc, S6I(b, k)) += a; else AT(d.bfl, S6I(b, k - 6)) += a;
  }
  sensors_vel(m, d, e, y);
}
// all lanes over dofs: qfrc_bias = S . f_subtree ; qfrc_passive = S . fluid_subtree + springs + dampers
FB_DEV void kvel_p3b(FB_PHASE_ARGS) {
  const float *damp = PRM(FB_P_DOF_DAMPING, m.dof_damping), *stiff = PRM(FB_P_JNT_STIFFNESS, m.jnt_stiffness);
  for (int k = y; k < m.nv; k += FB_NY) {
    int b = m.dof_bodyid[k];
    V3 Sa = ld3(d.Sang, k, d, e), Sl = ld3(d.Slin, k, d, e);
    S6 f = ld6(d.bfrc, b, d, e), fl = ld6(d.bfl, b, d, e);
    AT(d.qfrc_bias, k) = dot(Sa, f.a) + dot(Sl, f.l);
    float pas = dot(Sa, fl.a) + dot(Sl, fl.l) - damp[k] * AT(d.qvel, k);
    int j = m.dof_jntid[k];
    if (m.jnt_type[j] == FB_JNT_HINGE) { int qa = m.jnt_qposadr[j]; pas -= stiff[j] * (AT(d.qpos, qa) - m.qpos_spring[qa]); }
    AT(d.qfrc_passive, k) = pas;
  }
}
// gyro / velocimeter (MuJoCo mj_sensorVel; sensors fruitfly.xml:900-903)
FB_DEV void sensors_vel(const DevModel& m, const DevData& d, int e, int y) {
  for (int s = y; s < m.nsensor; s += FB_NY) {
    int tp = m.sensor_type[s];
    if (tp != FB_SENS_GYRO && tp != FB_SENS_VELOCIMETER) continue;
    int site = m.sensor_objid[s], adr = m.sensor_adr[s], b = m.site_bodyid[site];
    S6 v = ld6(d.bvel, b, d, e);
    M3 R = ld9(d.site_xmat, site, d, e);
    V3 out;
    if (tp == FB_SENS_GYRO) out = mulT(R, v.a);
    else out = mulT(R, v.l + cross(v.a, ld3(d.site_xpos, site, d, e)));
    AT(d.sensordata, adr) = out.x; AT(d.sensordata, adr + 1) = out.y; AT(d.sensordata, adr + 2) = out.z;
  }
}
