/* ik_reference.c -- fp64 restatement of the reference's multi-site inverse kinematics (flybody/inverse_kinematics.py:96-151:
 * qpos_from_site_xpos) for one problem, TEST INFRASTRUCTURE for tests/test_inverse_kinematics.py (compiled by tests/ik_reference.py).
 *
 * Kinematics as MuJoCo's mj_kinematics (hinge and free joints; a model with a ball joint is refused), the translational Jacobian of a
 * site as mj_jacSite, the step as mj_integratePos.  Objective: sum over included components of (site_xpos - target)^2 +
 * reg * |fitted hinge qpos|^2; gradient 2 diff^T J + 2 reg q_hinge; momentum u <- beta u + g; qpos <- integratePos(qpos, -lr u); every
 * 100 steps from step 0 the stopping test lr |u| / objective < thr.  Two deliberate differences from the reference, which the CUDA
 * solver shares: an objective of 0 counts as converged (the reference divides by it), and err_first is the site term at the returned
 * qpos (the reference's is one update stale when it stops at max_steps). */
#include <math.h>
#include <stdlib.h>
#include <string.h>
#include "../include/flybody_b200.h"

typedef struct IkProblem {
  int n_sites; const int* site_ids; int n_jnts; const int* jnt_ids;
  const unsigned char* include;        /* [3 n_sites] components in the objective, NULL = all */
  const double* target;                /* [n_sites][3] world frame; a NaN component is excluded */
  double reg, lr, beta, thr; int max_steps;
} IkProblem;

typedef struct {
  const FbModel* m; const IkProblem* k;
  double *qpos, *xpos, *xquat, *axis, *anchor, *site;   /* per body / per dof (world axis, point it turns about) / per program site */
  int *lin;                                              /* per dof: 1 for a free joint's translation */
  int *dof, *hq, nfd;                                    /* fitted dofs (joint order); qpos address of a fitted hinge, -1 otherwise */
  unsigned char* below;                                  /* [n_sites][nv]: the dof moves the site */
  double *r, *g, *u, *v;
} Ik;

static void qmul(double* r, const double* a, const double* b) {
  double w = a[0]*b[0]-a[1]*b[1]-a[2]*b[2]-a[3]*b[3], x = a[0]*b[1]+a[1]*b[0]+a[2]*b[3]-a[3]*b[2];
  double y = a[0]*b[2]-a[1]*b[3]+a[2]*b[0]+a[3]*b[1], z = a[0]*b[3]+a[1]*b[2]-a[2]*b[1]+a[3]*b[0];
  r[0]=w; r[1]=x; r[2]=y; r[3]=z;
}
static void qnorm(double* q) {
  double n = sqrt(q[0]*q[0]+q[1]*q[1]+q[2]*q[2]+q[3]*q[3]);
  if (n < 1e-15) { q[0]=1; q[1]=q[2]=q[3]=0; } else for (int i=0;i<4;i++) q[i]/=n;
}
static void q2m(double* R, const double* q) {
  double w=q[0], x=q[1], y=q[2], z=q[3];
  R[0]=w*w+x*x-y*y-z*z; R[1]=2*(x*y-w*z); R[2]=2*(x*z+w*y);
  R[3]=2*(x*y+w*z); R[4]=w*w-x*x+y*y-z*z; R[5]=2*(y*z-w*x);
  R[6]=2*(x*z-w*y); R[7]=2*(y*z+w*x); R[8]=w*w-x*x-y*y+z*z;
}
static void mv(double* r, const double* R, const double* v) {
  double x=R[0]*v[0]+R[1]*v[1]+R[2]*v[2], y=R[3]*v[0]+R[4]*v[1]+R[5]*v[2], z=R[6]*v[0]+R[7]*v[1]+R[8]*v[2];
  r[0]=x; r[1]=y; r[2]=z;
}
static void axisangle(double* q, const double* axis, double ang) {
  double s = sin(0.5*ang); q[0]=cos(0.5*ang); q[1]=axis[0]*s; q[2]=axis[1]*s; q[3]=axis[2]*s;
}

/* mj_kinematics for the bodies, the dofs' world axes / anchors, and the program's sites */
static void kinematics(Ik* s) {
  const FbModel* m = s->m;
  s->xpos[0]=s->xpos[1]=s->xpos[2]=0; s->xquat[0]=1; s->xquat[1]=s->xquat[2]=s->xquat[3]=0;
  for (int b=1;b<m->nbody;b++) {
    int p = m->body_parentid[b];
    double R[9], pos[3], quat[4], t[3];
    q2m(R, s->xquat+4*p); mv(t, R, m->body_pos+3*b);
    for (int i=0;i<3;i++) pos[i]=s->xpos[3*p+i]+t[i];
    qmul(quat, s->xquat+4*p, m->body_quat+4*b);
    for (int a=0;a<m->body_jntnum[b];a++) {
      int j=m->body_jntadr[b]+a, qa=m->jnt_qposadr[j], da=m->jnt_dofadr[j];
      if (m->jnt_type[j]==FB_JNT_FREE) {
        memcpy(pos, s->qpos+qa, 3*sizeof(double)); memcpy(quat, s->qpos+qa+3, 4*sizeof(double)); qnorm(quat);
        q2m(R, quat);
        for (int i=0;i<3;i++) {
          for (int c=0;c<3;c++) { s->axis[3*(da+i)+c]=(c==i); s->axis[3*(da+3+i)+c]=R[3*c+i]; s->anchor[3*(da+3+i)+c]=pos[c]; }
          s->lin[da+i]=1; s->lin[da+3+i]=0;
        }
      } else {
        double anchor[3], jq[4], nq[4];
        q2m(R, quat); mv(t, R, m->jnt_pos+3*j);
        for (int c=0;c<3;c++) anchor[c]=pos[c]+t[c];
        mv(s->axis+3*da, R, m->jnt_axis+3*j); memcpy(s->anchor+3*da, anchor, sizeof(anchor)); s->lin[da]=0;
        axisangle(jq, m->jnt_axis+3*j, s->qpos[qa]-m->qpos0[qa]); qmul(nq, quat, jq); memcpy(quat, nq, sizeof(nq));
        q2m(R, quat); mv(t, R, m->jnt_pos+3*j);
        for (int c=0;c<3;c++) pos[c]=anchor[c]-t[c];
      }
    }
    qnorm(quat);
    memcpy(s->xpos+3*b, pos, sizeof(pos)); memcpy(s->xquat+4*b, quat, sizeof(quat));
  }
  for (int q=0;q<s->k->n_sites;q++) {
    int sid=s->k->site_ids[q], b=m->site_bodyid[sid]; double R[9], t[3];
    q2m(R, s->xquat+4*b); mv(t, R, m->site_pos+3*sid);
    for (int c=0;c<3;c++) s->site[3*q+c]=s->xpos[3*b+c]+t[c];
  }
}
/* sum of squared included differences; r (may be NULL) <- 2 diff, 0 where excluded */
static double site_term(const Ik* s, double* r) {
  double e=0;
  for (int q=0;q<s->k->n_sites;q++) for (int c=0;c<3;c++) {
    double t=s->k->target[3*q+c];
    int inc=(!s->k->include || s->k->include[3*q+c]) && t==t;
    double df = inc ? s->site[3*q+c]-t : 0;
    e+=df*df; if (r) r[3*q+c]=2*df;
  }
  return e;
}
static double hinge_sq(const Ik* s) { double h=0; for (int i=0;i<s->nfd;i++) if (s->hq[i]>=0) h+=s->qpos[s->hq[i]]*s->qpos[s->hq[i]]; return h; }
/* gradient over the fitted dofs: column of mj_jacSite (axis x (site - anchor), or the axis for a translation) dotted with 2 diff */
static void gradient(Ik* s) {
  site_term(s, s->r);
  for (int i=0;i<s->nfd;i++) {
    int k=s->dof[i]; double g = s->hq[i]>=0 ? 2*s->k->reg*s->qpos[s->hq[i]] : 0;
    const double* a=s->axis+3*k;
    for (int q=0;q<s->k->n_sites;q++) {
      if (!s->below[(size_t)q*s->m->nv+k]) continue;
      double j[3];
      if (s->lin[k]) { j[0]=a[0]; j[1]=a[1]; j[2]=a[2]; }
      else { double d[3]={s->site[3*q]-s->anchor[3*k], s->site[3*q+1]-s->anchor[3*k+1], s->site[3*q+2]-s->anchor[3*k+2]};
             j[0]=a[1]*d[2]-a[2]*d[1]; j[1]=a[2]*d[0]-a[0]*d[2]; j[2]=a[0]*d[1]-a[1]*d[0]; }
      g += s->r[3*q]*j[0]+s->r[3*q+1]*j[1]+s->r[3*q+2]*j[2];
    }
    s->g[i]=g;
  }
}
/* mj_integratePos of the fitted joints with the step v over the fitted dofs (free joint: world-frame translation, body-frame rotation) */
static void integrate(Ik* s, const double* v) {
  const FbModel* m=s->m; int f=0;
  for (int a=0;a<s->k->n_jnts;a++) {
    int j=s->k->jnt_ids[a], qa=m->jnt_qposadr[j];
    if (m->jnt_type[j]==FB_JNT_HINGE) { s->qpos[qa]+=v[f++]; continue; }
    for (int c=0;c<3;c++) s->qpos[qa+c]+=v[f+c];
    double w[3]={v[f+3],v[f+4],v[f+5]}, qr[4], q[4], ang=sqrt(w[0]*w[0]+w[1]*w[1]+w[2]*w[2]);
    if (ang<1e-15) { w[0]=1; w[1]=w[2]=0; } else for (int c=0;c<3;c++) w[c]/=ang;
    axisangle(qr, w, ang);
    qnorm(s->qpos+qa+3); qmul(q, s->qpos+qa+3, qr); qnorm(q);
    memcpy(s->qpos+qa+3, q, sizeof(q));
    f+=6;
  }
}
static void release(Ik* s) {
  void* p[] = {s->xpos, s->xquat, s->axis, s->anchor, s->site, s->lin, s->dof, s->hq, s->below, s->r, s->g, s->u, s->v};
  for (size_t i=0;i<sizeof(p)/sizeof(p[0]);i++) free(p[i]);
}
static int setup(Ik* s, const FbModel* m, const IkProblem* k, double* qpos) {
  memset(s, 0, sizeof(*s));
  s->m=m; s->k=k; s->qpos=qpos;
  int nv=m->nv, nb=m->nbody, ns=k->n_sites;
  s->xpos=calloc(3*nb, sizeof(double)); s->xquat=calloc(4*nb, sizeof(double)); s->axis=calloc(3*nv+3, sizeof(double));
  s->anchor=calloc(3*nv+3, sizeof(double)); s->site=calloc(3*ns+3, sizeof(double)); s->lin=calloc(nv+1, sizeof(int));
  s->dof=calloc(nv+1, sizeof(int)); s->hq=calloc(nv+1, sizeof(int)); s->below=calloc((size_t)ns*nv+1, 1);
  s->r=calloc(3*ns+3, sizeof(double)); s->g=calloc(nv+1, sizeof(double)); s->u=calloc(nv+1, sizeof(double)); s->v=calloc(nv+1, sizeof(double));
  for (int j=0;j<m->njnt;j++) if (m->jnt_type[j]!=FB_JNT_FREE && m->jnt_type[j]!=FB_JNT_HINGE) return -1;
  for (int q=0;q<ns;q++) {
    if (k->site_ids[q]<0 || k->site_ids[q]>=m->nsite) return -1;
    for (int d=m->body_lastdof[m->site_bodyid[k->site_ids[q]]]; d>=0; d=m->dof_parentid[d]) s->below[(size_t)q*nv+d]=1;
  }
  for (int a=0;a<k->n_jnts;a++) {
    int j=k->jnt_ids[a];
    if (j<0 || j>=m->njnt) return -1;
    int nd = m->jnt_type[j]==FB_JNT_FREE ? 6 : 1;
    for (int i=0;i<nd;i++) { s->dof[s->nfd]=m->jnt_dofadr[j]+i; s->hq[s->nfd]=nd==1 ? m->jnt_qposadr[j] : -1; s->nfd++; }
  }
  return 0;
}

/* objective and its gradient over the fitted dofs (grad [nfd], may be NULL) at qpos; NaN for a refused problem */
double ikref_objective(const FbModel* m, const IkProblem* k, double* qpos, double* grad) {
  Ik s; double out=NAN;
  if (setup(&s, m, k, qpos)==0) {
    kinematics(&s); gradient(&s);
    if (grad) memcpy(grad, s.g, sizeof(double)*s.nfd);
    out=site_term(&s, NULL)+k->reg*hinge_sq(&s);
  }
  release(&s);
  return out;
}
/* the loop of qpos_from_site_xpos from qpos, which is left at the fit; 0, or -1 for a refused problem */
int ikref_solve(const FbModel* m, const IkProblem* k, double* qpos, double* err, double* err_first, int* steps, int* success) {
  Ik s; int rc=-1;
  if (setup(&s, m, k, qpos)==0 && k->max_steps>=1) {
    double e=NAN; int ok=0, step;
    kinematics(&s);
    for (step=0; step<k->max_steps; step++) {
      gradient(&s);
      for (int i=0;i<s.nfd;i++) { s.u[i]=k->beta*s.u[i]+s.g[i]; s.v[i]=-k->lr*s.u[i]; }
      integrate(&s, s.v);
      kinematics(&s);
      if (step%100==0) {
        e=site_term(&s, NULL)+k->reg*hinge_sq(&s);
        double un=0; for (int i=0;i<s.nfd;i++) un+=s.u[i]*s.u[i];
        if (e==0 || k->lr*sqrt(un)/e<k->thr) { ok=1; break; }
      }
    }
    if (step==k->max_steps) step=k->max_steps-1;
    *err=e; *err_first=site_term(&s, NULL); *steps=step; *success=ok; rc=0;
  }
  release(&s);
  return rc;
}
