/* fly_oracle.c -- CPU restatement (double precision, one environment, dense and simple) of the
 * physics step that runs under flybody.fly_envs: dm_control's `Physics.step()` with
 * legacy_step=True, i.e. MuJoCo `mj_step2; mj_step1` per substep, for the fly model.
 *
 * THIS IS TEST INFRASTRUCTURE.  Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
 * --impl reference legs may load it.  The product path (flybody_b200/csrc) never links or calls it.
 *
 * PARITY UNPINNED: neither `mujoco` nor `dm_control` is installable here (SURVEY.md 8(c)) and the
 * reference's tests hold no trajectory values, so this restatement follows the published MuJoCo
 * algorithms (engine_forward.c, engine_core_smooth.c, engine_passive.c, engine_collision_primitive.c,
 * engine_core_constraint.c, engine_solver.c, engine_sensor.c; mujoco is an un-pinned transitive
 * dependency of the reference, pyproject.toml:10) and is anchored by (a) the reference's model goldens
 * (tests/test_flybare.py:12-36, through the model compiler), (b) the in-tree Python restatement of the
 * ellipsoid fluid model (flybody/ellipsoid_fluid_model.py:88-310) and (c) physics invariants
 * (tests/test_oracle_invariants.py).
 *
 * Stage map (SURVEY.md 8(a) / App. A):
 *   K1 kinematics+comPos  orc_kinematics        K8  actuation      orc_actuation
 *   K2 crb+factor         orc_crb               K9  collision      orc_collision
 *   K3 tendon/transmission orc_transmission     K10 constraints    orc_make_constraint
 *   K4 comVel+rne bias    orc_bias              K11 solve+noslip   orc_solve / orc_noslip
 *   K5/K6/K7 passive      orc_passive           K12 sensors        orc_sensors
 *                                               K13 Euler          orc_euler
 * All spatial vectors are world-frame, referenced to the world origin, [angular; linear].
 */
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "../include/flybody_b200.h"

#define MINVAL 1e-15
#define ORC_MAXCON 256
#define ORC_MAXEFC 600
#define PI 3.14159265358979323846

typedef struct {
  double dist, pos[3], frame[9], includemargin, friction[5], solref[2], solimp[5], mu;
  int dim, geom1, geom2, exclude, efc_address;
} OrcContact;

typedef struct OrcData {
  const FbModel* m;
  /* state */
  double *qpos, *qvel, *act, *ctrl, *qacc, *qacc_warmstart, time;
  /* position stage */
  double *xpos, *xquat, *xmat, *xipos, *ximat, *geom_xpos, *geom_xmat, *site_xpos, *site_xmat, *subtree_com;
  double *Sang, *Slin;          /* per dof motion subspace */
  double *inert10;              /* per body: m, h[3], I_O[6] (xx,yy,zz,xy,xz,yz) about world origin */
  double *crb10;
  double *M, *L;                /* dense nv*nv, and its Cholesky factor (dense mode) */
  /* sparse mode (default; orc_set_dense(d, 1) selects the dense factor for the self-check tests): L^T D L of M in MuJoCo's
   * qLD layout (mj_factorM: row i = (i,i), (i,parent(i)), ... at dof_Madr[i]) and of M + h diag(damping) for the Euler step */
  int dense; int* chainlen; double *qLD, *qLDiagInv, *qLDe, *qLDeDiagInv;
  /* velocity stage */
  double *bvel, *bacc;          /* per body spatial velocity / bias acceleration */
  double *qfrc_bias, *qfrc_passive, *qfrc_actuator, *qfrc_smooth, *qacc_smooth, *qfrc_constraint;
  double *act_dot, *actuator_force, *actuator_length, *actuator_velocity, *moment; /* nu*nv */
  /* contacts / constraints */
  int ncon, nefc, nlimit;
  OrcContact con[ORC_MAXCON];
  double *efc_J;                /* nefc*nv dense */
  double efc_pos[ORC_MAXEFC], efc_margin[ORC_MAXEFC], efc_D[ORC_MAXEFC], efc_R[ORC_MAXEFC],
         efc_aref[ORC_MAXEFC], efc_vel[ORC_MAXEFC], efc_force[ORC_MAXEFC], efc_KBIP[4 * ORC_MAXEFC],
         efc_diagApprox[ORC_MAXEFC], efc_b[ORC_MAXEFC];
  int efc_type[ORC_MAXEFC], efc_id[ORC_MAXEFC], efc_state[ORC_MAXEFC];
  double *sensordata, *sensor_sum;
  int solver_niter, flags;
  double solver_tolerance;      /* <=0 -> use model opt_tolerance */
  double *wk;                   /* scratch nv*nv + ... */
  /* optional heightfield terrain (orc_set_hfield): geom id, grid, heights (scaled by hf_size[2]), geoms that can touch it */
  int hf_geom, hf_nrow, hf_ncol, hf_npair; int* hf_pair; double hf_size[4]; double* hf_data;
} OrcData;

enum { CT_LIMIT = 0, CT_CONTACT_FRICTIONLESS = 1, CT_CONTACT_ELLIPTIC = 2 };

/* ------------------------------------------------------------------------------------------ */
/* small math                                                                                   */
static inline double dot3(const double* a, const double* b) { return a[0]*b[0]+a[1]*b[1]+a[2]*b[2]; }
static inline void cross3(double* r, const double* a, const double* b) {
  double x = a[1]*b[2]-a[2]*b[1], y = a[2]*b[0]-a[0]*b[2], z = a[0]*b[1]-a[1]*b[0];
  r[0]=x; r[1]=y; r[2]=z;
}
static inline void add3(double* r, const double* a, const double* b) { r[0]=a[0]+b[0]; r[1]=a[1]+b[1]; r[2]=a[2]+b[2]; }
static inline void sub3(double* r, const double* a, const double* b) { r[0]=a[0]-b[0]; r[1]=a[1]-b[1]; r[2]=a[2]-b[2]; }
static inline void scl3(double* r, const double* a, double s) { r[0]=a[0]*s; r[1]=a[1]*s; r[2]=a[2]*s; }
static inline void addscl3(double* r, const double* a, double s) { r[0]+=a[0]*s; r[1]+=a[1]*s; r[2]+=a[2]*s; }
static inline void copy3(double* r, const double* a) { r[0]=a[0]; r[1]=a[1]; r[2]=a[2]; }
static inline double norm3(const double* a) { return sqrt(dot3(a,a)); }
static inline double normalize3(double* a) {
  double n = norm3(a);
  if (n < MINVAL) { a[0]=1; a[1]=0; a[2]=0; } else { a[0]/=n; a[1]/=n; a[2]/=n; }
  return n;
}
static void quat_mul(double* r, const double* a, const double* b) {
  double w = a[0]*b[0]-a[1]*b[1]-a[2]*b[2]-a[3]*b[3];
  double x = a[0]*b[1]+a[1]*b[0]+a[2]*b[3]-a[3]*b[2];
  double y = a[0]*b[2]-a[1]*b[3]+a[2]*b[0]+a[3]*b[1];
  double z = a[0]*b[3]+a[1]*b[2]-a[2]*b[1]+a[3]*b[0];
  r[0]=w; r[1]=x; r[2]=y; r[3]=z;
}
static void quat_norm(double* q) {
  double n = sqrt(q[0]*q[0]+q[1]*q[1]+q[2]*q[2]+q[3]*q[3]);
  if (n < MINVAL) { q[0]=1; q[1]=q[2]=q[3]=0; } else { q[0]/=n; q[1]/=n; q[2]/=n; q[3]/=n; }
}
static void quat2mat(double* R, const double* q) {   /* row-major 3x3 */
  double w=q[0], x=q[1], y=q[2], z=q[3];
  R[0]=w*w+x*x-y*y-z*z; R[1]=2*(x*y-w*z);       R[2]=2*(x*z+w*y);
  R[3]=2*(x*y+w*z);     R[4]=w*w-x*x+y*y-z*z;   R[5]=2*(y*z-w*x);
  R[6]=2*(x*z-w*y);     R[7]=2*(y*z+w*x);       R[8]=w*w-x*x-y*y+z*z;
}
static inline void mulmat3(double* r, const double* R, const double* v) {   /* r = R v */
  double x=R[0]*v[0]+R[1]*v[1]+R[2]*v[2], y=R[3]*v[0]+R[4]*v[1]+R[5]*v[2], z=R[6]*v[0]+R[7]*v[1]+R[8]*v[2];
  r[0]=x; r[1]=y; r[2]=z;
}
static inline void mulmatT3(double* r, const double* R, const double* v) {  /* r = R^T v */
  double x=R[0]*v[0]+R[3]*v[1]+R[6]*v[2], y=R[1]*v[0]+R[4]*v[1]+R[7]*v[2], z=R[2]*v[0]+R[5]*v[1]+R[8]*v[2];
  r[0]=x; r[1]=y; r[2]=z;
}
static void axisangle_quat(double* q, const double* axis, double ang) {
  double s = sin(0.5*ang);
  q[0]=cos(0.5*ang); q[1]=axis[0]*s; q[2]=axis[1]*s; q[3]=axis[2]*s;
}
static void matmul33(double* C, const double* A, const double* B) {
  double t[9];
  for (int i=0;i<3;i++) for (int j=0;j<3;j++) t[3*i+j]=A[3*i]*B[j]+A[3*i+1]*B[3+j]+A[3*i+2]*B[6+j];
  memcpy(C,t,sizeof(t));
}

/* 10-parameter spatial inertia about world origin applied to a motion vector [w; v]:
 * returns momentum [L; p].  I10 = m, h[3], Ixx,Iyy,Izz,Ixy,Ixz,Iyz */
static void inert_mul(double* L, double* p, const double* I10, const double* w, const double* v) {
  double m = I10[0]; const double* h = I10+1; const double* I = I10+4;
  double hv[3], wh[3];
  cross3(hv, h, v); cross3(wh, w, h);
  L[0] = I[0]*w[0]+I[3]*w[1]+I[4]*w[2] + hv[0];
  L[1] = I[3]*w[0]+I[1]*w[1]+I[5]*w[2] + hv[1];
  L[2] = I[4]*w[0]+I[5]*w[1]+I[2]*w[2] + hv[2];
  p[0] = m*v[0]+wh[0]; p[1] = m*v[1]+wh[1]; p[2] = m*v[2]+wh[2];
}

/* ------------------------------------------------------------------------------------------ */
static double* dalloc(size_t n) { double* p = (double*)calloc(n > 0 ? n : 1, sizeof(double)); return p; }

OrcData* orc_create(const FbModel* m) {
  /* K8 implements dynamics none (0) / filter (2, Euler) and bias none (0) / affine (1) with a fixed gain: refuse anything else
   * (e.g. filterexact, 3) instead of integrating it as a plain filter */
  for (int i=0;i<m->nu;i++) {
    int dt=m->actuator_dyntype[i], bt=m->actuator_biastype[i], aa=m->actuator_actadr[i];
    if ((dt!=0 && dt!=2) || (bt!=0 && bt!=1) || (dt==2)!=(aa>=0) || aa>=m->na) return NULL;
  }
  /* the touch ray test (orc_sensors_acc) knows capsule and sphere sites only: refuse a touch sensor on any other site type */
  for (int i=0;i<m->nsensor;i++)
    if (m->sensor_type[i]==FB_SENS_TOUCH && m->site_type[m->sensor_objid[i]]!=FB_GEOM_SPHERE && m->site_type[m->sensor_objid[i]]!=FB_GEOM_CAPSULE)
      return NULL;
  OrcData* d = (OrcData*)calloc(1, sizeof(OrcData));
  d->m = m;
  int nv=m->nv, nb=m->nbody;
  d->qpos=dalloc(m->nq); d->qvel=dalloc(nv); d->act=dalloc(m->na); d->ctrl=dalloc(m->nu);
  d->qacc=dalloc(nv); d->qacc_warmstart=dalloc(nv);
  d->xpos=dalloc(3*nb); d->xquat=dalloc(4*nb); d->xmat=dalloc(9*nb); d->xipos=dalloc(3*nb); d->ximat=dalloc(9*nb);
  d->geom_xpos=dalloc(3*m->ngeom); d->geom_xmat=dalloc(9*m->ngeom);
  d->site_xpos=dalloc(3*m->nsite); d->site_xmat=dalloc(9*m->nsite); d->subtree_com=dalloc(3*nb);
  d->Sang=dalloc(3*nv); d->Slin=dalloc(3*nv); d->inert10=dalloc(10*nb); d->crb10=dalloc(10*nb);
  d->M=dalloc((size_t)nv*nv); d->L=dalloc((size_t)nv*nv);
  d->qLD=dalloc(m->nM); d->qLDiagInv=dalloc(nv); d->qLDe=dalloc(m->nM); d->qLDeDiagInv=dalloc(nv);
  d->chainlen=(int*)calloc(nv>0?nv:1,sizeof(int));
  for (int i=0;i<nv;i++) { int c=0; for (int j=i;j>=0;j=m->dof_parentid[j]) c++; d->chainlen[i]=c; }
  d->bvel=dalloc(6*nb); d->bacc=dalloc(6*nb);
  d->qfrc_bias=dalloc(nv); d->qfrc_passive=dalloc(nv); d->qfrc_actuator=dalloc(nv); d->qfrc_smooth=dalloc(nv);
  d->qacc_smooth=dalloc(nv); d->qfrc_constraint=dalloc(nv);
  d->act_dot=dalloc(m->na); d->actuator_force=dalloc(m->nu); d->actuator_length=dalloc(m->nu);
  d->actuator_velocity=dalloc(m->nu); d->moment=dalloc((size_t)m->nu*nv);
  d->efc_J=dalloc((size_t)ORC_MAXEFC*nv);
  d->sensordata=dalloc(m->nsensordata); d->sensor_sum=dalloc(m->nsensordata);
  d->wk=dalloc((size_t)4*nv*nv + 64*nv + 4096);
  d->solver_tolerance = -1;
  memcpy(d->qpos, m->qpos0, sizeof(double)*m->nq);
  return d;
}
void orc_destroy(OrcData* d) {
  if (!d) return;
  double* ptrs[] = {d->qpos,d->qvel,d->act,d->ctrl,d->qacc,d->qacc_warmstart,d->xpos,d->xquat,d->xmat,d->xipos,d->ximat,
    d->geom_xpos,d->geom_xmat,d->site_xpos,d->site_xmat,d->subtree_com,d->Sang,d->Slin,d->inert10,d->crb10,d->M,d->L,
    d->bvel,d->bacc,d->qfrc_bias,d->qfrc_passive,d->qfrc_actuator,d->qfrc_smooth,d->qacc_smooth,d->qfrc_constraint,
    d->act_dot,d->actuator_force,d->actuator_length,d->actuator_velocity,d->moment,d->efc_J,d->sensordata,d->sensor_sum,d->wk};
  for (size_t i=0;i<sizeof(ptrs)/sizeof(ptrs[0]);i++) free(ptrs[i]);
  free(d->hf_data); free(d->hf_pair); free(d->qLD); free(d->qLDiagInv); free(d->qLDe); free(d->qLDeDiagInv); free(d->chainlen);
  free(d);
}

/* ------------------------------------------------------------------------------------------ */
/* K1: kinematics + comPos (MuJoCo mj_kinematics, mj_comPos; SURVEY.md A.1, A.2)               */
static void orc_kinematics(OrcData* d) {
  const FbModel* m = d->m;
  int nb = m->nbody;
  double* xpos=d->xpos; double* xquat=d->xquat;
  xpos[0]=xpos[1]=xpos[2]=0; xquat[0]=1; xquat[1]=xquat[2]=xquat[3]=0;
  quat2mat(d->xmat, xquat);
  for (int b=1;b<nb;b++) {
    int p = m->body_parentid[b];
    double pos[3], quat[4], t[3];
    mulmat3(t, d->xmat+9*p, m->body_pos+3*b);
    add3(pos, xpos+3*p, t);
    quat_mul(quat, xquat+4*p, m->body_quat+4*b);
    for (int k=0;k<m->body_jntnum[b];k++) {
      int j = m->body_jntadr[b]+k, qa = m->jnt_qposadr[j], da = m->jnt_dofadr[j];
      if (m->jnt_type[j]==FB_JNT_FREE) {
        copy3(pos, d->qpos+qa);
        memcpy(quat, d->qpos+qa+3, 4*sizeof(double));
        quat_norm(quat);
        double R[9]; quat2mat(R, quat);
        for (int i=0;i<3;i++) {
          double e[3]={0,0,0}; e[i]=1;
          d->Sang[3*(da+i)]=d->Sang[3*(da+i)+1]=d->Sang[3*(da+i)+2]=0;
          copy3(d->Slin+3*(da+i), e);
          double ax[3]={R[i],R[3+i],R[6+i]};
          copy3(d->Sang+3*(da+3+i), ax);
          cross3(d->Slin+3*(da+3+i), pos, ax);
        }
      } else {
        double R[9], anchor[3], axis[3], jq[4], nq[4];
        quat2mat(R, quat);
        mulmat3(t, R, m->jnt_pos+3*j); add3(anchor, pos, t);
        mulmat3(axis, R, m->jnt_axis+3*j);
        axisangle_quat(jq, m->jnt_axis+3*j, d->qpos[qa]-m->qpos0[qa]);
        quat_mul(nq, quat, jq); memcpy(quat, nq, sizeof(nq));
        quat2mat(R, quat);
        mulmat3(t, R, m->jnt_pos+3*j); sub3(pos, anchor, t);
        copy3(d->Sang+3*da, axis);
        cross3(d->Slin+3*da, anchor, axis);
      }
    }
    quat_norm(quat);
    copy3(xpos+3*b, pos); memcpy(xquat+4*b, quat, 4*sizeof(double));
    quat2mat(d->xmat+9*b, quat);
    mulmat3(t, d->xmat+9*b, m->body_ipos+3*b); add3(d->xipos+3*b, pos, t);
    double iq[4]; quat_mul(iq, quat, m->body_iquat+4*b); quat2mat(d->ximat+9*b, iq);
  }
  for (int g=0; g<m->ngeom; g++) {
    int b = m->geom_bodyid[g]; double t[3], q[4];
    mulmat3(t, d->xmat+9*b, m->geom_pos+3*g); add3(d->geom_xpos+3*g, xpos+3*b, t);
    quat_mul(q, xquat+4*b, m->geom_quat+4*g); quat2mat(d->geom_xmat+9*g, q);
  }
  for (int s=0; s<m->nsite; s++) {
    int b = m->site_bodyid[s]; double t[3], q[4];
    mulmat3(t, d->xmat+9*b, m->site_pos+3*s); add3(d->site_xpos+3*s, xpos+3*b, t);
    quat_mul(q, xquat+4*b, m->site_quat+4*s); quat2mat(d->site_xmat+9*s, q);
  }
  /* subtree com + 10-parameter inertias about the world origin */
  double* sm = d->wk;  /* nb */
  for (int b=0;b<nb;b++) { sm[b]=m->body_mass[b]; scl3(d->subtree_com+3*b, d->xipos+3*b, m->body_mass[b]); }
  for (int b=nb-1;b>0;b--) { int p=m->body_parentid[b]; sm[p]+=sm[b]; addscl3(d->subtree_com+3*p, d->subtree_com+3*b, 1.0); }
  for (int b=0;b<nb;b++) {
    if (sm[b]>MINVAL) scl3(d->subtree_com+3*b, d->subtree_com+3*b, 1.0/sm[b]);
    else copy3(d->subtree_com+3*b, d->xipos+3*b);
  }
  for (int b=0;b<nb;b++) {
    double* I10 = d->inert10+10*b; double mass=m->body_mass[b]; const double* c=d->xipos+3*b;
    const double* R=d->ximat+9*b; const double* di=m->body_inertia+3*b;
    double Ic[9];
    for (int i=0;i<3;i++) for (int j=0;j<3;j++) Ic[3*i+j]=R[3*i]*di[0]*R[3*j]+R[3*i+1]*di[1]*R[3*j+1]+R[3*i+2]*di[2]*R[3*j+2];
    double cc=dot3(c,c);
    I10[0]=mass; I10[1]=mass*c[0]; I10[2]=mass*c[1]; I10[3]=mass*c[2];
    I10[4]=Ic[0]+mass*(cc-c[0]*c[0]); I10[5]=Ic[4]+mass*(cc-c[1]*c[1]); I10[6]=Ic[8]+mass*(cc-c[2]*c[2]);
    I10[7]=Ic[1]-mass*c[0]*c[1]; I10[8]=Ic[2]-mass*c[0]*c[2]; I10[9]=Ic[5]-mass*c[1]*c[2];
  }
}

/* K2: composite rigid body inertia -> dense M, Cholesky (MuJoCo mj_crb + mj_factorM; A.3)      */
/* contiguous dot product; `omp simd` lets the compiler vectorise the reduction (-fopenmp-simd, no runtime) */
static inline double dotn(const double* a, const double* b, int n) {
  double s=0;
#pragma omp simd reduction(+:s)
  for (int k=0;k<n;k++) s+=a[k]*b[k];
  return s;
}
static int cholesky(double* L, const double* A, int n) {
  memcpy(L, A, sizeof(double)*n*n);
  for (int j=0;j<n;j++) {
    double s = L[j*n+j] - dotn(L+j*n, L+j*n, j);
    if (s < MINVAL) return -1;
    s = sqrt(s); L[j*n+j]=s;
    for (int i=j+1;i<n;i++) L[i*n+j]=(L[i*n+j]-dotn(L+i*n, L+j*n, j))/s;
  }
  return 0;
}
static void chol_solve(const double* L, double* x, int n) {   /* in place: x = (L L^T)^-1 x */
  for (int i=0;i<n;i++) x[i]=(x[i]-dotn(L+i*n,x,i))/L[i*n+i];
  for (int i=n-1;i>=0;i--) { double xi=x[i]/L[i*n+i]; x[i]=xi; const double* Li=L+i*n;     /* column sweep: rows of L stay contiguous */
#pragma omp simd
    for (int k=0;k<i;k++) x[k]-=Li[k]*xi; }
}
/* MuJoCo mj_factorI / mj_solveLD on the tree-sparse inertia (engine_core_smooth.c): qLD <- L^T D L of (M + diag(add)) */
static void factor_sparse(const OrcData* d, double* qLD, double* diaginv, const double* add) {
  const FbModel* m=d->m; int nv=m->nv;
  for (int i=0;i<nv;i++) { int a=m->dof_Madr[i], t=0; for (int j=i;j>=0;j=m->dof_parentid[j],t++) qLD[a+t]=d->M[(size_t)i*nv+j]; if (add) qLD[a]+=add[i]; }
  for (int k=nv-1;k>=0;k--) {
    int ak=m->dof_Madr[k], aki=ak+1, i=m->dof_parentid[k];
    while (i>=0) {
      double tmp=qLD[aki]/qLD[ak]; int ai=m->dof_Madr[i], cnt=d->chainlen[i];
      for (int c=0;c<cnt;c++) qLD[ai+c]-=tmp*qLD[aki+c];
      qLD[aki]=tmp; i=m->dof_parentid[i]; aki++;
    }
    diaginv[k]=1.0/qLD[ak];
  }
}
static void solve_sparse(const OrcData* d, const double* qLD, const double* diaginv, double* x) {
  const FbModel* m=d->m; int nv=m->nv;
  for (int i=nv-1;i>=0;i--) { double xi=x[i]; if (xi==0) continue; int a=m->dof_Madr[i]+1; for (int j=m->dof_parentid[i];j>=0;j=m->dof_parentid[j]) x[j]-=qLD[a++]*xi; }
  for (int i=0;i<nv;i++) x[i]*=diaginv[i];
  for (int i=0;i<nv;i++) { int a=m->dof_Madr[i]+1; double s=x[i]; for (int j=m->dof_parentid[i];j>=0;j=m->dof_parentid[j]) s-=qLD[a++]*x[j]; x[i]=s; }
}
/* x <- M^-1 x with whichever factor the mode keeps */
static void solve_M(const OrcData* d, double* x) { if (d->dense) chol_solve(d->L,x,d->m->nv); else solve_sparse(d,d->qLD,d->qLDiagInv,x); }
static void orc_crb(OrcData* d) {
  const FbModel* m=d->m; int nb=m->nbody, nv=m->nv;
  memcpy(d->crb10, d->inert10, sizeof(double)*10*nb);
  for (int b=nb-1;b>0;b--) { int p=m->body_parentid[b]; for (int k=0;k<10;k++) d->crb10[10*p+k]+=d->crb10[10*b+k]; }
  memset(d->M, 0, sizeof(double)*nv*nv);
  for (int i=0;i<nv;i++) {
    double L[3], p[3];
    inert_mul(L, p, d->crb10+10*m->dof_bodyid[i], d->Sang+3*i, d->Slin+3*i);
    for (int j=i;j>=0;j=m->dof_parentid[j]) {
      double v = dot3(d->Sang+3*j, L)+dot3(d->Slin+3*j, p);
      d->M[i*nv+j]=v; d->M[j*nv+i]=v;
    }
    d->M[i*nv+i] += m->dof_armature[i];
  }
  if (d->dense) cholesky(d->L, d->M, nv); else factor_sparse(d, d->qLD, d->qLDiagInv, NULL);
}

/* Jacobian of world point `p` attached to body b: jacp/jacr are 3 x nv dense (may be NULL) */
static void jac_point(const OrcData* d, int b, const double* p, double* jacp, double* jacr) {
  const FbModel* m=d->m; int nv=m->nv;
  if (jacp) memset(jacp,0,sizeof(double)*3*nv);
  if (jacr) memset(jacr,0,sizeof(double)*3*nv);
  for (int k=m->body_lastdof[b];k>=0;k=m->dof_parentid[k]) {
    if (jacr) for (int i=0;i<3;i++) jacr[i*nv+k]=d->Sang[3*k+i];
    if (jacp) { double t[3]; cross3(t, d->Sang+3*k, p); for (int i=0;i<3;i++) jacp[i*nv+k]=d->Slin[3*k+i]+t[i]; }
  }
}
/* qfrc += J^T [force at point; torque]  (MuJoCo mj_applyFT) */
static void apply_ft(const OrcData* d, int b, const double* point, const double* force, const double* torque, double* qfrc) {
  const FbModel* m=d->m;
  for (int k=m->body_lastdof[b];k>=0;k=m->dof_parentid[k]) {
    double t[3]; cross3(t, d->Sang+3*k, point); add3(t, t, d->Slin+3*k);
    qfrc[k] += dot3(t, force) + dot3(d->Sang+3*k, torque);
  }
}

/* K4: body velocities, bias accelerations, RNE bias force (MuJoCo mj_comVel + mj_rne; A.5)     */
static void motion_cross(double* r, const double* v, const double* Sa, const double* Sl) {
  /* r = v x_m S = [w x Sa; w x Sl + vO x Sa] */
  double t[3];
  cross3(r, v, Sa);
  cross3(r+3, v, Sl); cross3(t, v+3, Sa); add3(r+3, r+3, t);
}
/* forward pass: fills bvel and bacc; if qacc!=NULL adds S*qacc (full acceleration) */
static void rne_forward(OrcData* d, const double* qacc, double* bvel, double* bacc) {
  const FbModel* m=d->m; int nb=m->nbody;
  for (int k=0;k<6;k++) { bvel[k]=0; bacc[k]=0; }
  bacc[3]=-m->opt_gravity[0]; bacc[4]=-m->opt_gravity[1]; bacc[5]=-m->opt_gravity[2];
  for (int b=1;b<nb;b++) {
    int p=m->body_parentid[b];
    double v[6], a[6];
    memcpy(v, bvel+6*p, sizeof(v)); memcpy(a, bacc+6*p, sizeof(a));
    for (int k=0;k<m->body_jntnum[b];k++) {
      int j=m->body_jntadr[b]+k, da=m->jnt_dofadr[j];
      if (m->jnt_type[j]==FB_JNT_FREE) {
        double vlin[3]={d->qvel[da],d->qvel[da+1],d->qvel[da+2]}, w[3]={0,0,0};
        for (int i=0;i<6;i++) {
          double qd=d->qvel[da+i];
          addscl3(v, d->Sang+3*(da+i), qd); addscl3(v+3, d->Slin+3*(da+i), qd);
          if (i>=3) addscl3(w, d->Sang+3*(da+i), qd);
          if (qacc) { addscl3(a, d->Sang+3*(da+i), qacc[da+i]); addscl3(a+3, d->Slin+3*(da+i), qacc[da+i]); }
        }
        double t[3]; cross3(t, vlin, w); add3(a+3, a+3, t);   /* sum_i Sdot_i qd_i = [0; vlin x w] */
      } else {
        double qd=d->qvel[da], r[6];
        motion_cross(r, v, d->Sang+3*da, d->Slin+3*da);
        for (int i=0;i<6;i++) a[i]+=r[i]*qd;
        addscl3(v, d->Sang+3*da, qd); addscl3(v+3, d->Slin+3*da, qd);
        if (qacc) { addscl3(a, d->Sang+3*da, qacc[da]); addscl3(a+3, d->Slin+3*da, qacc[da]); }
      }
    }
    memcpy(bvel+6*b, v, sizeof(v)); memcpy(bacc+6*b, a, sizeof(a));
  }
}
/* per-body inertial force f = I a + v x* (I v) -> bfrc (6 per body, [torque about O; force]) */
static void rne_body_force(const OrcData* d, const double* bvel, const double* bacc, double* bfrc) {
  const FbModel* m=d->m;
  for (int b=0;b<m->nbody;b++) {
    double L[3],p[3],La[3],pa[3],t1[3],t2[3];
    const double* v=bvel+6*b; const double* a=bacc+6*b;
    inert_mul(L,p,d->inert10+10*b,v,v+3);
    inert_mul(La,pa,d->inert10+10*b,a,a+3);
    cross3(t1,v,L); cross3(t2,v+3,p);
    for (int i=0;i<3;i++) bfrc[6*b+i]=La[i]+t1[i]+t2[i];
    cross3(t1,v,p);
    for (int i=0;i<3;i++) bfrc[6*b+3+i]=pa[i]+t1[i];
  }
}
static void orc_bias(OrcData* d) {
  const FbModel* m=d->m; int nb=m->nbody, nv=m->nv;
  double* bfrc=d->wk;
  rne_forward(d, NULL, d->bvel, d->bacc);
  rne_body_force(d, d->bvel, d->bacc, bfrc);
  for (int b=nb-1;b>0;b--) { int p=m->body_parentid[b]; for (int k=0;k<6;k++) bfrc[6*p+k]+=bfrc[6*b+k]; }
  for (int i=0;i<nv;i++) { int b=m->dof_bodyid[i]; d->qfrc_bias[i]=dot3(d->Sang+3*i,bfrc+6*b)+dot3(d->Slin+3*i,bfrc+6*b+3); }
}

/* velocity of world point p moving with body b: w (world), v (world) */
static void point_velocity(const OrcData* d, int b, const double* p, double* w, double* v) {
  const double* bv=d->bvel+6*b; double t[3];
  copy3(w,bv); cross3(t,bv,p); add3(v,bv+3,t);
}

/* K5/K6/K7 passive forces (MuJoCo mj_passive: springs, dampers, inertia-box and ellipsoid fluid) */
static double ellipsoid_max_moment(const double* size, int dir) {
  double d0=size[dir], d1=size[(dir+1)%3], d2=size[(dir+2)%3]; double mx=d1>d2?d1:d2;
  return 8.0/15.0*PI*d0*mx*mx*mx*mx;
}
/* local-frame wrench [torque; force] of MuJoCo's ellipsoid fluid model on one geom, from its local angular (lw)
 * and linear (lv, wind subtracted) velocity.  Pinned against the reference's own Python restatement
 * (flybody/ellipsoid_fluid_model.py:88-209) by tests/test_reference_python_goldens.py. */
void orc_ellipsoid_local_force(const double* lw, const double* lv, const double* size, const double* coef,
                               double rho, double eta, double* lfrc) {
  for (int i=0;i<6;i++) lfrc[i]=0;
  double blunt=coef[1], slender=coef[2], angc=coef[3], kutta=coef[4], magnus=coef[5];
  const double* vmass=coef+6; const double* vinert=coef+9;
  /* added mass (ellipsoid_fluid_model.py:88-110) */
  double vlm[3],vam[3],f1[3],t1[3],t2[3];
  for (int i=0;i<3;i++) { vlm[i]=rho*vmass[i]*lv[i]; vam[i]=rho*vinert[i]*lw[i]; }
  cross3(f1,vlm,lw); cross3(t1,vlm,lv); cross3(t2,vam,lw);
  for (int i=0;i<3;i++) { lfrc[i]+=t1[i]+t2[i]; lfrc[3+i]+=f1[i]; }
  /* viscous forces (ellipsoid_fluid_model.py:113-209) */
  double volume=4.0/3.0*PI*size[0]*size[1]*size[2];
  double dmax=fmax(size[0],fmax(size[1],size[2])), dmin=fmin(size[0],fmin(size[1],size[2]));
  double dmid=size[0]+size[1]+size[2]-dmax-dmin;
  double A_max=PI*dmax*dmid;
  double magf[3]; cross3(magf,lw,lv); scl3(magf,magf,magnus*rho*volume);
  double s12=size[1]*size[2], s20=size[2]*size[0], s01=size[0]*size[1];
  double proj_denom=pow(s12,4)*lv[0]*lv[0]+pow(s20,4)*lv[1]*lv[1]+pow(s01,4)*lv[2]*lv[2];
  double proj_num=pow(s12*lv[0],2)+pow(s20*lv[1],2)+pow(s01*lv[2],2);
  double A_proj=PI*sqrt(proj_denom/fmax(MINVAL,proj_num));
  double nrm[3]={s12*s12*lv[0], s20*s20*lv[1], s01*s01*lv[2]};
  double speed=norm3(lv);
  double cos_alpha=proj_num/fmax(MINVAL,speed*proj_denom);
  double kc[3],kf[3]; cross3(kc,nrm,lv); scl3(kc,kc,kutta*rho*cos_alpha*A_proj); cross3(kf,kc,lv);
  double eqD=2.0/3.0*(size[0]+size[1]+size[2]);
  double lin_coef=3.0*PI*eqD, ang_coef=PI*eqD*eqD*eqD;
  double I_max=8.0/15.0*PI*dmid*pow(dmax,4);
  double II[3]={ellipsoid_max_moment(size,0),ellipsoid_max_moment(size,1),ellipsoid_max_moment(size,2)};
  double mom[3];
  for (int i=0;i<3;i++) mom[i]=lw[i]*(angc*II[i]+slender*(I_max-II[i]));
  double drag_lin=eta*lin_coef+rho*speed*(A_proj*blunt+slender*(A_max-A_proj));
  double drag_ang=eta*ang_coef+rho*norm3(mom);
  for (int i=0;i<3;i++) { lfrc[i]-=drag_ang*lw[i]; lfrc[3+i]+=magf[i]+kf[i]-drag_lin*lv[i]; }
  for (int i=0;i<6;i++) lfrc[i]*=coef[0];
}

static void orc_passive(OrcData* d) {
  const FbModel* m=d->m; int nv=m->nv;
  memset(d->qfrc_passive,0,sizeof(double)*nv);
  for (int j=0;j<m->njnt;j++) {
    if (m->jnt_type[j]==FB_JNT_HINGE) {
      int qa=m->jnt_qposadr[j], da=m->jnt_dofadr[j];
      d->qfrc_passive[da] -= m->jnt_stiffness[j]*(d->qpos[qa]-m->qpos_spring[qa]);
    }
  }
  for (int i=0;i<nv;i++) d->qfrc_passive[i] -= m->dof_damping[i]*d->qvel[i];
  double rho=m->opt_density, eta=m->opt_viscosity;
  if (rho<=0 && eta<=0) return;
  for (int b=1;b<m->nbody;b++) {
    double mass=m->body_mass[b];
    if (mass<MINVAL) continue;
    if (m->body_fluid_ellipsoid[b]) continue;
    /* inertia-box model (engine_passive.c mj_inertiaBoxFluidModel; SURVEY.md A.4) */
    const double* I=m->body_inertia+3*b; double box[3];
    box[0]=sqrt(fmax(MINVAL,I[1]+I[2]-I[0])/mass*6.0);
    box[1]=sqrt(fmax(MINVAL,I[0]+I[2]-I[1])/mass*6.0);
    box[2]=sqrt(fmax(MINVAL,I[0]+I[1]-I[2])/mass*6.0);
    double w[3],v[3],lw[3],lv[3],lfrc[6]={0,0,0,0,0,0};
    point_velocity(d,b,d->xipos+3*b,w,v);
    double vw[3]; sub3(vw,v,m->opt_wind);
    mulmatT3(lw,d->ximat+9*b,w); mulmatT3(lv,d->ximat+9*b,vw);
    if (eta>0) {
      double diam=(box[0]+box[1]+box[2])/3.0;
      for (int i=0;i<3;i++) { lfrc[i]=-PI*diam*diam*diam*eta*lw[i]; lfrc[3+i]=-3.0*PI*diam*eta*lv[i]; }
    }
    if (rho>0) {
      lfrc[3]-=0.5*rho*box[1]*box[2]*fabs(lv[0])*lv[0];
      lfrc[4]-=0.5*rho*box[0]*box[2]*fabs(lv[1])*lv[1];
      lfrc[5]-=0.5*rho*box[0]*box[1]*fabs(lv[2])*lv[2];
      lfrc[0]-=rho*box[0]*(pow(box[1],4)+pow(box[2],4))*fabs(lw[0])*lw[0]/64.0;
      lfrc[1]-=rho*box[1]*(pow(box[0],4)+pow(box[2],4))*fabs(lw[1])*lw[1]/64.0;
      lfrc[2]-=rho*box[2]*(pow(box[0],4)+pow(box[1],4))*fabs(lw[2])*lw[2]/64.0;
    }
    double tq[3],fr[3];
    mulmat3(tq,d->ximat+9*b,lfrc); mulmat3(fr,d->ximat+9*b,lfrc+3);
    apply_ft(d,b,d->xipos+3*b,fr,tq,d->qfrc_passive);
  }
  /* ellipsoid model (reference flybody/ellipsoid_fluid_model.py:88-310) */
  for (int g=0;g<m->nfluid;g++) {
    int b=m->fluid_bodyid[g];
    const double* coef=m->fluid_coef+12*g; const double* size=m->fluid_size+3*g;
    if (coef[0]==0.0) continue;
    double gpos[3],t[3],gq[4],gmat[9];
    mulmat3(t,d->xmat+9*b,m->fluid_pos+3*g); add3(gpos,d->xpos+3*b,t);
    quat_mul(gq,d->xquat+4*b,m->fluid_quat+4*g); quat2mat(gmat,gq);
    double w[3],v[3],lw[3],lv[3];
    point_velocity(d,b,gpos,w,v);
    double vw[3]; sub3(vw,v,m->opt_wind);
    mulmatT3(lw,gmat,w); mulmatT3(lv,gmat,vw);
    double lfrc[6];
    orc_ellipsoid_local_force(lw,lv,size,coef,rho,eta,lfrc);
    double tq[3],fr[3];
    mulmat3(tq,gmat,lfrc); mulmat3(fr,gmat,lfrc+3);
    apply_ft(d,b,gpos,fr,tq,d->qfrc_passive);
  }
}

/* ------------------------------------------------------------------------------------------ */
/* K9: collision (MuJoCo engine_collision_primitive.c restated; SURVEY.md A.7)                  */
static void make_frame(double* f) {   /* mju_makeFrame */
  normalize3(f);
  if (norm3(f+3)<0.5) { f[3]=f[4]=f[5]=0; if (f[1]<0.5 && f[1]>-0.5) f[4]=1; else f[5]=1; }
  double t=dot3(f,f+3); addscl3(f+3,f,-t); normalize3(f+3);
  cross3(f+6,f,f+3);
}
typedef struct { double dist, pos[3], normal[3], tangent[3]; } RawCon;

static int raw_sphere_sphere(RawCon* c, double margin, const double* p1, double r1, const double* p2, double r2) {
  double dif[3]; sub3(dif,p2,p1);
  double cd=dot3(dif,dif), lim=margin+r1+r2;
  if (cd>lim*lim) return 0;
  double len=sqrt(cd);
  c->dist=len-r1-r2;
  if (len<MINVAL) { c->normal[0]=1; c->normal[1]=c->normal[2]=0; } else scl3(c->normal,dif,1.0/len);
  copy3(c->pos,p1); addscl3(c->pos,c->normal,r1+0.5*c->dist);
  c->tangent[0]=c->tangent[1]=c->tangent[2]=0;
  return 1;
}
static int raw_plane_sphere(RawCon* c, double margin, const double* pp, const double* pmat, const double* sp, double r) {
  double n[3]={pmat[2],pmat[5],pmat[8]}, t[3]; sub3(t,sp,pp);
  double cd=dot3(t,n);
  if (cd>margin+r) return 0;
  c->dist=cd-r; copy3(c->normal,n);
  copy3(c->pos,sp); addscl3(c->pos,n,-(r+0.5*c->dist));
  c->tangent[0]=c->tangent[1]=c->tangent[2]=0;
  return 1;
}
static int col_plane_capsule(RawCon* c, double margin, const double* pp, const double* pmat, const double* cp, const double* cmat, const double* size) {
  double axis[3]={cmat[2],cmat[5],cmat[8]}, seg[3], e[3]; scl3(seg,axis,size[1]);
  int n=0;
  add3(e,cp,seg); n+=raw_plane_sphere(c+n,margin,pp,pmat,e,size[0]);
  sub3(e,cp,seg); n+=raw_plane_sphere(c+n,margin,pp,pmat,e,size[0]);
  for (int i=0;i<n;i++) copy3(c[i].tangent,axis);      /* align contact frames with capsule axis */
  return n;
}
static int col_plane_cylinder(RawCon* c, double margin, const double* pp, const double* pmat, const double* cp, const double* cmat, const double* size) {
  double n[3]={pmat[2],pmat[5],pmat[8]}, axis[3]={cmat[2],cmat[5],cmat[8]}, dif[3];
  sub3(dif,cp,pp);
  double dist0=dot3(dif,n), prjaxis=dot3(n,axis);
  if (prjaxis>0) { scl3(axis,axis,-1); prjaxis=-prjaxis; }
  double vec[3]; scl3(vec,axis,prjaxis); sub3(vec,vec,n);
  double len2=dot3(vec,vec);
  if (len2>=MINVAL) scl3(vec,vec,size[0]/sqrt(len2));
  else { vec[0]=cmat[0]*size[0]; vec[1]=cmat[3]*size[0]; vec[2]=cmat[6]*size[0]; }
  double prjvec=dot3(vec,n);
  scl3(axis,axis,size[1]); prjaxis*=size[1];
  int cnt=0;
  if (dist0+prjaxis+prjvec<=margin) {
    c[cnt].dist=dist0+prjaxis+prjvec;
    add3(c[cnt].pos,cp,vec); add3(c[cnt].pos,c[cnt].pos,axis); addscl3(c[cnt].pos,n,-0.5*c[cnt].dist);
    cnt++;
  } else return 0;
  if (dist0-prjaxis+prjvec<=margin) {
    c[cnt].dist=dist0-prjaxis+prjvec;
    add3(c[cnt].pos,cp,vec); sub3(c[cnt].pos,c[cnt].pos,axis); addscl3(c[cnt].pos,n,-0.5*c[cnt].dist);
    cnt++;
  }
  double prjvec1=-prjvec*0.5;
  if (dist0+prjaxis+prjvec1<=margin) {
    double vec1[3]; cross3(vec1,vec,axis); normalize3(vec1); scl3(vec1,vec1,size[0]*sqrt(3.0)*0.5);
    for (int s=0;s<2;s++) {
      c[cnt].dist=dist0+prjaxis+prjvec1;
      add3(c[cnt].pos,cp,axis); addscl3(c[cnt].pos,vec1,s?-1.0:1.0); addscl3(c[cnt].pos,vec,-0.5);
      addscl3(c[cnt].pos,n,-0.5*c[cnt].dist);
      cnt++;
    }
  }
  for (int i=0;i<cnt;i++) { copy3(c[i].normal,n); c[i].tangent[0]=c[i].tangent[1]=c[i].tangent[2]=0; }
  return cnt;
}
static int col_plane_ellipsoid(RawCon* c, double margin, const double* pp, const double* pmat, const double* ep, const double* emat, const double* size) {
  /* mjc_PlaneConvex with the ellipsoid support function in direction -normal */
  double n[3]={pmat[2],pmat[5],pmat[8]}, ln[3], s[3], sup[3], t[3];
  mulmatT3(ln,emat,n);
  for (int i=0;i<3;i++) s[i]=-size[i]*size[i]*ln[i];
  double den=sqrt(size[0]*size[0]*ln[0]*ln[0]+size[1]*size[1]*ln[1]*ln[1]+size[2]*size[2]*ln[2]*ln[2]);
  if (den<MINVAL) den=MINVAL;
  scl3(s,s,1.0/den);
  mulmat3(sup,emat,s); add3(sup,sup,ep);
  sub3(t,sup,pp);
  double dist=dot3(t,n);
  if (dist>margin) return 0;
  c->dist=dist; copy3(c->normal,n); copy3(c->pos,sup); addscl3(c->pos,n,-0.5*dist);
  c->tangent[0]=c->tangent[1]=c->tangent[2]=0;
  return 1;
}
static int col_sphere_capsule(RawCon* c, double margin, const double* sp, double sr, const double* cp, const double* cmat, const double* csize) {
  double axis[3]={cmat[2],cmat[5],cmat[8]}, vec[3]; sub3(vec,sp,cp);
  double x=dot3(axis,vec); if (x>csize[1]) x=csize[1]; if (x<-csize[1]) x=-csize[1];
  copy3(vec,cp); addscl3(vec,axis,x);
  return raw_sphere_sphere(c,margin,sp,sr,vec,csize[0]);
}
static double clipd(double x,double lo,double hi){ return x<lo?lo:(x>hi?hi:x); }
static int col_capsule_capsule(RawCon* c, double margin, const double* p1, const double* m1, const double* s1, const double* p2, const double* m2, const double* s2) {
  double a1[3]={m1[2],m1[5],m1[8]}, a2[3]={m2[2],m2[5],m2[8]}, dif[3]; sub3(dif,p1,p2);
  double ma=dot3(a1,a1), mb=-dot3(a1,a2), mc=dot3(a2,a2), u=-dot3(a1,dif), v=dot3(a2,dif);
  double det=ma*mc-mb*mb, v1[3], v2[3];
  if (fabs(det)>=MINVAL) {
    double x1=(mc*u-mb*v)/det, x2=(ma*v-mb*u)/det;
    if (x1>s1[1]) { x1=s1[1]; x2=(v-mb*s1[1])/mc; }
    else if (x1<-s1[1]) { x1=-s1[1]; x2=(v+mb*s1[1])/mc; }
    if (x2>s2[1]) { x2=s2[1]; x1=clipd((u-mb*s2[1])/ma,-s1[1],s1[1]); }
    else if (x2<-s2[1]) { x2=-s2[1]; x1=clipd((u+mb*s2[1])/ma,-s1[1],s1[1]); }
    copy3(v1,p1); addscl3(v1,a1,x1); copy3(v2,p2); addscl3(v2,a2,x2);
    return raw_sphere_sphere(c,margin,v1,s1[0],v2,s2[0]);
  }
  int n=0; double x;
  copy3(v1,p1); addscl3(v1,a1,s1[1]); x=clipd((v-mb*s1[1])/mc,-s2[1],s2[1]); copy3(v2,p2); addscl3(v2,a2,x);
  n+=raw_sphere_sphere(c+n,margin,v1,s1[0],v2,s2[0]);
  copy3(v1,p1); addscl3(v1,a1,-s1[1]); x=clipd((v+mb*s1[1])/mc,-s2[1],s2[1]); copy3(v2,p2); addscl3(v2,a2,x);
  n+=raw_sphere_sphere(c+n,margin,v1,s1[0],v2,s2[0]);
  if (n>=2) return n;
  copy3(v2,p2); addscl3(v2,a2,s2[1]); x=clipd((u-mb*s2[1])/ma,-s1[1],s1[1]); copy3(v1,p1); addscl3(v1,a1,x);
  n+=raw_sphere_sphere(c+n,margin,v1,s1[0],v2,s2[0]);
  if (n>=2) return n;
  copy3(v2,p2); addscl3(v2,a2,-s2[1]); x=clipd((u+mb*s2[1])/ma,-s1[1],s1[1]); copy3(v1,p1); addscl3(v1,a1,x);
  n+=raw_sphere_sphere(c+n,margin,v1,s1[0],v2,s2[0]);
  return n;
}

/* ------------------------------------------------------------------------------------------ */
/* Generic convex pairs (MuJoCo mjc_Convex, engine_collision_convex.c): Minkowski Portal Refinement as published in
 * libccd (src/mpr.c: ccdMPRPenetration -> discoverPortal / refinePortal / findPenetr / findPos, src/vec3.c:
 * ccdVec3PointTriDist2), which MuJoCo links for every pair without an analytic routine, with MuJoCo's support functions
 * (mjccd_support: each geom inflated by margin / 2), mpr_tolerance 1e-6, mpr_iterations 50, contact dist = margin - depth.
 * Restated from memory of libccd 2.1 / MuJoCo 2.3-3.1; multiccd is not restated (DESIGN.md).        */
#define CCD_EPS 2.220446049250313e-16
typedef struct { double v[3], v1[3], v2[3]; } MprPt;
typedef struct { const double *pos, *mat, *size; int type; double margin; } MprObj;
static int ccd_zero(double x) { return fabs(x)<CCD_EPS; }
static int ccd_eq(double a, double b) {
  double ab=fabs(a-b); if (ab<CCD_EPS) return 1;
  a=fabs(a); b=fabs(b); return (b>a) ? ab<CCD_EPS*b : ab<CCD_EPS*a;
}
static double sgn(double x) { return x>0 ? 1.0 : (x<0 ? -1.0 : 0.0); }
static void mpr_support1(const MprObj* o, const double* dir, double* out) {   /* mjccd_support */
  double ld[3], r[3]={0,0,0};
  mulmatT3(ld,o->mat,dir);
  if (o->type==FB_GEOM_SPHERE) { for (int i=0;i<3;i++) r[i]=ld[i]*o->size[0]; }
  else if (o->type==FB_GEOM_CAPSULE) { for (int i=0;i<3;i++) r[i]=ld[i]*o->size[0]; r[2]+=sgn(ld[2])*o->size[1]; }
  else if (o->type==FB_GEOM_ELLIPSOID) {
    double t[3]={ld[0]*o->size[0],ld[1]*o->size[1],ld[2]*o->size[2]}; double n=norm3(t);
    if (n>=MINVAL) for (int i=0;i<3;i++) r[i]=t[i]/n*o->size[i];
  } else if (o->type==FB_GEOM_CYLINDER) {
    double n=sqrt(ld[0]*ld[0]+ld[1]*ld[1]);
    if (n>MINVAL) { r[0]=ld[0]/n*o->size[0]; r[1]=ld[1]/n*o->size[0]; }
    r[2]=sgn(ld[2])*o->size[1];
  }
  for (int i=0;i<3;i++) r[i]+=ld[i]*0.5*o->margin;
  mulmat3(out,o->mat,r); add3(out,out,o->pos);
}
/* heightfield prism (mjc_ConvexHField): `size` points at its 6 vertices, given in the frame the test runs in */
#define FB_GEOM_PRISM 100
static void prism_support(const MprObj* o, const double* dir, double* out) {
  int best=0; double bd=dot3(o->size,dir);
  for (int k=1;k<6;k++) { double dd=dot3(o->size+3*k,dir); if (dd>bd) { bd=dd; best=k; } }
  copy3(out,o->size+3*best);
}
static void mpr_support(const MprObj* a, const MprObj* b, const double* dir, MprPt* p) {   /* __ccdSupport */
  double nd[3]={-dir[0],-dir[1],-dir[2]};
  if (a->type==FB_GEOM_PRISM) prism_support(a,dir,p->v1); else mpr_support1(a,dir,p->v1);
  mpr_support1(b,nd,p->v2); sub3(p->v,p->v1,p->v2);
}
static double seg_dist2(const double* P, const double* x0, const double* b, double* w) {     /* ccdVec3PointSegmentDist2 */
  double d[3],a[3],t; sub3(d,b,x0); sub3(a,x0,P);
  t=-dot3(a,d)/dot3(d,d);
  if (t<0 || ccd_zero(t)) { copy3(w,x0); }
  else if (t>1 || ccd_eq(t,1)) { copy3(w,b); }
  else { for (int i=0;i<3;i++) w[i]=x0[i]+t*d[i]; }
  double e[3]; sub3(e,w,P); return dot3(e,e);
}
static double tri_dist2(const double* P, const double* x0, const double* B, const double* C, double* w) {   /* ccdVec3PointTriDist2 */
  double d1[3],d2[3],a[3]; sub3(d1,B,x0); sub3(d2,C,x0); sub3(a,x0,P);
  double v=dot3(d1,d1), ww=dot3(d2,d2), pp=dot3(a,d1), q=dot3(a,d2), r=dot3(d1,d2);
  double s=(q*r-ww*pp)/(ww*v-r*r), t=(-s*r-q)/ww;
  if ((ccd_zero(s)||s>0) && (ccd_eq(s,1)||s<1) && (ccd_zero(t)||t>0) && (ccd_eq(t,1)||t<1) && (ccd_eq(t+s,1)||t+s<1)) {
    for (int i=0;i<3;i++) w[i]=x0[i]+s*d1[i]+t*d2[i];
    double e[3]; sub3(e,w,P); return dot3(e,e);
  }
  double w2[3], dist=seg_dist2(P,x0,B,w), d2_=seg_dist2(P,x0,C,w2);
  if (d2_<dist) { dist=d2_; copy3(w,w2); }
  d2_=seg_dist2(P,B,C,w2);
  if (d2_<dist) { dist=d2_; copy3(w,w2); }
  return dist;
}
static void portal_dir(const MprPt* s, double* dir) {
  double a[3],b[3]; sub3(a,s[2].v,s[1].v); sub3(b,s[3].v,s[1].v); cross3(dir,a,b); normalize3(dir);
}
static int portal_reach_tol(const MprPt* s, const MprPt* v4, const double* dir, double tol) {
  double dv1=dot3(s[1].v,dir), dv2=dot3(s[2].v,dir), dv3=dot3(s[3].v,dir), dv4=dot3(v4->v,dir);
  double d=fmin(dv4-dv1,fmin(dv4-dv2,dv4-dv3));
  return ccd_eq(d,tol) || d<tol;
}
static void expand_portal(MprPt* s, const MprPt* v4) {
  double v4v0[3]; cross3(v4v0,v4->v,s[0].v);
  double dot=dot3(s[1].v,v4v0);
  if (dot>0) { dot=dot3(s[2].v,v4v0); if (dot>0) s[1]=*v4; else s[3]=*v4; }
  else { dot=dot3(s[3].v,v4v0); if (dot>0) s[2]=*v4; else s[1]=*v4; }
}
/* returns 0 and depth / dir / pos when the (inflated) shapes intersect, -1 otherwise */
static int mpr_penetration(const MprObj* o1, const MprObj* o2, double tol, int max_iter, double* depth, double* pdir, double* pos) {
  MprPt s[4]; int size; double dir[3],va[3],vb[3],dot; MprPt v4;
  const double origin[3]={0,0,0};
  /* --- discoverPortal */
  copy3(s[0].v1,o1->pos); copy3(s[0].v2,o2->pos); sub3(s[0].v,s[0].v1,s[0].v2); size=1;
  if (ccd_eq(s[0].v[0],0)&&ccd_eq(s[0].v[1],0)&&ccd_eq(s[0].v[2],0)) { s[0].v[0]=CCD_EPS*10; s[0].v[1]=0; s[0].v[2]=0; }
  scl3(dir,s[0].v,-1); normalize3(dir);
  mpr_support(o1,o2,dir,&s[1]); size=2;
  dot=dot3(s[1].v,dir);
  if (ccd_zero(dot)||dot<0) return -1;
  cross3(dir,s[0].v,s[1].v);
  int res=0;
  if (ccd_zero(dot3(dir,dir))) res = (ccd_eq(s[1].v[0],0)&&ccd_eq(s[1].v[1],0)&&ccd_eq(s[1].v[2],0)) ? 1 : 2;
  if (res==0) {
    normalize3(dir);
    mpr_support(o1,o2,dir,&s[2]);
    dot=dot3(s[2].v,dir);
    if (ccd_zero(dot)||dot<0) return -1;
    size=3;
    sub3(va,s[1].v,s[0].v); sub3(vb,s[2].v,s[0].v); cross3(dir,va,vb); normalize3(dir);
    dot=dot3(dir,s[0].v);
    if (dot>0) { MprPt t=s[1]; s[1]=s[2]; s[2]=t; scl3(dir,dir,-1); }
    while (size<4) {
      mpr_support(o1,o2,dir,&s[3]);
      dot=dot3(s[3].v,dir);
      if (ccd_zero(dot)||dot<0) return -1;
      int cont=0;
      cross3(va,s[1].v,s[3].v); dot=dot3(va,s[0].v);
      if (dot<0 && !ccd_zero(dot)) { s[2]=s[3]; cont=1; }
      if (!cont) {
        cross3(va,s[3].v,s[2].v); dot=dot3(va,s[0].v);
        if (dot<0 && !ccd_zero(dot)) { s[1]=s[3]; cont=1; }
      }
      if (cont) { sub3(va,s[1].v,s[0].v); sub3(vb,s[2].v,s[0].v); cross3(dir,va,vb); normalize3(dir); }
      else size=4;
    }
  }
  if (res==1) {          /* findPenetrTouch: origin on v1 */
    *depth=0; copy3(pdir,origin);
    for (int i=0;i<3;i++) pos[i]=0.5*(s[1].v1[i]+s[1].v2[i]);
    return 0;
  }
  if (res==2) {          /* findPenetrSegment: origin on the segment v0-v1 */
    for (int i=0;i<3;i++) pos[i]=0.5*(s[1].v1[i]+s[1].v2[i]);
    copy3(pdir,s[1].v); *depth=norm3(pdir); normalize3(pdir);
    return 0;
  }
  /* --- refinePortal */
  for (;;) {
    portal_dir(s,dir);
    dot=dot3(dir,s[1].v);
    if (ccd_zero(dot)||dot>0) break;                 /* portalEncapsulesOrigin */
    mpr_support(o1,o2,dir,&v4);
    dot=dot3(v4.v,dir);
    if (!(ccd_zero(dot)||dot>0) || portal_reach_tol(s,&v4,dir,tol)) return -1;     /* portalCanEncapsuleOrigin */
    expand_portal(s,&v4);
  }
  /* --- findPenetr */
  for (int it=0;;it++) {
    portal_dir(s,dir);
    mpr_support(o1,o2,dir,&v4);
    if (portal_reach_tol(s,&v4,dir,tol) || it>max_iter) {
      *depth=sqrt(tri_dist2(origin,s[1].v,s[2].v,s[3].v,pdir));
      if (ccd_zero(pdir[0])&&ccd_zero(pdir[1])&&ccd_zero(pdir[2])) copy3(pdir,dir);
      normalize3(pdir);
      /* findPos: barycentric coordinates of the origin in the portal tetrahedron */
      double b[4],t[3],sum;
      cross3(t,s[1].v,s[2].v); b[0]=dot3(t,s[3].v);
      cross3(t,s[3].v,s[2].v); b[1]=dot3(t,s[0].v);
      cross3(t,s[0].v,s[1].v); b[2]=dot3(t,s[3].v);
      cross3(t,s[2].v,s[1].v); b[3]=dot3(t,s[0].v);
      sum=b[0]+b[1]+b[2]+b[3];
      if (ccd_zero(sum)||sum<0) {
        b[0]=0;
        cross3(t,s[2].v,s[3].v); b[1]=dot3(t,dir);
        cross3(t,s[3].v,s[1].v); b[2]=dot3(t,dir);
        cross3(t,s[1].v,s[2].v); b[3]=dot3(t,dir);
        sum=b[1]+b[2]+b[3];
      }
      double inv=1.0/sum, p1[3]={0,0,0}, p2[3]={0,0,0};
      for (int k=0;k<4;k++) for (int i=0;i<3;i++) { p1[i]+=b[k]*s[k].v1[i]; p2[i]+=b[k]*s[k].v2[i]; }
      for (int i=0;i<3;i++) pos[i]=0.5*inv*(p1[i]+p2[i]);
      return 0;
    }
    expand_portal(s,&v4);
  }
}
/* mjc_fixNormal (engine_collision_convex.c): MPR's portal normal is only as good as its 1e-6 tolerance (~1e-2 rad); for the
 * smooth primitives MuJoCo replaces it by the geometric surface normals at the contact point: n = normalize(n1 - n2) with
 * n_i the outward normal of geom i there (sphere: from the centre; capsule: from the axis segment; ellipsoid: gradient of the
 * implicit function; cylinder: side or cap, whichever the point is nearer to).  Restated from memory, see DESIGN.md.      */
static int surface_normal(int type, const double* pos, const double* mat, const double* size, const double* p, double* n) {
  double d[3], l[3]; sub3(d,p,pos); mulmatT3(l,mat,d);
  double nl[3]={0,0,0};
  if (type==FB_GEOM_SPHERE) { copy3(nl,l); }
  else if (type==FB_GEOM_CAPSULE) { double z=l[2]<-size[1]?-size[1]:(l[2]>size[1]?size[1]:l[2]); nl[0]=l[0]; nl[1]=l[1]; nl[2]=l[2]-z; }
  else if (type==FB_GEOM_ELLIPSOID) { for (int i=0;i<3;i++) nl[i]=l[i]/(size[i]*size[i]); }
  else if (type==FB_GEOM_CYLINDER) {
    double rad=sqrt(l[0]*l[0]+l[1]*l[1]);
    if (size[0]-rad < size[1]-fabs(l[2])) { nl[0]=l[0]; nl[1]=l[1]; }      /* nearer to the side */
    else nl[2]=l[2]>0?1.0:-1.0;                                            /* nearer to a cap */
  } else return 0;
  if (normalize3(nl)<MINVAL) return 0;
  mulmat3(n,mat,nl);
  return 1;
}
static void fix_normal(RawCon* c, int t1, const double* p1, const double* m1, const double* s1, int t2, const double* p2, const double* m2, const double* s2) {
  double n1[3], n2[3]; int h1=surface_normal(t1,p1,m1,s1,c->pos,n1), h2=surface_normal(t2,p2,m2,s2,c->pos,n2);
  double n[3];
  if (h1&&h2) sub3(n,n1,n2); else if (h1) copy3(n,n1); else if (h2) scl3(n,n2,-1); else return;
  if (normalize3(n)<MINVAL) return;
  copy3(c->normal,n);
}
static int col_convex(RawCon* c, double margin, int t1, const double* p1, const double* m1, const double* s1,
                      int t2, const double* p2, const double* m2, const double* s2) {
  MprObj a={p1,m1,s1,t1,margin}, b={p2,m2,s2,t2,margin};
  double depth,dir[3],pos[3];
  if (mpr_penetration(&a,&b,1e-6,50,&depth,dir,pos)!=0) return 0;
  if (ccd_eq(dir[0],0)&&ccd_eq(dir[1],0)&&ccd_eq(dir[2],0)) return 0;      /* normal undefined */
  c->dist=margin-depth; copy3(c->pos,pos); copy3(c->normal,dir); c->tangent[0]=c->tangent[1]=c->tangent[2]=0;
  fix_normal(c,t1,p1,m1,s1,t2,p2,m2,s2);
  return 1;
}
/* Convex geom against a heightfield (MuJoCo mjc_ConvexHField, engine_collision_convex.c, restated from memory): in the
 * heightfield's frame, the grid cells under the geom's bounding box are walked row by row as a triangle strip; every triangle is
 * the top of a prism that reaches down to the base (-size[3]), its top raised by the margin, and each prism runs through the same
 * MPR as any convex pair (the prism's support function is the farthest of its six vertices, its centre their mean).  Every
 * intersecting prism yields one contact (MuJoCo caps them at mjMAXCONPAIR = 50; orc_collision keeps 4 per geom, as the device
 * does): dist = margin - depth, normal from the heightfield into the geom.  orc_collision calls this for the terrain of a model
 * with a heightfield (orc_set_hfield); tests/test_hfield.py holds it against closed forms, tests/test_hfield_gates.py the device
 * code against it.  hf_size = (x half extent, y half extent, elevation scale, base depth); data [nrow][ncol] is scaled by
 * hf_size[2], row = y, col = x.  tri (may be null): per contact the triangle it came from, (row * ncol + column) * 2 + i, the
 * triangle completed at strip vertex (column, row + i).                                                                        */
int orc_convex_hfield_prisms(int type, const double* gpos, const double* gmat, const double* gsize, double margin,
                             const double* hf_pos, const double* hf_mat, const double* hf_size, int nrow, int ncol, const double* data,
                             double* out /* [max][7]: dist, pos[3], normal[3] */, int max, int* tri) {
  double pos[3], mat[9], tmp[3];
  sub3(tmp,gpos,hf_pos); mulmatT3(pos,hf_mat,tmp);
  for (int c=0;c<3;c++) { double col[3]={gmat[c],gmat[3+c],gmat[6+c]}, r[3]; mulmatT3(r,hf_mat,col); mat[c]=r[0]; mat[3+c]=r[1]; mat[6+c]=r[2]; }
  MprObj g={pos,mat,gsize,type,0.0};
  /* bounding box of the geom in the heightfield frame, from its support function */
  double lo[3], hi[3];
  for (int k=0;k<3;k++) { double d[3]={0,0,0}, p[3]; d[k]=1; mpr_support1(&g,d,p); hi[k]=p[k]; d[k]=-1; mpr_support1(&g,d,p); lo[k]=p[k]; }
  if (lo[0]>hf_size[0] || hi[0]<-hf_size[0] || lo[1]>hf_size[1] || hi[1]<-hf_size[1] || lo[2]>hf_size[2]+margin || hi[2]<-hf_size[3]) return 0;
  int cmin=(int)floor((lo[0]+hf_size[0])/(2*hf_size[0])*(ncol-1)), cmax=(int)ceil((hi[0]+hf_size[0])/(2*hf_size[0])*(ncol-1));
  int rmin=(int)floor((lo[1]+hf_size[1])/(2*hf_size[1])*(nrow-1)), rmax=(int)ceil((hi[1]+hf_size[1])/(2*hf_size[1])*(nrow-1));
  if (cmin<0) cmin=0; if (rmin<0) rmin=0; if (cmax>ncol-1) cmax=ncol-1; if (rmax>nrow-1) rmax=nrow-1;
  const double dx=2*hf_size[0]/(ncol-1), dy=2*hf_size[1]/(nrow-1);
  int cnt=0;
  for (int r=rmin;r<rmax;r++) {
    double prism[18]={0}; int nvert=0;
    for (int c=cmin;c<=cmax;c++) for (int i=0;i<2;i++) {
      /* next vertex of the strip: bottom copies in 0..2, top copies in 3..5 */
      for (int k=0;k<2;k++) { copy3(prism+3*k,prism+3*(k+1)); copy3(prism+3*(3+k),prism+3*(4+k)); }
      double x=dx*c-hf_size[0], y=dy*(r+i)-hf_size[1];
      prism[6]=x; prism[7]=y; prism[8]=-hf_size[3];
      prism[15]=x; prism[16]=y; prism[17]=data[(size_t)(r+i)*ncol+c]*hf_size[2]+margin;
      if (++nvert<3) continue;
      if (prism[11]<lo[2] && prism[14]<lo[2] && prism[17]<lo[2]) continue;        /* the geom is above this prism */
      double ctr[3]={0,0,0}; for (int k=0;k<6;k++) addscl3(ctr,prism+3*k,1.0/6.0);
      static const double eye[9]={1,0,0,0,1,0,0,0,1};
      MprObj pr={ctr,eye,prism,FB_GEOM_PRISM,0.0};
      double depth,dir[3],cp[3];
      if (mpr_penetration(&pr,&g,1e-6,50,&depth,dir,cp)!=0) continue;
      if (ccd_eq(dir[0],0)&&ccd_eq(dir[1],0)&&ccd_eq(dir[2],0)) continue;
      double* o=out+7*cnt;
      o[0]=margin-depth; mulmat3(tmp,hf_mat,cp); add3(o+1,tmp,hf_pos); mulmat3(o+4,hf_mat,dir);
      if (tri) tri[cnt]=(r*ncol+c)*2+i;
      if (++cnt>=max) return cnt;
    }
  }
  return cnt;
}
int orc_convex_hfield(int type, const double* gpos, const double* gmat, const double* gsize, double margin,
                      const double* hf_pos, const double* hf_mat, const double* hf_size, int nrow, int ncol, const double* data,
                      double* out, int max) {
  return orc_convex_hfield_prisms(type,gpos,gmat,gsize,margin,hf_pos,hf_mat,hf_size,nrow,ncol,data,out,max,NULL);
}
/* exported for the tests: one generic pair */
int orc_convex_pair(int t1, const double* p1, const double* m1, const double* s1, int t2, const double* p2, const double* m2, const double* s2,
                    double margin, double* out /* dist, pos[3], normal[3] */) {
  RawCon c; int n=col_convex(&c,margin,t1,p1,m1,s1,t2,p2,m2,s2);
  if (n) { out[0]=c.dist; copy3(out+1,c.pos); copy3(out+4,c.normal); }
  return n;
}

int orc_convex_hfield(int type, const double* gpos, const double* gmat, const double* gsize, double margin,
                      const double* hf_pos, const double* hf_mat, const double* hf_size, int nrow, int ncol, const double* data,
                      double* out, int max);
/* narrowphase dispatch of one geom pair (the lower type first, a plane first of all): up to 4 contacts into rc */
static int narrow_pair(RawCon* rc, double margin, int t1, const double* p1, const double* m1, const double* s1,
                       int t2, const double* p2, const double* m2, const double* s2) {
  if (t1==FB_GEOM_PLANE) {
    if (t2==FB_GEOM_SPHERE) return raw_plane_sphere(rc,margin,p1,m1,p2,s2[0]);
    if (t2==FB_GEOM_CAPSULE) return col_plane_capsule(rc,margin,p1,m1,p2,m2,s2);
    if (t2==FB_GEOM_CYLINDER) return col_plane_cylinder(rc,margin,p1,m1,p2,m2,s2);
    if (t2==FB_GEOM_ELLIPSOID) return col_plane_ellipsoid(rc,margin,p1,m1,p2,m2,s2);
    return 0;
  }
  if (t1==FB_GEOM_SPHERE && t2==FB_GEOM_SPHERE) return raw_sphere_sphere(rc,margin,p1,s1[0],p2,s2[0]);
  if (t1==FB_GEOM_SPHERE && t2==FB_GEOM_CAPSULE) return col_sphere_capsule(rc,margin,p1,s1[0],p2,m2,s2);
  if (t1==FB_GEOM_CAPSULE && t2==FB_GEOM_CAPSULE) return col_capsule_capsule(rc,margin,p1,m1,s1,p2,m2,s2);
  return col_convex(rc,margin,t1,p1,m1,s1,t2,p2,m2,s2);   /* generic convex pairs: MPR */
}
/* exported for the tests: one pair of any type through the collision stage's narrowphase and make_frame (no broadphase);
 * out [4][13] = dist, pos[3], frame[9] per contact */
int orc_pair(int t1, const double* p1, const double* m1, const double* s1, int t2, const double* p2, const double* m2, const double* s2,
             double margin, double* out) {
  RawCon rc[4]; int n=narrow_pair(rc,margin,t1,p1,m1,s1,t2,p2,m2,s2);
  for (int i=0;i<n;i++) {
    double* o=out+13*i; double f[9];
    copy3(f,rc[i].normal); copy3(f+3,rc[i].tangent); make_frame(f);
    o[0]=rc[i].dist; copy3(o+1,rc[i].pos); memcpy(o+4,f,sizeof f);
  }
  return n;
}
/* contacts of one geom pair -> d->con with mj_contactParam mixing */
static void add_contacts(OrcData* d, const RawCon* rc, int n, int g1, int g2, double margin, double gap) {
  const FbModel* m=d->m;
  for (int i=0;i<n && d->ncon<ORC_MAXCON;i++) {
    OrcContact* c=&d->con[d->ncon++];
    c->dist=rc[i].dist; copy3(c->pos,rc[i].pos); copy3(c->frame,rc[i].normal); copy3(c->frame+3,rc[i].tangent);
    make_frame(c->frame);
    c->geom1=g1; c->geom2=g2;
    /* mj_contactParam: equal priority -> max condim/friction, solmix-weighted solref/solimp */
    c->dim = m->geom_condim[g1]>m->geom_condim[g2]?m->geom_condim[g1]:m->geom_condim[g2];
    double f[3]; for (int q=0;q<3;q++) f[q]=fmax(m->geom_friction[3*g1+q],m->geom_friction[3*g2+q]);
    if (m->geom_priority[g1]!=m->geom_priority[g2]) {
      int gp=m->geom_priority[g1]>m->geom_priority[g2]?g1:g2;
      c->dim=m->geom_condim[gp]; for (int q=0;q<3;q++) f[q]=m->geom_friction[3*gp+q];
      for (int q=0;q<2;q++) c->solref[q]=m->geom_solref[2*gp+q];
      for (int q=0;q<5;q++) c->solimp[q]=m->geom_solimp[5*gp+q];
    } else {
      double mix1=m->geom_solmix[g1], mix2=m->geom_solmix[g2], mix;
      if (mix1>=MINVAL && mix2>=MINVAL) mix=mix1/(mix1+mix2);
      else if (mix1<MINVAL && mix2<MINVAL) mix=0.5; else if (mix1<MINVAL) mix=0.0; else mix=1.0;
      if (m->geom_solref[2*g1]>0 && m->geom_solref[2*g2]>0)
        for (int q=0;q<2;q++) c->solref[q]=mix*m->geom_solref[2*g1+q]+(1-mix)*m->geom_solref[2*g2+q];
      else for (int q=0;q<2;q++) c->solref[q]=fmin(m->geom_solref[2*g1+q],m->geom_solref[2*g2+q]);
      for (int q=0;q<5;q++) c->solimp[q]=mix*m->geom_solimp[5*g1+q]+(1-mix)*m->geom_solimp[5*g2+q];
    }
    c->friction[0]=c->friction[1]=f[0]; c->friction[2]=f[1]; c->friction[3]=c->friction[4]=f[2];
    c->includemargin=margin-gap;
    c->exclude = (c->dist<c->includemargin)?0:1;
    c->efc_address=-1; c->mu=f[0];
  }
}

static void orc_collision(OrcData* d) {
  const FbModel* m=d->m;
  d->ncon=0;
  for (int k=0;k<m->npair;k++) {
    int g1=m->pair_geom1[k], g2=m->pair_geom2[k];
    int t1=m->geom_type[g1], t2=m->geom_type[g2];
    double margin=fmax(m->geom_margin[g1],m->geom_margin[g2]);
    double gap=fmax(m->geom_gap[g1],m->geom_gap[g2]);
    const double *p1=d->geom_xpos+3*g1,*p2=d->geom_xpos+3*g2,*m1=d->geom_xmat+9*g1,*m2=d->geom_xmat+9*g2;
    const double *s1=m->geom_size+3*g1,*s2=m->geom_size+3*g2;
    /* broadphase: bounding spheres (plane: signed distance of centre) */
    if (t1==FB_GEOM_PLANE) {
      double n[3]={m1[2],m1[5],m1[8]}, t[3]; sub3(t,p2,p1);
      if (dot3(t,n)>margin+m->geom_rbound[g2]) continue;
    } else {
      double t[3]; sub3(t,p2,p1); double r=margin+m->geom_rbound[g1]+m->geom_rbound[g2];
      if (dot3(t,t)>r*r) continue;
    }
    RawCon rc[4]; int n=narrow_pair(rc,margin,t1,p1,m1,s1,t2,p2,m2,s2);
    add_contacts(d,rc,n,g1,g2,margin,gap);
  }
  /* terrain: every listed geom against the heightfield (mjc_ConvexHField), up to 4 contacts per geom, in list order */
  if (d->hf_data) {
    const int g1=d->hf_geom;
    for (int k=0;k<d->hf_npair;k++) {
      const int g2=d->hf_pair[k];
      const double margin=fmax(m->geom_margin[g1],m->geom_margin[g2]), gap=fmax(m->geom_gap[g1],m->geom_gap[g2]);
      double out[4*7]; RawCon rc[4];
      int n=orc_convex_hfield(m->geom_type[g2],d->geom_xpos+3*g2,d->geom_xmat+9*g2,m->geom_size+3*g2,margin,
                              d->geom_xpos+3*g1,d->geom_xmat+9*g1,d->hf_size,d->hf_nrow,d->hf_ncol,d->hf_data,out,4);
      for (int i=0;i<n;i++) { rc[i].dist=out[7*i]; copy3(rc[i].pos,out+7*i+1); copy3(rc[i].normal,out+7*i+4); rc[i].tangent[0]=rc[i].tangent[1]=rc[i].tangent[2]=0; }
      add_contacts(d,rc,n,g1,g2,margin,gap);
    }
  }
  if (d->ncon>=ORC_MAXCON) d->flags|=2;
}

/* ------------------------------------------------------------------------------------------ */
/* K10: constraint rows (MuJoCo mj_makeConstraint, mj_makeImpedance, mj_referenceConstraint; A.8) */
static void get_impedance(const double* solimp, double pos, double margin, double* imp) {
  if (solimp[0]==solimp[1] || solimp[2]<=MINVAL) { *imp=0.5*(solimp[0]+solimp[1]); return; }
  double x=(pos-margin)/solimp[2]; if (x<0) x=-x;
  if (x>=1 || x<=0) { *imp=(x>=1?solimp[1]:solimp[0]); return; }
  double y;
  if (solimp[4]==1) y=x;
  else if (x<=solimp[3]) { double a=1/pow(solimp[3],solimp[4]-1); y=a*pow(x,solimp[4]); }
  else { double b=1/pow(1-solimp[3],solimp[4]-1); y=1-b*pow(1-x,solimp[4]); }
  *imp=solimp[0]+y*(solimp[1]-solimp[0]);
}
static void contact_normal_jac(const OrcData* d, const OrcContact* c, int row, double* J) {
  /* J = frame[row] . (Jp(body2,pos) - Jp(body1,pos)) */
  const FbModel* m=d->m; int nv=m->nv;
  memset(J,0,sizeof(double)*nv);
  const double* f=c->frame+3*row;
  int b1=m->geom_bodyid[c->geom1], b2=m->geom_bodyid[c->geom2];
  for (int k=m->body_lastdof[b2];k>=0;k=m->dof_parentid[k]) {
    double t[3]; cross3(t,d->Sang+3*k,c->pos); add3(t,t,d->Slin+3*k); J[k]+=dot3(f,t);
  }
  for (int k=m->body_lastdof[b1];k>=0;k=m->dof_parentid[k]) {
    double t[3]; cross3(t,d->Sang+3*k,c->pos); add3(t,t,d->Slin+3*k); J[k]-=dot3(f,t);
  }
}
static void orc_make_constraint(OrcData* d) {
  const FbModel* m=d->m; int nv=m->nv; int n=0;
  double solref[2*ORC_MAXEFC], solimp[5*ORC_MAXEFC];
  /* joint limits (hinge) */
  for (int j=0;j<m->njnt;j++) {
    if (!m->jnt_limited[j] || m->jnt_type[j]!=FB_JNT_HINGE) continue;
    double value=d->qpos[m->jnt_qposadr[j]], margin=m->jnt_margin[j];
    for (int side=-1; side<=1; side+=2) {
      double dist=side*(m->jnt_range[2*j+(side+1)/2]-value);
      if (dist<margin && n<ORC_MAXEFC) {
        double* J=d->efc_J+(size_t)n*nv; memset(J,0,sizeof(double)*nv);
        J[m->jnt_dofadr[j]]=-side;
        d->efc_pos[n]=dist; d->efc_margin[n]=margin; d->efc_type[n]=CT_LIMIT; d->efc_id[n]=j;
        d->efc_diagApprox[n]=m->dof_invweight0[m->jnt_dofadr[j]];
        memcpy(solref+2*n,m->jnt_solref+2*j,2*sizeof(double)); memcpy(solimp+5*n,m->jnt_solimp+5*j,5*sizeof(double));
        n++;
      }
    }
  }
  d->nlimit=n;
  for (int ci=0;ci<d->ncon;ci++) {
    OrcContact* c=&d->con[ci];
    c->efc_address=-1;
    if (c->exclude) continue;
    int dim = (c->dim>=3)?3:1;
    if (n+dim>ORC_MAXEFC) { d->flags|=4; break; }
    c->efc_address=n;
    int b1=m->geom_bodyid[c->geom1], b2=m->geom_bodyid[c->geom2];
    double tran=m->body_invweight0[2*b1]+m->body_invweight0[2*b2];
    for (int r=0;r<dim;r++) {
      contact_normal_jac(d,c,r,d->efc_J+(size_t)(n+r)*nv);
      d->efc_pos[n+r]=(r==0)?c->dist:0.0; d->efc_margin[n+r]=(r==0)?c->includemargin:0.0;
      d->efc_type[n+r]=(dim==1)?CT_CONTACT_FRICTIONLESS:CT_CONTACT_ELLIPTIC; d->efc_id[n+r]=ci;
      d->efc_diagApprox[n+r]=tran;
      memcpy(solref+2*(n+r),c->solref,2*sizeof(double)); memcpy(solimp+5*(n+r),c->solimp,5*sizeof(double));
    }
    n+=dim;
  }
  d->nefc=n;
  /* mj_makeImpedance */
  double h=m->opt_timestep;
  for (int i=0;i<n;i++) {
    double* sr=solref+2*i; double* si=solimp+5*i;
    if (sr[0]>0 && sr[0]<2*h) sr[0]=2*h;      /* refsafe */
    double imp; int isfric = (d->efc_type[i]==CT_CONTACT_ELLIPTIC && d->con[d->efc_id[i]].efc_address!=i);
    double pos = isfric ? d->efc_pos[d->con[d->efc_id[i]].efc_address] : d->efc_pos[i];
    double mar = isfric ? d->efc_margin[d->con[d->efc_id[i]].efc_address] : d->efc_margin[i];
    get_impedance(si,pos,mar,&imp);
    if (imp<0.0001) imp=0.0001; if (imp>0.9999) imp=0.9999;
    d->efc_R[i]=fmax(MINVAL,(1-imp)*d->efc_diagApprox[i]/imp);
    double K,B;
    if (sr[0]>0) { double dmax=si[1]; K=1/fmax(MINVAL,dmax*dmax*sr[0]*sr[0]*sr[1]*sr[1]); B=2/fmax(MINVAL,dmax*sr[0]); }
    else { double dmax=si[1]; K=-sr[0]/fmax(MINVAL,dmax*dmax); B=-sr[1]/fmax(MINVAL,dmax); }
    if (isfric) K=0;
    d->efc_KBIP[4*i]=K; d->efc_KBIP[4*i+1]=B; d->efc_KBIP[4*i+2]=imp; d->efc_KBIP[4*i+3]=0;
  }
  /* elliptic friction rows: R_t = R_n/impratio, scaled so that R_j mu_j^2 is constant; con->mu */
  for (int ci=0;ci<d->ncon;ci++) {
    OrcContact* c=&d->con[ci]; int a=c->efc_address;
    if (a<0 || c->dim<3) continue;
    c->mu=c->friction[0]*sqrt(1.0/m->opt_impratio);
    d->efc_R[a+1]=d->efc_R[a]/fmax(MINVAL,m->opt_impratio);
    d->efc_R[a+2]=d->efc_R[a+1]*c->friction[0]*c->friction[0]/(c->friction[1]*c->friction[1]);
  }
  for (int i=0;i<n;i++) d->efc_D[i]=1.0/d->efc_R[i];
}
static void orc_reference_constraint(OrcData* d) {
  int nv=d->m->nv;
  for (int i=0;i<d->nefc;i++) {
    double v=0; const double* J=d->efc_J+(size_t)i*nv;
    for (int k=0;k<nv;k++) v+=J[k]*d->qvel[k];
    d->efc_vel[i]=v;
    d->efc_aref[i]=-d->efc_KBIP[4*i+1]*v-d->efc_KBIP[4*i]*d->efc_KBIP[4*i+2]*(d->efc_pos[i]-d->efc_margin[i]);
  }
}

/* K3: tendon + transmission (MuJoCo mj_tendon, mj_transmission; incl. adhesion/body) */
static void orc_transmission(OrcData* d) {
  const FbModel* m=d->m; int nv=m->nv;
  memset(d->moment,0,sizeof(double)*m->nu*nv);
  double* Jn=d->wk;
  for (int i=0;i<m->nu;i++) {
    double* mom=d->moment+(size_t)i*nv; int id=m->actuator_trnid[i];
    if (m->actuator_trntype[i]==FB_TRN_JOINT) {
      d->actuator_length[i]=d->qpos[m->jnt_qposadr[id]]; mom[m->jnt_dofadr[id]]=1.0;
    } else if (m->actuator_trntype[i]==FB_TRN_TENDON) {
      double len=0;
      for (int k=0;k<m->tendon_num[id];k++) { int w=m->tendon_adr[id]+k; len+=m->wrap_coef[w]*d->qpos[m->wrap_qposadr[w]]; mom[m->wrap_dofid[w]]=m->wrap_coef[w]; }
      d->actuator_length[i]=len;
    } else {
      /* adhesion: moment = - mean of contact-normal Jacobians of contacts touching this body,
       * including contacts inside the gap (exclude==1) */
      d->actuator_length[i]=0; int cnt=0;
      for (int ci=0;ci<d->ncon;ci++) {
        const OrcContact* c=&d->con[ci];
        int b1=m->geom_bodyid[c->geom1], b2=m->geom_bodyid[c->geom2];
        if (b1!=id && b2!=id) continue;
        contact_normal_jac(d,c,0,Jn);
        for (int k=0;k<nv;k++) mom[k]+=Jn[k];
        cnt++;
      }
      if (cnt) for (int k=0;k<nv;k++) mom[k]*=-1.0/cnt;
    }
  }
}

/* K8: actuation (MuJoCo mj_fwdActuation; A.6) */
static void orc_actuation(OrcData* d) {
  const FbModel* m=d->m; int nv=m->nv;
  memset(d->qfrc_actuator,0,sizeof(double)*nv);
  for (int i=0;i<m->nu;i++) {
    double ctrl=d->ctrl[i];
    if (m->actuator_ctrllimited[i]) ctrl=clipd(ctrl,m->actuator_ctrlrange[2*i],m->actuator_ctrlrange[2*i+1]);
    const double* mom=d->moment+(size_t)i*nv;
    double vel=0; for (int k=0;k<nv;k++) vel+=mom[k]*d->qvel[k];
    d->actuator_velocity[i]=vel;
    double input=ctrl; int aa=m->actuator_actadr[i];
    if (aa>=0) {
      double tau=fmax(MINVAL,m->actuator_dynprm[3*i]);
      d->act_dot[aa]=(ctrl-d->act[aa])/tau;
      input=d->act[aa];
    }
    double force=m->actuator_gainprm[3*i]*input;
    if (m->actuator_biastype[i]==1)
      force+=m->actuator_biasprm[3*i]+m->actuator_biasprm[3*i+1]*d->actuator_length[i]+m->actuator_biasprm[3*i+2]*vel;
    if (m->actuator_forcelimited[i]) force=clipd(force,m->actuator_forcerange[2*i],m->actuator_forcerange[2*i+1]);
    d->actuator_force[i]=force;
    for (int k=0;k<nv;k++) d->qfrc_actuator[k]+=mom[k]*force;
  }
}

/* ------------------------------------------------------------------------------------------ */
/* K11: primal Newton solver with exact line search, elliptic cones (MuJoCo mj_solNewton; A.9)  */
typedef struct { double cost; } CostOut;

/* evaluates constraint cost, forces and (optionally) per-row active weights / cone Hessians */
static double constraint_update(OrcData* d, const double* jar, double* force, int* state, double* hcone /* 9 per contact or NULL */) {
  double cost=0; int n=d->nefc;
  for (int i=0;i<n;i++) {
    if (d->efc_type[i]!=CT_CONTACT_ELLIPTIC) {
      if (jar[i]<0) { force[i]=-d->efc_D[i]*jar[i]; cost+=0.5*d->efc_D[i]*jar[i]*jar[i]; state[i]=1; }
      else { force[i]=0; state[i]=0; }
    } else {
      const OrcContact* c=&d->con[d->efc_id[i]];
      double mu=c->mu, fr[2]={c->friction[0],c->friction[1]};
      double U0=jar[i]*mu, U1=jar[i+1]*fr[0], U2=jar[i+2]*fr[1];
      double N=U0, T=sqrt(U1*U1+U2*U2);
      if (mu*N+T<=0 || (T<=0 && N<0)) {            /* bottom zone: quadratic */
        for (int r=0;r<3;r++) { force[i+r]=-d->efc_D[i+r]*jar[i+r]; cost+=0.5*d->efc_D[i+r]*jar[i+r]*jar[i+r]; state[i+r]=1; }
      } else if (N>=mu*T || (T<=0 && N>=0)) {      /* top zone: satisfied */
        for (int r=0;r<3;r++) { force[i+r]=0; state[i+r]=0; }
      } else {                                      /* middle zone: cone */
        double Dm=d->efc_D[i]/(mu*mu*(1+mu*mu)), NmT=N-mu*T;
        cost+=0.5*Dm*NmT*NmT;
        force[i]=-Dm*NmT*mu;
        force[i+1]=-force[i]/T*U1*fr[0];
        force[i+2]=-force[i]/T*U2*fr[1];
        state[i]=state[i+1]=state[i+2]=2;
        if (hcone) {
          double* H=hcone+9*d->efc_id[i]; double U[3]={U0,U1,U2}, sc[3]={mu,fr[0],fr[1]};
          double t=fmax(T,MINVAL), ttt=t*t*t;
          H[0]=1;
          for (int j=1;j<3;j++) H[j]=H[3*j]=-mu*U[j]/t;
          for (int k=1;k<3;k++) for (int j=1;j<3;j++) H[3*k+j]=mu*N/ttt*U[k]*U[j];
          for (int j=1;j<3;j++) H[3*j+j]+=mu*mu-mu*N/t;
          for (int k=0;k<3;k++) for (int j=0;j<3;j++) H[3*k+j]*=Dm*sc[k]*sc[j];
        }
      }
      i+=2;
    }
  }
  return cost;
}

/* 1-D cost along the search direction: value, first and second derivative at alpha */
static void ls_eval(const OrcData* d, double alpha, const double* jar, const double* jv, double quadG0, double quadG1, double quadG2,
                    double* val, double* d1, double* d2) {
  double c=quadG0+alpha*quadG1+alpha*alpha*quadG2, g=quadG1+2*alpha*quadG2, h=2*quadG2;
  int n=d->nefc;
  for (int i=0;i<n;i++) {
    if (d->efc_type[i]!=CT_CONTACT_ELLIPTIC) {
      double x=jar[i]+alpha*jv[i];
      if (x<0) { double D=d->efc_D[i]; c+=0.5*D*x*x; g+=D*x*jv[i]; h+=D*jv[i]*jv[i]; }
    } else {
      const OrcContact* cn=&d->con[d->efc_id[i]];
      double mu=cn->mu, f0=cn->friction[0], f1=cn->friction[1];
      double x0=jar[i]+alpha*jv[i], x1=jar[i+1]+alpha*jv[i+1], x2=jar[i+2]+alpha*jv[i+2];
      double U0=x0*mu, U1=x1*f0, U2=x2*f1, dU0=jv[i]*mu, dU1=jv[i+1]*f0, dU2=jv[i+2]*f1;
      double N=U0, T=sqrt(U1*U1+U2*U2);
      if (mu*N+T<=0 || (T<=0 && N<0)) {
        for (int r=0;r<3;r++) { double x=jar[i+r]+alpha*jv[i+r], D=d->efc_D[i+r]; c+=0.5*D*x*x; g+=D*x*jv[i+r]; h+=D*jv[i+r]*jv[i+r]; }
      } else if (N>=mu*T || (T<=0 && N>=0)) {
      } else {
        double Dm=d->efc_D[i]/(mu*mu*(1+mu*mu)), f=N-mu*T;
        double dT=(U1*dU1+U2*dU2)/T, ddT=(dU1*dU1+dU2*dU2-dT*dT)/T;
        double fp=dU0-mu*dT, fpp=-mu*ddT;
        c+=0.5*Dm*f*f; g+=Dm*f*fp; h+=Dm*(fp*fp+f*fpp);
      }
      i+=2;
    }
  }
  *val=c; *d1=g; *d2=h;
}

static void mul_M(const OrcData* d, double* r, const double* x) {
  int nv=d->m->nv;
  for (int i=0;i<nv;i++) r[i]=dotn(d->M+(size_t)i*nv,x,nv);
}

/* Newton direction in sparse mode.  H = M + U U^T with one column of U per active constraint direction: sqrt(D_r) J_r for an
 * active plain / bottom-zone row, and J_c^T G_c for a contact in the cone's middle zone, G_c G_c^T its 3x3 PSD Hessian block
 * (pivoted Cholesky, rank <= 3).  Then  H^-1 g = M^-1 g - W (I + U^T W)^-1 U^T M^-1 g,  W = M^-1 U  (Woodbury), with M^-1 from the
 * tree-sparse factor: nc sparse solves + an nc x nc Cholesky instead of an nv x nv one.  Same direction as the dense path to
 * round-off (tests/test_oracle_invariants.py holds the two modes against each other); MuJoCo reaches the same H^-1 g with a
 * Cholesky of H that it updates by rank-1 steps as constraint states change (engine_solver.c).  Returns -1 if nc > nv. */
static int newton_direction_lowrank(OrcData* d, int n, const int* state, const double* hcone, const double* grad, double* search, double* work) {
  const FbModel* m=d->m; int nv=m->nv, nc=0;
  double* U=work;                                   /* [nc][nv], then W [nc][nv], then S [nc][nc], t[nc] */
  int cap=nv;                                        /* work holds 2 nv^2 doubles */
  for (int r=0;r<n;r++) {
    if (state[r]==1) {
      if (nc>=cap) return -1;
      double e=sqrt(d->efc_D[r]); const double* J=d->efc_J+(size_t)r*nv; double* u=U+(size_t)nc*nv;
      for (int k=0;k<nv;k++) u[k]=e*J[k];
      nc++;
    } else if (state[r]==2 && d->con[d->efc_id[r]].efc_address==r) {
      const double* Hc=hcone+9*d->efc_id[r]; double G[9]={0}, A[9]; memcpy(A,Hc,sizeof(A));
      double scale=fabs(A[0])+fabs(A[4])+fabs(A[8]);
      for (int j=0;j<3;j++) {                         /* outer-product Cholesky; a vanishing pivot drops the column (PSD, rank-deficient) */
        double piv=A[3*j+j];
        if (piv<=1e-14*scale) continue;
        double sq=sqrt(piv);
        for (int i=j;i<3;i++) G[3*i+j]=A[3*i+j]/sq;
        for (int i=j;i<3;i++) for (int k=j;k<3;k++) A[3*i+k]-=G[3*i+j]*G[3*k+j];
        if (nc>=cap) return -1;
        double* u=U+(size_t)nc*nv; memset(u,0,sizeof(double)*nv);
        for (int p=j;p<3;p++) { double g=G[3*p+j]; if (g==0) continue; const double* J=d->efc_J+(size_t)(r+p)*nv; for (int k=0;k<nv;k++) u[k]+=g*J[k]; }
        nc++;
      }
    }
  }
  double* W=U+(size_t)nc*nv; double* S=W+(size_t)nc*nv; double* t=S+(size_t)nc*nc; double* LS=t+nc;
  if ((size_t)(LS-work)+(size_t)nc*nc > (size_t)2*nv*nv) return -1;
  for (int c=0;c<nc;c++) { memcpy(W+(size_t)c*nv,U+(size_t)c*nv,sizeof(double)*nv); solve_sparse(d,d->qLD,d->qLDiagInv,W+(size_t)c*nv); }
  for (int a=0;a<nc;a++) for (int b=0;b<=a;b++) { double v=dotn(U+(size_t)a*nv,W+(size_t)b*nv,nv); if (a==b) v+=1.0; S[a*nc+b]=v; S[b*nc+a]=v; }
  for (int i=0;i<nv;i++) search[i]=-grad[i];
  solve_sparse(d,d->qLD,d->qLDiagInv,search);
  if (nc==0) return 0;
  for (int c=0;c<nc;c++) t[c]=dotn(U+(size_t)c*nv,search,nv);
  if (cholesky(LS,S,nc)!=0) return -1;
  chol_solve(LS,t,nc);
  for (int c=0;c<nc;c++) { double tc=t[c]; const double* w=W+(size_t)c*nv; for (int k=0;k<nv;k++) search[k]-=w[k]*tc; }
  return 0;
}

static void orc_solve(OrcData* d) {
  const FbModel* m=d->m; int nv=m->nv, n=d->nefc;
  /* qacc_smooth */
  for (int i=0;i<nv;i++) { d->qfrc_smooth[i]=d->qfrc_passive[i]-d->qfrc_bias[i]+d->qfrc_actuator[i]; d->qacc_smooth[i]=d->qfrc_smooth[i]; }
  solve_M(d,d->qacc_smooth);
  d->solver_niter=0;
  if (n==0) {
    memcpy(d->qacc,d->qacc_smooth,sizeof(double)*nv); memset(d->qfrc_constraint,0,sizeof(double)*nv);
    return;
  }
  for (int i=0;i<n;i++) { const double* J=d->efc_J+(size_t)i*nv; d->efc_b[i]=dotn(J,d->qacc_smooth,nv)-d->efc_aref[i]; }
  double* wk=d->wk; double *Ma=wk, *grad=wk+nv, *search=wk+2*nv, *Mv=wk+3*nv, *tmp=wk+4*nv, *H=wk+8*nv, *LH=H+(size_t)nv*nv;
  double jar[ORC_MAXEFC], jv[ORC_MAXEFC], force[ORC_MAXEFC]; int state[ORC_MAXEFC];
  double* hcone=(double*)malloc(sizeof(double)*9*(d->ncon+1));
  double tol = d->solver_tolerance>0 ? d->solver_tolerance : m->opt_tolerance;
  double scale=1.0/(m->stat_meaninertia*(nv>1?nv:1));
  /* warm start: the better of qacc_warmstart and qacc_smooth (MuJoCo warmstart()) */
  double cost_ws, cost_sm;
  {
    double* a=d->qacc_warmstart;
    for (int i=0;i<n;i++) { const double* J=d->efc_J+(size_t)i*nv; jar[i]=dotn(J,a,nv)-d->efc_aref[i]; }
    cost_ws=constraint_update(d,jar,force,state,NULL);
    mul_M(d,Ma,a);
    double g=0; for (int i=0;i<nv;i++) g+=0.5*(Ma[i]-d->qfrc_smooth[i])*(a[i]-d->qacc_smooth[i]);
    cost_ws+=g;
    cost_sm=constraint_update(d,d->efc_b,force,state,NULL);
    if (cost_ws<cost_sm && isfinite(cost_ws)) memcpy(d->qacc,a,sizeof(double)*nv); else memcpy(d->qacc,d->qacc_smooth,sizeof(double)*nv);
  }
  int maxiter=m->opt_iterations;
  double cost=0;
  for (int iter=0; iter<maxiter; iter++) {
    for (int i=0;i<n;i++) { const double* J=d->efc_J+(size_t)i*nv; jar[i]=dotn(J,d->qacc,nv)-d->efc_aref[i]; }
    cost=constraint_update(d,jar,force,state,hcone);
    mul_M(d,Ma,d->qacc);
    double gauss=0; for (int i=0;i<nv;i++) gauss+=0.5*(Ma[i]-d->qfrc_smooth[i])*(d->qacc[i]-d->qacc_smooth[i]);
    cost+=gauss;
    /* gradient = M a - qfrc_smooth - J^T force */
    for (int i=0;i<nv;i++) grad[i]=Ma[i]-d->qfrc_smooth[i];
    for (int r=0;r<n;r++) { if (force[r]==0) continue; const double* J=d->efc_J+(size_t)r*nv; for (int k=0;k<nv;k++) grad[k]-=J[k]*force[r]; }
    double gnorm=0; for (int i=0;i<nv;i++) gnorm+=grad[i]*grad[i]; gnorm=sqrt(gnorm);
    if (scale*gnorm<tol) break;
    if (!d->dense && newton_direction_lowrank(d,n,state,hcone,grad,search,H)==0) {
      /* search = -H^-1 grad through the low-rank form of H (below); falls through to the dense factor when it does not apply */
    } else {
    /* Hessian H = M + J^T D_active J + cone blocks */
      memcpy(H,d->M,sizeof(double)*nv*nv);
      for (int r=0;r<n;r++) {
        if (state[r]==1) {
          const double* J=d->efc_J+(size_t)r*nv; double D=d->efc_D[r];
          for (int a=0;a<nv;a++) { if (J[a]==0) continue; double t=D*J[a]; for (int b=0;b<nv;b++) H[a*nv+b]+=t*J[b]; }
        } else if (state[r]==2 && d->con[d->efc_id[r]].efc_address==r) {
          const double* Hc=hcone+9*d->efc_id[r];
          for (int p=0;p<3;p++) for (int q=0;q<3;q++) {
            const double* Jp=d->efc_J+(size_t)(r+p)*nv; const double* Jq=d->efc_J+(size_t)(r+q)*nv; double hc=Hc[3*p+q];
            if (hc==0) continue;
            for (int a=0;a<nv;a++) { if (Jp[a]==0) continue; double t=hc*Jp[a]; for (int b=0;b<nv;b++) H[a*nv+b]+=t*Jq[b]; }
          }
        }
      }
      if (cholesky(LH,H,nv)!=0) { d->flags|=1; break; }
      for (int i=0;i<nv;i++) search[i]=-grad[i];
      chol_solve(LH,search,nv);
    }
    /* exact line search on phi(alpha) = cost(qacc + alpha*search) */
    for (int i=0;i<n;i++) { const double* J=d->efc_J+(size_t)i*nv; jv[i]=dotn(J,search,nv); }
    mul_M(d,Mv,search);
    double q1=0,q2=0; for (int i=0;i<nv;i++) { q1+=search[i]*(Ma[i]-d->qfrc_smooth[i]); q2+=0.5*search[i]*Mv[i]; }
    double v0,g0,h0; ls_eval(d,0.0,jar,jv,gauss,q1,q2,&v0,&g0,&h0);
    double alpha=0, lo=0, hi=-1, glo=g0;
    if (g0>=0 || h0<=0) { d->solver_niter=iter+1; break; }
    alpha=-g0/h0;
    for (int ls=0; ls<m->opt_ls_iterations*2; ls++) {
      double v,g,h; ls_eval(d,alpha,jar,jv,gauss,q1,q2,&v,&g,&h);
      if (fabs(g)<1e-14*fabs(g0)+1e-300) break;
      if (g<0) { lo=alpha; glo=g; } else hi=alpha;
      double na=alpha-g/h;
      if (hi>=0 && (na<=lo || na>=hi)) na=0.5*(lo+hi);
      else if (hi<0 && na<=lo) na=2*alpha+1e-12;
      if (fabs(na-alpha)<=1e-15*fabs(alpha)) { alpha=na; break; }
      alpha=na;
    }
    (void)glo;
    double v1,g1,h1; ls_eval(d,alpha,jar,jv,gauss,q1,q2,&v1,&g1,&h1);
    for (int i=0;i<nv;i++) d->qacc[i]+=alpha*search[i];
    d->solver_niter=iter+1;
    double improvement=scale*(v0-v1);
    if (improvement<tol) {
      /* final gradient check happens at loop top on next pass only if iterations remain */
      for (int i=0;i<n;i++) { const double* J=d->efc_J+(size_t)i*nv; jar[i]=dotn(J,d->qacc,nv)-d->efc_aref[i]; }
      constraint_update(d,jar,force,state,NULL);
      break;
    }
    (void)tmp;
  }
  /* final forces at the solution */
  for (int i=0;i<n;i++) { const double* J=d->efc_J+(size_t)i*nv; jar[i]=dotn(J,d->qacc,nv)-d->efc_aref[i]; }
  constraint_update(d,jar,force,state,NULL);
  memcpy(d->efc_force,force,sizeof(double)*n); memcpy(d->efc_state,state,sizeof(int)*n);
  memset(d->qfrc_constraint,0,sizeof(double)*nv);
  for (int r=0;r<n;r++) { if (force[r]==0) continue; const double* J=d->efc_J+(size_t)r*nv; for (int k=0;k<nv;k++) d->qfrc_constraint[k]+=J[k]*force[r]; }
  free(hcone);
}

/* mju_QCQP2: min 0.5 x'Ax + x'b  s.t. sum (x_i/d_i)^2 <= r^2 ; returns 1 if constraint active */
static int qcqp2(double* res, const double* Ain, const double* bin, const double* dd, double r) {
  double A11=Ain[0]*dd[0]*dd[0], A22=Ain[3]*dd[1]*dd[1], A12=Ain[1]*dd[0]*dd[1];
  double b1=bin[0]*dd[0], b2=bin[1]*dd[1];
  double P11,P22,P12,det,v1,v2,la=0,val,deriv,detinv;
  for (int iter=0; iter<20; iter++) {
    det=(A11+la)*(A22+la)-A12*A12;
    if (det<1e-10) { res[0]=res[1]=0; return 0; }
    detinv=1/det; P11=(A22+la)*detinv; P22=(A11+la)*detinv; P12=-A12*detinv;
    v1=-P11*b1-P12*b2; v2=-P12*b1-P22*b2;
    val=v1*v1+v2*v2-r*r;
    if (val<1e-10) break;
    deriv=-2*(P11*v1*v1+2*P12*v1*v2+P22*v2*v2);
    double delta=-val/deriv;
    if (delta<1e-10) break;
    la+=delta;
  }
  res[0]=v1*dd[0]; res[1]=v2*dd[1];
  return la!=0;
}

/* noslip post-processing (MuJoCo mj_solNoSlip; A.9): PGS sweeps on contact friction dims with the
 * unregularised Delassus rows A = J M^-1 J^T */
static void orc_noslip(OrcData* d) {
  const FbModel* m=d->m; int nv=m->nv, n=d->nefc;
  if (m->opt_noslip_iterations<=0 || n==0) return;
  int any=0; for (int i=0;i<n;i++) if (d->efc_type[i]==CT_CONTACT_ELLIPTIC) any=1;
  if (!any) return;
  /* A rows for friction dims: A[i][:] = J_i M^-1 J^T */
  double* MinvJT=(double*)malloc(sizeof(double)*nv);
  double* A=(double*)calloc((size_t)n*n,sizeof(double));
  for (int i=0;i<n;i++) {
    if (d->efc_type[i]!=CT_CONTACT_ELLIPTIC) continue;
    memcpy(MinvJT,d->efc_J+(size_t)i*nv,sizeof(double)*nv);
    solve_M(d,MinvJT);
    for (int j=0;j<n;j++) A[(size_t)i*n+j]=dotn(d->efc_J+(size_t)j*nv,MinvJT,nv);
  }
  double* f=d->efc_force;
  double scale=1.0/(m->stat_meaninertia*(nv>1?nv:1));
  for (int iter=0; iter<m->opt_noslip_iterations; iter++) {
    double improvement=0;
    if (iter==0) for (int i=0;i<n;i++) improvement+=0.5*f[i]*f[i]*d->efc_R[i];
    for (int i=0;i<n;i++) {
      if (d->efc_type[i]!=CT_CONTACT_ELLIPTIC) continue;
      const OrcContact* c=&d->con[d->efc_id[i]];
      /* residual of friction rows without regulariser */
      double res[2], old[2]={f[i+1],f[i+2]}, Ac[4], bc[2], v[2];
      for (int r=0;r<2;r++) { double s=d->efc_b[i+1+r]; const double* Ar=A+(size_t)(i+1+r)*n; for (int j=0;j<n;j++) s+=Ar[j]*f[j]; res[r]=s; }
      Ac[0]=A[(size_t)(i+1)*n+i+1]; Ac[1]=A[(size_t)(i+1)*n+i+2]; Ac[2]=A[(size_t)(i+2)*n+i+1]; Ac[3]=A[(size_t)(i+2)*n+i+2];
      bc[0]=res[0]-Ac[0]*old[0]-Ac[1]*old[1]; bc[1]=res[1]-Ac[2]*old[0]-Ac[3]*old[1];
      if (f[i]<MINVAL) { v[0]=v[1]=0; }
      else {
        int active=qcqp2(v,Ac,bc,c->friction,f[i]);
        if (active) {
          double s=(v[0]/c->friction[0])*(v[0]/c->friction[0])+(v[1]/c->friction[1])*(v[1]/c->friction[1]);
          s=sqrt(f[i]*f[i]/fmax(MINVAL,s)); v[0]*=s; v[1]*=s;
        }
      }
      f[i+1]=v[0]; f[i+2]=v[1];
      double dl[2]={v[0]-old[0],v[1]-old[1]};
      /* costChange = 0.5 d'A d + d'res */
      double change=0.5*(dl[0]*(Ac[0]*dl[0]+Ac[1]*dl[1])+dl[1]*(Ac[2]*dl[0]+Ac[3]*dl[1]))+dl[0]*res[0]+dl[1]*res[1];
      if (change>1e-10) { f[i+1]=old[0]; f[i+2]=old[1]; change=0; }
      improvement-=change;
      i+=2;
    }
    improvement*=scale;
    if (improvement<m->opt_noslip_tolerance) break;
  }
  /* qfrc_constraint = J^T f ; qacc = qacc_smooth + M^-1 qfrc_constraint */
  memset(d->qfrc_constraint,0,sizeof(double)*nv);
  for (int r=0;r<n;r++) { if (f[r]==0) continue; const double* J=d->efc_J+(size_t)r*nv; for (int k=0;k<nv;k++) d->qfrc_constraint[k]+=J[k]*f[r]; }
  memcpy(MinvJT,d->qfrc_constraint,sizeof(double)*nv);
  solve_M(d,MinvJT);
  for (int k=0;k<nv;k++) d->qacc[k]=d->qacc_smooth[k]+MinvJT[k];
  free(MinvJT); free(A);
}

/* ------------------------------------------------------------------------------------------ */
/* K12 sensors (MuJoCo mj_sensorVel / mj_sensorAcc + mj_rnePostConstraint; A.10)               */
static double ray_quad(double a, double b, double c, double* x) {
  double det=b*b-a*c;
  if (det<MINVAL) { x[0]=x[1]=-1; return -1; }
  det=sqrt(det);
  x[0]=(-b-det)/a; x[1]=(-b+det)/a;
  if (x[0]>=0) return x[0]; if (x[1]>=0) return x[1]; return -1;
}
static double ray_capsule(const double* pos, const double* mat, const double* size, const double* pnt, const double* vec) {
  double dif[3], lp[3], lv[3], xx[2]; sub3(dif,pnt,pos);
  double ssz=size[0]+size[1];
  if (ray_quad(dot3(vec,vec),dot3(vec,dif),dot3(dif,dif)-ssz*ssz,xx)<0) return -1;
  mulmatT3(lp,mat,dif); mulmatT3(lv,mat,vec);
  double x=-1;
  double a=lv[0]*lv[0]+lv[1]*lv[1], b=lv[0]*lp[0]+lv[1]*lp[1], c=lp[0]*lp[0]+lp[1]*lp[1]-size[0]*size[0];
  double sol=ray_quad(a,b,c,xx);
  if (sol>=0 && fabs(lp[2]+sol*lv[2])<=size[1]) { if (x<0||sol<x) x=sol; }
  double ld[3]={lp[0],lp[1],lp[2]-size[1]};
  ray_quad(dot3(lv,lv),dot3(lv,ld),dot3(ld,ld)-size[0]*size[0],xx);
  for (int i=0;i<2;i++) if (xx[i]>=0 && lp[2]+xx[i]*lv[2]>=size[1]) { if (x<0||xx[i]<x) x=xx[i]; }
  ld[2]=lp[2]+size[1];
  ray_quad(dot3(lv,lv),dot3(lv,ld),dot3(ld,ld)-size[0]*size[0],xx);
  for (int i=0;i<2;i++) if (xx[i]>=0 && lp[2]+xx[i]*lv[2]<=-size[1]) { if (x<0||xx[i]<x) x=xx[i]; }
  return x;
}
static double ray_sphere(const double* pos, double r, const double* pnt, const double* vec) {
  double dif[3], xx[2]; sub3(dif,pnt,pos);
  return ray_quad(dot3(vec,vec),dot3(vec,dif),dot3(dif,dif)-r*r,xx);
}
/* position/velocity-stage sensors (read the current bvel) */
static void orc_sensors_vel(OrcData* d) {
  const FbModel* m=d->m;
  for (int s=0;s<m->nsensor;s++) {
    int tp=m->sensor_type[s], site=m->sensor_objid[s], adr=m->sensor_adr[s], b=m->site_bodyid[site];
    if (tp==FB_SENS_GYRO) mulmatT3(d->sensordata+adr,d->site_xmat+9*site,d->bvel+6*b);
    else if (tp==FB_SENS_VELOCIMETER) { double w[3],v[3]; point_velocity(d,b,d->site_xpos+3*site,w,v); mulmatT3(d->sensordata+adr,d->site_xmat+9*site,v); }
  }
}
/* acceleration-stage sensors: accelerometer, force, touch */
static void orc_sensors_acc(OrcData* d) {
  const FbModel* m=d->m; int nb=m->nbody;
  int need_rne=0;
  for (int s=0;s<m->nsensor;s++) { int tp=m->sensor_type[s]; if (tp==FB_SENS_ACCELEROMETER||tp==FB_SENS_FORCE) need_rne=1; }
  double* bacc=d->wk; double* bfrc=d->wk+6*nb; double* bvel=d->wk+12*nb;
  if (need_rne) {
    rne_forward(d,d->qacc,bvel,bacc);
    rne_body_force(d,bvel,bacc,bfrc);
    /* subtract external (contact) forces: cfrc_ext */
    for (int ci=0;ci<d->ncon;ci++) {
      const OrcContact* c=&d->con[ci]; if (c->efc_address<0) continue;
      int dim=(c->dim>=3)?3:1; double F[3]={0,0,0};
      for (int r=0;r<dim;r++) addscl3(F,c->frame+3*r,d->efc_force[c->efc_address+r]);
      double tq[3]; cross3(tq,c->pos,F);
      int b1=m->geom_bodyid[c->geom1], b2=m->geom_bodyid[c->geom2];
      for (int i=0;i<3;i++) { bfrc[6*b2+i]-=tq[i]; bfrc[6*b2+3+i]-=F[i]; bfrc[6*b1+i]+=tq[i]; bfrc[6*b1+3+i]+=F[i]; }
    }
    for (int b=nb-1;b>0;b--) { int p=m->body_parentid[b]; for (int k=0;k<6;k++) bfrc[6*p+k]+=bfrc[6*b+k]; }
  }
  for (int s=0;s<m->nsensor;s++) {
    int tp=m->sensor_type[s], site=m->sensor_objid[s], adr=m->sensor_adr[s], b=m->site_bodyid[site];
    if (tp==FB_SENS_ACCELEROMETER) {
      const double* a=bacc+6*b; const double* v=bvel+6*b; const double* p=d->site_xpos+3*site;
      double vp[3],t[3],acc[3];
      cross3(t,v,p); add3(vp,v+3,t);              /* velocity of the site point */
      cross3(t,a,p); add3(acc,a+3,t);             /* aO + alpha x p */
      cross3(t,v,vp); add3(acc,acc,t);            /* + w x v_p */
      mulmatT3(d->sensordata+adr,d->site_xmat+9*site,acc);
    } else if (tp==FB_SENS_FORCE) {
      mulmatT3(d->sensordata+adr,d->site_xmat+9*site,bfrc+6*b+3);
    } else if (tp==FB_SENS_TOUCH) {
      double sum=0;
      for (int ci=0;ci<d->ncon;ci++) {
        const OrcContact* c=&d->con[ci]; if (c->efc_address<0) continue;
        int b1=m->geom_bodyid[c->geom1], b2=m->geom_bodyid[c->geom2];
        if (b!=b1 && b!=b2) continue;
        double fn=d->efc_force[c->efc_address]; if (fn<=0) continue;
        double ray[3]; copy3(ray,c->frame); normalize3(ray);
        if (b==b2) scl3(ray,ray,-1);
        double hit;
        if (m->site_type[site]==FB_GEOM_CAPSULE) hit=ray_capsule(d->site_xpos+3*site,d->site_xmat+9*site,m->site_size+3*site,c->pos,ray);
        else hit=ray_sphere(d->site_xpos+3*site,m->site_size[3*site],c->pos,ray);
        if (hit>=0) sum+=fn;
      }
      d->sensordata[adr]=sum;
    }
  }
}

/* ------------------------------------------------------------------------------------------ */
/* K13 Euler with implicit joint damping (MuJoCo mj_Euler; A.11)                                */
static void orc_euler(OrcData* d) {
  const FbModel* m=d->m; int nv=m->nv; double h=m->opt_timestep;
  double* qacc=d->wk; int anydamp=0;
  for (int i=0;i<nv;i++) if (m->dof_damping[i]>0) anydamp=1;
  if (anydamp && !d->dense) {          /* implicit joint damping: (M + h D) qacc' = f, tree-sparse factor */
    double* hd=d->wk+nv; for (int i=0;i<nv;i++) hd[i]=h*m->dof_damping[i];
    factor_sparse(d,d->qLDe,d->qLDeDiagInv,hd);
    for (int i=0;i<nv;i++) qacc[i]=d->qfrc_smooth[i]+d->qfrc_constraint[i];
    solve_sparse(d,d->qLDe,d->qLDeDiagInv,qacc);
  } else if (anydamp) {
    double* H=d->wk+nv; double* LH=H+(size_t)nv*nv;
    memcpy(H,d->M,sizeof(double)*nv*nv);
    for (int i=0;i<nv;i++) H[i*nv+i]+=h*m->dof_damping[i];
    cholesky(LH,H,nv);
    for (int i=0;i<nv;i++) qacc[i]=d->qfrc_smooth[i]+d->qfrc_constraint[i];
    chol_solve(LH,qacc,nv);
  } else memcpy(qacc,d->qacc,sizeof(double)*nv);
  for (int i=0;i<m->na;i++) d->act[i]+=h*d->act_dot[i];
  for (int i=0;i<nv;i++) d->qvel[i]+=h*qacc[i];
  for (int j=0;j<m->njnt;j++) {
    int qa=m->jnt_qposadr[j], da=m->jnt_dofadr[j];
    if (m->jnt_type[j]==FB_JNT_FREE) {
      for (int i=0;i<3;i++) d->qpos[qa+i]+=h*d->qvel[da+i];
      double w[3]={d->qvel[da+3],d->qvel[da+4],d->qvel[da+5]};
      double ang=norm3(w)*h;
      if (ang>0) { double ax[3]; copy3(ax,w); normalize3(ax); double dq[4],nq[4]; axisangle_quat(dq,ax,ang); quat_mul(nq,d->qpos+qa+3,dq); quat_norm(nq); memcpy(d->qpos+qa+3,nq,sizeof(nq)); }
      else quat_norm(d->qpos+qa+3);
    } else d->qpos[qa]+=h*d->qvel[da];
  }
  d->time+=h;
  memcpy(d->qacc_warmstart,d->qacc,sizeof(double)*nv);
}

/* ------------------------------------------------------------------------------------------ */
/* pipeline (MuJoCo engine_forward.c: mj_step1 / mj_step2 / mj_forward)                         */
static void check_state(OrcData* d) {
  const FbModel* m=d->m; double s=0;
  for (int i=0;i<m->nv;i++) { if (!isfinite(d->qacc[i])||!isfinite(d->qvel[i])) d->flags|=1; s+=d->qacc[i]*d->qacc[i]; }
  for (int i=0;i<m->nq;i++) if (!isfinite(d->qpos[i])) d->flags|=1;
  if (sqrt(s)>1e14) d->flags|=1;
}
void orc_step1(OrcData* d) {
  orc_kinematics(d); orc_crb(d); orc_collision(d); orc_make_constraint(d); orc_transmission(d);
  /* velocity stage */
  orc_bias(d); orc_passive(d); orc_reference_constraint(d); orc_sensors_vel(d);
}
void orc_step2(OrcData* d) {
  orc_actuation(d); orc_solve(d); orc_noslip(d); orc_sensors_acc(d); check_state(d); orc_euler(d);
}
void orc_forward(OrcData* d) {
  orc_step1(d); orc_actuation(d); orc_solve(d); orc_noslip(d); orc_sensors_acc(d);
}
void orc_step(OrcData* d) { orc_step1(d); orc_step2(d); }
/* n x physics.step() of dm_control with legacy_step=True: (mj_step2; mj_step1), accumulating the
 * per-substep sensor mean (observable buffer_size = n, aggregator mean; fruitfly.py:626-665).  */
void orc_control_step(OrcData* d, int nsub, double* sensor_mean) {
  int ns=d->m->nsensordata;
  memset(d->sensor_sum,0,sizeof(double)*ns);
  for (int k=0;k<nsub;k++) {
    orc_step2(d); orc_step1(d);
    for (int i=0;i<ns;i++) d->sensor_sum[i]+=d->sensordata[i];
  }
  if (sensor_mean) for (int i=0;i<ns;i++) sensor_mean[i]=d->sensor_sum[i]/nsub;
}
void orc_reset(OrcData* d, const double* qpos, const double* qvel) {
  const FbModel* m=d->m;
  memcpy(d->qpos, qpos?qpos:m->qpos0, sizeof(double)*m->nq);
  if (qvel) memcpy(d->qvel,qvel,sizeof(double)*m->nv); else memset(d->qvel,0,sizeof(double)*m->nv);
  memset(d->act,0,sizeof(double)*m->na); memset(d->ctrl,0,sizeof(double)*m->nu);
  memset(d->qacc,0,sizeof(double)*m->nv); memset(d->qacc_warmstart,0,sizeof(double)*m->nv);
  d->time=0; d->flags=0;
  orc_forward(d);
}

/* accessors for the ctypes test harness */
int orc_get(OrcData* d, int field, double* out) {
  const FbModel* m=d->m; int nv=m->nv;
  switch (field) {
    case FB_QPOS: memcpy(out,d->qpos,sizeof(double)*m->nq); return m->nq;
    case FB_QVEL: memcpy(out,d->qvel,sizeof(double)*nv); return nv;
    case FB_ACT: memcpy(out,d->act,sizeof(double)*m->na); return m->na;
    case FB_CTRL: memcpy(out,d->ctrl,sizeof(double)*m->nu); return m->nu;
    case FB_QACC: memcpy(out,d->qacc,sizeof(double)*nv); return nv;
    case FB_QACC_WARMSTART: memcpy(out,d->qacc_warmstart,sizeof(double)*nv); return nv;
    case FB_SENSORDATA: memcpy(out,d->sensordata,sizeof(double)*m->nsensordata); return m->nsensordata;
    case FB_XPOS: memcpy(out,d->xpos,sizeof(double)*3*m->nbody); return 3*m->nbody;
    case FB_XMAT: memcpy(out,d->xmat,sizeof(double)*9*m->nbody); return 9*m->nbody;
    case FB_SITE_XPOS: memcpy(out,d->site_xpos,sizeof(double)*3*m->nsite); return 3*m->nsite;
    case FB_SITE_XMAT: memcpy(out,d->site_xmat,sizeof(double)*9*m->nsite); return 9*m->nsite;
    case FB_SUBTREE_COM: memcpy(out,d->subtree_com,sizeof(double)*3*m->nbody); return 3*m->nbody;
    case FB_NCON: out[0]=d->ncon; return 1;
    case FB_NEFC: out[0]=d->nefc; return 1;
    case FB_TIME: out[0]=d->time; return 1;
    case FB_QFRC_SMOOTH: memcpy(out,d->qfrc_smooth,sizeof(double)*nv); return nv;
    case FB_QM_DENSE: memcpy(out,d->M,sizeof(double)*nv*nv); return nv*nv;
    case FB_QFRC_CONSTRAINT: memcpy(out,d->qfrc_constraint,sizeof(double)*nv); return nv;
    case FB_SOLVER_NITER: out[0]=d->solver_niter; return 1;
    case FB_QFRC_PASSIVE: memcpy(out,d->qfrc_passive,sizeof(double)*nv); return nv;
    case FB_QFRC_BIAS: memcpy(out,d->qfrc_bias,sizeof(double)*nv); return nv;
    case FB_QFRC_ACTUATOR: memcpy(out,d->qfrc_actuator,sizeof(double)*nv); return nv;
    case FB_CONTACT:
      for (int i=0;i<d->ncon && i<FB_MAXCON;i++) {
        const OrcContact* c=&d->con[i]; double* o=out+16*i;
        o[0]=c->dist; copy3(o+1,c->pos); copy3(o+4,c->frame); o[7]=c->geom1; o[8]=c->geom2; o[9]=c->dim;
        o[10]=c->exclude?0:1; o[11]=c->mu; o[12]=c->efc_address; copy3(o+13,c->frame+3);
      }
      return 16*(d->ncon<FB_MAXCON?d->ncon:FB_MAXCON);
    case FB_EFC_FORCE: memcpy(out,d->efc_force,sizeof(double)*d->nefc); return d->nefc;
    case FB_FLAGS: out[0]=d->flags; return 1;
    default: return -1;
  }
}
int orc_set(OrcData* d, int field, const double* in) {
  const FbModel* m=d->m;
  switch (field) {
    case FB_QPOS: memcpy(d->qpos,in,sizeof(double)*m->nq); return 0;
    case FB_QVEL: memcpy(d->qvel,in,sizeof(double)*m->nv); return 0;
    case FB_ACT: memcpy(d->act,in,sizeof(double)*m->na); return 0;
    case FB_CTRL: memcpy(d->ctrl,in,sizeof(double)*m->nu); return 0;
    case FB_QACC_WARMSTART: memcpy(d->qacc_warmstart,in,sizeof(double)*m->nv); return 0;
    case FB_QACC: memcpy(d->qacc,in,sizeof(double)*m->nv); return 0;
    default: return -1;
  }
}
/* heightfield terrain for the collision stage (tests of the vision-flight groundwork); data is copied */
void orc_set_hfield(OrcData* d, int geom, const double* size, int nrow, int ncol, const double* data, const int* pair_geom, int npair) {
  free(d->hf_data); free(d->hf_pair);
  d->hf_geom=geom; d->hf_nrow=nrow; d->hf_ncol=ncol; d->hf_npair=npair;
  for (int k=0;k<4;k++) d->hf_size[k]=size[k];
  d->hf_data=(double*)malloc(sizeof(double)*(size_t)nrow*ncol); memcpy(d->hf_data,data,sizeof(double)*(size_t)nrow*ncol);
  d->hf_pair=(int*)malloc(sizeof(int)*npair); memcpy(d->hf_pair,pair_geom,sizeof(int)*npair);
}
void orc_set_tolerance(OrcData* d, double tol) { d->solver_tolerance=tol; }
/* 1: dense Cholesky of M and of M + h D (the original, simplest statement); 0 (default): MuJoCo's tree-sparse L^T D L */
void orc_set_dense(OrcData* d, int dense) { d->dense=dense; }
/* efc row data for tests: J (dense), aref, D, R ; returns nefc */
int orc_get_efc(OrcData* d, double* J, double* aref, double* D, double* R, double* pos, int* type) {
  int nv=d->m->nv, n=d->nefc;
  if (J) memcpy(J,d->efc_J,sizeof(double)*(size_t)n*nv);
  if (aref) memcpy(aref,d->efc_aref,sizeof(double)*n);
  if (D) memcpy(D,d->efc_D,sizeof(double)*n);
  if (R) memcpy(R,d->efc_R,sizeof(double)*n);
  if (pos) memcpy(pos,d->efc_pos,sizeof(double)*n);
  if (type) memcpy(type,d->efc_type,sizeof(int)*n);
  return n;
}
