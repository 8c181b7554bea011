// fb_constraint.h -- collision, constraint rows, Delassus projection, actuation, the dual-space
// Newton solver with elliptic cones + noslip, acceleration-stage sensors and the Euler integrator.
#pragma once
#include "fb_tree.h"

// contact record: con_pos[3], con_frame[9] per slot (positions relative to ref)
#define CON_F(arr, slot, k, K) AT(arr, (slot) * (K) + (k))
#define EFC(arr, r) AT(arr, r)
// efc_J / efc_Z rows are stored CHAIN-SPARSE: a row touches the ancestor chain of one dof (limit) or of two (contact: chain a
// of body 2, chain b of body 1).  Slot p < FB_ZCAP holds the p-th element of chain a counted from its end dof upwards
// (= chainlen[la] - chainlen[k] for dof k on the chain); slot FB_ZCAP + p the p-th element of chain b, used only below the point
// where b joins a (the common ancestors carry the sum J_a - J_b in their chain-a slot).  48 floats per row instead of nv = 114.
#define FB_ZCAP 24      // longest dof chain a row may have (fly: 20)
#define FB_JROW (2 * FB_ZCAP)
#define EJC(arr, r, slot) AT(arr, (r) * FB_JROW + (slot))

// ---------------------------------------------------------------------------------------------
// K9 collision: one warp per env.  A bounding-sphere broadphase over the static pair list, then the analytic narrowphase
// one candidate per lane (kcol_broad .. kcol_compact below); the contacts come out in pair-list order, which the Gauss-Seidel
// noslip sweeps depend on.
struct ShCol { int cnt; int njobs, slice; /* candidates of this env; MPR jobs of this env; byte stride between the warps' slices (GPU) */ };
struct RawCon { float dist; V3 pos, n, t; };

FB_DEV int raw_sphere_sphere(RawCon* c, float margin, V3 p1, float r1, V3 p2, float r2) {
  V3 dif = p2 - p1; float cd = dot(dif, dif), lim = margin + r1 + r2;
  if (cd > lim * lim) return 0;
  float len = sqrtf(cd);
  c->dist = len - r1 - r2;
  c->n = (len < 1e-20f) ? v3(1, 0, 0) : dif * (1.0f / len);
  c->pos = p1 + c->n * (r1 + 0.5f * c->dist);
  c->t = v3(0, 0, 0);
  return 1;
}
FB_DEV int raw_plane_sphere(RawCon* c, float margin, V3 pp, V3 n, V3 sp, float r) {
  float cd = dot(sp - pp, n);
  if (cd > margin + r) return 0;
  c->dist = cd - r; c->n = n; c->pos = sp - n * (r + 0.5f * c->dist); c->t = v3(0, 0, 0);
  return 1;
}
FB_DEV int col_plane_capsule(RawCon* c, float margin, V3 pp, V3 n, V3 cp, const M3& cm, V3 size) {
  V3 axis = col(cm, 2), seg = axis * size.y; int k = 0;
  k += raw_plane_sphere(c + k, margin, pp, n, cp + seg, size.x);
  k += raw_plane_sphere(c + k, margin, pp, n, cp - seg, size.x);
  for (int i = 0; i < k; i++) c[i].t = axis;
  return k;
}
// |axis (n.axis) - n|^2 below which a cylinder stands upright on the plane (MuJoCo: 1e-15).  On a plane whose normal is a
// coordinate axis (the floor) its part across n has no cancellation and fp32 resolves it down to 1e-15 as well; on a tilted
// plane fp32 resolves it to ~1e-14 only (DESIGN.md section 2)
#define FB_CYLINDER_UPRIGHT 1e-15f
FB_DEV int col_plane_cylinder(RawCon* c, float margin, V3 pp, V3 n, V3 cp, const M3& cm, V3 size) {
  V3 axis = col(cm, 2);
  float dist0 = dot(cp - pp, n), prjaxis = dot(n, axis);
  if (prjaxis > 0) { axis = axis * -1.0f; prjaxis = -prjaxis; }
  V3 vec = axis * prjaxis - n;
  float len2 = dot(vec, vec);
  if (len2 >= FB_CYLINDER_UPRIGHT) vec = vec * (size.x / sqrtf(len2)); else vec = col(cm, 0) * size.x;
  float prjvec = dot(vec, n);
  axis = axis * size.y; prjaxis *= size.y;
  int cnt = 0;
  if (dist0 + prjaxis + prjvec <= margin) {
    c[cnt].dist = dist0 + prjaxis + prjvec; c[cnt].pos = cp + vec + axis - n * (0.5f * c[cnt].dist); cnt++;
  } else return 0;
  if (dist0 - prjaxis + prjvec <= margin) {
    c[cnt].dist = dist0 - prjaxis + prjvec; c[cnt].pos = cp + vec - axis - n * (0.5f * c[cnt].dist); cnt++;
  }
  float prjvec1 = -prjvec * 0.5f;
  if (dist0 + prjaxis + prjvec1 <= margin) {
    V3 vec1 = normalized(cross(vec, axis)) * (size.x * 0.8660254038f);
    for (int s = 0; s < 2; s++) {
      c[cnt].dist = dist0 + prjaxis + prjvec1;
      c[cnt].pos = cp + axis + vec1 * (s ? -1.0f : 1.0f) - vec * 0.5f - n * (0.5f * c[cnt].dist);
      cnt++;
    }
  }
  for (int i = 0; i < cnt; i++) { c[i].n = n; c[i].t = v3(0, 0, 0); }
  return cnt;
}
FB_DEV int col_plane_ellipsoid(RawCon* c, float margin, V3 pp, V3 n, V3 ep, const M3& em, V3 size) {
  V3 ln = mulT(em, n);
  V3 s = v3(-size.x * size.x * ln.x, -size.y * size.y * ln.y, -size.z * size.z * ln.z);
  float den = sqrtf(size.x * size.x * ln.x * ln.x + size.y * size.y * ln.y * ln.y + size.z * size.z * ln.z * ln.z);
  s = s * (1.0f / fmaxf(den, 1e-30f));
  V3 sup = mul(em, s) + ep;
  float dist = dot(sup - pp, n);
  if (dist > margin) return 0;
  c->dist = dist; c->n = n; c->pos = sup - n * (0.5f * dist); c->t = v3(0, 0, 0);
  return 1;
}
FB_DEV int col_sphere_capsule(RawCon* c, float margin, V3 sp, float sr, V3 cp, const M3& cm, V3 csize) {
  V3 axis = col(cm, 2);
  float x = clampf(dot(axis, sp - cp), -csize.y, csize.y);
  return raw_sphere_sphere(c, margin, sp, sr, cp + axis * x, csize.x);
}
#define FB_CAPSULE_PARALLEL 1e-15f     // |a1 x a2|^2 below which two capsule axes count as parallel
FB_DEV int col_capsule_capsule(RawCon* c, float margin, V3 p1, const M3& m1, V3 s1, V3 p2, const M3& m2, V3 s2) {
  V3 a1 = col(m1, 2), a2 = col(m2, 2), dif = p1 - p2;
  float ma = dot(a1, a1), mb = -dot(a1, a2), mc = dot(a2, a2), u = -dot(a1, dif), v = dot(a2, dif);
  // det = ma mc - mb^2 = |a1 x a2|^2, and the closest-point numerators mc u - mb v = n.(a2 x dif), ma v - mb u = n.(a1 x dif)
  // with n = a1 x a2 (Binet-Cauchy).  In the cross-product form they keep their relative precision for nearly parallel axes,
  // where ma mc - mb^2 cancels in fp32 (5 % off at 1e-3 rad, exactly 0 below 2.4e-4 rad).  DESIGN.md section 2 gives the
  // angles at which fp32 and the fp64 reference still take different branches.
  const V3 n = cross(a1, a2);
  const float det = dot(n, n);
  if (det >= FB_CAPSULE_PARALLEL) {
    float x1 = dot(n, cross(a2, dif)) / det, x2 = dot(n, cross(a1, dif)) / det;
    if (x1 > s1.y) { x1 = s1.y; x2 = (v - mb * s1.y) / mc; }
    else if (x1 < -s1.y) { x1 = -s1.y; x2 = (v + mb * s1.y) / mc; }
    if (x2 > s2.y) { x2 = s2.y; x1 = clampf((u - mb * s2.y) / ma, -s1.y, s1.y); }
    else if (x2 < -s2.y) { x2 = -s2.y; x1 = clampf((u + mb * s2.y) / ma, -s1.y, s1.y); }
    return raw_sphere_sphere(c, margin, p1 + a1 * x1, s1.x, p2 + a2 * x2, s2.x);
  }
  int k = 0; float x;
  x = clampf((v - mb * s1.y) / mc, -s2.y, s2.y); k += raw_sphere_sphere(c + k, margin, p1 + a1 * s1.y, s1.x, p2 + a2 * x, s2.x);
  x = clampf((v + mb * s1.y) / mc, -s2.y, s2.y); k += raw_sphere_sphere(c + k, margin, p1 - a1 * s1.y, s1.x, p2 + a2 * x, s2.x);
  if (k >= 2) return k;
  x = clampf((u - mb * s2.y) / ma, -s1.y, s1.y); k += raw_sphere_sphere(c + k, margin, p1 + a1 * x, s1.x, p2 + a2 * s2.y, s2.x);
  if (k >= 2) return k;
  x = clampf((u + mb * s2.y) / ma, -s1.y, s1.y); k += raw_sphere_sphere(c + k, margin, p1 + a1 * x, s1.x, p2 - a2 * s2.y, s2.x);
  return k;
}
// ---------------------------------------------------------------------------------------------
// Generic convex pairs (MuJoCo mjc_Convex): Minkowski Portal Refinement as in libccd (mpr.c: discoverPortal /
// refinePortal / findPenetr / findPos, vec3.c: point-triangle distance), with MuJoCo's support functions (each geom
// inflated by margin / 2), tolerance 1e-6, 50 iterations, dist = margin - depth.
#ifdef FB_EMU
static long g_convex_stats[4];     // host emulation only: generic candidates, past the pre-tests, contacts, support evaluations
#define CONVEX_STAT(i) g_convex_stats[i]++
#else
#define CONVEX_STAT(i)
#endif
// MPR runs in single precision.  libccd's zero tests compare against an ABSOLUTE machine epsilon, which in double (1e-16) is far below
// any geometric quantity but in single precision (1e-7) is not: with centimetre-scale geometry |v0 x v1|^2 ~ 1e-7 sin^2 and
// the portal discovery mis-classifies ordinary configurations as degenerate (6 % of shallow contacts came out 10x too deep).
// The fp32 code therefore keeps the RELATIVE comparisons at FLT_EPSILON and makes the absolute zero test scale-free
// (1e-30); with that it agrees with the fp64 oracle as often as a double-precision copy fed with the same fp32 inputs does
// (tests/test_emu_parity.py).  MPR in double was 3x slower on the GPU (the FP64 pipe is narrow).
#define MPR_EPS 1.1920929e-7f
#define MPR_ZERO 1e-30f
struct D3 { float x, y, z; };
FB_DEV D3 d3(float x, float y, float z) { D3 r; r.x = x; r.y = y; r.z = z; return r; }
FB_DEV D3 operator+(D3 a, D3 b) { return d3(a.x + b.x, a.y + b.y, a.z + b.z); }
FB_DEV D3 operator-(D3 a, D3 b) { return d3(a.x - b.x, a.y - b.y, a.z - b.z); }
FB_DEV D3 operator*(D3 a, float s) { return d3(a.x * s, a.y * s, a.z * s); }
FB_DEV float ddot(D3 a, D3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
FB_DEV D3 dcross(D3 a, D3 b) { return d3(a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x); }
FB_DEV float dnorm(D3 a) { return sqrtf(ddot(a, a)); }
// 1/sqrtf(x): a single-precision seed + two Newton steps (full single precision without the IEEE sqrt and divide sequences; this
// sits in the inner loop of MPR).  GPU: the hardware reciprocal square root as the seed
#ifdef __CUDACC__
FB_DEV float fast_rsqrt(float x) { float y = rsqrtf(x); y = y * (1.5f - 0.5f * x * y * y); return y * (1.5f - 0.5f * x * y * y); }
#else
FB_DEV float fast_rsqrt(float x) { float y = (float)(1.0f / sqrtf((float)x)); y = y * ((float)1.5 - (float)0.5 * x * y * y); return y * ((float)1.5 - (float)0.5 * x * y * y); }
#endif
FB_DEV D3 dnormalized(D3 a) { float n2 = ddot(a, a); if (n2 < 1e-36) { float n = sqrtf(n2); if (n < 1e-300) return d3(1, 0, 0); return a * (1.0 / n); } return a * fast_rsqrt(n2); }
FB_DEV D3 dsel(bool c, D3 a, D3 b) { return d3(c ? a.x : b.x, c ? a.y : b.y, c ? a.z : b.z); }
struct MprPt { D3 v, v1, v2; };
// e / zoff: per-type coefficients of the branch-free support function below (set by mpr_obj_coefs)
struct MprObj { D3 pos; float mat[9]; D3 size; int type; float margin; D3 e; float zoff; bool round; };
FB_DEV void mpr_obj_coefs(MprObj& o) {
  const bool round = o.type == FB_GEOM_SPHERE || o.type == FB_GEOM_CAPSULE, cyl = o.type == FB_GEOM_CYLINDER;
  o.round = round;
  o.e = (round || cyl) ? d3(o.size.x, o.size.x, cyl ? 0 : o.size.x) : o.size;
  o.zoff = (o.type == FB_GEOM_CAPSULE || cyl) ? o.size.y : 0;
}
FB_DEV bool mpr_zero(float x) { return fabsf(x) < MPR_ZERO; }
FB_DEV bool mpr_eq(float a, float b) { float ab = fabsf(a - b); if (ab < MPR_ZERO) return true; a = fabsf(a); b = fabsf(b); return (b > a) ? ab < MPR_EPS * b : ab < MPR_EPS * a; }
FB_DEV float mpr_sgn(float x) { return x > 0 ? 1.0 : (x < 0 ? -1.0 : 0.0); }
// mjccd_support for sphere / capsule / ellipsoid / cylinder as ONE expression: in the geom frame the support point is
//   e (.) normalize(e (.) d) + sgn(d_z) zoff e_z        e = (r, r, r) sphere, capsule; semi-axes ellipsoid; (r, r, 0) cylinder
// (a sphere is an ellipsoid with equal axes, a capsule a sphere swept by +-zoff, a cylinder a disc swept by +-zoff).  The MPR
// jobs of a warp's lanes are different geom pairs: with a switch over the type every lane pays for every type present.
FB_DEV D3 mpr_support1(const MprObj& o, D3 dir) {
  const float* R = o.mat;
  D3 ld = d3(R[0] * dir.x + R[3] * dir.y + R[6] * dir.z, R[1] * dir.x + R[4] * dir.y + R[7] * dir.z, R[2] * dir.x + R[5] * dir.y + R[8] * dir.z);
  D3 t = d3(ld.x * o.e.x, ld.y * o.e.y, ld.z * o.e.z);
  float n2 = ddot(t, t), in = n2 >= (float)1e-30 ? fast_rsqrt(n2) : (float)0;
  D3 r = d3(t.x * in * o.e.x, t.y * in * o.e.y, t.z * in * o.e.z);
  r = dsel(o.round, ld * o.e.x, r);                 // spheres / capsule caps: radius * d exactly (no normalisation of the unit d)
  r.z += mpr_sgn(ld.z) * o.zoff;
  r = r + ld * ((float)0.5 * o.margin);
  return d3(R[0] * r.x + R[1] * r.y + R[2] * r.z, R[3] * r.x + R[4] * r.y + R[5] * r.z, R[6] * r.x + R[7] * r.y + R[8] * r.z) + o.pos;
}
FB_DEV MprPt mpr_support(const MprObj& a, const MprObj& b, D3 dir) { MprPt p;
  CONVEX_STAT(3);
 p.v1 = mpr_support1(a, dir); p.v2 = mpr_support1(b, d3(0, 0, 0) - dir); p.v = p.v1 - p.v2; return p; }
FB_DEV float mpr_seg_dist2(D3 P, D3 x0, D3 b, D3& w) {
  D3 dd = b - x0, a = x0 - P; float t = -ddot(a, dd) / ddot(dd, dd);
  if (t < 0 || mpr_zero(t)) w = x0; else if (t > 1 || mpr_eq(t, 1)) w = b; else w = x0 + dd * t;
  D3 ee = w - P; return ddot(ee, ee);
}
FB_DEV float mpr_tri_dist2(D3 P, D3 x0, D3 B, D3 C, D3& w) {
  D3 d1 = B - x0, d2 = C - x0, a = x0 - P;
  float v = ddot(d1, d1), ww = ddot(d2, d2), pp = ddot(a, d1), q = ddot(a, d2), r = ddot(d1, d2);
  float s = (q * r - ww * pp) / (ww * v - r * r), t = (-s * r - q) / ww;
  if ((mpr_zero(s) || s > 0) && (mpr_eq(s, 1) || s < 1) && (mpr_zero(t) || t > 0) && (mpr_eq(t, 1) || t < 1) && (mpr_eq(t + s, 1) || t + s < 1)) {
    w = x0 + d1 * s + d2 * t; D3 ee = w - P; return ddot(ee, ee);
  }
  D3 w2; float dist = mpr_seg_dist2(P, x0, B, w), dd = mpr_seg_dist2(P, x0, C, w2);
  if (dd < dist) { dist = dd; w = w2; }
  dd = mpr_seg_dist2(P, B, C, w2);
  if (dd < dist) { dist = dd; w = w2; }
  return dist;
}
// The portal lives in registers: v0..v3 are the Minkowski-difference vertices, p1[i] the first object's support point of
// vertex i (the second's is p1[i] - v_i; only read for the contact position at the very end, so it may sit in local memory).
// Vertex replacement is a chain of selects, not a branch per case: the lanes of a warp refine different pairs.
FB_DEV D3 mpr_portal_dir3(D3 v1, D3 v2, D3 v3) { return dnormalized(dcross(v2 - v1, v3 - v1)); }
FB_DEV bool mpr_reach_tol3(D3 v1, D3 v2, D3 v3, D3 v4, D3 dir, float tol) {
  float dv4 = ddot(v4, dir), dmin = fminf(dv4 - ddot(v1, dir), fminf(dv4 - ddot(v2, dir), dv4 - ddot(v3, dir)));
  return mpr_eq(dmin, tol) || dmin < tol;
}
#define MPR_EXPAND() { D3 v4v0 = dcross(n.v, v0); const bool c1 = ddot(v1, v4v0) > 0, c2 = ddot(v2, v4v0) > 0, c3 = ddot(v3, v4v0) > 0; \
    const int k = c1 ? (c2 ? 1 : 3) : (c3 ? 2 : 1); v1 = dsel(k == 1, n.v, v1); v2 = dsel(k == 2, n.v, v2); v3 = dsel(k == 3, n.v, v3); p1[k] = n.v1; }
// 0 and depth / dir / pos when the inflated shapes intersect, -1 otherwise
FB_DEVN int mpr_penetration(const MprObj& o1, const MprObj& o2, float tol, int max_iter, float& depth, D3& pdir, D3& pos) {
  D3 p1[4], v0, v1, v2, v3, dir; float dt; MprPt n;
  v2 = v3 = d3(0, 0, 0); p1[2] = p1[3] = d3(0, 0, 0);
  p1[0] = o1.pos; v0 = o1.pos - o2.pos;
  if (mpr_eq(v0.x, 0) && mpr_eq(v0.y, 0) && mpr_eq(v0.z, 0)) v0 = d3(MPR_EPS * 10, 0, 0);
  dir = dnormalized(d3(0, 0, 0) - v0);
  n = mpr_support(o1, o2, dir); v1 = n.v; p1[1] = n.v1;
  dt = ddot(v1, dir);
  if (mpr_zero(dt) || dt < 0) return -1;
  dir = dcross(v0, v1);
  int res = 0;
  if (mpr_zero(ddot(dir, dir))) res = (mpr_eq(v1.x, 0) && mpr_eq(v1.y, 0) && mpr_eq(v1.z, 0)) ? 1 : 2;
  if (res == 1) { depth = 0; pdir = d3(0, 0, 0); pos = (p1[1] + p1[1] - v1) * 0.5; return 0; }
  if (res == 2) { pos = (p1[1] + p1[1] - v1) * 0.5; depth = dnorm(v1); pdir = dnormalized(v1); return 0; }
  dir = dnormalized(dir);
  n = mpr_support(o1, o2, dir); v2 = n.v; p1[2] = n.v1;
  dt = ddot(v2, dir);
  if (mpr_zero(dt) || dt < 0) return -1;
  dir = dnormalized(dcross(v1 - v0, v2 - v0));
  if (ddot(dir, v0) > 0) { D3 tv = v1; v1 = v2; v2 = tv; tv = p1[1]; p1[1] = p1[2]; p1[2] = tv; dir = d3(0, 0, 0) - dir; }
  for (int guard = 0;; guard++) {                // discoverPortal
    n = mpr_support(o1, o2, dir); v3 = n.v; p1[3] = n.v1;
    dt = ddot(v3, dir);
    if (mpr_zero(dt) || dt < 0) return -1;
    dt = ddot(dcross(v1, v3), v0);
    const bool r2 = dt < 0 && !mpr_zero(dt);
    dt = ddot(dcross(v3, v2), v0);
    const bool r1 = !r2 && dt < 0 && !mpr_zero(dt);
    if (!(r1 || r2)) break;
    v2 = dsel(r2, v3, v2); v1 = dsel(r1, v3, v1); p1[r2 ? 2 : 1] = p1[3];
    dir = dnormalized(dcross(v1 - v0, v2 - v0));
    if (guard > 1000) return -1;                 // (libccd loops without a bound here)
  }
  for (int guard = 0;; guard++) {                // refinePortal
    dir = mpr_portal_dir3(v1, v2, v3);
    dt = ddot(dir, v1);
    if (mpr_zero(dt) || dt > 0) break;
    n = mpr_support(o1, o2, dir);
    dt = ddot(n.v, dir);
    if (!(mpr_zero(dt) || dt > 0) || mpr_reach_tol3(v1, v2, v3, n.v, dir, tol) || guard > 1000) return -1;
    MPR_EXPAND()
  }
  for (int it = 0;; it++) {                      // findPenetr
    dir = mpr_portal_dir3(v1, v2, v3);
    n = mpr_support(o1, o2, dir);
    if (mpr_reach_tol3(v1, v2, v3, n.v, dir, tol) || it > max_iter) {
      depth = sqrtf(mpr_tri_dist2(d3(0, 0, 0), v1, v2, v3, pdir));
      if (mpr_zero(pdir.x) && mpr_zero(pdir.y) && mpr_zero(pdir.z)) pdir = dir;
      pdir = dnormalized(pdir);
      float b0 = ddot(dcross(v1, v2), v3), b1 = ddot(dcross(v3, v2), v0);
      float b2 = ddot(dcross(v0, v1), v3), b3 = ddot(dcross(v2, v1), v0);
      float sum = b0 + b1 + b2 + b3;
      if (mpr_zero(sum) || sum < 0) {
        b0 = 0; b1 = ddot(dcross(v2, v3), dir); b2 = ddot(dcross(v3, v1), dir); b3 = ddot(dcross(v1, v2), dir);
        sum = b1 + b2 + b3;
      }
      float inv = 0.5 / sum;
      // sum_i b_i (first_i + second_i): vertex 0 = the two centres, vertices 1..3 second_i = first_i - v_i
      pos = ((o1.pos + o2.pos) * b0 + (p1[1] + p1[1] - v1) * b1 + (p1[2] + p1[2] - v2) * b2 + (p1[3] + p1[3] - v3) * b3) * inv;
      return 0;
    }
    MPR_EXPAND()
  }
}
// bounding capsule (axis index, half length, radius) of a convex geom: contains the shape, so that disjoint bounding capsules
// (segment-segment distance > radii + margin) mean "no contact" without running MPR
FB_DEV void bound_capsule(int type, V3 size, int& axis, float& h, float& r) {
  axis = 2; h = 0; r = size.x;
  if (type == FB_GEOM_CAPSULE || type == FB_GEOM_CYLINDER) { h = size.y; }
  else if (type == FB_GEOM_ELLIPSOID) {
    axis = (size.x >= size.y && size.x >= size.z) ? 0 : (size.y >= size.z ? 1 : 2);
    float L = comp(size, axis); r = fmaxf(comp(size, (axis + 1) % 3), comp(size, (axis + 2) % 3)); h = fmaxf(L - r, 0.0f);
  }
}
FB_DEV float seg_seg_dist2(V3 p1, V3 a1, float h1, V3 p2, V3 a2, float h2) {       // distance^2 between two centred segments
  V3 dif = p1 - p2;
  float mb = -dot(a1, a2), u = -dot(a1, dif), v = dot(a2, dif), det = 1.0f - mb * mb, x1, x2;
  if (det > 1e-6f) { x1 = clampf((u - mb * v) / det, -h1, h1); } else x1 = 0;
  x2 = clampf(v - mb * x1, -h2, h2);
  x1 = clampf(u - mb * x2, -h1, h1);
  x2 = clampf(v - mb * x1, -h2, h2);
  V3 dd = (p1 + a1 * x1) - (p2 + a2 * x2); return dot(dd, dd);
}
// mjc_fixNormal: the portal normal is replaced by the geometric surface normals at the contact point (see the oracle)
FB_DEV bool surface_normal(int type, V3 pos, const M3& mat, V3 size, V3 p, V3& n) {
  V3 l = mulT(mat, p - pos), nl = v3(0, 0, 0);
  if (type == FB_GEOM_SPHERE) nl = l;
  else if (type == FB_GEOM_CAPSULE) { float z = clampf(l.z, -size.y, size.y); nl = v3(l.x, l.y, l.z - z); }
  else if (type == FB_GEOM_ELLIPSOID) nl = v3(l.x / (size.x * size.x), l.y / (size.y * size.y), l.z / (size.z * size.z));
  else if (type == FB_GEOM_CYLINDER) {
    float rad = sqrtf(l.x * l.x + l.y * l.y);
    if (size.x - rad < size.y - fabsf(l.z)) nl = v3(l.x, l.y, 0); else nl = v3(0, 0, l.z > 0 ? 1.0f : -1.0f);
  } else return false;
  float nn = norm(nl);
  if (nn < FB_MINVAL) return false;
  n = mul(mat, nl * (1.0f / nn));
  return true;
}
// half width of a convex geom along the unit direction d (its support function measured from the centre)
FB_DEV float support_width(int type, V3 size, const M3& R, V3 d) {
  V3 ld = mulT(R, d);
  if (type == FB_GEOM_SPHERE) return size.x;
  if (type == FB_GEOM_CAPSULE) return size.x + fabsf(ld.z) * size.y;
  if (type == FB_GEOM_ELLIPSOID) return sqrtf(ld.x * ld.x * size.x * size.x + ld.y * ld.y * size.y * size.y + ld.z * ld.z * size.z * size.z);
  return size.x * sqrtf(fmaxf(0.0f, 1.0f - ld.z * ld.z)) + fabsf(ld.z) * size.y;      // cylinder
}
// true if the plane orthogonal to d separates the two geoms by more than the margin (conservative, fp32 with a safety band)
FB_DEV bool separated_along(V3 d, V3 dc, float margin, int t1, V3 s1, const M3& m1, int t2, V3 s2, const M3& m2) {
  float gap = fabsf(dot(dc, d)) - support_width(t1, s1, m1, d) - support_width(t2, s2, m2, d);
  return gap > margin + 1e-5f;
}
// cheap tests that prove "no contact" for a generic convex pair: disjoint bounding capsules, or a separating plane along
// the centre line / a principal axis of either geom.  MPR would report no intersection in these cases, so pruning here does
// not change any result; it leaves ~4 of ~77 generic candidates per env-substep for MPR.
FB_DEV bool convex_prefilter(float margin, int t1, V3 p1, const M3& m1, V3 s1, int t2, V3 p2, const M3& m2, V3 s2) {
  CONVEX_STAT(0);
  int ax1, ax2; float h1, r1, h2, r2;
  bound_capsule(t1, s1, ax1, h1, r1); bound_capsule(t2, s2, ax2, h2, r2);
  float lim = r1 + r2 + margin; lim *= 1.0001f;
  if (seg_seg_dist2(p1, col(m1, ax1), h1, p2, col(m2, ax2), h2) > lim * lim) return false;
  V3 dc = p2 - p1; float n = norm(dc);
  if (n > 1e-9f && separated_along(dc * (1.0f / n), dc, margin, t1, s1, m1, t2, s2, m2)) return false;
  for (int k = 0; k < 3; k++) {
    if (separated_along(col(m1, k), dc, margin, t1, s1, m1, t2, s2, m2)) return false;
    if (separated_along(col(m2, k), dc, margin, t1, s1, m1, t2, s2, m2)) return false;
  }
  return true;
}
FB_DEV int convex_mpr(RawCon* c, float margin, int t1, V3 p1, const M3& m1, V3 s1, int t2, V3 p2, const M3& m2, V3 s2) {
  CONVEX_STAT(1);
  // MPR works on differences of support points: move the origin to the middle of the two centres first, so that the
  // coordinates are of the size of the geoms (fp32 resolution) rather than of their distance to the env's reference point
  const V3 mid = (p1 + p2) * 0.5f;
  MprObj a, b;
  a.pos = d3(p1.x - mid.x, p1.y - mid.y, p1.z - mid.z); a.size = d3(s1.x, s1.y, s1.z); a.type = t1; a.margin = margin;
  b.pos = d3(p2.x - mid.x, p2.y - mid.y, p2.z - mid.z); b.size = d3(s2.x, s2.y, s2.z); b.type = t2; b.margin = margin;
  for (int k = 0; k < 9; k++) { a.mat[k] = m1.m[k]; b.mat[k] = m2.m[k]; }
  mpr_obj_coefs(a); mpr_obj_coefs(b);
  float depth; D3 dir, pos;
  if (mpr_penetration(a, b, (float)1e-6, 50, depth, dir, pos) != 0) return 0;
  if (mpr_eq(dir.x, 0) && mpr_eq(dir.y, 0) && mpr_eq(dir.z, 0)) return 0;
  CONVEX_STAT(2);
  c->dist = (float)(margin - depth); c->pos = v3((float)pos.x, (float)pos.y, (float)pos.z) + mid; c->n = v3((float)dir.x, (float)dir.y, (float)dir.z); c->t = v3(0, 0, 0);
  { V3 n1, n2, nf; bool h1 = surface_normal(t1, p1, m1, s1, c->pos, n1), h2 = surface_normal(t2, p2, m2, s2, c->pos, n2);
    if (h1 || h2) { nf = (h1 && h2) ? n1 - n2 : (h1 ? n1 : v3(0, 0, 0) - n2); float nn = norm(nf); if (nn >= FB_MINVAL) c->n = nf * (1.0f / nn); } }
  return 1;
}
FB_DEV int col_convex(RawCon* c, float margin, int t1, V3 p1, const M3& m1, V3 s1, int t2, V3 p2, const M3& m2, V3 s2) {
  if (!convex_prefilter(margin, t1, p1, m1, s1, t2, p2, m2, s2)) return 0;
  return convex_mpr(c, margin, t1, p1, m1, s1, t2, p2, m2, s2);
}
FB_DEV void make_frame(V3 n, V3 t, V3& f1, V3& f2) {   // mju_makeFrame
  if (norm(t) < 0.5f) { t = (n.y < 0.5f && n.y > -0.5f) ? v3(0, 1, 0) : v3(0, 0, 1); }
  t = normalized(t - n * dot(n, t));
  f1 = t; f2 = cross(n, t);
}

#define FB_COL_ARGS const DevModel& m, const DevData& d, ShCol& sh, int e, int y
// geom positions of this env into shared memory (coalesced), so that the pair loop does not touch the record
FB_DEV void kcol_stage(FB_COL_ARGS) {
  float* gx = sh_dyn(sh); float* gn = gx + 3 * m.ngeom;      // positions; normals (z axes) of the plane geoms
  for (int g = y; g < m.ngeom; g += FB_NY) {
    V3 p = ld3(d.geom_xpos, g, d, e); gx[3 * g] = p.x; gx[3 * g + 1] = p.y; gx[3 * g + 2] = p.z;
    if (m.geom_type[g] == FB_GEOM_PLANE) for (int c = 0; c < 3; c++) gn[3 * g + c] = AT(d.geom_xmat, FB_M3S * g + 3 * c + 2);
  }
}
// Collision in three converged phases.  Broadphase and narrowphase are separated on purpose: in a fused pair loop the
// whole warp pays for the narrowphase whenever ANY lane has a candidate in that iteration (68 iterations x ~1300 cycles);
// here the lanes first only filter their pairs, and the candidates are then narrow-phased one per lane.
#define FB_MAXCAND 192                 // candidates per env (4 contact slots each in tmp_con)
#define FB_COL_DYN(m) (6 * (m).ngeom + 3 * FB_MAXCAND)
#define FB_COL_PTRS float* gx = sh_dyn(sh); float* gn = gx + 3 * m.ngeom; int* flat = reinterpret_cast<int*>(gn + 3 * m.ngeom); \
  int* ccnt = flat + FB_MAXCAND; [[maybe_unused]] int* jobs = ccnt + FB_MAXCAND; (void)gx; (void)gn; (void)flat; (void)ccnt;
// 1. broadphase: lane l tests the pairs l, l + 32, ... of the static pair list (packed record: geoms, plane flag; margin +
// bounding radii -- one coalesced line per step), four steps loaded ahead of the tests.  The hits are ranked with ballots,
// so the candidate list comes out in pair order without per-lane lists.
FB_WARPFN void kcol_broad(const DevModel& m, const DevData& d, ShCol& sh, int e) {
  LREG(int, h0); LREG(int, h1); LREG(int, h2); LREG(int, h3);
  int base = 0;
  const int nstep = (m.npair + 31) / 32;
  for (int i0 = 0; i0 < nstep; i0 += 4) {
    WPAR_BEGIN { FB_COL_PTRS
      int pw[4]; float rs[4]; int hit[4];
#pragma unroll
      for (int u = 0; u < 4; u++) { int k = 32 * (i0 + u) + lane; bool ok = k < m.npair; pw[u] = ok ? m.pair_info[k] : -1; rs[u] = ok ? m.pair_rsum[k] : 0.0f; }
#pragma unroll
      for (int u = 0; u < 4; u++) {
        hit[u] = 0;
        if (pw[u] < 0) continue;
        const int g1 = pw[u] & 0x7fff, g2 = (pw[u] >> 15) & 0x7fff; const bool plane = (pw[u] >> 30) & 1;
        V3 x1 = v3(gx[3 * g1], gx[3 * g1 + 1], gx[3 * g1 + 2]), x2 = v3(gx[3 * g2], gx[3 * g2 + 1], gx[3 * g2 + 2]);
        V3 df = x2 - x1;
        if (plane) hit[u] = dot(df, v3(gn[3 * g1], gn[3 * g1 + 1], gn[3 * g1 + 2])) <= rs[u];
        else hit[u] = dot(df, df) <= rs[u] * rs[u];
      }
      L(h0) = hit[0]; L(h1) = hit[1]; L(h2) = hit[2]; L(h3) = hit[3];
    } WPAR_END
    unsigned m0, m1, m2, m3;
    BALLOT(m0, h0, != 0); BALLOT(m1, h1, != 0); BALLOT(m2, h2, != 0); BALLOT(m3, h3, != 0);
    WPAR_BEGIN { FB_COL_PTRS
      const unsigned lt = (1u << lane) - 1u; int b = base, pos;
      if (L(h0)) { pos = b + POPC(m0 & lt); if (pos < FB_MAXCAND) flat[pos] = 32 * i0 + lane; } b += POPC(m0);
      if (L(h1)) { pos = b + POPC(m1 & lt); if (pos < FB_MAXCAND) flat[pos] = 32 * (i0 + 1) + lane; } b += POPC(m1);
      if (L(h2)) { pos = b + POPC(m2 & lt); if (pos < FB_MAXCAND) flat[pos] = 32 * (i0 + 2) + lane; } b += POPC(m2);
      if (L(h3)) { pos = b + POPC(m3 & lt); if (pos < FB_MAXCAND) flat[pos] = 32 * (i0 + 3) + lane; }
    } WPAR_END
    base += POPC(m0) + POPC(m1) + POPC(m2) + POPC(m3);
  }
  WPAR_BEGIN { if (lane == 0) { sh.cnt = base > FB_MAXCAND ? FB_MAXCAND : base; if (base > FB_MAXCAND) FB_FLAG_OR(2); } } WPAR_END
}
FB_DEV void col_store(const DevModel& m, const DevData& d, int e, int j, const RawCon* rc, int n, int g1, int g2) {
  for (int i = 0; i < n; i++) {
    int slot = 4 * j + i;
    V3 f1, f2; make_frame(rc[i].n, rc[i].t, f1, f2);
    CON_F(d.tmp_con, slot, 0, 13) = rc[i].dist;
    CON_F(d.tmp_con, slot, 1, 13) = rc[i].pos.x; CON_F(d.tmp_con, slot, 2, 13) = rc[i].pos.y; CON_F(d.tmp_con, slot, 3, 13) = rc[i].pos.z;
    CON_F(d.tmp_con, slot, 4, 13) = rc[i].n.x; CON_F(d.tmp_con, slot, 5, 13) = rc[i].n.y; CON_F(d.tmp_con, slot, 6, 13) = rc[i].n.z;
    CON_F(d.tmp_con, slot, 7, 13) = f1.x; CON_F(d.tmp_con, slot, 8, 13) = f1.y; CON_F(d.tmp_con, slot, 9, 13) = f1.z;
    CON_F(d.tmp_con, slot, 10, 13) = f2.x; CON_F(d.tmp_con, slot, 11, 13) = f2.y; CON_F(d.tmp_con, slot, 12, 13) = f2.z;
    AT(d.tmp_geom, 2 * slot) = g1; AT(d.tmp_geom, 2 * slot + 1) = g2;
  }
}
// narrowphase dispatch of one pair (the lower type first, a plane first of all; pn: the plane's normal): its contacts into
// rc[0..3], or -1 for a generic convex pair that the cheap tests cannot rule out (its MPR runs as a job of kcol_mpr).  `g` gives
// a geom's size and rotation (k = 1, 2), loaded only where the pair type needs them.  kcol_narrow and the test hook
// fb_emu_pair both call this, so the hook runs the kernel's own decisions.
template <class G>
FB_DEV int col_narrow_pair(RawCon* rc, float margin, bool plane, int t1, V3 x1, int t2, V3 x2, V3 pn, const G& g) {
  int n = 0;
  if (plane) {
    V3 s2 = g.size(2);
    if (t2 == FB_GEOM_SPHERE) n = raw_plane_sphere(rc, margin, x1, pn, x2, s2.x);
    else { M3 R2 = g.rot(2);
      if (t2 == FB_GEOM_CAPSULE) n = col_plane_capsule(rc, margin, x1, pn, x2, R2, s2);
      else if (t2 == FB_GEOM_CYLINDER) n = col_plane_cylinder(rc, margin, x1, pn, x2, R2, s2);
      else if (t2 == FB_GEOM_ELLIPSOID) n = col_plane_ellipsoid(rc, margin, x1, pn, x2, R2, s2); }
  } else {
    V3 s1 = g.size(1), s2 = g.size(2);
    if (t1 == FB_GEOM_SPHERE && t2 == FB_GEOM_SPHERE) n = raw_sphere_sphere(rc, margin, x1, s1.x, x2, s2.x);
    else if (t1 == FB_GEOM_SPHERE && t2 == FB_GEOM_CAPSULE) { M3 R2 = g.rot(2); n = col_sphere_capsule(rc, margin, x1, s1.x, x2, R2, s2); }
    else if (t1 == FB_GEOM_CAPSULE && t2 == FB_GEOM_CAPSULE) { M3 R1 = g.rot(1), R2 = g.rot(2); n = col_capsule_capsule(rc, margin, x1, R1, s1, x2, R2, s2); }
    else { M3 R1 = g.rot(1), R2 = g.rot(2);      // generic convex pair: MPR job if the cheap tests cannot rule it out
      n = convex_prefilter(margin, t1, x1, R1, s1, t2, x2, R2, s2) ? -1 : 0; }
  }
  return n;
}
struct ColGeoms {         // col_narrow_pair's geoms in the kernel: sizes from the model, rotations from the env's record
  const DevModel& m; const DevData& d; int e, g1, g2;
  FB_DEVM V3 size(int k) const { return mld3(m.geom_size, k == 1 ? g1 : g2); }
  FB_DEVM M3 rot(int k) const { return ld9(d.geom_xmat, k == 1 ? g1 : g2, d, e); }
};
// 2. narrowphase: one candidate per lane, up to 4 contacts each into tmp_con[4 j + i]
FB_DEV void kcol_narrow(FB_COL_ARGS) {
  FB_COL_PTRS
  const int T = sh.cnt;
  for (int j = y; j < T; j += FB_NY) {
    const int k = flat[j], pw = m.pair_info[k];
    const int g1 = pw & 0x7fff, g2 = (pw >> 15) & 0x7fff; const bool plane = (pw >> 30) & 1;
    V3 x1 = v3(gx[3 * g1], gx[3 * g1 + 1], gx[3 * g1 + 2]), x2 = v3(gx[3 * g2], gx[3 * g2 + 1], gx[3 * g2 + 2]);
    const int t1 = m.geom_type[g1], t2 = m.geom_type[g2];
    const float margin = fmaxf(m.geom_margin[g1], m.geom_margin[g2]);
    RawCon rc[4];
    const V3 pn = plane ? v3(gn[3 * g1], gn[3 * g1 + 1], gn[3 * g1 + 2]) : v3(0, 0, 0);
    const int n = col_narrow_pair(rc, margin, plane, t1, x1, t2, x2, pn, ColGeoms{m, d, e, g1, g2});
    col_store(m, d, e, j, rc, n, g1, g2);
    ccnt[j] = n;
  }
}
// 2b. the generic pairs that survived the cheap tests, compacted with ballots and run through MPR one per lane: in the
// candidate loop above a single such pair would stall the other 31 lanes of its round
FB_WARPFN void kcol_mpr(const DevModel& m, const DevData& d, ShCol& sh, int e) {
  LREG(int, pend);
  const int T = sh.cnt;
  int njobs = 0;
  for (int base = 0; base < T; base += 32) {
    WPAR_BEGIN { FB_COL_PTRS L(pend) = (base + lane < T && ccnt[base + lane] < 0) ? 1 : 0; } WPAR_END
    unsigned mk; BALLOT(mk, pend, != 0);
    WPAR_BEGIN { FB_COL_PTRS if (L(pend)) jobs[njobs + POPC(mk & ((1u << lane) - 1u))] = base + lane; } WPAR_END
    njobs += POPC(mk);
  }
#ifdef __CUDACC__
  // The block's envs pool their jobs: an env has ~3 of them, so a warp working on its own list keeps 3 of 32 lanes busy
  // through the longest MPR of the three.  Warp 0 takes the jobs of all FB_WPB envs of the block (one per lane, reading the
  // other warps' lists and geom positions in their shared slices) while the other warps wait at the barrier and leave
  // their issue slots to the rest of the SM.  (Dealing the pooled jobs out to all four warps was measured too: 1.32 ms
  // per control step against 1.03 ms -- four diverging instruction streams per block instead of one.)  All warps of a block
  // are live: env ranges are multiples of FB_WPB.
  if (threadIdx.x == 0) sh.njobs = njobs;
  __syncthreads();
  if (threadIdx.y == 0) {
    const int lane = threadIdx.x, e_first = e;
    unsigned char* base = reinterpret_cast<unsigned char*>(&sh);
    int nj[FB_WPB], tot = 0;
#pragma unroll
    for (int w = 0; w < FB_WPB; w++) { nj[w] = reinterpret_cast<ShCol*>(base + (size_t)w * sh.slice)->njobs; tot += nj[w]; }
    for (int q = lane; q < tot; q += 32) {
      int w = 0, r = q;
      while (r >= nj[w]) { r -= nj[w]; w++; }
      ShCol& o = *reinterpret_cast<ShCol*>(base + (size_t)w * sh.slice);
      const float* gx = sh_dyn(o); const int* flat = reinterpret_cast<const int*>(gx + 6 * m.ngeom); int* ccnt = const_cast<int*>(flat) + FB_MAXCAND; const int* jobs = ccnt + FB_MAXCAND;
      const int e = e_first + w;                                  // env of that warp (AT() and the loads below index by `e`)
      const int j = jobs[r], k = flat[j], pw = m.pair_info[k];
      const int g1 = pw & 0x7fff, g2 = (pw >> 15) & 0x7fff;
      V3 x1 = v3(gx[3 * g1], gx[3 * g1 + 1], gx[3 * g1 + 2]), x2 = v3(gx[3 * g2], gx[3 * g2 + 1], gx[3 * g2 + 2]);
      M3 R1 = ld9(d.geom_xmat, g1, d, e), R2 = ld9(d.geom_xmat, g2, d, e);
      RawCon rc[1];
      int n = convex_mpr(rc, fmaxf(m.geom_margin[g1], m.geom_margin[g2]), m.geom_type[g1], x1, R1, mld3(m.geom_size, g1), m.geom_type[g2], x2, R2, mld3(m.geom_size, g2));
      col_store(m, d, e, j, rc, n, g1, g2);
      ccnt[j] = n;
    }
  }
  __syncthreads();
#else
  // host emulation: each env runs its own jobs
  WPAR_BEGIN { FB_COL_PTRS
    for (int q = lane; q < njobs; q += 32) {
      const int j = jobs[q], k = flat[j], pw = m.pair_info[k];
      const int g1 = pw & 0x7fff, g2 = (pw >> 15) & 0x7fff;
      V3 x1 = v3(gx[3 * g1], gx[3 * g1 + 1], gx[3 * g1 + 2]), x2 = v3(gx[3 * g2], gx[3 * g2 + 1], gx[3 * g2 + 2]);
      M3 R1 = ld9(d.geom_xmat, g1, d, e), R2 = ld9(d.geom_xmat, g2, d, e);
      RawCon rc[1];
      int n = convex_mpr(rc, fmaxf(m.geom_margin[g1], m.geom_margin[g2]), m.geom_type[g1], x1, R1, mld3(m.geom_size, g1), m.geom_type[g2], x2, R2, mld3(m.geom_size, g2));
      col_store(m, d, e, j, rc, n, g1, g2);
      ccnt[j] = n;
    } } WPAR_END
#endif
}
// 3. compaction into the contact list, in candidate order
FB_DEV void kcol_compact(FB_COL_ARGS) {
  FB_COL_PTRS
  const int T = sh.cnt;
  int off = 0, jj = 0;
  for (int j = y; j < T; j += FB_NY) {
    for (; jj < j; jj++) off += ccnt[jj];
    int cnt = ccnt[j];
    for (int i = 0; i < cnt; i++) {
      int dst = off + i, src = 4 * j + i;
      if (dst >= FB_MAXCON) { FB_FLAG_OR(2); break; }
      AT(d.con_dist, dst) = CON_F(d.tmp_con, src, 0, 13);
      for (int k = 0; k < 3; k++) CON_F(d.con_pos, dst, k, 3) = CON_F(d.tmp_con, src, 1 + k, 13);
      for (int k = 0; k < 9; k++) CON_F(d.con_frame, dst, k, 9) = CON_F(d.tmp_con, src, 4 + k, 13);
      AT(d.con_geom1, dst) = AT(d.tmp_geom, 2 * src); AT(d.con_geom2, dst) = AT(d.tmp_geom, 2 * src + 1);
    }
  }
  if (y == 0) { int tot = 0; for (int j = 0; j < T; j++) tot += ccnt[j]; AT(d.ncon, 0) = tot > FB_MAXCON ? FB_MAXCON : tot; }
}

// ---------------------------------------------------------------------------------------------
// K10 constraint rows (MuJoCo mj_makeConstraint + mj_makeImpedance)
FB_DEV float impedance(const float* si, float pos, float margin) {
  if (si[0] == si[1] || si[2] <= FB_MINVAL) return 0.5f * (si[0] + si[1]);
  float x = fabsf((pos - margin) / si[2]);
  if (x >= 1 || x <= 0) return x >= 1 ? si[1] : si[0];
  float yv;
  if (si[4] == 1) yv = x;
  else if (x <= si[3]) yv = powf(x, si[4]) / powf(si[3], si[4] - 1);
  else yv = 1 - powf(1 - x, si[4]) / powf(1 - si[3], si[4] - 1);
  return si[0] + yv * (si[1] - si[0]);
}
FB_DEV void row_params(const DevModel& m, const DevData& d, int e, int r, const float* sr_in, const float* si, float pos, float margin,
                       float diagApprox, bool isfric) {
  float sr0 = sr_in[0], sr1 = sr_in[1];
  if (sr0 > 0 && sr0 < 2 * m.timestep) sr0 = 2 * m.timestep;    // refsafe
  float imp = clampf(impedance(si, pos, margin), 0.0001f, 0.9999f);
  float R = fmaxf(FB_MINVAL, (1 - imp) * diagApprox / imp);
  float K, B, dmax = si[1];
  if (sr0 > 0) { K = 1 / fmaxf(FB_MINVAL, dmax * dmax * sr0 * sr0 * sr1 * sr1); B = 2 / fmaxf(FB_MINVAL, dmax * sr0); }
  else { K = -sr0 / fmaxf(FB_MINVAL, dmax * dmax); B = -sr1 / fmaxf(FB_MINVAL, dmax); }
  if (isfric) K = 0;
  EFC(d.efc_R, r) = R; EFC(d.efc_D, r) = 1.0f / R; EFC(d.efc_K, r) = K; EFC(d.efc_B, r) = B; EFC(d.efc_imp, r) = imp;
}
struct ShCon { int cnt[FB_ROWPAR]; int base; };
#define FB_CON_ARGS const DevModel& m, const DevData& d, ShCon& sh, int e, int y
FB_DEV bool limit_active(const DevModel& m, const DevData& d, int e, int j, int side, float& dist) {
  float value = AT(d.qpos, m.jnt_qposadr[j]);
  dist = side * (m.jnt_range[2 * j + (side + 1) / 2] - value);
  return dist < m.jnt_margin[j];
}
// phase 0/1: joint-limit rows (joints split into contiguous ranges over y so that rows stay in joint order)
FB_DEV void kcon_p0(FB_CON_ARGS) {
  prefetch_rec(d.qLD, m.nM, d, e, y); prefetch_rec(d.Sang, FB_V3S * m.nv, d, e, y); prefetch_rec(d.Slin, FB_V3S * m.nv, d, e, y);   // for the projection phases
  if (y >= FB_ROWPAR) return;
  int j0 = (int)((long)y * m.njnt / FB_ROWPAR), j1 = (int)((long)(y + 1) * m.njnt / FB_ROWPAR), c = 0; float dist;
  for (int j = j0; j < j1; j++) { if (!m.jnt_limited[j] || m.jnt_type[j] != FB_JNT_HINGE) continue; for (int side = -1; side <= 1; side += 2) c += limit_active(m, d, e, j, side, dist) ? 1 : 0; }
  sh.cnt[y] = c;
}
FB_DEV void kcon_p1(FB_CON_ARGS) {
  if (y >= FB_ROWPAR) return;
  int n = 0; for (int yy = 0; yy < y; yy++) n += sh.cnt[yy];
  int j0 = (int)((long)y * m.njnt / FB_ROWPAR), j1 = (int)((long)(y + 1) * m.njnt / FB_ROWPAR); float dist;
  for (int j = j0; j < j1; j++) {
    if (!m.jnt_limited[j] || m.jnt_type[j] != FB_JNT_HINGE) continue;
    for (int side = -1; side <= 1; side += 2) {
      if (limit_active(m, d, e, j, side, dist) && n < FB_MAXEFC) {
        EFC(d.efc_type, n) = FB_CT_LIMIT; EFC(d.efc_id, n) = (side < 0) ? j : -(j + 1);   // sign encodes the side
        EFC(d.efc_pos, n) = dist; EFC(d.efc_margin, n) = m.jnt_margin[j];
        row_params(m, d, e, n, m.jnt_solref + 2 * j, m.jnt_solimp + 5 * j, dist, m.jnt_margin[j], m.dof_invweight0[m.jnt_dofadr[j]], false);
        n++;
      }
    }
  }
  if (y == FB_ROWPAR - 1) sh.base = n < FB_MAXEFC ? n : FB_MAXEFC;
}
// contact -> (dim, included)
FB_DEV int contact_dim(const DevModel& m, const DevData& d, int e, int ci, float& includemargin, bool& incl) {
  int g1 = AT(d.con_geom1, ci), g2 = AT(d.con_geom2, ci);
  float margin = fmaxf(m.geom_margin[g1], m.geom_margin[g2]), gap = fmaxf(m.geom_gap[g1], m.geom_gap[g2]);
  includemargin = margin - gap;
  int dim = m.geom_condim[g1] > m.geom_condim[g2] ? m.geom_condim[g1] : m.geom_condim[g2];
  incl = AT(d.con_dist, ci) < includemargin;
  return dim >= 3 ? 3 : 1;
}
FB_DEV void kcon_p2(FB_CON_ARGS) {
  if (y >= FB_ROWPAR) return;
  int ncon = AT(d.ncon, 0);
  int c0 = y * ncon / FB_ROWPAR, c1 = (y + 1) * ncon / FB_ROWPAR, rows = 0;
  for (int ci = c0; ci < c1; ci++) { float im; bool incl; int dim = contact_dim(m, d, e, ci, im, incl); if (incl) rows += dim; }
  sh.cnt[y] = rows;
}
FB_DEV void kcon_p3(FB_CON_ARGS) {
  if (y >= FB_ROWPAR) return;
  int ncon = AT(d.ncon, 0);
  int n = sh.base; for (int yy = 0; yy < y; yy++) n += sh.cnt[yy];
  int c0 = y * ncon / FB_ROWPAR, c1 = (y + 1) * ncon / FB_ROWPAR;
  const float* fric = PRM(FB_P_GEOM_FRICTION, m.geom_friction);
  for (int ci = c0; ci < c1; ci++) {
    float includemargin; bool incl; int dim = contact_dim(m, d, e, ci, includemargin, incl);
    int g1 = AT(d.con_geom1, ci), g2 = AT(d.con_geom2, ci);
    float dist = AT(d.con_dist, ci);
    float fr0 = fmaxf(fric[3 * g1], fric[3 * g2]);
    AT(d.con_dim, ci) = dim; AT(d.con_mu, ci) = fr0 * sqrtf(1.0f / m.impratio);
    CON_F(d.con_fric, ci, 0, 2) = fr0; CON_F(d.con_fric, ci, 1, 2) = fr0;
    AT(d.con_efcadr, ci) = -1;
    if (!incl) continue;                            // detected, but inside the gap: adhesion only
    if (n + dim > FB_MAXEFC) { FB_FLAG_OR(4); n += dim; continue; }
    float mix1 = m.geom_solmix[g1], mix2 = m.geom_solmix[g2], mix;
    if (mix1 >= FB_MINVAL && mix2 >= FB_MINVAL) mix = mix1 / (mix1 + mix2);
    else if (mix1 < FB_MINVAL && mix2 < FB_MINVAL) mix = 0.5f; else mix = (mix1 < FB_MINVAL) ? 0.0f : 1.0f;
    float sr[2], si[5];
    if (m.geom_solref[2 * g1] > 0 && m.geom_solref[2 * g2] > 0) for (int q = 0; q < 2; q++) sr[q] = mix * m.geom_solref[2 * g1 + q] + (1 - mix) * m.geom_solref[2 * g2 + q];
    else for (int q = 0; q < 2; q++) sr[q] = fminf(m.geom_solref[2 * g1 + q], m.geom_solref[2 * g2 + q]);
    for (int q = 0; q < 5; q++) si[q] = mix * m.geom_solimp[5 * g1 + q] + (1 - mix) * m.geom_solimp[5 * g2 + q];
    int b1 = m.geom_bodyid[g1], b2 = m.geom_bodyid[g2];
    float tran = m.body_invweight0[2 * b1] + m.body_invweight0[2 * b2];
    AT(d.con_efcadr, ci) = n;
    for (int r = 0; r < dim; r++) {
      EFC(d.efc_type, n + r) = dim == 1 ? FB_CT_FRICTIONLESS : FB_CT_ELLIPTIC; EFC(d.efc_id, n + r) = ci;
      EFC(d.efc_pos, n + r) = r == 0 ? dist : 0.0f; EFC(d.efc_margin, n + r) = r == 0 ? includemargin : 0.0f;
      row_params(m, d, e, n + r, sr, si, dist, includemargin, tran, r > 0);
    }
    if (dim == 3) {   // friction rows: R_t = R_n / impratio (both tangents share mu here)
      float Rn = EFC(d.efc_R, n), Rt = Rn / fmaxf(FB_MINVAL, m.impratio);
      EFC(d.efc_R, n + 1) = Rt; EFC(d.efc_D, n + 1) = 1.0f / Rt; EFC(d.efc_R, n + 2) = Rt; EFC(d.efc_D, n + 2) = 1.0f / Rt;
    }
    n += dim;
  }
  if (y == FB_ROWPAR - 1) {
    // rows are contiguous up to the first overflowing contact; later ones were all dropped
    int tot = n;
    if (tot > FB_MAXEFC) { tot = sh.base; for (int ci = 0; ci < ncon; ci++) { int a = AT(d.con_efcadr, ci); if (a >= 0 && a + AT(d.con_dim, ci) > tot) tot = a + AT(d.con_dim, ci); } }
    AT(d.nefc, 0) = tot;
  }
}

// ---------------------------------------------------------------------------------------------
// Row dof sets.  A limit row touches the ancestor chain of its dof; a contact row the union of the
// chains of its two bodies.  `RowDofs` walks that union in descending dof order.
struct RowChains { int la, lb; };
FB_DEV RowChains row_chains(const DevModel& m, const DevData& d, int e, int r, int& ci, int& frow, float& sign) {
  RowChains rc; int tp = EFC(d.efc_type, r), id = EFC(d.efc_id, r);
  if (tp == FB_CT_LIMIT) {
    int j = id >= 0 ? id : -(id + 1);
    sign = id >= 0 ? 1.0f : -1.0f;        // lower limit: J = +1, upper: J = -1
    rc.la = m.jnt_dofadr[j]; rc.lb = -1; ci = -1; frow = 0;
  } else {
    ci = id; frow = r - AT(d.con_efcadr, ci); sign = 1.0f;
    rc.la = m.body_lastdof[m.geom_bodyid[AT(d.con_geom2, ci)]];
    rc.lb = m.body_lastdof[m.geom_bodyid[AT(d.con_geom1, ci)]];
  }
  return rc;
}

// Jacobian entry of contact `ci`, frame row `frow`, on dof k of chain side s (+1 body2, -1 body1)
FB_DEV float contact_J(const DevModel& m, const DevData& d, int e, V3 f, V3 pos, int k) {
  V3 t = ld3(d.Slin, k, d, e) + cross(ld3(d.Sang, k, d, e), pos);
  return dot(f, t);
}

// K10b projection: one warp per env, rows dealt to the lanes.
//   phase 0: J (dense-by-dof storage), Z = D^-1/2 L^-T J^T restricted to the row's dof set
//   phase 1: A = Z Z^T  (= J M^-1 J^T, the unregularised Delassus matrix)
struct ShNone { int dummy; };
#define FB_ROW_ARGS const DevModel& m, const DevData& d, ShCon& sh, int e, int y
// one dof chain of a row: Jacobian entries along the chain, then z = D^-1/2 L^-T j by a dense back-sweep over the
// chain (the ancestors of the p-th chain element are the elements p+1.. and L[k_p][k_q] sits at qLD[Madr[k_p] + q - p])
FB_DEV void proj_chain(const DevModel& m, const DevData& d, int e, int r, int last, float sgn, bool contact, V3 f, V3 pos, float* zc,
                       int other_last, bool accumulate) {
  if (last < 0) return;
  int adr0 = m.dof_Madr[last], L = m.dof_chainlen[last];
  if (L > FB_ZCAP) { FB_FLAG_OR(4); L = FB_ZCAP; }
  const int Lo = other_last >= 0 ? m.dof_chainlen[other_last] : 0, base = accumulate ? FB_ZCAP : 0;
  // chain b joins chain a at its first common ancestor: from there up the entries are added to chain a's slots
  const int join = (accumulate && other_last >= 0) ? L - m.dof_lca[last * m.nv + other_last] : L;
  for (int p = 0; p < L; p++) {
    int k = m.dof_anc[adr0 + p];
    float v = contact ? sgn * contact_J(m, d, e, f, pos, k) : (p == 0 ? sgn : 0.0f);
    zc[p] = v;
    if (p >= join) EJC(d.efc_J, r, Lo - (L - p)) += v; else EJC(d.efc_J, r, base + p) = v;      // chainlen[k] = L - p
  }
  for (int p = 0; p < L; p++) {
    int k = m.dof_anc[adr0 + p], row = m.dof_Madr[k];
    float zk = zc[p], D = AT(d.qLD, row), zs = zk / D;          // unscaled rows: L[k][anc] z[k] = M'[k][anc] (z[k] / D[k])
    for (int q = p + 1; q < L; q++) zc[q] -= AT(d.qLD, row + (q - p)) * zs;
    float zf = zk / sqrtf(D);
    if (p >= join) EJC(d.efc_Z, r, Lo - (L - p)) += zf; else EJC(d.efc_Z, r, base + p) = zf;
  }
}
// all 32 lanes over rows: J (chain-sparse storage, see EJC) and Z = D^-1/2 L^-T J^T, chain by chain (a contact row is the
// difference of two single-chain rows; the sweep is linear)
FB_DEV void kproj_p0(FB_ROW_ARGS) {
  int n = AT(d.nefc, 0);
  float* zc = sh_dyn(sh) + (size_t)y * FB_ZCAP;
  for (int r = y; r < n; r += FB_NY) {
    int ci, frow; float sign;
    RowChains rc = row_chains(m, d, e, r, ci, frow, sign);
    AT(d.efc_la, r) = rc.la; AT(d.efc_lb, r) = rc.lb;
    {   // row identity for the warm start: limit -> (joint, side); contact -> (geom pair, ordinal within the pair, frame row)
      int key;
      if (ci < 0) key = 0x40000000 | (EFC(d.efc_id, r) + FB_MAXEFC * 4);
      else { int g1 = AT(d.con_geom1, ci), g2 = AT(d.con_geom2, ci), ord = 0;
        while (ci - ord - 1 >= 0 && AT(d.con_geom1, ci - ord - 1) == g1 && AT(d.con_geom2, ci - ord - 1) == g2) ord++;
        key = (((g1 * m.ngeom + g2) * 4 + (ord & 3)) * 3 + frow); }
      AT(d.efc_key, r) = key;
    }
    V3 f = v3(0, 0, 0), pos = v3(0, 0, 0);
    if (ci >= 0) { f = v3(CON_F(d.con_frame, ci, 3 * frow, 9), CON_F(d.con_frame, ci, 3 * frow + 1, 9), CON_F(d.con_frame, ci, 3 * frow + 2, 9));
                   pos = v3(CON_F(d.con_pos, ci, 0, 3), CON_F(d.con_pos, ci, 1, 3), CON_F(d.con_pos, ci, 2, 3)); }
    proj_chain(m, d, e, r, rc.la, ci >= 0 ? 1.0f : sign, ci >= 0, f, pos, zc, -1, false);
    if (ci >= 0) proj_chain(m, d, e, r, rc.lb, -1.0f, true, f, pos, zc, rc.la, true);
  }
}
// A = Z Z^T (= J M^-1 J^T, the unregularised Delassus matrix), packed lower triangle; pairs dealt to all lanes
// Z[r] . Z[c] over the dofs one chain of row r shares with one chain of row c.  Two ancestor chains share exactly their common TAIL
// (from the lowest common ancestor up), m.dof_lca gives its length, and with the chain-sparse row layout (EJC) the shared dofs are
// a CONTIGUOUS slot range in both rows: a plain dot product, no membership tests and no chain walk.  (x, y) in {a, b}: `base` is
// the chain's slot base (0 / FB_ZCAP), `lim` how many of its leading slots the row stores (chain a: all of it; chain b: only the
// part below its join with chain a -- the common ancestors carry the summed entry in their chain-a slot).
FB_DEV float zdot_tail(const DevModel& m, const DevData& d, int e, int r, int lx, int Lx, int xbase, int xlim, int c, int ly, int Ly, int ybase, int ylim) {
  if (lx < 0 || ly < 0) return 0.0f;
  const int mlen = m.dof_lca[lx * m.nv + ly];
  if (mlen == 0) return 0.0f;
  const int sh = Lx - Ly;                                   // slot in chain x = slot in chain y + sh (both count from the chain's end dof upwards)
  int p = Ly - mlen, p_hi = Ly < ylim ? Ly : ylim;
  if (xlim - sh < p_hi) p_hi = xlim - sh;
  float s = 0;
  for (; p < p_hi; p++) s += EJC(d.efc_Z, r, xbase + p + sh) * EJC(d.efc_Z, c, ybase + p);
  return s;
}
FB_DEV void kproj_p1(FB_ROW_ARGS) {
  int n = AT(d.nefc, 0), npair = n * (n + 1) / 2;
  for (int idx = y; idx < npair; idx += FB_NY) {
    int r = (int)((sqrtf(8.0f * idx + 1.0f) - 1.0f) * 0.5f);
    while (r * (r + 1) / 2 > idx) r--;
    while ((r + 1) * (r + 2) / 2 <= idx) r++;
    int c = idx - r * (r + 1) / 2;
    const int rla = AT(d.efc_la, r), rlb = AT(d.efc_lb, r), cla = AT(d.efc_la, c), clb = AT(d.efc_lb, c);
    const int Lra = rla >= 0 ? m.dof_chainlen[rla] : 0, Lrb = rlb >= 0 ? m.dof_chainlen[rlb] : 0;
    const int Lca = cla >= 0 ? m.dof_chainlen[cla] : 0, Lcb = clb >= 0 ? m.dof_chainlen[clb] : 0;
    const int jr = (rlb >= 0 && rla >= 0) ? Lrb - m.dof_lca[rlb * m.nv + rla] : Lrb;      // slots of chain b below its join with chain a
    const int jc = (clb >= 0 && cla >= 0) ? Lcb - m.dof_lca[clb * m.nv + cla] : Lcb;
    AT(d.efc_A, idx) = zdot_tail(m, d, e, r, rla, Lra, 0, Lra, c, cla, Lca, 0, Lca) + zdot_tail(m, d, e, r, rla, Lra, 0, Lra, c, clb, Lcb, FB_ZCAP, jc)
                     + zdot_tail(m, d, e, r, rlb, Lrb, FB_ZCAP, jr, c, cla, Lca, 0, Lca) + zdot_tail(m, d, e, r, rlb, Lrb, FB_ZCAP, jr, c, clb, Lcb, FB_ZCAP, jc);
  }
}
// aref and b = J qacc_smooth - aref for every row.  J qacc_smooth = Z (D^-1/2 L^-T qfrc_smooth); that vector is
// in shared memory (XS) from the half solve; the chains are walked through dof_anc (no pointer chasing), chain b stops where it
// joins chain a.
FB_DEV void kref(FB_PHASE_ARGS) {
  const float* xs = sh_dyn(sh);
  int n = AT(d.nefc, 0);
  for (int r = y; r < n; r += FB_NY) {
    int ci, frow; float sign;
    RowChains rc = row_chains(m, d, e, r, ci, frow, sign);
    float vel = 0, as = 0; const int la = rc.la, lb = rc.lb;
    if (la >= 0) {
      int adr = m.dof_Madr[la], len = m.dof_chainlen[la];
      for (int t = 0; t < len; t++) { int k = m.dof_anc[adr + t]; vel += EJC(d.efc_J, r, t) * AT(d.qvel, k); as += EJC(d.efc_Z, r, t) * XS(k); }
    }
    if (lb >= 0) {
      int adr = m.dof_Madr[lb], len = m.dof_chainlen[lb] - (la >= 0 ? m.dof_lca[lb * m.nv + la] : 0);      // common ancestors were counted with chain a
      for (int t = 0; t < len; t++) {
        int k = m.dof_anc[adr + t];
        vel += EJC(d.efc_J, r, FB_ZCAP + t) * AT(d.qvel, k); as += EJC(d.efc_Z, r, FB_ZCAP + t) * XS(k);
      }
    }
    float aref = -EFC(d.efc_B, r) * vel - EFC(d.efc_K, r) * EFC(d.efc_imp, r) * (EFC(d.efc_pos, r) - EFC(d.efc_margin, r));
    EFC(d.efc_aref, r) = aref; EFC(d.efc_b, r) = as - aref;
  }
}

// ---------------------------------------------------------------------------------------------
// K3 + K8 transmission and actuation (MuJoCo mj_transmission, mj_fwdActuation)
FB_DEV void kact_p0(FB_PHASE_ARGS) {
  tsolve_stage_issue(m, d, sh, e, y, d.qLD); for (int k = y; k < m.nv; k += FB_NY) AT(d.qfrc_actuator, k) = 0; }
FB_DEV void kact_p1(FB_PHASE_ARGS) {
  const float *gain = PRM(FB_P_ACTUATOR_GAINPRM, m.actuator_gainprm), *bias = PRM(FB_P_ACTUATOR_BIASPRM, m.actuator_biasprm);
  for (int i = y; i < m.nu; i += FB_NY) {
    float ctrl = AT(d.ctrl, i);
    if (MLD(m.actuator_ctrllimited[i])) ctrl = clampf(ctrl, MLD(m.actuator_ctrlrange[2 * i]), MLD(m.actuator_ctrlrange[2 * i + 1]));
    int id = MLD(m.actuator_trnid[i]), tt = MLD(m.actuator_trntype[i]);
    float len = 0, vel = 0;
    if (tt == FB_TRN_JOINT) { len = AT(d.qpos, MLD(m.jnt_qposadr[id])); vel = AT(d.qvel, MLD(m.jnt_dofadr[id])); }
    else if (tt == FB_TRN_TENDON) {
      for (int w = MLD(m.tendon_adr[id]); w < MLD(m.tendon_adr[id]) + MLD(m.tendon_num[id]); w++) { len += MLD(m.wrap_coef[w]) * AT(d.qpos, MLD(m.wrap_qposadr[w])); vel += MLD(m.wrap_coef[w]) * AT(d.qvel, MLD(m.wrap_dofid[w])); }
    }
    float input = ctrl; int aa = MLD(m.actuator_actadr[i]);
    if (aa >= 0) { AT(d.act_dot, aa) = (ctrl - AT(d.act, aa)) / fmaxf(FB_MINVAL, MLD(m.actuator_dynprm[3 * i])); input = AT(d.act, aa); }
    float force = MLD(gain[3 * i]) * input;
    if (MLD(m.actuator_biastype[i]) == 1) force += MLD(bias[3 * i]) + MLD(bias[3 * i + 1]) * len + MLD(bias[3 * i + 2]) * vel;
    if (MLD(m.actuator_forcelimited[i])) force = clampf(force, MLD(m.actuator_forcerange[2 * i]), MLD(m.actuator_forcerange[2 * i + 1]));
    AT(d.actuator_force, i) = force;
    // joint / tendon transmissions touch disjoint dofs (one actuator per joint or tendon in the fly model)
    if (tt == FB_TRN_JOINT) AT(d.qfrc_actuator, MLD(m.jnt_dofadr[id])) += force;
    else if (tt == FB_TRN_TENDON) { for (int w = MLD(m.tendon_adr[id]); w < MLD(m.tendon_adr[id]) + MLD(m.tendon_num[id]); w++) AT(d.qfrc_actuator, MLD(m.wrap_dofid[w])) += MLD(m.wrap_coef[w]) * force; }
  }
}
// adhesion (body transmission): moment = - mean of the contact-normal Jacobians of all detected contacts of the
// body (incl. those inside the gap).  Chains share the root dofs, so this part runs on one thread.
FB_DEV void kact_p2(FB_PHASE_ARGS) {       // force per contact of every adhesion body: -force / (number of its contacts)
  float* xs = sh_dyn(sh);
  int ncon = AT(d.ncon, 0);
  for (int b = y; b < m.nbody; b += FB_NY) {
    int i = m.body_adhesion[b]; float sc = 0;
    if (i >= 0 && ncon > 0) {
      float force = AT(d.actuator_force, i); int cnt = 0;
      if (force != 0.0f) for (int ci = 0; ci < ncon; ci++) { if (m.geom_bodyid[AT(d.con_geom1, ci)] == b || m.geom_bodyid[AT(d.con_geom2, ci)] == b) cnt++; }
      if (cnt > 0) sc = -force / cnt;
    }
    XS(b) = sc;
  }
}
// ... applied along the chains of the two bodies of each such contact; lanes over the dofs (a dof on both chains gets
// +J - J = 0, as in the sequential formulation)
FB_DEV void kact_p2b(FB_PHASE_ARGS) {
  const float* xs = sh_dyn(sh);
  int ncon = AT(d.ncon, 0);
  if (ncon == 0) return;
  for (int k = y; k < m.nv; k += FB_NY) {
    const int se = m.dof_subend[k]; float s = 0;
    for (int ci = 0; ci < ncon; ci++) {
      int b1 = m.geom_bodyid[AT(d.con_geom1, ci)], b2 = m.geom_bodyid[AT(d.con_geom2, ci)];
      float sc = XS(b1) + XS(b2);
      if (sc == 0.0f) continue;
      int l1 = m.body_lastdof[b1], l2 = m.body_lastdof[b2];
      int sgn = ((l2 >= 0 && k <= l2 && l2 <= se) ? 1 : 0) - ((l1 >= 0 && k <= l1 && l1 <= se) ? 1 : 0);
      if (sgn == 0) continue;
      V3 f = v3(CON_F(d.con_frame, ci, 0, 9), CON_F(d.con_frame, ci, 1, 9), CON_F(d.con_frame, ci, 2, 9));
      V3 pos = v3(CON_F(d.con_pos, ci, 0, 3), CON_F(d.con_pos, ci, 1, 3), CON_F(d.con_pos, ci, 2, 3));
      s += sgn * sc * contact_J(m, d, e, f, pos, k);
    }
    if (s != 0.0f) AT(d.qfrc_actuator, k) += s;
  }
}
// qfrc_applied[k] + the dof-k row of J^T xfrc_applied (MuJoCo mj_xfrcAccumulate / mj_applyFT): a body's wrench, force at its CoM
// xipos, reaches the dofs of its ancestor chain, the dofs k with k <= body_lastdof[b] <= dof_subend[k].  Inlined: an out-of-line call
// would take DevModel / DevData by address and copy the kernel parameters to the stack on every launch, null path included.
FB_DEV float applied_force(const DevModel& m, const DevData& d, int e, int k) {
  float s = d.qfrc_applied[(size_t)e * m.nv + k];
  const float* xf = d.xfrc_applied + (size_t)e * m.nbody * 6;
  const int se = m.dof_subend[k];
  const V3 sa = ld3(d.Sang, k, d, e), sl = ld3(d.Slin, k, d, e);
  for (int b = 1; b < m.nbody; b++) {
    const int l = m.body_lastdof[b];
    if (l < k || l > se) continue;
    const float* w = xf + 6 * b;
    if (w[0] == 0.0f && w[1] == 0.0f && w[2] == 0.0f && w[3] == 0.0f && w[4] == 0.0f && w[5] == 0.0f) continue;
    const V3 f = v3(w[0], w[1], w[2]), t = v3(w[3], w[4], w[5]);
    s += dot(f, sl + cross(sa, ld3(d.xipos, b, d, e))) + dot(t, sa);
  }
  return s;
}
FB_DEV void kact_p3(FB_PHASE_ARGS) {
  float* xs = sh_dyn(sh);
  for (int k = y; k < m.nv; k += FB_NY) {
    float s = AT(d.qfrc_passive, k) - AT(d.qfrc_bias, k) + AT(d.qfrc_actuator, k);
    if (d.qfrc_applied) s += applied_force(m, d, e, k);      // uniform over the launch: null unless the handle has applied forces
    AT(d.qfrc_smooth, k) = s; XS(k) = s;
  }
}
// ---------------------------------------------------------------------------------------------
// K11 constraint solve in the dual (force) space.
//
// With a = qacc_smooth + M^-1 J^T lam the primal cost of MuJoCo's Newton solver becomes
//   c(lam) = 1/2 lam^T A lam + s(b + A lam),   A = J M^-1 J^T, b = J qacc_smooth - aref,
// s = the same per-row cost (half-quadratic for limits / frictionless contacts, three-zone elliptic
// cone for frictional contacts).  Newton steps on the primal problem map to
//   dlam = -(I + C A)^-1 (lam - f(lam)),   C = Hessian of s = E E^T,
// solved through the small SPD system G = I + E^T A E (Cholesky), followed by the same exact line
// search.  The minimiser is the one MuJoCo's primal Newton converges to (strictly convex problem).
FB_DEV int qcqp2(float* res, const float* A, const float* b, float d0, float d1, float r) {   // mju_QCQP2
  float A11 = A[0] * d0 * d0, A22 = A[3] * d1 * d1, A12 = A[1] * d0 * d1, b1 = b[0] * d0, b2 = b[1] * d1;
  float la = 0, v1 = 0, v2 = 0;
  for (int it = 0; it < 20; it++) {
    float det = (A11 + la) * (A22 + la) - A12 * A12;
    if (det < 1e-10f) { res[0] = 0; res[1] = 0; return 0; }
    float di = 1 / det, P11 = (A22 + la) * di, P22 = (A11 + la) * di, P12 = -A12 * di;
    v1 = -P11 * b1 - P12 * b2; v2 = -P12 * b1 - P22 * b2;
    float val = v1 * v1 + v2 * v2 - r * r;
    if (val < 1e-10f) break;
    float deriv = -2 * (P11 * v1 * v1 + 2 * P12 * v1 * v2 + P22 * v2 * v2);
    float delta = -val / deriv;
    if (delta < 1e-10f) break;
    la += delta;
  }
  res[0] = v1 * d0; res[1] = v2 * d1;
  return la != 0;
}

// ---------------------------------------------------------------------------------------------
// K12 acceleration-stage sensors + K13 Euler: the "finish" kernel of step2.
//   F1 all lanes : XS <- qfrc_constraint ; ext wrench array cleared
//   F2..F4       : tree solve  XS <- M^-1 J^T f
//   F5 all lanes : qacc = qacc_smooth + XS ; XS <- qfrc_smooth + qfrc_constraint (Euler rhs) ; lane 0: contact wrenches
//   F6 lists     : Euler solve phase a (M + hD factor)       | root: delta-acceleration of the roots
//   F7 lists     : delta-acceleration chains + body forces    | root: Euler solve phase b
//   F8 lists     : subtree force sums ; Euler solve phase c ; integrate
//   F9 all lanes : sensors (accelerometer, force, touch), state check
// The sensor pass reuses the velocity stage: with the bias accelerations a0_b (bacc) and per-body bias forces
// f0_b (bfrc0) of the same state, the full quantities are a_b = a0_b + delta_b, f_b = f0_b + I_b delta_b with
// delta_b = delta_parent + sum_d S_d qacc_d (MuJoCo mj_rnePostConstraint restated).
FB_DEV void kfin_f1(FB_PHASE_ARGS) {
  float* xs = sh_dyn(sh);
  tsolve_stage_issue(m, d, sh, e, y, d.qLD);
  prefetch_rec(d.Sang, FB_V3S * m.nv, d, e, y); prefetch_rec(d.Slin, FB_V3S * m.nv, d, e, y); prefetch_rec(d.inert10, FB_I10S * m.nbody, d, e, y); prefetch_rec(d.bfrc0, FB_S6S * m.nbody, d, e, y);
  if (d.do_integrate) prefetch_rec(d.qLDe, m.nM, d, e, y);   // second factor, staged after the first solve
  for (int i = y; i < m.nv; i += FB_NY) XS(i) = AT(d.qtmp, i) + AT(d.dof_isd, i) * AT(d.qfrc_zf, i);      // D^-1 u + D^-1/2 Z^T f
  for (int k = y; k < FB_S6S * m.nbody; k += FB_NY) AT(d.bfl, k) = 0;
}
FB_WARPFN void kfin_solve(const DevModel& m, const DevData& d, ShTree& sh, int e) {      // qacc = L^-1 (...)
  WPAR_BEGIN tsolve_stage_wait(m, d, sh, e, lane); WPAR_END
  tsolve_c(m, d, sh, e);
}
// Euler with implicit joint damping: qacc' = (M + h D)^-1 (qfrc_smooth + qfrc_constraint), second factor qLDe
FB_WARPFN void kfin_solve_euler(const DevModel& m, const DevData& d, ShTree& sh, int e) { if (d.do_integrate) tri_solve(m, d, sh, e); }
FB_DEV void kfin_f5(FB_PHASE_ARGS) {
  float* xs = sh_dyn(sh);
  if (d.do_integrate) tsolve_stage_issue(m, d, sh, e, y, d.qLDe);      // overlaps the sensor sweeps below
  for (int i = y; i < m.nv; i += FB_NY) { AT(d.qacc, i) = XS(i); XS(i) = AT(d.qfrc_smooth, i) + AT(d.qfrc_constraint, i); }
  if (y != 0) return;
  // external (contact) wrench per body into bfl (about ref)
  int ncon = AT(d.ncon, 0);
  for (int ci = 0; ci < ncon; ci++) {
    int adr = AT(d.con_efcadr, ci); if (adr < 0) continue;
    int dim = AT(d.con_dim, ci);
    V3 F = v3(0, 0, 0);
    for (int r = 0; r < dim; r++) F = F + v3(CON_F(d.con_frame, ci, 3 * r, 9), CON_F(d.con_frame, ci, 3 * r + 1, 9), CON_F(d.con_frame, ci, 3 * r + 2, 9)) * EFC(d.efc_force, adr + r);
    V3 pos = v3(CON_F(d.con_pos, ci, 0, 3), CON_F(d.con_pos, ci, 1, 3), CON_F(d.con_pos, ci, 2, 3));
    V3 tq = cross(pos, F);
    int b1 = m.geom_bodyid[AT(d.con_geom1, ci)], b2 = m.geom_bodyid[AT(d.con_geom2, ci)];
    S6 w2 = ld6(d.bfl, b2, d, e); w2.a = w2.a + tq; w2.l = w2.l + F; st6(d.bfl, b2, d, e, w2);
    S6 w1 = ld6(d.bfl, b1, d, e); w1.a = w1.a - tq; w1.l = w1.l - F; st6(d.bfl, b1, d, e, w1);
  }
}
// delta acceleration of body b from its parent's delta: dl += sum_d S_d qacc_d
FB_DEV void delta_from_parent(const DevModel& m, const DevData& d, int e, int b, S6& dl) {
  for (int kk = 0; kk < m.body_dofnum[b]; kk++) {
    int k = m.body_dofadr[b] + kk; float qa = AT(d.qacc, k);
    dl.a = dl.a + ld3(d.Sang, k, d, e) * qa; dl.l = dl.l + ld3(d.Slin, k, d, e) * qa;
  }
}
FB_DEV void kfin_f6(FB_PHASE_ARGS) {
  if (y == 0) for (int r = 0; r < m.nroot; r++) { int b = m.root_body[r]; S6 dl; dl.a = dl.l = v3(0, 0, 0); delta_from_parent(m, d, e, b, dl); st6(d.bdel, b, d, e, dl); }
}
FB_DEV void kfin_f7(FB_PHASE_ARGS) {
  if (y >= m.nlist) return;
  int prev = -1; S6 cd; cd.a = cd.l = v3(0, 0, 0);
  FB_LIST_LOOP_FWD {
    if (!m.body_sensacc[b]) { prev = -1; continue; }
    int p = m.body_parentid[b];
    if (p != prev) cd = ld6(d.bdel, p, d, e);
    delta_from_parent(m, d, e, b, cd);
    st6(d.bdel, b, d, e, cd);
    prev = b;
    if (m.body_sensfrc[b]) {   // f_b = f0_b + I_b delta_b - ext_b
      I10 I = ld10(d.inert10, b, d, e); V3 L, pm; inert_mul(I, cd.a, cd.l, L, pm);
      S6 f = ld6(d.bfrc0, b, d, e), x = ld6(d.bfl, b, d, e);
      f.a = f.a + L - x.a; f.l = f.l + pm - x.l;
      st6(d.bfrc, b, d, e, f);
    }
  }
}
FB_DEV void integrate_body(const DevModel& m, const DevData& d, int e, const float* xs, int b);
FB_DEV void kfin_f8(FB_PHASE_ARGS) {
  float* xs = sh_dyn(sh);
  if (y < m.nlist) {
    FB_LIST_LOOP_REV {      // cfrc_int of the force-sensor bodies: sums over their subtrees
      if (!m.body_sensfrc[b]) continue;
      int p = m.body_parentid[b];
      if (!m.body_sensfrc[p]) continue;
      S6 f = ld6(d.bfrc, b, d, e), pf = ld6(d.bfrc, p, d, e);
      pf.a = pf.a + f.a; pf.l = pf.l + f.l; st6(d.bfrc, p, d, e, pf);
    }
  }
  if (!d.do_integrate) return;
  if (AT(d.hold, 0)) return;          // env staged for reset: recompute (forward) but do not integrate
  // semi-implicit Euler: the free joints one lane per root (quaternion update), every other dof on its own lane -- walking the lists
  // body by body put a chain of dependent read-modify-writes of qvel / qpos on one lane per list
  if (y < m.nroot) integrate_body(m, d, e, xs, m.root_body[y]);
  if (y == 0) AT(d.time, 0) += m.timestep;
  const float h = m.timestep;
  for (int k = y; k < m.nv; k += FB_NY) {
    const int j = m.dof_jntid[k];
    if (m.jnt_type[j] != FB_JNT_HINGE) continue;          // free and ball joints: integrate_body
    const float v = AT(d.qvel, k) + h * XS(k);
    AT(d.qvel, k) = v; AT(d.qpos, m.jnt_qposadr[j]) += h * v;
  }
}
FB_DEV float ray_quad(float a, float b, float c, float* x) {
  float det = b * b - a * c;
  if (det < 1e-30f) { x[0] = -1; x[1] = -1; return -1; }
  det = sqrtf(det); x[0] = (-b - det) / a; x[1] = (-b + det) / a;
  if (x[0] >= 0) return x[0]; if (x[1] >= 0) return x[1]; return -1;
}
FB_DEV float ray_capsule(V3 pos, const M3& mat, V3 size, V3 pnt, V3 vec) {
  V3 dif = pnt - pos; float xx[2]; float ssz = size.x + size.y;
  if (ray_quad(dot(vec, vec), dot(vec, dif), dot(dif, dif) - ssz * ssz, xx) < 0) return -1;
  V3 lp = mulT(mat, dif), lv = mulT(mat, vec);
  float x = -1;
  float sol = ray_quad(lv.x * lv.x + lv.y * lv.y, lv.x * lp.x + lv.y * lp.y, lp.x * lp.x + lp.y * lp.y - size.x * size.x, xx);
  if (sol >= 0 && fabsf(lp.z + sol * lv.z) <= size.y) { if (x < 0 || sol < x) x = sol; }
  V3 ld = v3(lp.x, lp.y, lp.z - size.y);
  ray_quad(dot(lv, lv), dot(lv, ld), dot(ld, ld) - size.x * size.x, xx);
  for (int i = 0; i < 2; i++) if (xx[i] >= 0 && lp.z + xx[i] * lv.z >= size.y) { if (x < 0 || xx[i] < x) x = xx[i]; }
  ld.z = lp.z + size.y;
  ray_quad(dot(lv, lv), dot(lv, ld), dot(ld, ld) - size.x * size.x, xx);
  for (int i = 0; i < 2; i++) if (xx[i] >= 0 && lp.z + xx[i] * lv.z <= -size.y) { if (x < 0 || xx[i] < x) x = xx[i]; }
  return x;
}
FB_DEV void kfin_f9(FB_PHASE_ARGS) {
  int ncon = AT(d.ncon, 0);
  for (int s = y; s < m.nsensor; s += FB_NY) {
    int tp = m.sensor_type[s], site = m.sensor_objid[s], adr = m.sensor_adr[s], b = m.site_bodyid[site];
    if (tp == FB_SENS_ACCELEROMETER) {
      S6 a = ld6(d.bacc, b, d, e), dl = ld6(d.bdel, b, d, e), v = ld6(d.bvel, b, d, e);
      a.a = a.a + dl.a; a.l = a.l + dl.l;
      V3 p = ld3(d.site_xpos, site, d, e);
      V3 vp = v.l + cross(v.a, p);
      V3 acc = a.l + cross(a.a, p) + cross(v.a, vp);
      V3 out = mulT(ld9(d.site_xmat, site, d, e), acc);
      AT(d.sensordata, adr) = out.x; AT(d.sensordata, adr + 1) = out.y; AT(d.sensordata, adr + 2) = out.z;
    } else if (tp == FB_SENS_FORCE) {
      V3 out = mulT(ld9(d.site_xmat, site, d, e), ld3(d.bfrc, 2 * b + 1, d, e));
      AT(d.sensordata, adr) = out.x; AT(d.sensordata, adr + 1) = out.y; AT(d.sensordata, adr + 2) = out.z;
    } else if (tp == FB_SENS_TOUCH) {
      float sum = 0;
      for (int ci = 0; ci < ncon; ci++) {
        int ea = AT(d.con_efcadr, ci); if (ea < 0) continue;
        int b1 = m.geom_bodyid[AT(d.con_geom1, ci)], b2 = m.geom_bodyid[AT(d.con_geom2, ci)];
        if (b != b1 && b != b2) continue;
        float fn = EFC(d.efc_force, ea); if (fn <= 0) continue;
        V3 ray = v3(CON_F(d.con_frame, ci, 0, 9), CON_F(d.con_frame, ci, 1, 9), CON_F(d.con_frame, ci, 2, 9));
        if (b == b2) ray = ray * -1.0f;
        V3 pos = v3(CON_F(d.con_pos, ci, 0, 3), CON_F(d.con_pos, ci, 1, 3), CON_F(d.con_pos, ci, 2, 3));
        V3 ssz = mld3(m.site_size, site);
        float hit;
        if (m.site_type[site] == FB_GEOM_CAPSULE) hit = ray_capsule(ld3(d.site_xpos, site, d, e), ld9(d.site_xmat, site, d, e), ssz, pos, ray);
        else { float xx[2]; V3 dif = pos - ld3(d.site_xpos, site, d, e); hit = ray_quad(dot(ray, ray), dot(ray, dif), dot(dif, dif) - ssz.x * ssz.x, xx); }
        if (hit >= 0) sum += fn;
      }
      AT(d.sensordata, adr) = sum;
    }
  }
  // state check (|qacc| > 1e14 or non-finite: reference tasks/base.py:222-225): each lane sums its dofs, kfin_f10 adds the lanes up
  float s2 = 0; bool bad = false;
  for (int k = y; k < m.nv; k += FB_NY) { float a = AT(d.qacc, k); s2 += a * a; if (!isfinite(a) || !isfinite(AT(d.qvel, k))) bad = true; }
  sh.red[y] = bad ? INFINITY : s2;
  if (d.do_integrate && !AT(d.hold, 0)) for (int i = y; i < m.na; i += FB_NY) AT(d.act, i) += m.timestep * AT(d.act_dot, i);
}
FB_DEV void kfin_f10(FB_PHASE_ARGS) {
  if (y != 0) return;
  float s2 = 0; for (int l = 0; l < FB_NY; l++) s2 += sh.red[l];
  if (!(s2 < 1e28f)) FB_FLAG_OR(1);
}
// a ball joint: qvel += h qacc, then the quaternion qpos[qa .. qa + 3] turned by the body-frame angular velocity over one step (MuJoCo
// mju_quatIntegrate; the free joint's branch restates it)
FB_DEV void integrate_ball(const DevData& d, int e, const float* xs, int qa, int da, float h) {
  for (int i = 0; i < 3; i++) { AT(d.qvel, da + i) += h * XS(da + i); }
  V3 w = v3(AT(d.qvel, da), AT(d.qvel, da + 1), AT(d.qvel, da + 2));
  float ang = norm(w) * h;
  Q4 q = q4(AT(d.qpos, qa), AT(d.qpos, qa + 1), AT(d.qpos, qa + 2), AT(d.qpos, qa + 3));
  if (ang > 0) q = qmul(q, axisangle(normalized(w), ang));
  q = qnormalize(q);
  AT(d.qpos, qa) = q.w; AT(d.qpos, qa + 1) = q.x; AT(d.qpos, qa + 2) = q.y; AT(d.qpos, qa + 3) = q.z;
}
FB_DEV void integrate_body(const DevModel& m, const DevData& d, int e, const float* xs, int b) {
  float h = m.timestep;
  for (int k = 0; k < m.body_jntnum[b]; k++) {
    int j = m.body_jntadr[b] + k, qa = m.jnt_qposadr[j], da = m.jnt_dofadr[j];
    if (m.jnt_type[j] == FB_JNT_FREE) {
      for (int i = 0; i < 6; i++) { AT(d.qvel, da + i) += h * XS(da + i); }
      for (int i = 0; i < 3; i++) AT(d.qpos, qa + i) += h * AT(d.qvel, da + i);
      V3 w = v3(AT(d.qvel, da + 3), AT(d.qvel, da + 4), AT(d.qvel, da + 5));
      float ang = norm(w) * h;
      Q4 q = q4(AT(d.qpos, qa + 3), AT(d.qpos, qa + 4), AT(d.qpos, qa + 5), AT(d.qpos, qa + 6));
      if (ang > 0) q = qmul(q, axisangle(normalized(w), ang));
      q = qnormalize(q);
      AT(d.qpos, qa + 3) = q.w; AT(d.qpos, qa + 4) = q.x; AT(d.qpos, qa + 5) = q.y; AT(d.qpos, qa + 6) = q.z;
    } else if (m.jnt_type[j] == FB_JNT_BALL) {
      FB_NO_MERGE(); integrate_ball(d, e, xs, qa, da, h); FB_NO_MERGE();
    } else {
      AT(d.qvel, da) += h * XS(da);
      AT(d.qpos, qa) += h * AT(d.qvel, da);
    }
  }
}
// last phase of the velocity kernel: per-substep sensor accumulation (d.sens_mode: 1 first substep, 0 next, -1 off)
FB_DEV void kvel_p4(FB_PHASE_ARGS) {
  if (d.sens_mode < 0) return;
  for (int i = y; i < m.nsensordata; i += FB_NY) AT(d.sensor_sum, i) = (d.sens_mode ? 0.0f : AT(d.sensor_sum, i)) + AT(d.sensordata, i);
}

// ---------------------------------------------------------------------------------------------
// packed per-env observation record (AoS, one row per env) for the host task code / NCCL gather:
//   qpos[nq] qvel[nv] act[na] sensor_mean[nsd] sensordata[nsd] root_xpos[3] root_xmat[9] site_xpos[3*nsite]
//   flags[1] qacc_sq[1] time[1]
FB_DEV void kpack(const DevModel& m, const DevData& d, int e, int y, float inv_nsub) {
  if (e >= d.N) return;
  float* o = d.obs + (size_t)e * d.obs_dim;
  int k = 0;
  for (int i = y; i < m.nq; i += FB_NY) o[k + i] = AT(d.qpos, i);
  k += m.nq;
  for (int i = y; i < m.nv; i += FB_NY) o[k + i] = AT(d.qvel, i);
  k += m.nv;
  for (int i = y; i < m.na; i += FB_NY) o[k + i] = AT(d.act, i);
  k += m.na;
  for (int i = y; i < m.nsensordata; i += FB_NY) { o[k + i] = AT(d.sensor_sum, i) * inv_nsub; o[k + m.nsensordata + i] = AT(d.sensordata, i); }
  k += 2 * m.nsensordata;
  int rb = m.root_body[0];
  if (y < 3) o[k + y] = AT(d.xpos, FB_V3S * rb + y) + AT(d.ref, y);
  k += 3;
  if (y < 9) o[k + y] = AT(d.xmat, FB_M3S * rb + y);
  k += 9;
  for (int i = y; i < 3 * m.nsite; i += FB_NY) o[k + i] = AT(d.site_xpos, FB_V3S * (i / 3) + i % 3) + AT(d.ref, i % 3);
  k += 3 * m.nsite;
  if (y == 0) { o[k] = (float)AT(d.flags, 0); float s2 = 0; for (int i = 0; i < m.nv; i++) { float a = AT(d.qacc, i); s2 += a * a; } o[k + 1] = s2; o[k + 2] = AT(d.time, 0); }
}
// ---------------------------------------------------------------------------------------------
// task observation program: evaluates the reference task's observables (FruitFlyObservables,
// fruitfly.py:585-756; ref_displacement / ref_root_quat, tasks/base.py:245-268) on the device.
FB_DEV void ktaskobs(const DevModel& m, const DevData& d, int e, int y) {
  if (!d.tobs || e >= d.N) return;
  float* o = d.tobs + (size_t)e * d.tobs_dim;
  int rb = d.op_root_body;
  V3 ref = v3(AT(d.ref, 0), AT(d.ref, 1), AT(d.ref, 2));
  V3 rpos = ld3(d.xpos, rb, d, e);
  M3 R = ld9(d.xmat, rb, d, e);
  bool first = d.op_first ? d.op_first[e] != 0 : false;
  float inv = d.op_nsub > 0 ? 1.0f / d.op_nsub : 1.0f;
  int step = d.op_step ? d.op_step[e] : 0;
  int rj = m.body_jntadr[rb], rq = rj >= 0 ? m.jnt_qposadr[rj] : 0;
  const float* rtab = d.op_ref_slot ? d.op_ref + (size_t)e * 7 * d.op_ref_len : d.op_ref;      // the env's own reference snippet, or the shared one
  for (int it = 0; it < d.op_n; it++) {
    int kind = d.op_kind[it], a = d.op_a[it], b = d.op_b[it], k = d.op_off[it];
    switch (kind) {
      case FB_OBS_SENSOR_MEAN: for (int i = y; i < b; i += FB_NY) o[k + i] = first ? AT(d.sensordata, a + i) * inv : AT(d.sensor_sum, a + i) * inv; break;
      case FB_OBS_SENSOR_NOW: for (int i = y; i < b; i += FB_NY) o[k + i] = AT(d.sensordata, a + i); break;
      case FB_OBS_ACT: for (int i = y; i < b; i += FB_NY) o[k + i] = AT(d.act, a + i); break;
      case FB_OBS_QPOS: for (int i = y; i < b; i += FB_NY) o[k + i] = AT(d.qpos, d.op_list[a + i]); break;
      case FB_OBS_QVEL: for (int i = y; i < b; i += FB_NY) o[k + i] = AT(d.qvel, d.op_list[a + i]); break;
      case FB_OBS_SITES_EGO: for (int i = y; i < b; i += FB_NY) { V3 v = mulT(R, ld3(d.site_xpos, d.op_list[a + i], d, e) - rpos); o[k + 3 * i] = v.x; o[k + 3 * i + 1] = v.y; o[k + 3 * i + 2] = v.z; } break;
      case FB_OBS_DOF_AXIS_EGO: for (int i = y; i < b; i += FB_NY) { V3 v = mulT(R, ld3(d.Sang, d.op_list[a + i], d, e)); o[k + 3 * i] = v.x; o[k + 3 * i + 1] = v.y; o[k + 3 * i + 2] = v.z; } break;
      case FB_OBS_ROOT_ZAXIS: if (y < 3) o[k + y] = R.m[6 + y]; break;
      case FB_OBS_REF_DISP: {
        V3 fly = v3(AT(d.qpos, rq), AT(d.qpos, rq + 1), AT(d.qpos, rq + 2));
        for (int i = y; i < b; i += FB_NY) { int t = step + i; if (t > d.op_ref_len - 1) t = d.op_ref_len - 1; const float* rr = rtab + 7 * t;
          V3 v = mulT(R, v3(rr[0], rr[1], rr[2]) - fly); o[k + 3 * i] = v.x; o[k + 3 * i + 1] = v.y; o[k + 3 * i + 2] = v.z; }
      } break;
      case FB_OBS_REF_QUAT: {
        Q4 q = q4(AT(d.qpos, rq + 3), AT(d.qpos, rq + 4), AT(d.qpos, rq + 5), AT(d.qpos, rq + 6));
        float n2 = q.w * q.w + q.x * q.x + q.y * q.y + q.z * q.z; float s = 1.0f / n2;
        Q4 qi = q4(q.w * s, -q.x * s, -q.y * s, -q.z * s);
        for (int i = y; i < b; i += FB_NY) { int t = step + i; if (t > d.op_ref_len - 1) t = d.op_ref_len - 1; const float* rr = rtab + 7 * t;
          Q4 r4 = qmul(qi, q4(rr[3], rr[4], rr[5], rr[6])); o[k + 4 * i] = r4.w; o[k + 4 * i + 1] = r4.x; o[k + 4 * i + 2] = r4.y; o[k + 4 * i + 3] = r4.z; }
      } break;
      case FB_OBS_SCALARS: if (y == 0) { o[k] = (float)AT(d.flags, 0); float s2 = 0; for (int i = 0; i < m.nv; i++) { float x = AT(d.qacc, i); s2 += x * x; } o[k + 1] = s2; o[k + 2] = AT(d.time, 0); } break;
      case FB_OBS_ROOT_POSE: if (y < 3) o[k + y] = comp(rpos + ref, y); else if (y < 7) o[k + y] = AT(d.qpos, rq + y); break;
      case FB_OBS_SUBTREE_COM: if (y < 3) { float mass = AT(d.crb10, FB_I10S * a); o[k + y] = (mass > 0 ? AT(d.crb10, FB_I10S * a + 1 + y) / mass : 0.0f) + AT(d.ref, y); } break;
      case FB_OBS_TASK_TARGET: if (d.task && d.task->target) for (int i = y; i < b; i += FB_NY) o[k + i] = d.task->target[2 * e + i]; break;
      case FB_OBS_WORLD_CONTACT: if (y == 0) { int nc = AT(d.ncon, 0); float hit = 0.0f;
          for (int ci = 0; ci < nc; ci++) if (AT(d.con_efcadr, ci) >= 0 && (m.geom_bodyid[AT(d.con_geom1, ci)] == 0 || m.geom_bodyid[AT(d.con_geom2, ci)] == 0)) hit = 1.0f;
          o[k] = hit; } break;
      default: break;
    }
  }
}
// mj_resetData zeroes qfrc_applied and xfrc_applied: the rows of a resetting env (no-op while the handle has none)
FB_DEV void zero_applied(const DevModel& m, const DevData& d, int e, int y) {
  if (!d.qfrc_applied) return;
  for (int i = y; i < m.nv; i += FB_NY) d.qfrc_applied[(size_t)e * m.nv + i] = 0.0f;
  for (int i = y; i < 6 * m.nbody; i += FB_NY) d.xfrc_applied[(size_t)e * 6 * m.nbody + i] = 0.0f;
}
// partial reset staged by fb_reset / fb_reset_hold: warp w of the launch rewrites env rst_ids[w]
FB_DEV void kreset_scatter(const DevModel& m, const DevData& d, int w, int y) {
  if (w >= d.rst_n) return;
  int e = d.rst_ids[w];
  for (int i = y; i < m.nq; i += FB_NY) AT(d.qpos, i) = d.rst_qpos[(size_t)w * m.nq + i];
  for (int i = y; i < m.nv; i += FB_NY) { AT(d.qvel, i) = d.rst_has_qvel ? d.rst_qvel[(size_t)w * m.nv + i] : 0.0f; AT(d.qacc, i) = 0; }
  for (int i = y; i < m.na; i += FB_NY) AT(d.act, i) = 0;
  for (int i = y; i < m.nu; i += FB_NY) AT(d.ctrl, i) = 0;         // mj_resetData zeroes ctrl (reference: physics.reset() before initialize_episode)
  zero_applied(m, d, e, y);
  if (y == 0) { AT(d.time, 0) = 0; AT(d.flags, 0) = 0; AT(d.hold, 0) = d.rst_hold; AT(d.prev_n, 0) = 0; }
}
FB_DEV void kclear_hold(const DevModel& m, const DevData& d, int e, int y) { if (y == 0) AT(d.hold, 0) = 0; }
// generic column scatter (fb_write_state / fb_set_ctrl): field[idx[c]] of env e <- vals[e][c]
FB_DEV void kscatter(const DevModel& m, const DevData& d, int e, int y) {
  if (e >= d.Np) return;
  const int src = (e >= d.N) ? 0 : e;                  // pad envs mirror env 0
  // an env held for its reset ignores the action of the step() call that resets it (dm_env: the action passed with a reset is
  // dropped), so its FIRST observation is computed with ctrl = 0 whatever the caller sent
  const bool drop = d.sc_field == d.ctrl && AT(d.hold, 0) != 0;
  for (int c = y; c < d.sc_k; c += FB_NY) {
    int t = d.sc_idx ? d.sc_idx[c] : c;
    if (t < 0) continue;                                 // column without a target (e.g. a user action)
    float v = d.sc_vals[(size_t)src * d.sc_k + c];
    if (d.sc_nan0 && !(v == v)) v = 0.0f;                // NaN actions act as 0 (reference tasks/base.py:199)
    if (d.sc_stride) d.sc_field[(size_t)e * d.sc_stride + t] = v;      // compact per-env array (applied forces)
    else AT(d.sc_field, t) = drop ? 0.0f : v;
  }
}
