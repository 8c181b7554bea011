// fb_math.h -- small fp32 vector / quaternion / spatial helpers used by every stage.
#pragma once
#include <math.h>
#include "fb_types.h"

struct V3 { float x, y, z; };
struct Q4 { float w, x, y, z; };
struct M3 { float m[9]; };       // row-major

FB_DEV V3 v3(float x, float y, float z) { V3 r; r.x = x; r.y = y; r.z = z; return r; }
FB_DEV V3 operator+(V3 a, V3 b) { return v3(a.x + b.x, a.y + b.y, a.z + b.z); }
FB_DEV V3 operator-(V3 a, V3 b) { return v3(a.x - b.x, a.y - b.y, a.z - b.z); }
FB_DEV V3 operator*(V3 a, float s) { return v3(a.x * s, a.y * s, a.z * s); }
FB_DEV V3 operator*(float s, V3 a) { return v3(a.x * s, a.y * s, a.z * s); }
FB_DEV float dot(V3 a, V3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
FB_DEV V3 cross(V3 a, V3 b) { return v3(a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x); }
FB_DEV float norm(V3 a) { return sqrtf(dot(a, a)); }
FB_DEV V3 normalized(V3 a) { float n = norm(a); if (n < 1e-30f) return v3(1, 0, 0); float s = 1.0f / n; return a * s; }
FB_DEV float comp(V3 a, int i) { return i == 0 ? a.x : (i == 1 ? a.y : a.z); }

FB_DEV Q4 q4(float w, float x, float y, float z) { Q4 q; q.w = w; q.x = x; q.y = y; q.z = z; return q; }
FB_DEV Q4 qmul(Q4 a, Q4 b) {
  return q4(a.w * b.w - a.x * b.x - a.y * b.y - a.z * b.z, a.w * b.x + a.x * b.w + a.y * b.z - a.z * b.y,
            a.w * b.y - a.x * b.z + a.y * b.w + a.z * b.x, a.w * b.z + a.x * b.y - a.y * b.x + a.z * b.w);
}
FB_DEV Q4 qnormalize(Q4 q) {
  float n = sqrtf(q.w * q.w + q.x * q.x + q.y * q.y + q.z * q.z);
  if (n < 1e-30f) return q4(1, 0, 0, 0);
  float s = 1.0f / n; return q4(q.w * s, q.x * s, q.y * s, q.z * s);
}
FB_DEV M3 q2m(Q4 q) {
  M3 R; float w = q.w, x = q.x, y = q.y, z = q.z;
  R.m[0] = w * w + x * x - y * y - z * z; R.m[1] = 2 * (x * y - w * z); R.m[2] = 2 * (x * z + w * y);
  R.m[3] = 2 * (x * y + w * z); R.m[4] = w * w - x * x + y * y - z * z; R.m[5] = 2 * (y * z - w * x);
  R.m[6] = 2 * (x * z - w * y); R.m[7] = 2 * (y * z + w * x); R.m[8] = w * w - x * x - y * y + z * z;
  return R;
}
FB_DEV V3 mul(const M3& R, V3 v) {
  return v3(R.m[0] * v.x + R.m[1] * v.y + R.m[2] * v.z, R.m[3] * v.x + R.m[4] * v.y + R.m[5] * v.z,
            R.m[6] * v.x + R.m[7] * v.y + R.m[8] * v.z);
}
FB_DEV V3 mulT(const M3& R, V3 v) {
  return v3(R.m[0] * v.x + R.m[3] * v.y + R.m[6] * v.z, R.m[1] * v.x + R.m[4] * v.y + R.m[7] * v.z,
            R.m[2] * v.x + R.m[5] * v.y + R.m[8] * v.z);
}
FB_DEV V3 col(const M3& R, int i) { return v3(R.m[i], R.m[3 + i], R.m[6 + i]); }
FB_DEV Q4 axisangle(V3 axis, float ang) {
  float s, c;
#ifdef __CUDACC__
  sincosf(0.5f * ang, &s, &c);
#else
  s = sinf(0.5f * ang); c = cosf(0.5f * ang);
#endif
  return q4(c, axis.x * s, axis.y * s, axis.z * s);
}
FB_DEV float clampf(float x, float lo, float hi) { return x < lo ? lo : (x > hi ? hi : x); }

// record accessor: slot i of array `arr` of env e (arr = record base + array offset).  32-bit index
// arithmetic: rec * Np stays below 2^32 (checked in fb_create).
#define AT(arr, i) (arr)[(unsigned)e * d.rec + (unsigned)(i)]
// model parameter p (enum FbParam) of env e: its row of the overlay when the handle has one (fb_param_*), else the compiled table.
// One test, uniform over the launch; the element index is the table's.
#define PRM(p, table) (d.prm ? (const float*)d.prm + (unsigned)e * d.prm_stride + (unsigned)d.prm_off[p] : (table))
// ... a scalar one (mjModel.opt), `val` the compiled value
#define PRMS(p, k, val) (d.prm ? d.prm[(unsigned)e * d.prm_stride + (unsigned)d.prm_off[p] + (k)] : (val))

// Record arrays of 3-vectors, quaternions, 3x3 matrices, spatial 6-vectors and 10-parameter inertias are PADDED to multiples of
// four floats (V3 -> 4, M3 -> 12, S6 -> 2 x 4, I10 -> 12) and start on 16-byte boundaries (alloc_data), so that every element is
// read / written with 128-bit accesses: one LDG.128 instead of three or four LDG.32 -- the L1TEX / LSU pipe is the busiest unit of
// the tree kernels (profiles/README.md).  FB_V3S / FB_M3S / FB_S6S / FB_I10S are the element strides for the few direct indexers.
#define FB_V3S 4
#define FB_M3S 12
#define FB_S6S 8
#define FB_I10S 12
#define S6I(b, k) (FB_S6S * (b) + (k) + ((k) >= 3 ? 1 : 0))      // slot of component k (0..5: angular xyz, linear xyz) of body b
#ifdef __CUDACC__
struct __align__(16) F4 { float x, y, z, w; };
FB_DEV F4 ldf4(const float* p) { return *reinterpret_cast<const F4*>(p); }
FB_DEV void stf4(float* p, float x, float y, float z, float w) { F4 v; v.x = x; v.y = y; v.z = z; v.w = w; *reinterpret_cast<F4*>(p) = v; }
#else
struct F4 { float x, y, z, w; };
FB_DEV F4 ldf4(const float* p) { F4 v; v.x = p[0]; v.y = p[1]; v.z = p[2]; v.w = p[3]; return v; }
FB_DEV void stf4(float* p, float x, float y, float z, float w) { p[0] = x; p[1] = y; p[2] = z; p[3] = w; }
#endif
FB_DEV V3 ld3(const float* arr, int i, const DevData& d, int e) { F4 v = ldf4(&AT(arr, FB_V3S * i)); return v3(v.x, v.y, v.z); }
FB_DEV void st3(float* arr, int i, const DevData& d, int e, V3 v) { stf4(&AT(arr, FB_V3S * i), v.x, v.y, v.z, 0.0f); }
FB_DEV Q4 ld4(const float* arr, int i, const DevData& d, int e) { F4 v = ldf4(&AT(arr, 4 * i)); return q4(v.x, v.y, v.z, v.w); }
FB_DEV void st4(float* arr, int i, const DevData& d, int e, Q4 q) { stf4(&AT(arr, 4 * i), q.w, q.x, q.y, q.z); }
FB_DEV M3 ld9(const float* arr, int i, const DevData& d, int e) {
  const float* p = &AT(arr, FB_M3S * i); F4 a = ldf4(p), b = ldf4(p + 4), c = ldf4(p + 8); M3 R;
  R.m[0] = a.x; R.m[1] = a.y; R.m[2] = a.z; R.m[3] = a.w; R.m[4] = b.x; R.m[5] = b.y; R.m[6] = b.z; R.m[7] = b.w; R.m[8] = c.x; return R;
}
FB_DEV void st9(float* arr, int i, const DevData& d, int e, const M3& R) {
  float* p = &AT(arr, FB_M3S * i);
  stf4(p, R.m[0], R.m[1], R.m[2], R.m[3]); stf4(p + 4, R.m[4], R.m[5], R.m[6], R.m[7]); stf4(p + 8, R.m[8], 0.0f, 0.0f, 0.0f);
}
// model tables of 3-vectors are uploaded padded to four floats (build_model: upf3), quaternion tables are four wide anyway
// (no kernel writes a model table: the read-only path lets the compiler move these loads above stores to the record)
#ifdef __CUDACC__
#define MLD(x) __ldg(&(x))
#else
#define MLD(x) (x)
#endif
#ifdef __CUDACC__
FB_DEV V3 mld3(const float* a, int i) { const float4 v = __ldg(reinterpret_cast<const float4*>(a + 4 * i)); return v3(v.x, v.y, v.z); }
FB_DEV Q4 mld4(const float* a, int i) { const float4 v = __ldg(reinterpret_cast<const float4*>(a + 4 * i)); return q4(v.x, v.y, v.z, v.w); }
#else
FB_DEV V3 mld3(const float* a, int i) { F4 v = ldf4(a + 4 * i); return v3(v.x, v.y, v.z); }
FB_DEV Q4 mld4(const float* a, int i) { F4 v = ldf4(a + 4 * i); return q4(v.x, v.y, v.z, v.w); }
#endif

// 10-parameter spatial inertia about the reference point: m, h[3], Ixx Iyy Izz Ixy Ixz Iyz
struct I10 { float v[10]; };
FB_DEV void inert_mul(const I10& I, V3 w, V3 v, V3& L, V3& p) {
  V3 h = v3(I.v[1], I.v[2], I.v[3]);
  V3 hv = cross(h, v), wh = cross(w, h);
  L = v3(I.v[4] * w.x + I.v[7] * w.y + I.v[8] * w.z + hv.x, I.v[7] * w.x + I.v[5] * w.y + I.v[9] * w.z + hv.y,
         I.v[8] * w.x + I.v[9] * w.y + I.v[6] * w.z + hv.z);
  p = v3(I.v[0] * v.x + wh.x, I.v[0] * v.y + wh.y, I.v[0] * v.z + wh.z);
}
FB_DEV I10 ld10(const float* arr, int b, const DevData& d, int e) {
  const float* p = &AT(arr, FB_I10S * b); F4 a = ldf4(p), q = ldf4(p + 4), c = ldf4(p + 8); I10 I;
  I.v[0] = a.x; I.v[1] = a.y; I.v[2] = a.z; I.v[3] = a.w; I.v[4] = q.x; I.v[5] = q.y; I.v[6] = q.z; I.v[7] = q.w; I.v[8] = c.x; I.v[9] = c.y; return I;
}
FB_DEV void st10(float* arr, int b, const DevData& d, int e, const float* v) {
  float* p = &AT(arr, FB_I10S * b);
  stf4(p, v[0], v[1], v[2], v[3]); stf4(p + 4, v[4], v[5], v[6], v[7]); stf4(p + 8, v[8], v[9], 0.0f, 0.0f);
}

// spatial 6-vector [angular; linear]
struct S6 { V3 a, l; };
FB_DEV S6 ld6(const float* arr, int b, const DevData& d, int e) { S6 s; s.a = ld3(arr, 2 * b, d, e); s.l = ld3(arr, 2 * b + 1, d, e); return s; }
FB_DEV void st6(float* arr, int b, const DevData& d, int e, const S6& s) { st3(arr, 2 * b, d, e, s.a); st3(arr, 2 * b + 1, d, e, s.l); }

// L2 prefetch of a record array (one request per 128-byte line, lanes take consecutive lines): used in the first phase of
// a kernel for arrays it will read later through dependent, scattered loads
FB_DEV void prefetch_l2(const void* p) {
#ifdef __CUDACC__
  asm volatile("prefetch.global.L2 [%0];" ::"l"(p));
#else
  (void)p;
#endif
}
FB_DEV void prefetch_rec(const float* arr, int n, const DevData& d, int e, int y) {
  for (int k = 32 * y; k < n; k += 32 * FB_NY) prefetch_l2(&AT(arr, k));
}
