// fb_hfield.h -- convex geom against a heightfield (MuJoCo mjc_ConvexHField, engine_collision_convex.c; restated from memory).
// The heightfield stage of the step (fb_hf_kernel / fb_hf_kernel_ids, models with a terrain geom: the `vision` variant) calls
// col_convex_hfield through khf_narrow; the test hook fb_emu_convex_hfield runs it alone.  Both are held against the fp64 CPU
// restatement (`orc_convex_hfield`) prism by prism and contact by contact in tests/test_hfield_gates.py.
//
// In the heightfield's frame the grid cells under the geom's bounding box are walked row by row as a triangle strip; every
// triangle tops a prism that reaches down to the base, its top raised by the margin; each prism goes through MPR against the
// geom (prism support = the farthest of its six vertices, prism centre = their mean).  The MPR loops are a copy of
// fb_constraint.h: mpr_penetration with the first object's support replaced -- kept separate so that the code generated for the
// walking / flight step kernels does not depend on this file.
#pragma once
#include "fb_constraint.h"

struct HfPrism { D3 v[6]; };
FB_DEV MprPt hf_support(const HfPrism& pr, const MprObj& g, D3 dir) {
  MprPt p; int best = 0; float bd = ddot(pr.v[0], dir);
#pragma unroll
  for (int k = 1; k < 6; k++) { float dd = ddot(pr.v[k], dir); if (dd > bd) { bd = dd; best = k; } }
  p.v1 = pr.v[best]; p.v2 = mpr_support1(g, d3(0, 0, 0) - dir); p.v = p.v1 - p.v2; return p;
}
FB_DEVN int hf_mpr_penetration(const HfPrism& o1, D3 c1, const MprObj& o2, float tol, int max_iter, float& depth, D3& pdir, D3& pos) {
  D3 p1[4], v0, v1, v2, v3, dir; float dt; MprPt n;
  v2 = v3 = d3(0, 0, 0); p1[2] = p1[3] = d3(0, 0, 0);
  p1[0] = c1; v0 = c1 - o2.pos;
  if (mpr_eq(v0.x, 0) && mpr_eq(v0.y, 0) && mpr_eq(v0.z, 0)) v0 = d3(MPR_EPS * 10, 0, 0);
  dir = dnormalized(d3(0, 0, 0) - v0);
  n = hf_support(o1, o2, dir); v1 = n.v; p1[1] = n.v1;
  dt = ddot(v1, dir);
  if (mpr_zero(dt) || dt < 0) return -1;
  dir = dcross(v0, v1);
  int res = 0;
  if (mpr_zero(ddot(dir, dir))) res = (mpr_eq(v1.x, 0) && mpr_eq(v1.y, 0) && mpr_eq(v1.z, 0)) ? 1 : 2;
  if (res == 1) { depth = 0; pdir = d3(0, 0, 0); pos = (p1[1] + p1[1] - v1) * 0.5; return 0; }
  if (res == 2) { pos = (p1[1] + p1[1] - v1) * 0.5; depth = dnorm(v1); pdir = dnormalized(v1); return 0; }
  dir = dnormalized(dir);
  n = hf_support(o1, o2, dir); v2 = n.v; p1[2] = n.v1;
  dt = ddot(v2, dir);
  if (mpr_zero(dt) || dt < 0) return -1;
  dir = dnormalized(dcross(v1 - v0, v2 - v0));
  if (ddot(dir, v0) > 0) { D3 tv = v1; v1 = v2; v2 = tv; tv = p1[1]; p1[1] = p1[2]; p1[2] = tv; dir = d3(0, 0, 0) - dir; }
  for (int guard = 0;; guard++) {                // discoverPortal
    n = hf_support(o1, o2, dir); v3 = n.v; p1[3] = n.v1;
    dt = ddot(v3, dir);
    if (mpr_zero(dt) || dt < 0) return -1;
    dt = ddot(dcross(v1, v3), v0);
    const bool r2 = dt < 0 && !mpr_zero(dt);
    dt = ddot(dcross(v3, v2), v0);
    const bool r1 = !r2 && dt < 0 && !mpr_zero(dt);
    if (!(r1 || r2)) break;
    v2 = dsel(r2, v3, v2); v1 = dsel(r1, v3, v1); p1[r2 ? 2 : 1] = p1[3];
    dir = dnormalized(dcross(v1 - v0, v2 - v0));
    if (guard > 1000) return -1;
  }
  for (int guard = 0;; guard++) {                // refinePortal
    dir = mpr_portal_dir3(v1, v2, v3);
    dt = ddot(dir, v1);
    if (mpr_zero(dt) || dt > 0) break;
    n = hf_support(o1, o2, dir);
    dt = ddot(n.v, dir);
    if (!(mpr_zero(dt) || dt > 0) || mpr_reach_tol3(v1, v2, v3, n.v, dir, tol) || guard > 1000) return -1;
    MPR_EXPAND()
  }
  for (int it = 0;; it++) {                      // findPenetr
    dir = mpr_portal_dir3(v1, v2, v3);
    n = hf_support(o1, o2, dir);
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
      pos = ((c1 + o2.pos) * b0 + (p1[1] + p1[1] - v1) * b1 + (p1[2] + p1[2] - v2) * b2 + (p1[3] + p1[3] - v3) * b3) * inv;
      return 0;
    }
    MPR_EXPAND()
  }
}
// contacts of one geom with the heightfield, in world coordinates; returns their number (<= max).  prism (optional, the tests'
// hook): per contact the triangle it came from, (row * ncol + column) * 2 + i, the triangle completed at strip vertex (column, row + i)
struct HfCon { float dist; V3 pos, n; };
FB_DEV int col_convex_hfield(HfCon* out, int max, float margin, int type, V3 gp, const M3& gm, V3 gs,
                             V3 hp, const M3& hm, const float* hf_size, int nrow, int ncol, const float* data, int* prism = nullptr) {
  // the geom in the heightfield's frame, origin shifted to the geom's footprint for fp32 resolution
  const V3 rel = mulT(hm, gp - hp);
  MprObj g; g.size = d3(gs.x, gs.y, gs.z); g.type = type; g.margin = 0;
  for (int c = 0; c < 3; c++) { V3 col = mulT(hm, v3(gm.m[c], gm.m[3 + c], gm.m[6 + c])); g.mat[c] = col.x; g.mat[3 + c] = col.y; g.mat[6 + c] = col.z; }
  mpr_obj_coefs(g);
  g.pos = d3(0, 0, 0);
  D3 lo, hi;
  { D3 p = mpr_support1(g, d3(1, 0, 0)); hi.x = p.x; p = mpr_support1(g, d3(-1, 0, 0)); lo.x = p.x;
    p = mpr_support1(g, d3(0, 1, 0)); hi.y = p.y; p = mpr_support1(g, d3(0, -1, 0)); lo.y = p.y;
    p = mpr_support1(g, d3(0, 0, 1)); hi.z = p.z; p = mpr_support1(g, d3(0, 0, -1)); lo.z = p.z; }
  const float sx = hf_size[0], sy = hf_size[1];
  if (lo.x + rel.x > sx || hi.x + rel.x < -sx || lo.y + rel.y > sy || hi.y + rel.y < -sy || lo.z + rel.z > hf_size[2] + margin || hi.z + rel.z < -hf_size[3]) return 0;
  int cmin = (int)floorf((lo.x + rel.x + sx) / (2 * sx) * (ncol - 1)), cmax = (int)ceilf((hi.x + rel.x + sx) / (2 * sx) * (ncol - 1));
  int rmin = (int)floorf((lo.y + rel.y + sy) / (2 * sy) * (nrow - 1)), rmax = (int)ceilf((hi.y + rel.y + sy) / (2 * sy) * (nrow - 1));
  cmin = cmin < 0 ? 0 : cmin; rmin = rmin < 0 ? 0 : rmin; cmax = cmax > ncol - 1 ? ncol - 1 : cmax; rmax = rmax > nrow - 1 ? nrow - 1 : rmax;
  const float dx = 2 * sx / (ncol - 1), dy = 2 * sy / (nrow - 1);
  int cnt = 0;
  for (int r = rmin; r < rmax; r++) {
    HfPrism pr; int nvert = 0;
    for (int k = 0; k < 6; k++) pr.v[k] = d3(0, 0, 0);
    for (int c = cmin; c <= cmax; c++) for (int i = 0; i < 2; i++) {
      pr.v[0] = pr.v[1]; pr.v[1] = pr.v[2]; pr.v[3] = pr.v[4]; pr.v[4] = pr.v[5];
      const float x = dx * c - sx - rel.x, y = dy * (r + i) - sy - rel.y;            // relative to the geom centre
      pr.v[2] = d3(x, y, -hf_size[3] - rel.z);
      pr.v[5] = d3(x, y, data[(size_t)(r + i) * ncol + c] * hf_size[2] + margin - rel.z);
      if (++nvert < 3) continue;
      if (pr.v[3].z < lo.z && pr.v[4].z < lo.z && pr.v[5].z < lo.z) continue;        // the geom is above this prism
      D3 ctr = (pr.v[0] + pr.v[1] + pr.v[2] + pr.v[3] + pr.v[4] + pr.v[5]) * (float)(1.0 / 6.0);
      float depth; D3 dir, cp;
      if (hf_mpr_penetration(pr, ctr, g, (float)1e-6, 50, depth, dir, cp) != 0) continue;
      if (mpr_eq(dir.x, 0) && mpr_eq(dir.y, 0) && mpr_eq(dir.z, 0)) continue;
      HfCon& o = out[cnt];
      o.dist = (float)(margin - depth);
      o.pos = mul(hm, v3((float)cp.x, (float)cp.y, (float)cp.z) + rel) + hp;
      o.n = mul(hm, v3((float)dir.x, (float)dir.y, (float)dir.z));
      if (prism) prism[cnt] = (r * ncol + c) * 2 + i;
      if (++cnt >= max) return cnt;
    }
  }
  return cnt;
}

// ---------------------------------------------------------------------------------------------
// Heightfield contacts of one env, appended to the contact list after the collision kernel (fb_hfield_collision).  Runs as
// its own launch between `col` and `proj`, and only for models that carry a heightfield: the step kernels of the other
// models are untouched.  Phase 0: lane l takes the pairs l, l + 32, ... (terrain, geom): bounding-sphere test against the
// highest point under the geom's footprint, then the prism walk; up to FB_HF_PER_GEOM contacts per geom go to the staging
// slots 4 k + i of pair k (free again after the collision kernel's compaction), and the first unused slot of the four is marked
// with geom id -1.  Phase 1: lane 0 appends them in pair order, each pair up to its mark.  The staging record holds the 4 slots
// of all FB_MAXCAND pairs and nothing else, so every npair the ABI accepts keeps its contacts apart.
#define FB_HF_PER_GEOM 4
struct DevHf { int geom, nrow, ncol, npair; float size[4]; const int* pair_geom; const float* data; const float* hmax; };
FB_DEV void khf_narrow(const DevModel& m, const DevData& d, const DevHf& p, int e, int y) {
  // (geom positions are stored relative to the env's reference point, like every spatial quantity of the step: only
  // differences enter the test, and the contact positions come out in the same relative coordinates)
  const V3 hp = ld3(d.geom_xpos, p.geom, d, e); const M3 hm = ld9(d.geom_xmat, p.geom, d, e);
  const float* data = p.data + (size_t)e * p.nrow * p.ncol;
  for (int k = y; k < p.npair; k += FB_NY) {
    const int g = p.pair_geom[k];
    const V3 gp = ld3(d.geom_xpos, g, d, e);
    const float margin = fmaxf(m.geom_margin[p.geom], m.geom_margin[g]);
    int n = 0;
    // bounding sphere against the highest grid point under its footprint (the arena's rim rises to "horizon mountains" of 4-5
    // length units, so the terrain-wide maximum would never reject a fly cruising at 0.5-0.8).  The test runs in the terrain's
    // frame, as the prism walk does: the sphere is the same in every frame, only its centre is carried over.
    const float rb = m.geom_rbound[g] + margin;
    const V3 rel = mulT(hm, gp - hp);
    bool near = rel.z - rb <= p.hmax[e] * p.size[2];
    if (near) {
      const float fx0 = (rel.x - rb + p.size[0]) / (2 * p.size[0]) * (p.ncol - 1), fx1 = (rel.x + rb + p.size[0]) / (2 * p.size[0]) * (p.ncol - 1);
      const float fy0 = (rel.y - rb + p.size[1]) / (2 * p.size[1]) * (p.nrow - 1), fy1 = (rel.y + rb + p.size[1]) / (2 * p.size[1]) * (p.nrow - 1);
      int c0 = (int)floorf(fx0), c1 = (int)ceilf(fx1), r0 = (int)floorf(fy0), r1 = (int)ceilf(fy1);
      if (c1 < 0 || r1 < 0 || c0 > p.ncol - 1 || r0 > p.nrow - 1) near = false;            // beside the terrain
      else {
        c0 = c0 < 0 ? 0 : c0; r0 = r0 < 0 ? 0 : r0; c1 = c1 > p.ncol - 1 ? p.ncol - 1 : c1; r1 = r1 > p.nrow - 1 ? p.nrow - 1 : r1;
        float top = 0.0f;
        if ((c1 - c0 + 1) * (r1 - r0 + 1) <= 64) { for (int r = r0; r <= r1; r++) for (int c = c0; c <= c1; c++) top = fmaxf(top, data[(size_t)r * p.ncol + c]); }
        else top = p.hmax[e];
        near = rel.z - rb <= top * p.size[2];
      }
    }
    if (near) {
      HfCon c[FB_HF_PER_GEOM]; RawCon rc[FB_HF_PER_GEOM];
      n = col_convex_hfield(c, FB_HF_PER_GEOM, margin, m.geom_type[g], gp, ld9(d.geom_xmat, g, d, e), mld3(m.geom_size, g), hp, hm, p.size, p.nrow, p.ncol, data);
      for (int i = 0; i < n; i++) { rc[i].dist = c[i].dist; rc[i].pos = c[i].pos; rc[i].n = c[i].n; rc[i].t = v3(0, 0, 0); }
      col_store(m, d, e, k, rc, n, p.geom, g);
    }
    if (n < FB_HF_PER_GEOM) AT(d.tmp_geom, 2 * (FB_HF_PER_GEOM * k + n)) = -1;
  }
}
FB_DEV void khf_append(const DevModel& m, const DevData& d, const DevHf& p, int e, int y) {
  if (y != 0) return;
  int dst = AT(d.ncon, 0);
  for (int k = 0; k < p.npair; k++) {
    for (int i = 0; i < FB_HF_PER_GEOM; i++, dst++) {
      const int src = FB_HF_PER_GEOM * k + i;
      if (AT(d.tmp_geom, 2 * src) < 0) break;
      if (dst >= FB_MAXCON) { FB_FLAG_OR(2); AT(d.ncon, 0) = FB_MAXCON; return; }
      AT(d.con_dist, dst) = CON_F(d.tmp_con, src, 0, 13);
      for (int c = 0; c < 3; c++) CON_F(d.con_pos, dst, c, 3) = CON_F(d.tmp_con, src, 1 + c, 13);
      for (int c = 0; c < 9; c++) CON_F(d.con_frame, dst, c, 9) = CON_F(d.tmp_con, src, 4 + c, 13);
      AT(d.con_geom1, dst) = AT(d.tmp_geom, 2 * src); AT(d.con_geom2, dst) = AT(d.tmp_geom, 2 * src + 1);
    }
  }
  AT(d.ncon, 0) = dst;
}
