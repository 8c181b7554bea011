// fb_solver_reg.h -- K11 constraint solve for nefc <= 32: ONE ROW PER LANE, row state in registers.
//
// Same mathematics as ksolve_impl (fb_solver.h: dual Newton on the constraint forces, exact line search, noslip,
// force gather); what changes is where the data lives.  Lane r owns row r: its constants (D, b, R, friction), its
// work values (lam, jar, f, residual, search direction ...) are registers; vectors are "read" with warp shuffles.
// Shared memory only holds what is indexed irregularly: the Delassus matrix A as a full 32 x 33 array (row stride 33:
// lane r reading A[r][j] for a common j is bank-conflict free), the Hessian block G (up to FB_CHOL_REG columns: larger
// blocks are rare and are assembled and factorised in the env's record, efc_G) with its right-hand sides, and mirrors of
// E / u for the Hessian assembly.  Matrix-vector products cost one shuffle, one shared load and one FMA
// per element instead of a packed-index computation and two shared loads.
//
// Host emulation (-DFB_EMU): a lane register is an array over the 32 lanes and a shuffle is an indexed read.  WPAR
// sections run lane after lane there, so a value that is shuffled must have been written in an EARLIER section
// (or, for reads from lower lanes only, earlier in the same one).
#pragma once
#include "fb_solver.h"

#define A_(r, c) A[(r) * 33 + (c)]
#define GP(p, q) G[TRI(p, q)]                    // p >= q
#ifndef FB_CHOL_REG
#define FB_CHOL_REG 24                           // Hessian blocks up to this size are factorised in registers (steady-state walk: 8 - 23 columns)
#endif
// one warp's slice: A, G of up to FB_CHOL_REG columns, P XQ XO E0s E1s Us ECR ECK.  6448 bytes: 4 warps + the 1 KB the system
// reserves per CTA fit 8 CTAs on an sm_90 SM (228 KB; tests/test_smem_budget.py)
#define FB_SOLVE_WARP_FLOATS (32 * 33 + TRI(FB_CHOL_REG, 0) + 8 * 32)
#ifdef __CUDACC__
#define FB_RSQRT(x) rsqrtf(x)
#else
#define FB_RSQRT(x) (1.0f / sqrtf(x))
#endif

// forces / cost / Hessian factors of the rows headed by one lane: a plain row (kind 0) or the normal row of an elliptic
// contact (kind 1) with its two friction rows (values j1, j2, D1, D2 of lanes +1, +2)
struct RegHead { float f0, f1, f2, cost, e0, e01, e02, e11, e12; int st, stt; };
FB_DEV void reg_head(int kind, float jar, float j1, float j2, float D, float D1, float D2, float mu, float c1, float c2, RegHead& o) {
  o.f0 = o.f1 = o.f2 = o.cost = o.e0 = o.e01 = o.e02 = o.e11 = o.e12 = 0; o.st = 0; o.stt = 0;
  if (kind == 0) {
    if (jar < 0) { o.f0 = -D * jar; o.cost = 0.5f * D * jar * jar; o.st = 1; o.e0 = sqrtf(D); }
    return;
  }
  float U0 = jar * mu, U1 = j1 * c1, U2 = j2 * c2, N = U0, T = sqrtf(U1 * U1 + U2 * U2);
  if (mu * N + T <= 0 || (T <= 0 && N < 0)) {             // bottom zone: quadratic, three independent columns
    o.f0 = -D * jar; o.f1 = -D1 * j1; o.f2 = -D2 * j2;
    o.cost = 0.5f * (D * jar * jar + D1 * j1 * j1 + D2 * j2 * j2);
    o.st = 1; o.stt = 1; o.e0 = sqrtf(D); o.e01 = sqrtf(D1); o.e02 = sqrtf(D2);
  } else if (N >= mu * T || (T <= 0 && N >= 0)) {          // top zone: satisfied
  } else {                                                  // middle zone: cone, two columns shared by the three rows
    float Dm = D / (mu * mu * (1 + mu * mu)), NmT = N - mu * T;
    o.cost = 0.5f * Dm * NmT * NmT;
    float f0 = -Dm * NmT * mu;
    o.f0 = f0; o.f1 = -f0 / T * U1 * c1; o.f2 = -f0 / T * U2 * c2;
    float sD = sqrtf(Dm), k2 = sqrtf(fmaxf(0.0f, Dm * (-NmT) * mu / T));
    o.st = 2; o.stt = 3;
    o.e0 = sD * mu; o.e01 = -sD * c1 * mu * U1 / T; o.e02 = -sD * c2 * mu * U2 / T;
    o.e11 = -k2 * c1 * U2 / T; o.e12 = k2 * c2 * U1 / T;
  }
}
// line-search contribution (value, slope, curvature) of the rows headed by one lane at step alpha
FB_DEV void reg_head_ls(int kind, float alpha, float jar, float jv, float ja1, float jv1, float ja2, float jv2, float D, float D1, float D2,
                        float mu, float c1, float c2, float& c, float& g, float& h) {
  float x = jar + alpha * jv;
  if (kind == 0) { if (x < 0) { c += 0.5f * D * x * x; g += D * x * jv; h += D * jv * jv; } return; }
  float x1 = ja1 + alpha * jv1, x2 = ja2 + alpha * jv2;
  float U0 = x * mu, U1 = x1 * c1, U2 = x2 * c2, dU0 = jv * mu, dU1 = jv1 * c1, dU2 = jv2 * c2;
  float N = U0, T = sqrtf(U1 * U1 + U2 * U2);
  if (mu * N + T <= 0 || (T <= 0 && N < 0)) {
    c += 0.5f * (D * x * x + D1 * x1 * x1 + D2 * x2 * x2); g += D * x * jv + D1 * x1 * jv1 + D2 * x2 * jv2;
    h += D * jv * jv + D1 * jv1 * jv1 + D2 * jv2 * jv2;
  } else if (N >= mu * T || (T <= 0 && N >= 0)) {
  } else {
    float Dm = D / (mu * mu * (1 + mu * mu)), f = N - mu * T;
    float dT = (U1 * dU1 + U2 * dU2) / T, ddT = (dU1 * dU1 + dU2 * dU2 - dT * dT) / T;
    float fp = dU0 - mu * dT, fpp = -mu * ddT;
    c += 0.5f * Dm * f * f; g += Dm * f * fp; h += Dm * (fp * fp + f * fpp);
  }
}

// p = E^T u ; G = I + E^T A E (packed lower triangle, nc columns) -- one lane's share
FB_DEV void reg_assemble(const float* A, const float* E0s, const float* E1s, const float* Us, const int* ECR, const int* ECK,
                         float* P, float* G, int nc, int lane) {
  NOUNROLL for (int p = lane; p < nc; p += 32) {
    int rp = ECR[p], kd = ECK[p], np = kd == 0 ? 1 : 3; const float* Ep = kd == 2 ? E1s : E0s;
    float pv = 0; NOUNROLL for (int a = 0; a < np; a++) pv += Ep[rp + a] * Us[rp + a];
    P[p] = pv;
  }
  const int npairs = nc * (nc + 1) / 2;
  NOUNROLL for (int t = lane; t < npairs; t += 32) {
    int p = (int)((sqrtf(8.0f * t + 1.0f) - 1.0f) * 0.5f);
    while ((p + 1) * (p + 2) / 2 <= t) p++;
    while (p * (p + 1) / 2 > t) p--;
    int q = t - p * (p + 1) / 2;
    int rp = ECR[p], np = ECK[p] == 0 ? 1 : 3, rq = ECR[q], nq = ECK[q] == 0 ? 1 : 3;
    const float* Ep = ECK[p] == 2 ? E1s : E0s; const float* Eq = ECK[q] == 2 ? E1s : E0s;
    float s = (p == q) ? 1.0f : 0.0f;
    NOUNROLL for (int a = 0; a < np; a++) { float va = Ep[rp + a]; if (va == 0.0f) continue; NOUNROLL for (int bb = 0; bb < nq; bb++) s += va * A_(rp + a, rq + bb) * Eq[rq + bb]; }
    GP(p, q) = s;
  }
}
// out = sum_j A[lane][j] * x[j]   (x: lane register written in an earlier section)
#define REG_MATVEC(out, xname) { float s_ = 0; _Pragma("unroll 4") for (int j = 0; j < n; j++) s_ += A_(lane, j) * SHF(xname, j); out = lane < n ? s_ : 0.0f; }
// evaluate the rows headed by this lane from the current jar; tails take their values from the head (lanes -1 / -2)
#define REG_HEADS(costvar, build)                                                                                     \
  WPAR_BEGIN { L(j1) = SHF(jar, lane + 1); L(j2) = SHF(jar, lane + 2); } WPAR_END                                       \
  WPAR_BEGIN { RegHead o; float cc_ = 0;                                                                              \
      if (L(kind) <= 1) { reg_head(L(kind), L(jar), L(j1), L(j2), L(D), L(D1), L(D2), L(mu), L(c1), L(c2), o); cc_ = o.cost;   \
        L(f) = o.f0; L(hf1) = o.f1; L(hf2) = o.f2;                                                                    \
        if (build) { L(state) = o.st; L(e0) = o.e0; L(e1) = 0; L(hst) = o.stt; L(he01) = o.e01; L(he02) = o.e02; L(he11) = o.e11; L(he12) = o.e12; } }   \
      WSUM_PUT(costvar, cc_); } WPAR_END                                                                              \
  WPAR_BEGIN { float a1 = SHF(hf1, lane - 1), a2 = SHF(hf2, lane - 2);                                               \
      if (L(kind) == 2) L(f) = a1; else if (L(kind) == 3) L(f) = a2;                                                  \
      if (build) { int s1 = SHF(hst, lane - 1), s2 = SHF(hst, lane - 2);                                              \
        float x1 = SHF(he01, lane - 1), x2 = SHF(he02, lane - 2), y1 = SHF(he11, lane - 1), y2 = SHF(he12, lane - 2); \
        if (L(kind) == 2) { L(state) = s1; L(e0) = x1; L(e1) = y1; } else if (L(kind) == 3) { L(state) = s2; L(e0) = x2; L(e1) = y2; } } } WPAR_END

FB_WARPFN void ksolve_reg(const DevModel& m, const DevData& d, float* wsm, int e, int n) {
  const float scale = 1.0f / (m.meaninertia * (m.nv > 1 ? m.nv : 1));
  float* A = wsm; float* G = A + 32 * 33; float* P = G + TRI(FB_CHOL_REG, 0); float* XQ = P + 32; float* XO = XQ + 32;
  float* E0s = XO + 32; float* E1s = E0s + 32; float* Us = E1s + 32;
  int* ECR = reinterpret_cast<int*>(Us + 32); int* ECK = ECR + 32;
  [[maybe_unused]] SolveMem sm; sm.v = nullptr; sm.A = nullptr; sm.G = nullptr; sm.cap = 32; sm.red = nullptr;
#ifndef __CUDACC__
  float red_[4 * 32]; sm.red = red_;                // WSUM staging of the host emulation (warp shuffles on the GPU)
#endif
  float tot[4] = {0, 0, 0, 0}; (void)tot;
  LREG(float, D); LREG(float, D1); LREG(float, D2); LREG(float, b); LREG(float, Rr); LREG(float, mu); LREG(float, c1); LREG(float, c2);
  LREG(float, lam); LREG(float, jar); LREG(float, f); LREG(float, res); LREG(float, dl); LREG(float, adl); LREG(float, e0); LREG(float, e1);
  LREG(float, j1); LREG(float, j2); LREG(float, hf1); LREG(float, hf2); LREG(float, he01); LREG(float, he02); LREG(float, he11); LREG(float, he12);
  LREG(float, ja1); LREG(float, ja2); LREG(float, jv1); LREG(float, jv2); LREG(float, tmp); LREG(float, tmp2); LREG(float, chg);
  LREG(int, kind); LREG(int, state); LREG(int, hst); LREG(int, colx); LREG(int, la); LREG(int, lb); LREG(int, cla); LREG(int, clb);
  int niter = 0;
  if (n > 0) {
    // ---- stage: row constants into registers, A into shared memory (full, symmetric), warm start from the previous forces
    WPAR_BEGIN {
      const int r = lane;
      // the J / Z rows are read once, at the very end (J^T f gather); ask for them now: without this the gather sits on DRAM misses
      // for a quarter of the kernel's stall samples (profiles/r02_ncu_full_v8_summary.json, by-line)
      prefetch_rec(d.efc_J, n * FB_JROW, d, e, lane); prefetch_rec(d.efc_Z, n * FB_JROW, d, e, lane);
      L(kind) = 0; L(D) = 0; L(b) = 0; L(Rr) = 0; L(mu) = 0; L(c1) = 0; L(c2) = 0; L(lam) = 0; L(la) = -1; L(lb) = -1; L(cla) = 0; L(clb) = 0;
      L(state) = 0; L(hst) = 0; L(f) = 0; L(hf1) = 0; L(hf2) = 0; L(e0) = 0; L(e1) = 0; L(he01) = 0; L(he02) = 0; L(he11) = 0; L(he12) = 0; L(chg) = 0;
      if (r < n) {
        int tp = EFC(d.efc_type, r);
        if (tp == FB_CT_ELLIPTIC) { int ci = EFC(d.efc_id, r); L(kind) = 1 + (r - AT(d.con_efcadr, ci)); L(mu) = AT(d.con_mu, ci); L(c1) = CON_F(d.con_fric, ci, 0, 2); L(c2) = CON_F(d.con_fric, ci, 1, 2); }
        L(D) = EFC(d.efc_D, r); L(b) = EFC(d.efc_b, r); L(Rr) = EFC(d.efc_R, r);
        L(la) = AT(d.efc_la, r); L(lb) = AT(d.efc_lb, r);
        L(cla) = L(la) >= 0 ? m.dof_chainlen[L(la)] : 0; L(clb) = L(lb) >= 0 ? m.dof_chainlen[L(lb)] : 0;
        int key = AT(d.efc_key, r), pn = AT(d.prev_n, 0); float l0 = 0;
        NOUNROLL for (int q = 0; q < pn; q++) if (AT(d.prev_key, q) == key) { l0 = AT(d.prev_lam, q); break; }
        L(lam) = l0;
      }
      L(jar) = L(b);
      const int nt = TRI(n, 0);
      NOUNROLL for (int t = lane; t < nt; t += 32) {
        int p = (int)((sqrtf(8.0f * t + 1.0f) - 1.0f) * 0.5f);
        while ((p + 1) * (p + 2) / 2 <= t) p++;
        while (p * (p + 1) / 2 > t) p--;
        int q = t - p * (p + 1) / 2; float v = AT(d.efc_A, t);
        A_(p, q) = v; A_(q, p) = v;
      }
    } WPAR_END
    WPAR_BEGIN { L(D1) = SHF(D, lane + 1); L(D2) = SHF(D, lane + 2); } WPAR_END
    // ---- warm start kept only if cheaper than lam = 0 (jar holds b here)
    REG_HEADS(0, false)
    const float cost0 = WSUM_GET(0);
    WPAR_BEGIN WPAR_END
    WPAR_BEGIN { float s; REG_MATVEC(s, lam) L(tmp) = s; WSUM_PUT(0, 0.5f * L(lam) * s); } WPAR_END
    float quad = WSUM_GET(0);
    WPAR_BEGIN { L(jar) = L(b) + L(tmp); } WPAR_END
    REG_HEADS(1, false)
    const float cost_ws = quad + WSUM_GET(1);
    WPAR_BEGIN WPAR_END
    if (!(cost_ws < cost0)) { WPAR_BEGIN { L(lam) = 0; L(jar) = L(b); } WPAR_END quad = 0; }
    // ---- Newton iterations (jar and quad are carried along, see ksolve_impl)
    NOUNROLL for (int iter = 0; iter < m.max_iter; iter++) {
      REG_HEADS(1, true)
      WPAR_BEGIN { float rv = L(lam) - L(f); L(res) = rv; WSUM_PUT(2, rv * rv); WSUM_PUT(3, L(f) * L(f)); E0s[lane] = L(e0); E1s[lane] = L(e1); } WPAR_END
      const float cost = quad + WSUM_GET(1), rr = WSUM_GET(2), ll = WSUM_GET(3);
      WPAR_BEGIN WPAR_END
      if (rr <= 1e-12f * (ll + 1e-30f)) break;
      // columns of E: one per active plain / bottom-zone row, two per cone (shared by its three rows)
      unsigned m1, m2;
      BALLOT(m1, state, == 1); BALLOT(m2, state, == 2);
      const int nc = POPC(m1) + 2 * POPC(m2);
      WPAR_BEGIN { unsigned lt = (1u << lane) - 1u; int c0 = POPC(m1 & lt) + 2 * POPC(m2 & lt);
          L(colx) = L(state) == 0 ? -1 : c0;
          if (L(state) == 1) { ECR[c0] = lane; ECK[c0] = 0; }
          else if (L(state) == 2) { ECR[c0] = lane; ECK[c0] = 1; ECR[c0 + 1] = lane; ECK[c0 + 1] = 2; } } WPAR_END
      WPAR_BEGIN { int c1_ = SHF(colx, lane - 1), c2_ = SHF(colx, lane - 2); if (L(state) == 3) L(colx) = (L(kind) == 2) ? c1_ : c2_; } WPAR_END
      // u = A r, then p and G (reg_assemble)
      WPAR_BEGIN { float s; REG_MATVEC(s, res) Us[lane] = s; } WPAR_END
#if FB_CHOL_REG > 0
      if (nc <= FB_CHOL_REG) {
        WPAR_BEGIN reg_assemble(A, E0s, E1s, Us, ECR, ECK, P, G, nc, lane); WPAR_END
        // Cholesky G = L L^T with ROW i OF G / L IN THE REGISTERS OF LANE i (right-looking: after step j every lane has subtracted
        // column j's outer product from its row; L[k][j] travels by shuffle).  Register indices must be static, so the row lives
        // in slots that shift by one per step (below).  The forward substitution L y = p rides along (y in a lane register); L is
        // written back to the packed triangle (triangular numbers mod 32 are a permutation: conflict-free) for the backward
        // substitution, where lane i needs column i of L.  All lanes < nc work in every step -- the column-by-column shared-memory
        // form below kept 2.4 - 4.6 lanes busy (profiles/r02_ncu_full_v9_summary.json).
        LREGA(float, g, FB_CHOL_REG); LREG(float, yv); LREG(float, lcol); LREG(float, yjr); LREG(float, dinv);
        WPAR_BEGIN {
#pragma unroll
          for (int k = 0; k < FB_CHOL_REG; k++) LA(g, k) = (k < nc && lane < nc && k <= lane) ? GP(lane, k) : 0.0f;      // (an early exit at k >= nc costs registers: measured 18 % slower)
          L(yv) = lane < nc ? P[lane] : 0.0f; L(dinv) = 0.0f;
        } WPAR_END
        // slot s of the register row always holds column j + s: every step works on slot 0 and writes the updated column j + q into
        // slot q - 1 (update and shift in one FMA), so the loop over the columns stays rolled -- one copy of the step in the
        // instruction cache.  (First version: both loops unrolled, 24 copies; a third of the kernel's stall samples waited for
        // instructions, profiles/r02_ncu_full_v13_summary.json.)  The exit test of the inner loop comes once per four columns: columns
        // >= nc hold zeros, their updates are no-ops (per column: 1.94 ms per control step; per four: 1.73; rolled: 1.71).  Entries
        // above the diagonal (slot index > row) carry values nobody reads.
        NOUNROLL for (int j = 0; j < nc; j++) {
          WPAR_BEGIN {
            const float inv = FB_RSQRT(fmaxf(SHFA(g, 0, j), 1e-12f));
            L(lcol) = LA(g, 0) * inv;                      // lane j: L[j][j]; lanes above: L[i][j]
            L(yjr) = SHF(yv, j) * inv;
            if (lane == j) L(dinv) = inv;
          } WPAR_END
          WPAR_BEGIN {
            const float l = L(lcol), yj = L(yjr);
            if (lane >= j && lane < nc) GP(lane, j) = l;
            if (lane == j) L(yv) = yj; else if (lane > j) L(yv) -= l * yj;
            const int rem = nc - 1 - j;
#pragma unroll
            for (int q = 1; q < FB_CHOL_REG; q++) {
              if ((q - 1) % 4 == 0 && q > rem) break;          // (columns >= nc hold zeros: lanes >= nc have lcol = 0)
              LA(g, q - 1) = LA(g, q) - l * SHF(lcol, j + q);
            }
          } WPAR_END
        }
        NOUNROLL for (int i = nc - 1; i > 0; i--) {      // backward: L^T x = y; x_i = y_i / L[i][i] once the rows above are subtracted
          WPAR_BEGIN { const float xi = SHF(yv, i) * SHF(dinv, i); if (lane < i) L(yv) -= GP(i, lane) * xi; } WPAR_END
        }
        WPAR_BEGIN { if (lane < nc) XO[lane] = L(yv) * L(dinv); } WPAR_END
      } else
#endif
      {
        // larger blocks (rare, see FB_CHOL_REG) in the env's record, which keeps the shared slice at the size of the register
        // form's G: column by column (two warp barriers per column); the forward substitution L y = p rides along on lane 0
        float* Gr = &AT(d.efc_G, 0);
        WPAR_BEGIN reg_assemble(A, E0s, E1s, Us, ECR, ECK, P, Gr, nc, lane); WPAR_END
        NOUNROLL for (int j = 0; j < nc; j++) {
          WPAR_BEGIN NOUNROLL for (int i = j + lane; i < nc; i += 32) {
              float t = Gr[TRI(i, j)]; NOUNROLL for (int k = 0; k < j; k++) t -= Gr[TRI(i, k)] * Gr[TRI(j, k)];
              Gr[TRI(i, j)] = (i == j) ? sqrtf(fmaxf(t, 1e-12f)) : t; }
          WPAR_END
          WPAR_BEGIN const float dg = Gr[TRI(j, j)];
            NOUNROLL for (int i = j + 1 + lane; i < nc; i += 32) Gr[TRI(i, j)] = Gr[TRI(i, j)] / dg;
            if (lane == 0) { float yv = P[j]; NOUNROLL for (int k = 0; k < j; k++) yv -= Gr[TRI(j, k)] * XQ[k]; XQ[j] = yv / dg; }
          WPAR_END
        }
        NOUNROLL for (int j = nc - 1; j >= 0; j--) {     // backward: L^T out = y
          WPAR_BEGIN float xj = XQ[j] / Gr[TRI(j, j)];
            NOUNROLL for (int i = lane; i < j; i += 32) XQ[i] -= Gr[TRI(j, i)] * xj;
            if (lane == 0) XO[j] = xj;
          WPAR_END
        }
      }
      // dlam = -r + E q ; A dlam ; quadratic coefficients of the Gauss term along dlam
      WPAR_BEGIN { float v = -L(res); int stt = L(state), c0 = L(colx);
          if (stt == 1) v += L(e0) * XO[c0];
          else if (stt >= 2) v += L(e0) * XO[c0] + L(e1) * XO[c0 + 1];
          L(dl) = v; } WPAR_END
      WPAR_BEGIN { float s; REG_MATVEC(s, dl) L(adl) = s; WSUM_PUT(0, L(dl) * (L(jar) - L(b))); WSUM_PUT(1, 0.5f * L(dl) * s); } WPAR_END
      const float q1 = WSUM_GET(0), q2 = WSUM_GET(1);
      WPAR_BEGIN { L(ja1) = SHF(jar, lane + 1); L(ja2) = SHF(jar, lane + 2); L(jv1) = SHF(adl, lane + 1); L(jv2) = SHF(adl, lane + 2); } WPAR_END
      // exact line search: safeguarded Newton on the derivative of the 1-D cost
      float alpha = 0, lo = 0, hi = -1, g0 = 0, cbest = cost; bool stop = false, nodescent = false;
      NOUNROLL for (int ls = 0; ls <= m.ls_iter && !stop; ls++) {
        WPAR_BEGIN { float c = 0, g = 0, h = 0;
            if (L(kind) <= 1) reg_head_ls(L(kind), alpha, L(jar), L(adl), L(ja1), L(jv1), L(ja2), L(jv2), L(D), L(D1), L(D2), L(mu), L(c1), L(c2), c, g, h);
            WSUM_PUT(0, c); WSUM_PUT(1, g); WSUM_PUT(2, h); } WPAR_END
        float c = quad + alpha * q1 + alpha * alpha * q2 + WSUM_GET(0), g = q1 + 2 * alpha * q2 + WSUM_GET(1), h = 2 * q2 + WSUM_GET(2);
        WPAR_BEGIN WPAR_END
        if (ls == 0) {
          g0 = g;
          if (!(g < 0) || !(h > 0)) { alpha = 0; stop = true; nodescent = true; }
          else alpha = -g / h;
        } else {
          cbest = c;
          if (fabsf(g) < m.ls_tolerance * fabsf(g0) || ls == m.ls_iter) stop = true;
          else {
            if (g < 0) lo = alpha; else hi = alpha;
            float na = alpha - g / h;
            if (hi >= 0 && (na <= lo || na >= hi)) na = 0.5f * (lo + hi);
            else if (hi < 0 && na <= lo) na = 2 * alpha;
            if (fabsf(na - alpha) <= 1e-7f * fabsf(alpha)) stop = true;
            alpha = na;
          }
        }
      }
      if (nodescent) break;                               // converged to fp32 resolution
      WPAR_BEGIN { L(lam) += alpha * L(dl); L(jar) += alpha * L(adl); } WPAR_END
      quad += alpha * q1 + alpha * alpha * q2;
      niter = iter + 1;
      if (scale * (cost - cbest) < m.tolerance || (cost - cbest) < m.solve_rtol * fabsf(cost)) break;
    }
    // ---- forces at the solution: f(b + A lam), recomputed from scratch
    WPAR_BEGIN { float s; REG_MATVEC(s, lam) L(tmp) = s; } WPAR_END
    WPAR_BEGIN { L(jar) = L(b) + L(tmp); } WPAR_END
    REG_HEADS(1, false)
    // ---- noslip (MuJoCo mj_solNoSlip): Gauss-Seidel over the frictional contacts with the unregularised A; the residual
    // b + A f of every row is kept current in a register, the head lane of the contact solves its 2x2 QCQP
    if (m.noslip_iterations > 0) {
      unsigned heads;
      BALLOT(heads, kind, == 1);
      WPAR_BEGIN { float s; REG_MATVEC(s, f) L(tmp) = s; } WPAR_END
      WPAR_BEGIN { L(res) = L(b) + L(tmp); L(chg) = 0.5f * L(f) * L(f) * L(Rr); } WPAR_END       // res doubles as the noslip residual
      NOUNROLL for (int it = 0; it < m.noslip_iterations; it++) {
        if (heads == 0) break;
        unsigned todo = heads;
        while (todo) {
          const int i = FFS(todo) - 1; todo &= todo - 1;
          WPAR_BEGIN { L(j1) = SHF(f, lane + 1); L(j2) = SHF(f, lane + 2); L(ja1) = SHF(res, lane + 1); L(ja2) = SHF(res, lane + 2); } WPAR_END
          WPAR_BEGIN { L(tmp) = 0; L(tmp2) = 0; L(jv1) = L(j1); L(jv2) = L(j2);
            if (lane == i) {
              float fn = L(f), old0 = L(j1), old1 = L(j2), res0 = L(ja1), res1 = L(ja2), Ac[4], bc[2], v[2];
              Ac[0] = A_(i + 1, i + 1); Ac[1] = A_(i + 2, i + 1); Ac[2] = Ac[1]; Ac[3] = A_(i + 2, i + 2);
              bc[0] = res0 - Ac[0] * old0 - Ac[1] * old1; bc[1] = res1 - Ac[2] * old0 - Ac[3] * old1;
              if (fn < FB_MINVAL) { v[0] = 0; v[1] = 0; }
              else {
                int active = qcqp2(v, Ac, bc, L(c1), L(c2), fn);
                if (active) { float s = (v[0] / L(c1)) * (v[0] / L(c1)) + (v[1] / L(c2)) * (v[1] / L(c2)); s = sqrtf(fn * fn / fmaxf(FB_MINVAL, s)); v[0] *= s; v[1] *= s; }
              }
              float d0 = v[0] - old0, d1 = v[1] - old1;
              float change = 0.5f * (d0 * (Ac[0] * d0 + Ac[1] * d1) + d1 * (Ac[2] * d0 + Ac[3] * d1)) + d0 * res0 + d1 * res1;
              if (change > 1e-10f) { v[0] = old0; v[1] = old1; change = 0; d0 = 0; d1 = 0; }
              L(chg) -= change; L(tmp) = d0; L(tmp2) = d1; L(jv1) = v[0]; L(jv2) = v[1];
            } } WPAR_END
          WPAR_BEGIN { float d0 = SHF(tmp, i), d1 = SHF(tmp2, i), v0 = SHF(jv1, i), v1 = SHF(jv2, i);
            if (lane == i + 1) L(f) = v0; else if (lane == i + 2) L(f) = v1;
            if (lane < n) L(res) += A_(lane, i + 1) * d0 + A_(lane, i + 2) * d1; } WPAR_END
        }
        WPAR_BEGIN { WSUM_PUT(0, L(chg)); L(chg) = 0; } WPAR_END
        const float improvement = WSUM_GET(0);
        WPAR_BEGIN WPAR_END
        if (improvement * scale < m.noslip_tolerance) break;
      }
    }
    WPAR_BEGIN { const int r = lane; if (r < n) { EFC(d.efc_force, r) = L(f); AT(d.prev_lam, r) = L(lam); AT(d.prev_key, r) = AT(d.efc_key, r); } } WPAR_END
  }
  // ---- qfrc_constraint = J^T f and Z^T f.  The rows are chain-sparse (fb_constraint.h: EJC): lane s takes slot s of a row's chain a
  // (dof = s-th ancestor of the row's last dof, m.dof_anc) and adds its product to per-dof accumulators in shared memory (A is dead
  // by now), row after row -- within a row the dofs are distinct, a warp barrier orders the rows, so every dof sums in row order.
  // Loads of four rows are in flight together.  Chain b (the second body of a self-contact, below its join with chain a) follows
  // for the few rows that have one.  (Before: every lane scanned every row for its four dofs -- 8 loads per row and lane, most of
  // them masked; 25 % of the kernel's stall samples, profiles/r02_ncu_full_v10_summary.json.)
  float* QJ = wsm; float* QZ = wsm + 128;
  LREG(int, jb);
  WPAR_BEGIN
    if (lane == 0) { AT(d.niter, 0) = niter; if (d.do_integrate) AT(d.prev_n, 0) = n; }
#pragma unroll
    for (int i = 0; i < 4; i++) { QJ[lane + 32 * i] = 0.0f; QZ[lane + 32 * i] = 0.0f; }
    L(jb) = (n > 0 && lane < n && L(lb) >= 0) ? L(clb) - (L(la) >= 0 ? (int)m.dof_lca[L(lb) * m.nv + L(la)] : 0) : 0;
  WPAR_END
  NOUNROLL for (int r0 = 0; r0 < n; r0 += 4) {
    LREGA(float, gj, 4); LREGA(float, gz, 4); LREGA(int, gd, 4);
    WPAR_BEGIN
#pragma unroll
      for (int u = 0; u < 4; u++) {
        const int r = r0 + u, la_ = SHF(la, r), La_ = SHF(cla, r);
        const bool on = r < n && lane < La_;
        LA(gd, u) = on ? m.dof_anc[m.dof_Madr[la_] + lane] : -1;
        LA(gj, u) = on ? AT(d.efc_J, r * FB_JROW + lane) : 0.0f; LA(gz, u) = on ? AT(d.efc_Z, r * FB_JROW + lane) : 0.0f;
      }
    WPAR_END
#pragma unroll
    for (int u = 0; u < 4; u++) {
      WPAR_BEGIN { const int r = r0 + u, dd = LA(gd, u); const float fr = SHF(f, r);
        if (r < n && dd >= 0) { QJ[dd] += LA(gj, u) * fr; QZ[dd] += LA(gz, u) * fr; } } WPAR_END
    }
  }
  unsigned mb;
  BALLOT(mb, jb, > 0);
  while (mb) {
    const int r = FFS(mb) - 1; mb &= mb - 1;
    WPAR_BEGIN { const int lb_ = SHF(lb, r), J_ = SHF(jb, r); const float fr = SHF(f, r);
      if (lane < J_) { const int dd = m.dof_anc[m.dof_Madr[lb_] + lane];
        QJ[dd] += AT(d.efc_J, r * FB_JROW + FB_ZCAP + lane) * fr; QZ[dd] += AT(d.efc_Z, r * FB_JROW + FB_ZCAP + lane) * fr; } } WPAR_END
  }
  WPAR_BEGIN
#pragma unroll
    for (int i = 0; i < 4; i++) { int k = lane + 32 * i; if (k < m.nv) { AT(d.qfrc_constraint, k) = QJ[k]; AT(d.qfrc_zf, k) = QZ[k]; } }
  WPAR_END
}

// one env; `wsm` = this warp's shared-memory slice (FB_SOLVE_WARP_FLOATS floats).  Envs with more rows than the register path
// holds (nefc > 32: freshly reset flies, flies pressed against their joint limits -- 0.05 - 1 % of a batch) run the generic code
// on their record in global memory, inline in this kernel: there their solve overlaps with the other envs' solves.
FB_WARPFN void ksolve_warp(const DevModel& m, const DevData& d, float* wsm, int e) {
  const int n = AT(d.nefc, 0);
  if (n <= m.solve_ncap) { ksolve_reg(m, d, wsm, e, n); return; }
  SolveMem sm;
  sm.red = wsm; sm.v = &AT(d.efc_w, 0); sm.A = &AT(d.efc_A, 0); sm.G = &AT(d.efc_G, 0); sm.cap = FB_MAXEFC;
  ksolve_impl(m, d, sm, e, n);
}
