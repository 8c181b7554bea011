// fb_solver.h -- K11 constraint solve, one WARP per environment.
//
// Thread mapping: blockDim = (32, FB_SOLVE_WPB); warp (threadIdx.y) owns one env, its 32 lanes split the
// rows of that env's dual problem (rows of the Delassus matrix-vector products, columns of the Hessian
// factor, line-search partial sums).  Every env therefore runs exactly its own number of Newton
// iterations on its own problem size -- no divergence between envs -- and synchronisation is
// __syncwarp only.  This generic form solves the problems the register path (fb_solver_reg.h) does not
// hold (nefc > solve_ncap): the working set of an env (row constants, 12 work vectors, the packed Delassus
// matrix A and the packed Hessian factor G) stays in the env's record; only the warp-sum staging RED
// uses the warp's shared-memory slice.
//
// Math (see DESIGN.md "Solver"): with a = qacc_smooth + M^-1 J^T lam the primal cost of MuJoCo's Newton
// solver becomes  c(lam) = 1/2 lam^T A lam + s(b + A lam),  A = J M^-1 J^T,  b = J qacc_smooth - aref,
// s = per-row cost (half-quadratic for limits / frictionless contacts, three-zone elliptic cone for
// frictional contacts).  Primal Newton steps map to  dlam = -(I + C A)^-1 (lam - f(lam)),  C = Hess s =
// E E^T, solved through the SPD system G = I + E^T A E (Cholesky) + the same exact line search.
//
// Written as WPAR sections (each ends in a warp barrier); code between sections is warp-uniform and is
// executed redundantly by all lanes on the GPU / once by the host emulation, where a WPAR section is a
// loop over the 32 lanes.
#pragma once
#include "fb_constraint.h"

#define FB_SOLVE_WPB 4          // warps (envs) per block
#define FB_SOLVE_NCAP 32        // rows that fit the shared-memory slice

enum { W_LAM = 0, W_JAR, W_F, W_R, W_U, W_DL, W_ADL, W_P, X_E0, X_E1, X_XQ, X_OUT,
       // row constants staged once per solve (so the Newton phases never chase global metadata)
       S_D, S_B, S_R, S_TYPE /* 0 plain, 1 elliptic head, 2 elliptic tail */, S_MU, S_F1, S_F2, S_LA, S_LB,
       S_STATE, S_COLIDX, S_ECROW, S_ECKIND, S_NSLOT };
#define TRI(r, c) ((r) * ((r) + 1) / 2 + (c))

// memory of one env's problem: work vectors v [S_NSLOT][cap], packed Delassus matrix A and packed Hessian factor G in the env's
// record (efc_w, efc_A, efc_G; cap = FB_MAXEFC), warp-sum staging red [4][32] in the warp's shared-memory slice
struct SolveMem { float* v; float* A; float* G; float* red; int cap; };
#define SV(slot, r) sm.v[(slot) * sm.cap + (r)]
#define AM(r, c) sm.A[(r) >= (c) ? TRI(r, c) : TRI(c, r)]
#define GM(p, q) sm.G[TRI(p, q)]        // p >= q
#define RED(k, l) sm.red[(k) * 32 + (l)]

#define NOUNROLL _Pragma("unroll 1")
#define WROWS NOUNROLL for (int r = lane; r < n; r += 32)
FB_DEV float red_total(const SolveMem& sm, int k) { float s = 0; for (int l = 0; l < 32; l++) s += RED(k, l); return s; }
// warp sums: butterfly shuffles on the GPU (every lane gets the total, no shared-memory round trip);
// the host emulation runs lanes one after the other, so it stages partials in RED and sums afterwards
#ifdef __CUDACC__
FB_DEV float wsum(float v) { for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o); return v; }
#define WSUM_PUT(k, v) tot[k] = wsum(v)
#define WSUM_GET(k) (tot[k])
#else
#define WSUM_PUT(k, v) RED(k, lane) = (v)
#define WSUM_GET(k) red_total(sm, k)
#endif
#define IS_HEAD(r) (SV(S_TYPE, r) < 1.5f)

// forces / cost of the rows headed at r (a plain row, or the first row of an elliptic contact)
FB_DEVN float head_update(const SolveMem sm, int r, bool build) {
  int tp = (int)SV(S_TYPE, r);
  float jar = SV(W_JAR, r), D = SV(S_D, r), cost = 0;
  if (tp == 0) {
    if (jar < 0) { SV(W_F, r) = -D * jar; cost = 0.5f * D * jar * jar; if (build) { SV(S_STATE, r) = 1; SV(X_E0, r) = sqrtf(D); } }
    else { SV(W_F, r) = 0; if (build) SV(S_STATE, r) = 0; }
    return cost;
  }
  float mu = SV(S_MU, r), f1 = SV(S_F1, r), f2 = SV(S_F2, r);
  float j1 = SV(W_JAR, r + 1), j2 = SV(W_JAR, r + 2), D1 = SV(S_D, r + 1), D2 = SV(S_D, r + 2);
  float U0 = jar * mu, U1 = j1 * f1, U2 = j2 * f2, N = U0, T = sqrtf(U1 * U1 + U2 * U2);
  if (mu * N + T <= 0 || (T <= 0 && N < 0)) {             // bottom zone: quadratic
    SV(W_F, r) = -D * jar; SV(W_F, r + 1) = -D1 * j1; SV(W_F, r + 2) = -D2 * j2;
    cost = 0.5f * (D * jar * jar + D1 * j1 * j1 + D2 * j2 * j2);
    if (build) { SV(S_STATE, r) = 1; SV(S_STATE, r + 1) = 1; SV(S_STATE, r + 2) = 1; SV(X_E0, r) = sqrtf(D); SV(X_E0, r + 1) = sqrtf(D1); SV(X_E0, r + 2) = sqrtf(D2); }
  } else if (N >= mu * T || (T <= 0 && N >= 0)) {          // top zone: satisfied
    SV(W_F, r) = 0; SV(W_F, r + 1) = 0; SV(W_F, r + 2) = 0;
    if (build) { SV(S_STATE, r) = 0; SV(S_STATE, r + 1) = 0; SV(S_STATE, r + 2) = 0; }
  } else {                                                  // middle zone: cone
    float Dm = D / (mu * mu * (1 + mu * mu)), NmT = N - mu * T;
    cost = 0.5f * Dm * NmT * NmT;
    float f0 = -Dm * NmT * mu;
    SV(W_F, r) = f0; SV(W_F, r + 1) = -f0 / T * U1 * f1; SV(W_F, r + 2) = -f0 / T * U2 * f2;
    if (build) {
      // C = Dm [ (S g)(S g)^T + (-f mu / T)(S t)(S t)^T ],  g = (1, -mu U1/T, -mu U2/T), t = (0, -U2, U1)/T
      float sD = sqrtf(Dm), k2 = sqrtf(fmaxf(0.0f, Dm * (-NmT) * mu / T));
      SV(S_STATE, r) = 2; SV(S_STATE, r + 1) = 3; SV(S_STATE, r + 2) = 3;
      SV(X_E0, r) = sD * mu; SV(X_E0, r + 1) = -sD * f1 * mu * U1 / T; SV(X_E0, r + 2) = -sD * f2 * mu * U2 / T;
      SV(X_E1, r) = 0; SV(X_E1, r + 1) = -k2 * f1 * U2 / T; SV(X_E1, r + 2) = k2 * f2 * U1 / T;
    }
  }
  return cost;
}
// line-search contribution (value, 1st, 2nd derivative) of the rows headed at r
FB_DEVN void head_ls(const SolveMem sm, int r, float alpha, float& c, float& g, float& h) {
  int tp = (int)SV(S_TYPE, r);
  float jv = SV(W_ADL, r), x = SV(W_JAR, r) + alpha * jv, D = SV(S_D, r);
  if (tp == 0) { if (x < 0) { c += 0.5f * D * x * x; g += D * x * jv; h += D * jv * jv; } return; }
  float mu = SV(S_MU, r), f1 = SV(S_F1, r), f2 = SV(S_F2, r);
  float jv1 = SV(W_ADL, r + 1), jv2 = SV(W_ADL, r + 2);
  float x1 = SV(W_JAR, r + 1) + alpha * jv1, x2 = SV(W_JAR, r + 2) + alpha * jv2;
  float D1 = SV(S_D, r + 1), D2 = SV(S_D, r + 2);
  float U0 = x * mu, U1 = x1 * f1, U2 = x2 * f2, dU0 = jv * mu, dU1 = jv1 * f1, dU2 = jv2 * f2;
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
FB_DEV float ecol_val(const SolveMem& sm, int p, int a) {   // a-th entry of column p of E
  int kind = (int)SV(S_ECKIND, p), r = (int)SV(S_ECROW, p);
  return kind == 2 ? SV(X_E1, r + a) : SV(X_E0, r + a);
}

// dst[r] = (addb ? b[r] : 0) + sum_j A[r][j] src[j] for this lane's rows; returns sum_r src[r]*(dst[r]-b[r]) partial
// (one loop over j with a select for the packed index: splitting it at the diagonal makes the lanes diverge)
FB_DEVN float matvec_rows(const SolveMem sm, int n, int lane, int src, int dst, bool addb) {
  float acc = 0;
  NOUNROLL for (int r = lane; r < n; r += 32) {
    float s = 0;
#pragma unroll 2
    for (int j = 0; j < n; j++) s += AM(r, j) * SV(src, j);
    acc += SV(src, r) * s;
    SV(dst, r) = addb ? s + SV(S_B, r) : s;
  }
  return acc;
}


FB_WARPFN void ksolve_impl(const DevModel& m, const DevData& d, const SolveMem& sm, int e, int n) {
  const float scale = 1.0f / (m.meaninertia * (m.nv > 1 ? m.nv : 1));
  float tot[4] = {0, 0, 0, 0}; (void)tot;
  int niter = 0;
  if (n > 0) {
    // ---- stage row constants (and A) next to the work vectors
    WPAR_BEGIN WROWS {
      int tp = EFC(d.efc_type, r), tcode = 0; float mu = 0, f1 = 0, f2 = 0;
      if (tp == FB_CT_ELLIPTIC) { int ci = EFC(d.efc_id, r); tcode = (AT(d.con_efcadr, ci) == r) ? 1 : 2; mu = AT(d.con_mu, ci); f1 = CON_F(d.con_fric, ci, 0, 2); f2 = CON_F(d.con_fric, ci, 1, 2); }
      SV(S_TYPE, r) = (float)tcode; SV(S_MU, r) = mu; SV(S_F1, r) = f1; SV(S_F2, r) = f2;
      SV(S_D, r) = EFC(d.efc_D, r); SV(S_B, r) = EFC(d.efc_b, r); SV(S_R, r) = EFC(d.efc_R, r);
      SV(S_LA, r) = (float)AT(d.efc_la, r); SV(S_LB, r) = (float)AT(d.efc_lb, r);
      // warm start: force of the same row in the previous solve (0 for new rows)
      { int key = AT(d.efc_key, r), pn = AT(d.prev_n, 0); float l0 = 0;
        NOUNROLL for (int q = 0; q < pn; q++) if (AT(d.prev_key, q) == key) { l0 = AT(d.prev_lam, q); break; }
        SV(W_LAM, r) = l0; }
    }
    WPAR_END
    // ---- warm start: the previous solve's forces (matched by row identity), kept if cheaper than lam = 0.
    // jar = b + A lam and quad = 1/2 lam^T A lam are carried along the iterations: a step lam += alpha dlam changes them by
    // alpha * (A dlam) and alpha q1 + alpha^2 q2, both already known from the line search (the forces at the solution are
    // recomputed from scratch after the loop)
    WPAR_BEGIN WROWS SV(W_JAR, r) = SV(S_B, r); WPAR_END
    WPAR_BEGIN float c = 0; WROWS if (IS_HEAD(r)) c += head_update(sm, r, false); WSUM_PUT(0, c); WPAR_END
    const float cost0 = WSUM_GET(0);
    WPAR_BEGIN WPAR_END
    WPAR_BEGIN float q = 0.5f * matvec_rows(sm, n, lane, W_LAM, W_JAR, true); WSUM_PUT(0, q); WPAR_END
    WPAR_BEGIN float c = 0; WROWS if (IS_HEAD(r)) c += head_update(sm, r, false); WSUM_PUT(1, c); WPAR_END
    float quad = WSUM_GET(0);
    const float cost_ws = quad + WSUM_GET(1);
    WPAR_BEGIN WPAR_END
    if (!(cost_ws < cost0)) { WPAR_BEGIN WROWS { SV(W_LAM, r) = 0; SV(W_JAR, r) = SV(S_B, r); } WPAR_END quad = 0; }
    // ---- Newton iterations
    NOUNROLL for (int iter = 0; iter < m.max_iter; iter++) {
      WPAR_BEGIN float c = 0; WROWS if (IS_HEAD(r)) c += head_update(sm, r, true); WSUM_PUT(1, c); WPAR_END
      WPAR_BEGIN float rr = 0, ll = 0; WROWS { float f = SV(W_F, r), rv = SV(W_LAM, r) - f; SV(W_R, r) = rv; rr += rv * rv; ll += f * f; } WSUM_PUT(2, rr); WSUM_PUT(3, ll); WPAR_END
      float cost = quad + WSUM_GET(1);
      float rr = WSUM_GET(2), ll = WSUM_GET(3);
      WPAR_BEGIN WPAR_END              // all lanes have read RED before it is reused
      if (rr <= 1e-12f * (ll + 1e-30f)) break;
      // column bookkeeping (prefix over rows) by lane 0; nc is left in RED(0, 0)
      WPAR_BEGIN if (lane == 0) { int nc = 0;
        NOUNROLL for (int r = 0; r < n; r++) { int stt = (int)SV(S_STATE, r);
          if (stt == 1) { SV(S_COLIDX, r) = (float)nc; SV(S_ECROW, nc) = (float)r; SV(S_ECKIND, nc) = 0; nc++; }
          else if (stt == 2) { SV(S_COLIDX, r) = (float)nc; SV(S_COLIDX, r + 1) = (float)nc; SV(S_COLIDX, r + 2) = (float)nc; SV(S_ECROW, nc) = (float)r; SV(S_ECKIND, nc) = 1; SV(S_ECROW, nc + 1) = (float)r; SV(S_ECKIND, nc + 1) = 2; nc += 2; }
          else if (stt == 0) SV(S_COLIDX, r) = -1.0f; }
        RED(0, 0) = (float)nc; }
      WPAR_END
      const int nc = (int)RED(0, 0);
      // u = A r
      WPAR_BEGIN matvec_rows(sm, n, lane, W_R, W_U, false); WPAR_END
      // p = E^T u ; G = I + E^T A E (packed lower triangle)
      WPAR_BEGIN
        NOUNROLL for (int p = lane; p < nc; p += 32) {
          int rp = (int)SV(S_ECROW, p), np = SV(S_ECKIND, p) == 0 ? 1 : 3;
          float pv = 0; NOUNROLL for (int a = 0; a < np; a++) pv += ecol_val(sm, p, a) * SV(W_U, rp + a);
          SV(W_P, p) = pv;
        }
        const int npairs = nc * (nc + 1) / 2;                 // lanes over the entries (p >= q) of the packed triangle
        NOUNROLL for (int t = lane; t < npairs; t += 32) {
          int p = (int)((sqrtf(8.0f * t + 1.0f) - 1.0f) * 0.5f);
          while ((p + 1) * (p + 2) / 2 <= t) p++;
          while (p * (p + 1) / 2 > t) p--;
          int q = t - p * (p + 1) / 2;
          int rp = (int)SV(S_ECROW, p), np = SV(S_ECKIND, p) == 0 ? 1 : 3;
          int rq = (int)SV(S_ECROW, q), nq = SV(S_ECKIND, q) == 0 ? 1 : 3;
          float s = (p == q) ? 1.0f : 0.0f;
          NOUNROLL for (int a = 0; a < np; a++) { float va = ecol_val(sm, p, a); if (va == 0.0f) continue; NOUNROLL for (int bb = 0; bb < nq; bb++) s += va * AM(rp + a, rq + bb) * ecol_val(sm, q, bb); }
          GM(p, q) = s;
        }
      WPAR_END
      // Cholesky G = L L^T, column by column; the forward substitution L y = p rides along (lane 0)
      NOUNROLL for (int j = 0; j < nc; j++) {
        WPAR_BEGIN NOUNROLL for (int i = j + lane; i < nc; i += 32) {
            float t = GM(i, j); NOUNROLL for (int k = 0; k < j; k++) t -= GM(i, k) * GM(j, k);
            GM(i, j) = t; if (i == j) RED(1, 0) = sqrtf(fmaxf(t, 1e-12f)); }
        WPAR_END
        WPAR_BEGIN float dg = RED(1, 0);
          NOUNROLL for (int i = j + lane; i < nc; i += 32) GM(i, j) = (i == j) ? dg : GM(i, j) / dg;
          if (lane == 0) { float yv = SV(W_P, j); NOUNROLL for (int k = 0; k < j; k++) yv -= GM(j, k) * SV(X_XQ, k); SV(X_XQ, j) = yv / dg; }
        WPAR_END
      }
      NOUNROLL for (int j = nc - 1; j >= 0; j--) {     // backward: L^T out = y
        WPAR_BEGIN float xj = SV(X_XQ, j) / GM(j, j);
          NOUNROLL for (int i = lane; i < j; i += 32) SV(X_XQ, i) -= GM(j, i) * xj;
          if (lane == 0) SV(X_OUT, j) = xj;
        WPAR_END
      }
      // dlam = -r + E q ;  A dlam ; quadratic coefficients of the Gauss term along dlam
      WPAR_BEGIN WROWS { float v = -SV(W_R, r); int stt = (int)SV(S_STATE, r), c0 = (int)SV(S_COLIDX, r);
          if (stt == 1) v += SV(X_E0, r) * SV(X_OUT, c0);
          else if (stt >= 2) v += SV(X_E0, r) * SV(X_OUT, c0) + SV(X_E1, r) * SV(X_OUT, c0 + 1);
          SV(W_DL, r) = v; }
      WPAR_END
      WPAR_BEGIN float q2 = 0.5f * matvec_rows(sm, n, lane, W_DL, W_ADL, false), q1 = 0;
          WROWS q1 += SV(W_DL, r) * (SV(W_JAR, r) - SV(S_B, r)); WSUM_PUT(0, q1); WSUM_PUT(1, q2); WPAR_END
      const float q1 = WSUM_GET(0), q2 = WSUM_GET(1);
      WPAR_BEGIN WPAR_END
      // exact line search: safeguarded Newton on the derivative of the 1-D cost
      float alpha = 0, lo = 0, hi = -1, g0 = 0, cbest = cost; bool stop = false, nodescent = false;
      NOUNROLL for (int ls = 0; ls <= m.ls_iter && !stop; ls++) {
        WPAR_BEGIN float c = 0, g = 0, h = 0; WROWS if (IS_HEAD(r)) head_ls(sm, r, alpha, c, g, h); WSUM_PUT(0, c); WSUM_PUT(1, g); WSUM_PUT(2, h); WPAR_END
        float c = quad + alpha * q1 + alpha * alpha * q2 + WSUM_GET(0), g = q1 + 2 * alpha * q2 + WSUM_GET(1), h = 2 * q2 + WSUM_GET(2);
        WPAR_BEGIN WPAR_END          // keep RED reads of all lanes ahead of the next section's writes
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
      WPAR_BEGIN WROWS { SV(W_LAM, r) += alpha * SV(W_DL, r); SV(W_JAR, r) += alpha * SV(W_ADL, r); } WPAR_END
      quad += alpha * q1 + alpha * alpha * q2;
      niter = iter + 1;
      // MuJoCo's absolute criterion, plus a relative one: Newton converges quadratically, so a step whose
      // improvement is below 1e-7 of the cost has already landed within fp32 resolution of the minimiser
      if (scale * (cost - cbest) < m.tolerance || (cost - cbest) < m.solve_rtol * fabsf(cost)) break;
    }
    // ---- forces at the solution: lam = f(b + A lam)
    WPAR_BEGIN matvec_rows(sm, n, lane, W_LAM, W_JAR, true); WPAR_END
    WPAR_BEGIN WROWS if (IS_HEAD(r)) head_update(sm, r, false); WPAR_END
    // ---- noslip (MuJoCo mj_solNoSlip): sequential Gauss-Seidel over the friction rows with the unregularised A
    if (m.noslip_iterations > 0) {
      // residual res = b + A f of every row, kept current in W_U: the contact being updated reads its two friction
      // entries, then all lanes apply the rank-2 change -- no O(n) dot products on a single lane
      WPAR_BEGIN matvec_rows(sm, n, lane, W_F, W_U, true); WPAR_END
      WPAR_BEGIN if (lane == 0) { float imp = 0; NOUNROLL for (int i = 0; i < n; i++) imp += 0.5f * SV(W_F, i) * SV(W_F, i) * SV(S_R, i); RED(1, 0) = imp; } WPAR_END
      NOUNROLL for (int it = 0; it < m.noslip_iterations; it++) {
        bool any = false;
        NOUNROLL for (int i = 0; i < n; i++) {
          if (SV(S_TYPE, i) < 0.5f || SV(S_TYPE, i) > 1.5f) continue;        // heads of frictional contacts only
          any = true;
          WPAR_BEGIN if (lane == 0) {
            float fn = SV(W_F, i), old0 = SV(W_F, i + 1), old1 = SV(W_F, i + 2);
            float res0 = SV(W_U, i + 1), res1 = SV(W_U, i + 2), Ac[4], bc[2], v[2];
            Ac[0] = AM(i + 1, i + 1); Ac[1] = AM(i + 2, i + 1); Ac[2] = Ac[1]; Ac[3] = AM(i + 2, i + 2);
            bc[0] = res0 - Ac[0] * old0 - Ac[1] * old1; bc[1] = res1 - Ac[2] * old0 - Ac[3] * old1;
            float fr0 = SV(S_F1, i), fr1 = SV(S_F2, i);
            if (fn < FB_MINVAL) { v[0] = 0; v[1] = 0; }
            else {
              int active = qcqp2(v, Ac, bc, fr0, fr1, fn);
              if (active) { float s = (v[0] / fr0) * (v[0] / fr0) + (v[1] / fr1) * (v[1] / fr1); s = sqrtf(fn * fn / fmaxf(FB_MINVAL, s)); v[0] *= s; v[1] *= s; }
            }
            float d0 = v[0] - old0, d1 = v[1] - old1;
            float change = 0.5f * (d0 * (Ac[0] * d0 + Ac[1] * d1) + d1 * (Ac[2] * d0 + Ac[3] * d1)) + d0 * res0 + d1 * res1;
            if (change > 1e-10f) { v[0] = old0; v[1] = old1; change = 0; d0 = 0; d1 = 0; }
            SV(W_F, i + 1) = v[0]; SV(W_F, i + 2) = v[1];
            RED(1, 0) -= change; RED(0, 0) = d0; RED(0, 1) = d1;
          } WPAR_END
          const float d0 = RED(0, 0), d1 = RED(0, 1);
          WPAR_BEGIN WPAR_END          // every lane has read RED(0, .) before lane 0 writes it again for the next contact (racecheck, r2)
          if (d0 != 0.0f || d1 != 0.0f) { WPAR_BEGIN WROWS SV(W_U, r) += AM(r, i + 1) * d0 + AM(r, i + 2) * d1; WPAR_END }
        }
        const float improvement = RED(1, 0);
        WPAR_BEGIN WPAR_END            // ... and RED(1, 0) before it is cleared (racecheck, r2)
        WPAR_BEGIN if (lane == 0) RED(1, 0) = 0; WPAR_END
        if (!any) break;
        if (improvement * scale < m.noslip_tolerance) break;
      }
    }
    WPAR_BEGIN WROWS { EFC(d.efc_force, r) = SV(W_F, r); AT(d.prev_lam, r) = SV(W_LAM, r); AT(d.prev_key, r) = AT(d.efc_key, r); } WPAR_END
  }
  // ---- qfrc_constraint = J^T f and Z^T f (the constraint part of qacc before the L^-1 sweep of the finish kernel).
  // Lane l owns the dofs l, l + 32, l + 64, l + 96 (nv <= 128, checked in fb_create).  A row touches dof k iff k lies on
  // the ancestor chain of one of its two end dofs.  The loads are unconditional (rows not touching k read row 0, always a
  // valid address, and are discarded by a select), so two rows x four dofs x {J, Z} are in flight together.
  WPAR_BEGIN
    if (lane == 0) { AT(d.niter, 0) = niter; if (d.do_integrate) AT(d.prev_n, 0) = n; }
    float sj[4] = {0, 0, 0, 0}, sz[4] = {0, 0, 0, 0}; int se[4], ck[4];
#pragma unroll
    for (int i = 0; i < 4; i++) { int k = lane + 32 * i; se[i] = k < m.nv ? m.dof_subend[k] : -1; ck[i] = k < m.nv ? m.dof_chainlen[k] : 0; }
#pragma unroll 2
    for (int r = 0; r < n; r++) {
      const int la = (int)SV(S_LA, r), lb = (int)SV(S_LB, r); const float f = SV(W_F, r);
      const int La = la >= 0 ? m.dof_chainlen[la] : 0, Lb = lb >= 0 ? m.dof_chainlen[lb] : 0;
#pragma unroll
      for (int i = 0; i < 4; i++) {
        const int k = lane + 32 * i;
        const bool ina = (k <= la && la <= se[i]), in = ina || (k <= lb && lb <= se[i]);
        const int idx = in ? r * FB_JROW + (ina ? La - ck[i] : FB_ZCAP + Lb - ck[i]) : 0;      // chain-sparse rows (fb_constraint.h: EJC)
        const float vj = AT(d.efc_J, idx), vz = AT(d.efc_Z, idx);
        sj[i] += in ? vj * f : 0.0f; sz[i] += in ? vz * f : 0.0f;
      }
    }
#pragma unroll
    for (int i = 0; i < 4; i++) { int k = lane + 32 * i; if (k < m.nv) { AT(d.qfrc_constraint, k) = sj[i]; AT(d.qfrc_zf, k) = sz[i]; } }
  WPAR_END
}

