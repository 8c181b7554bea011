// fb_lqr.h -- the iLQR backward pass (Tassa, Erez & Todorov 2012; fb_lqr), batched over L problems, all in fp64: for t = T-1 .. 0 from
// s = q_T, P = diag(Qf),
//   Qx = q_t + A's          Qu = r_t + B's
//   Qxx = diag(Q) + A'PA    Quu = diag(R) + B'PB + mu I    Qux = B'PA
//   chol(Quu)               (failure: status = t + 1 and the problem stops)
//   k = -Quu^-1 Qu          K = -Quu^-1 Qux
//   dV1 += k'Qu             dV2 += k'Quu k / 2
//   s = Qx + K'Quu k + K'Qu + Qux'k
//   P = sym(Qxx + K'Quu K + K'Qux + Qux'K),  sym(X) = (X + X') / 2
// with A [nx][nx] and B [nx][nu] the fp32 Jacobians fb_fd_read writes.  Five launches per step, one warp per work unit, no atomics;
// every element is one fixed-order sum of its problem's data, so a problem's bits depend on neither its index nor L.  nz = nx + nu;
// M = [A B] (nx x nz).  Per problem, in its own slices of the workspace:
//   W [nx][nz+1] = P M, and column nz = s           (klqr_w; tiles of LQR_ROWS rows x 32 columns)
//   H [nz][nz+1] = M'W + diag(Q, R + mu), and column nz + (q_t, r_t): rows < nx are (Qxx | Qxu | Qx), rows >= nx (Qux | Quu | Qu)  (klqr_h)
//   C [nu][nu] the lower Cholesky factor of Quu     (klqr_chol; one warp per problem, column after column)
//   X [nu][nx+1] = (K | k) and G [nu][nx+1] = Quu X + (Qux | Qu)   (klqr_solve; lane j solves column j in place)
//   P, s and dV from X and G: P_ij and P_ji take the same two sums, so P stays exactly symmetric   (klqr_p)
#pragma once
#include "fb_types.h"

#define LQR_ROWS 8               // rows of a tile: one fp64 accumulator per row and lane

struct DevLqr {
  int L, T, t, nx, nu;                      // problems, steps, the step a launch serves, state and control sizes
  const float *A, *B;                       // [L][T][nx][nx], [L][T][nx][nu]
  const double *q, *r, *Q, *R, *Qf, *mu;    // [L][T+1][nx], [L][T][nu], [nx], [nu], [nx], [L]
  double *P, *s, *W, *H, *C, *X, *G;        // workspace per problem: [nx][nx], [nx], [nx][nz+1], [nz][nz+1], [nu][nu], [nu][nx+1] x 2
  double *K, *k, *dV;                       // outputs: [L][T][nu][nx], [L][T][nu], [L][2]
  int* status;                              // [L]: 0, or t + 1 for a Cholesky failure at step t
};

// work unit w of a launch over L problems x the tiles of a rows x cols matrix -> the problem, the tile's first row and first column
FB_DEV int lqr_tile(int w, int rows, int cols, int* i0, int* j0) {
  const int nrb = (rows + LQR_ROWS - 1) / LQR_ROWS, ncb = (cols + 31) / 32, per = nrb * ncb, u = w % per;
  *i0 = (u / ncb) * LQR_ROWS; *j0 = (u % ncb) * 32;
  return w / per;
}
FB_HD inline int lqr_tiles(int rows, int cols) { return ((rows + LQR_ROWS - 1) / LQR_ROWS) * ((cols + 31) / 32); }

// P = diag(Qf), s = q_T, dV = 0, status = 0
FB_WARPFN void klqr_init(const DevLqr& p, int l) {
  const int nx = p.nx;
  double* P = p.P + (size_t)l * nx * nx;
  const double* qT = p.q + ((size_t)l * (p.T + 1) + p.T) * nx;
  WPAR_BEGIN
    for (int i = lane; i < nx * nx; i += FB_NY) P[i] = i % (nx + 1) == 0 ? p.Qf[i / (nx + 1)] : 0.0;
    for (int i = lane; i < nx; i += FB_NY) p.s[(size_t)l * nx + i] = qT[i];
    if (lane == 0) { p.dV[2 * l] = 0.0; p.dV[2 * l + 1] = 0.0; p.status[l] = 0; }
  WPAR_END
}

// W = P M over the tiles of nx x (nz + 1); column nz is a copy of s
FB_WARPFN void klqr_w(const DevLqr& p, int w) {
  const int nx = p.nx, nu = p.nu, nz = nx + nu, ncol = nz + 1;
  int i0, j0;
  const int l = lqr_tile(w, nx, ncol, &i0, &j0);
  if (p.status[l]) return;
  const double* P = p.P + (size_t)l * nx * nx;
  const float* A = p.A + ((size_t)l * p.T + p.t) * nx * nx;
  const float* B = p.B + ((size_t)l * p.T + p.t) * nx * nu;
  double* W = p.W + (size_t)l * nx * ncol;
  const int nr = nx - i0 < LQR_ROWS ? nx - i0 : LQR_ROWS;
  WPAR_BEGIN
    const int j = j0 + lane;
    if (j == nz) {
      for (int r = 0; r < nr; r++) W[(size_t)(i0 + r) * ncol + j] = p.s[(size_t)l * nx + i0 + r];
    } else if (j < nz) {
      const float* mc = j < nx ? A + j : B + (j - nx);
      const int ms = j < nx ? nx : nu;
      const double* pr[LQR_ROWS];
#pragma unroll
      for (int r = 0; r < LQR_ROWS; r++) pr[r] = P + (size_t)(r < nr ? i0 + r : i0) * nx;
      double acc[LQR_ROWS] = {};
      for (int c = 0; c < nx; c++) {
        const double m = mc[(size_t)c * ms];
#pragma unroll
        for (int r = 0; r < LQR_ROWS; r++) acc[r] = fma(pr[r][c], m, acc[r]);
      }
      for (int r = 0; r < nr; r++) W[(size_t)(i0 + r) * ncol + j] = acc[r];
    }
  WPAR_END
}

// H = M'W + diag(Q, R + mu), column nz + (q_t, r_t), over the tiles of nz x (nz + 1)
FB_WARPFN void klqr_h(const DevLqr& p, int w) {
  const int nx = p.nx, nu = p.nu, nz = nx + nu, ncol = nz + 1;
  int i0, j0;
  const int l = lqr_tile(w, nz, ncol, &i0, &j0);
  if (p.status[l]) return;
  const float* A = p.A + ((size_t)l * p.T + p.t) * nx * nx;
  const float* B = p.B + ((size_t)l * p.T + p.t) * nx * nu;
  const double* W = p.W + (size_t)l * nx * ncol;
  double* H = p.H + (size_t)l * nz * ncol;
  const int nr = nz - i0 < LQR_ROWS ? nz - i0 : LQR_ROWS;
  WPAR_BEGIN
    const int j = j0 + lane;
    if (j < ncol) {
      const float* mr[LQR_ROWS]; int ms[LQR_ROWS];      // column i0 + r of M
#pragma unroll
      for (int r = 0; r < LQR_ROWS; r++) {
        const int i = r < nr ? i0 + r : i0;
        mr[r] = i < nx ? A + i : B + (i - nx); ms[r] = i < nx ? nx : nu;
      }
      double acc[LQR_ROWS] = {};
      for (int c = 0; c < nx; c++) {
        const double x = W[(size_t)c * ncol + j];
#pragma unroll
        for (int r = 0; r < LQR_ROWS; r++) acc[r] = fma((double)mr[r][(size_t)c * ms[r]], x, acc[r]);
      }
      for (int r = 0; r < nr; r++) {
        const int i = i0 + r;
        double v = acc[r];
        if (i == j) v += i < nx ? p.Q[i] : p.R[i - nx] + p.mu[l];
        if (j == nz) v += i < nx ? p.q[((size_t)l * (p.T + 1) + p.t) * nx + i] : p.r[((size_t)l * p.T + p.t) * nu + i - nx];
        H[(size_t)i * ncol + j] = v;
      }
    }
  WPAR_END
}

// C C' = Quu (the lower triangle of H's block), column after column; a pivot that is not positive and finite stops the problem
FB_WARPFN void klqr_chol(const DevLqr& p, int l) {
  const int nx = p.nx, nu = p.nu, ncol = nx + nu + 1;
  if (p.status[l]) return;
  const double* Quu = p.H + (size_t)l * (nx + nu) * ncol + (size_t)nx * ncol + nx;
  double* C = p.C + (size_t)l * nu * nu;
  for (int j = 0; j < nu; j++) {
    WPAR_BEGIN
      if (lane == 0) {
        double d = Quu[(size_t)j * ncol + j];
        for (int c = 0; c < j; c++) d = fma(-C[j * nu + c], C[j * nu + c], d);
        C[j * nu + j] = d > 0.0 && d < HUGE_VAL ? sqrt(d) : 0.0;
      }
    WPAR_END
    const double cjj = C[j * nu + j];
    if (!(cjj > 0.0)) {
      WPAR_BEGIN if (lane == 0) p.status[l] = p.t + 1; WPAR_END
      return;
    }
    WPAR_BEGIN
      for (int i = j + 1 + lane; i < nu; i += FB_NY) {
        double v = Quu[(size_t)i * ncol + j];
        for (int c = 0; c < j; c++) v = fma(-C[i * nu + c], C[j * nu + c], v);
        C[i * nu + j] = v / cjj;
      }
    WPAR_END
  }
}

// lane j of a block of 32 columns of (Qux | Qu): X_j = -Quu^-1 b_j by the two triangular solves in place, G_j = Quu X_j + b_j; K_t and
// k_t to the outputs
FB_WARPFN void klqr_solve(const DevLqr& p, int w) {
  const int nx = p.nx, nu = p.nu, nz = nx + nu, ncol = nz + 1, ncx = nx + 1, ncb = (ncx + 31) / 32;
  const int l = w / ncb, j0 = (w % ncb) * 32;
  if (p.status[l]) return;
  const double* H = p.H + (size_t)l * nz * ncol;
  const double* C = p.C + (size_t)l * nu * nu;
  double* X = p.X + (size_t)l * nu * ncx;
  double* G = p.G + (size_t)l * nu * ncx;
  WPAR_BEGIN
    const int j = j0 + lane;
    if (j < ncx) {
      const int jh = j < nx ? j : nz;                   // the column of H: Qux_j, or Qu
      double* x = X + j;
      for (int u = 0; u < nu; u++) {
        double v = H[(size_t)(nx + u) * ncol + jh];
        for (int c = 0; c < u; c++) v = fma(-C[u * nu + c], x[(size_t)c * ncx], v);
        x[(size_t)u * ncx] = v / C[u * nu + u];
      }
      for (int u = nu - 1; u >= 0; u--) {
        double v = x[(size_t)u * ncx];
        for (int c = u + 1; c < nu; c++) v = fma(-C[c * nu + u], x[(size_t)c * ncx], v);
        x[(size_t)u * ncx] = v / C[u * nu + u];
      }
      const size_t lt = (size_t)l * p.T + p.t;
      for (int u = 0; u < nu; u++) {
        const double v = -x[(size_t)u * ncx];
        x[(size_t)u * ncx] = v;
        if (j < nx) p.K[(lt * nu + u) * nx + j] = v; else p.k[lt * nu + u] = v;
      }
      for (int u = 0; u < nu; u++) {
        double g = H[(size_t)(nx + u) * ncol + jh];
        const double* quu = H + (size_t)(nx + u) * ncol + nx;
        for (int c = 0; c < nu; c++) g = fma(quu[c], x[(size_t)c * ncx], g);
        G[(size_t)u * ncx + j] = g;
      }
    }
  WPAR_END
}

// over the tiles of nx x (nx + 1): V_ij = H_ij + sum_u X_ui G_uj + sum_u Qux_ui X_uj (column nx: Qx, k, Quu k + Qu), so P = sym(V) on
// columns < nx and s = column nx; the first tile's lane 0 adds the step's dV
FB_WARPFN void klqr_p(const DevLqr& p, int w) {
  const int nx = p.nx, nu = p.nu, nz = nx + nu, ncol = nz + 1, ncx = nx + 1;
  int i0, j0;
  const int l = lqr_tile(w, nx, ncx, &i0, &j0);
  if (p.status[l]) return;
  const double* H = p.H + (size_t)l * nz * ncol;
  const double* X = p.X + (size_t)l * nu * ncx;
  const double* G = p.G + (size_t)l * nu * ncx;
  double* P = p.P + (size_t)l * nx * nx;
  const int nr = nx - i0 < LQR_ROWS ? nx - i0 : LQR_ROWS;
  WPAR_BEGIN
    const int j = j0 + lane;
    if (j < ncx) {
      const int jh = j < nx ? j : nz;
      for (int r = 0; r < nr; r++) {
        const int i = i0 + r;
        double v = H[(size_t)i * ncol + jh];
        for (int u = 0; u < nu; u++) v = fma(X[(size_t)u * ncx + i], G[(size_t)u * ncx + j], v);
        for (int u = 0; u < nu; u++) v = fma(H[(size_t)(nx + u) * ncol + i], X[(size_t)u * ncx + j], v);
        if (j == nx) { p.s[(size_t)l * nx + i] = v; continue; }
        double vt = H[(size_t)j * ncol + i];
        for (int u = 0; u < nu; u++) vt = fma(X[(size_t)u * ncx + j], G[(size_t)u * ncx + i], vt);
        for (int u = 0; u < nu; u++) vt = fma(H[(size_t)(nx + u) * ncol + j], X[(size_t)u * ncx + i], vt);
        P[(size_t)i * nx + j] = 0.5 * (v + vt);
      }
    }
    if (i0 == 0 && j0 == 0 && lane == 0) {
      double d1 = 0.0, d2 = 0.0;
      for (int u = 0; u < nu; u++) {
        const double ku = X[(size_t)u * ncx + nx];
        double g = 0.0;
        for (int c = 0; c < nu; c++) g = fma(H[(size_t)(nx + u) * ncol + nx + c], X[(size_t)c * ncx + nx], g);
        d1 = fma(ku, H[(size_t)(nx + u) * ncol + nz], d1);
        d2 = fma(ku, g, d2);
      }
      p.dV[2 * l] += d1; p.dV[2 * l + 1] += 0.5 * d2;
    }
  WPAR_END
}

// ---- control-limited DDP (Tassa, Mansard & Todorov 2014; fb_lqr_box): klqr_chol and klqr_solve give way to
//   klqr_boxqp      k = argmin 1/2 x'Quu x + Qu'x subject to lower_t <= x <= upper_t, by the projected Newton method of Tassa's boxQP;
//                   C the Cholesky factor of the free block Quu_ff, with identity rows and columns on the clamped controls
//   klqr_solve_box  K = -Quu_ff^-1 Qux_f on the free rows, 0 on the clamped ones; X = (K | k) and G = Quu X + (Qux | Qu) as klqr_solve
// and klqr_p's general value update holds for that K and k as it is.  The bounds are on the control change du = u - ubar.
// boxQP's constants:
#define BOXQP_MAX_ITER 100       // Newton iterations
#define BOXQP_MIN_GRAD 1e-8      // stop when |g_free|_2 is below
#define BOXQP_MIN_REL 1e-8       // stop when an accepted step lowers the objective by less than this times |objective|
#define BOXQP_STEP_DEC 0.6       // the projected line search's step factor
#define BOXQP_MIN_STEP 1e-22     // the line search gives up below this step
#define BOXQP_ARMIJO 0.1         // accept a step when (f_try - f) / (step dx'g) >= this
// stop reasons (qp[1]), Tassa's numbering: -1 a free block that is not positive definite (status = t + 1), 0 no descent direction,
// 1 BOXQP_MAX_ITER iterations, 2 the line search gave up, 4 a small improvement, 5 a small free gradient, 6 every control clamped

struct DevLqrBox {
  const double *lower, *upper;              // [L][T][nu] bounds on du (+-inf allowed)
  int *clamped, *qp;                        // outputs: [L][T][nu] -1 at lower, +1 at upper, 0 free; [L][T][2] accepted steps, stop reason
  double *x, *dx, *g, *xt;                  // workspace per problem [nu]: the iterate, the Newton direction, the gradient, the trial point
  int* set;                                 // [nu] per problem: the clamped set C was last factored for (1 clamped)
};

// one problem step's QP: Quu and Qu in H's rows (stride ncol), its bounds, workspace and outputs
struct LqrQp {
  int nu, ncol;
  const double *Quu, *Qu, *lo, *hi;
  double *x, *dx, *g, *xt, *C;
  int *cl, *set;
};

// 1/2 x'Quu x + Qu'x: lane partials over rows, added in lane order (every lane returns the same value)
FB_WARPFN double boxqp_value(const LqrQp& q, const double* x) {
  LREG(double, part);
  WPAR_BEGIN
    double a = 0.0;
    for (int i = lane; i < q.nu; i += FB_NY) {
      const double* h = q.Quu + (size_t)i * q.ncol;
      double v = 0.0;
      for (int c = 0; c < q.nu; c++) v = fma(h[c], x[c], v);
      a = fma(x[i], fma(0.5, v, q.Qu[(size_t)i * q.ncol]), a);
    }
    L(part) = a;
  WPAR_END
  double f = 0.0;
  WPAR_BEGIN
    double sum = 0.0;
    for (int y = 0; y < FB_NY; y++) sum += SHF(part, y);
    f = sum;
  WPAR_END
  return f;
}

// g = Qu + Quu x and the clamped set at x (into cl) -> the number of free controls; *changed: the set differs from the factored one;
// *gsq: |g_free|^2
FB_WARPFN int boxqp_set(const LqrQp& q, bool* changed, double* gsq) {
  LREG(int, nf); LREG(int, ch); LREG(double, gs);
  WPAR_BEGIN
    int a = 0, b = 0;
    double s = 0.0;
    for (int i = lane; i < q.nu; i += FB_NY) {
      const double* h = q.Quu + (size_t)i * q.ncol;
      double v = q.Qu[(size_t)i * q.ncol];
      for (int c = 0; c < q.nu; c++) v = fma(h[c], q.x[c], v);
      q.g[i] = v;
      const double xi = q.x[i];
      const int c = xi == q.lo[i] && v > 0.0 ? -1 : xi == q.hi[i] && v < 0.0 ? 1 : 0;
      q.cl[i] = c;
      b |= (c != 0) != (q.set[i] != 0);
      if (c == 0) { a++; s = fma(v, v, s); }
    }
    L(nf) = a; L(ch) = b; L(gs) = s;
  WPAR_END
  int n = 0, d = 0;
  double s = 0.0;
  WPAR_BEGIN
    int a = 0, b = 0;
    double t = 0.0;
    for (int y = 0; y < FB_NY; y++) { a += SHF(nf, y); b |= SHF(ch, y); t += SHF(gs, y); }
    n = a; d = b; s = t;
  WPAR_END
  *changed = d != 0; *gsq = s;
  return n;
}

// C C' = the free block of Quu (klqr_chol's column order and arithmetic; identity rows and columns on clamped controls), and the set it
// was factored for -> false on a pivot that is not positive and finite
FB_WARPFN bool boxqp_factor(const LqrQp& q) {
  const int nu = q.nu;
  double* C = q.C;
  for (int j = 0; j < nu; j++) {
    const bool cj = q.cl[j] != 0;
    WPAR_BEGIN
      if (lane == 0) {
        double d = 1.0;
        if (!cj) {
          d = q.Quu[(size_t)j * q.ncol + j];
          for (int c = 0; c < j; c++) d = fma(-C[j * nu + c], C[j * nu + c], d);
          d = d > 0.0 && d < HUGE_VAL ? sqrt(d) : 0.0;
        }
        C[j * nu + j] = d;
      }
    WPAR_END
    const double cjj = C[j * nu + j];
    if (!(cjj > 0.0)) return false;
    WPAR_BEGIN
      for (int i = j + 1 + lane; i < nu; i += FB_NY) {
        double v = 0.0;
        if (!cj && q.cl[i] == 0) {
          v = q.Quu[(size_t)i * q.ncol + j];
          for (int c = 0; c < j; c++) v = fma(-C[i * nu + c], C[j * nu + c], v);
          v = v / cjj;
        }
        C[i * nu + j] = v;
      }
    WPAR_END
  }
  WPAR_BEGIN
    for (int i = lane; i < nu; i += FB_NY) q.set[i] = q.cl[i] != 0;
  WPAR_END
  return true;
}

// problem l's box QP at step p.t: k_t into the workspace's x, C, the clamped set and the QP record; a failed factor sets status = t + 1
FB_WARPFN void klqr_boxqp(const DevLqr& p, const DevLqrBox& b, int l) {
  if (p.status[l]) return;
  const int nx = p.nx, nu = p.nu, ncol = nx + nu + 1;
  const size_t lt = (size_t)l * p.T + p.t, ln = (size_t)l * nu;
  const double* Hu = p.H + (size_t)l * (nx + nu) * ncol + (size_t)nx * ncol;     // the rows of (Qux | Quu | Qu)
  const LqrQp q = {nu, ncol, Hu + nx, Hu + nx + nu, b.lower + lt * nu, b.upper + lt * nu, b.x + ln, b.dx + ln, b.g + ln, b.xt + ln,
                   p.C + ln * nu, b.clamped + lt * nu, b.set + ln};
  WPAR_BEGIN
    for (int i = lane; i < nu; i += FB_NY) { const double v = 0.0 < q.lo[i] ? q.lo[i] : 0.0; q.x[i] = v > q.hi[i] ? q.hi[i] : v; }
  WPAR_END
  double f = boxqp_value(q, q.x);
  int steps = 0, reason = 1;
  bool factored = false, changed;
  double gsq;
  LREG(double, sd);
  for (int it = 0; it < BOXQP_MAX_ITER; it++) {
    if (boxqp_set(q, &changed, &gsq) == 0) { reason = 6; break; }
    if (!factored || changed) {
      if (!boxqp_factor(q)) { reason = -1; break; }
      factored = true;
    }
    if (sqrt(gsq) < BOXQP_MIN_GRAD) { reason = 5; break; }
    // the Newton direction on the free controls, dx_f = -Quu_ff^-1 g_f (dx_c = 0), and dx'g
    WPAR_BEGIN
      if (lane == 0) {
        const double* C = q.C;
        for (int u = 0; u < nu; u++) {
          double v = q.cl[u] ? 0.0 : -q.g[u];
          for (int c = 0; c < u; c++) v = fma(-C[u * nu + c], q.dx[c], v);
          q.dx[u] = v / C[u * nu + u];
        }
        double s = 0.0;
        for (int u = nu - 1; u >= 0; u--) {
          double v = q.dx[u];
          for (int c = u + 1; c < nu; c++) v = fma(-C[c * nu + u], q.dx[c], v);
          q.dx[u] = v / C[u * nu + u];
        }
        for (int u = 0; u < nu; u++) s = fma(q.dx[u], q.g[u], s);
        L(sd) = s;
      }
    WPAR_END
    double sdotg = 0.0;
    WPAR_BEGIN sdotg = SHF(sd, 0); WPAR_END
    if (!(sdotg < 0.0)) { reason = 0; break; }
    // the projected Armijo search
    double step = 1.0, ft = 0.0;
    bool found = false;
    for (;;) {
      WPAR_BEGIN
        for (int i = lane; i < nu; i += FB_NY) {
          const double v = fma(step, q.dx[i], q.x[i]);
          q.xt[i] = v < q.lo[i] ? q.lo[i] : v > q.hi[i] ? q.hi[i] : v;
        }
      WPAR_END
      ft = boxqp_value(q, q.xt);
      if ((ft - f) / (step * sdotg) >= BOXQP_ARMIJO) { found = true; break; }
      step *= BOXQP_STEP_DEC;
      if (step < BOXQP_MIN_STEP) break;
    }
    if (!found) { reason = 2; break; }
    WPAR_BEGIN
      for (int i = lane; i < nu; i += FB_NY) q.x[i] = q.xt[i];
    WPAR_END
    const double f0 = f;
    f = ft;
    steps++;
    if (f0 - f < BOXQP_MIN_REL * fabs(f0)) { reason = 4; break; }
  }
  // the set at the final x, with the factor of its free block
  if (reason != -1) {
    boxqp_set(q, &changed, &gsq);
    if ((!factored || changed) && !boxqp_factor(q)) reason = -1;
  }
  WPAR_BEGIN
    if (lane == 0) {
      b.qp[2 * lt] = steps; b.qp[2 * lt + 1] = reason;
      if (reason == -1) p.status[l] = p.t + 1;
    }
  WPAR_END
}

// klqr_solve on the free block: lane j of a block of 32 columns of (Qux | Qu); the right-hand side is 0 on clamped rows, so with the
// masked factor those rows of K are 0; the k column is the QP's x; G_j = Quu X_j + b_j with the full Quu
FB_WARPFN void klqr_solve_box(const DevLqr& p, const DevLqrBox& b, int w) {
  const int nx = p.nx, nu = p.nu, nz = nx + nu, ncol = nz + 1, ncx = nx + 1, ncb = (ncx + 31) / 32;
  const int l = w / ncb, j0 = (w % ncb) * 32;
  if (p.status[l]) return;
  const size_t lt = (size_t)l * p.T + p.t;
  const double* H = p.H + (size_t)l * nz * ncol;
  const double* C = p.C + (size_t)l * nu * nu;
  const int* cl = b.clamped + lt * nu;
  double* X = p.X + (size_t)l * nu * ncx;
  double* G = p.G + (size_t)l * nu * ncx;
  WPAR_BEGIN
    const int j = j0 + lane;
    if (j < ncx) {
      const int jh = j < nx ? j : nz;
      double* x = X + j;
      if (j < nx) {
        for (int u = 0; u < nu; u++) {
          double v = cl[u] ? 0.0 : H[(size_t)(nx + u) * ncol + jh];
          for (int c = 0; c < u; c++) v = fma(-C[u * nu + c], x[(size_t)c * ncx], v);
          x[(size_t)u * ncx] = v / C[u * nu + u];
        }
        for (int u = nu - 1; u >= 0; u--) {
          double v = x[(size_t)u * ncx];
          for (int c = u + 1; c < nu; c++) v = fma(-C[c * nu + u], x[(size_t)c * ncx], v);
          x[(size_t)u * ncx] = v / C[u * nu + u];
        }
      }
      for (int u = 0; u < nu; u++) {
        const double v = j == nx ? b.x[(size_t)l * nu + u] : cl[u] ? 0.0 : -x[(size_t)u * ncx];
        x[(size_t)u * ncx] = v;
        if (j < nx) p.K[(lt * nu + u) * nx + j] = v; else p.k[lt * nu + u] = v;
      }
      for (int u = 0; u < nu; u++) {
        double g = H[(size_t)(nx + u) * ncol + jh];
        const double* quu = H + (size_t)(nx + u) * ncol + nx;
        for (int c = 0; c < nu; c++) g = fma(quu[c], x[(size_t)c * ncx], g);
        G[(size_t)u * ncx + j] = g;
      }
    }
  WPAR_END
}
