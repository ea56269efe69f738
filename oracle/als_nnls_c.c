/* als_nnls_c.c - oracle/als_nnls.py's nonnegative ALS half-step (NNLSSolver) in plain C, for full runs
 * (DESIGN.md 4.21).
 *
 * THIS IS TEST / MEASUREMENT INFRASTRUCTURE, NOT PRODUCT.  Single-threaded.  Every floating-point statement rounds
 * once: build with -ffp-contract=off and without -ffast-math (oracle/als_nnls_cext.py does).  The accumulation is
 * oracle/als_c.c's (explicit) or oracle/als_implicit_c.c's (implicit, from the YtY that its srs_oracle_als_yty
 * returns); the solve is NNLS.solve's loop with reference BLAS's ddot, dgemv "N" and daxpy for the arguments it
 * passes them. */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

/* ddot from 0, i ascending */
static double ddot(int n, const double* x, const double* y) {
  double s = 0.0;
  for (int i = 0; i < n; ++i) s = s + x[i] * y[i];
  return s;
}

/* dgemv("N", n, n, 1.0, a, n, x, 1, 0.0, y, 1): y = 0, then column j with x(j) != 0 adds (1.0 x(j)) a(:, j) */
static void dgemv(int n, const double* a, const double* x, double* y) {
  for (int i = 0; i < n; ++i) y[i] = 0.0;
  for (int j = 0; j < n; ++j) {
    if (x[j] == 0.0) continue;
    const double t = 1.0 * x[j];
    for (int i = 0; i < n; ++i) y[i] = y[i] + t * a[(size_t)j * n + i];
  }
}

/* daxpy(n, da, x, 1, y, 1): returns at once for da == 0 */
static void daxpy(int n, double da, const double* x, double* y) {
  if (da == 0.0) return;
  for (int i = 0; i < n; ++i) y[i] = y[i] + da * x[i];
}

static int stop(double step, double ndir, double nx) {
  return isnan(step) || step < 1e-7 || step > 1e40 || ndir < 1e-12 * nx || ndir < 1e-32;
}

/* steplen(d, res) = ddot(d, res) / (ddot(A d, d) + 1e-20); scratch [n] */
static double steplen(int n, const double* ata, const double* d, const double* res, double* scratch) {
  const double top = ddot(n, d, res);
  dgemv(n, ata, d, scratch);
  return top / (ddot(n, scratch, d) + 1e-20);
}

/* NNLS.solve(ata [n][n], atb [n]) into x [n]; ws [5 n].  Returns the iterations run (iterMax: never stopped). */
static int32_t nnls(int n, const double* ata, const double* atb, double* x, double* ws) {
  double *grad = ws, *dir = ws + n, *last_dir = ws + 2 * n, *res = ws + 3 * n, *scratch = ws + 4 * n;
  for (int i = 0; i < 5 * n; ++i) ws[i] = 0.0;
  for (int i = 0; i < n; ++i) x[i] = 0.0;
  const int iter_max = n * 20 > 400 ? n * 20 : 400;
  double last_norm = 0.0;
  int iterno = 0, last_wall = 0;
  while (iterno < iter_max) {
    dgemv(n, ata, x, res);
    daxpy(n, -1.0, atb, res);
    memcpy(grad, res, sizeof(double) * n);
    for (int i = 0; i < n; ++i)
      if (grad[i] > 0.0 && x[i] == 0.0) grad[i] = 0.0;
    const double ngrad = ddot(n, grad, grad);
    memcpy(dir, grad, sizeof(double) * n);
    double step = steplen(n, ata, grad, res, scratch);
    double ndir = 0.0;
    const double nx = ddot(n, x, x);
    if (iterno > last_wall + 1) {
      const double alpha = ngrad / last_norm;
      daxpy(n, alpha, last_dir, dir);
      const double dstep = steplen(n, ata, dir, res, scratch);
      ndir = ddot(n, dir, dir);
      if (stop(dstep, ndir, nx)) {
        memcpy(dir, grad, sizeof(double) * n);
        ndir = ddot(n, dir, dir);
      } else {
        step = dstep;
      }
    } else {
      ndir = ddot(n, dir, dir);
    }
    if (stop(step, ndir, nx)) return iterno;
    for (int i = 0; i < n; ++i)
      if (step * dir[i] > x[i]) step = x[i] / dir[i];
    for (int i = 0; i < n; ++i) {
      if (step * dir[i] > x[i] * (1 - 1e-14)) {
        x[i] = 0.0;
        last_wall = iterno;
      } else {
        x[i] = x[i] - step * dir[i];
      }
    }
    ++iterno;
    memcpy(last_dir, dir, sizeof(double) * n);
    last_norm = ngrad;
  }
  return iterno;
}

/* One half-step with NNLSSolver: entity e's ratings are src[off[e] .. off[e+1]) with ratings r over the source
 * factors srcF.  yty null: explicit (ata from 0, dspr(1.0) and daxpy(r) per rating, lambda = reg * count); else
 * implicit from the packed YtY [k (k + 1) / 2] (dspr(alpha |r|), daxpy(1 + alpha |r|) for r > 0, lambda = reg *
 * (ratings > 0)).  fillAtA, NNLS.solve, toFloat -> dst [nE][k]; iters [nE], when not null, the NNLS iterations.
 * Returns 0, or -2 when out of memory. */
int32_t srs_oracle_als_solve_nnls(const int32_t* off, const int32_t* src, const float* r, int32_t nE,
                                  const float* srcF, const double* yty, float* dstF, int32_t k, double reg,
                                  double alpha, int32_t* iters) {
  const int nA = k * (k + 1) / 2;
  double* ap = malloc(sizeof(double) * nA);
  double* b = malloc(sizeof(double) * k);
  double* x = malloc(sizeof(double) * k);
  double* ata = malloc(sizeof(double) * k * k);
  double* sol = malloc(sizeof(double) * k);
  double* ws = malloc(sizeof(double) * 5 * k);
  if (!ap || !b || !x || !ata || !sol || !ws) {
    free(ap); free(b); free(x); free(ata); free(sol); free(ws);
    return -2;
  }
  for (int32_t e = 0; e < nE; ++e) {
    for (int i = 0; i < nA; ++i) ap[i] = yty ? 0.0 + 1.0 * yty[i] : 0.0;
    for (int i = 0; i < k; ++i) b[i] = 0.0;
    int32_t n = 0;
    for (int32_t p = off[e]; p < off[e + 1]; ++p) {
      const float* f = srcF + (size_t)src[p] * k;
      for (int i = 0; i < k; ++i) x[i] = (double)f[i];
      const double rv = (double)r[p];
      const double c = yty ? alpha * fabs(rv) : 1.0;             /* dspr's scalar */
      const double w = yty ? (rv > 0.0 ? 1.0 + c : 0.0) : rv;     /* daxpy's scalar */
      n += yty ? rv > 0.0 : 1;
      if (c != 0.0)
        for (int j = 0, kk = 0; j < k; kk += j + 1, ++j) {
          if (x[j] == 0.0) continue;
          const double t = c * x[j];
          for (int i = 0; i <= j; ++i) ap[kk + i] = ap[kk + i] + x[i] * t;
        }
      if (w != 0.0)
        for (int i = 0; i < k; ++i) b[i] = b[i] + w * x[i];
    }
    const double lambda = (double)n * reg;
    for (int i = 0, pos = 0; i < k; ++i) {                       /* fillAtA */
      for (int j = 0; j <= i; ++j, ++pos) {
        ata[i * k + j] = ap[pos];
        ata[j * k + i] = ap[pos];
      }
      ata[i * k + i] += lambda;
    }
    const int32_t it = nnls(k, ata, b, sol, ws);
    if (iters) iters[e] = it;
    for (int i = 0; i < k; ++i) dstF[(size_t)e * k + i] = (float)sol[i];
  }
  free(ap); free(b); free(x); free(ata); free(sol); free(ws);
  return 0;
}
