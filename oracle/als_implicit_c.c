/* als_implicit_c.c - oracle/als_implicit.py's implicit ALS half-step and RankingMetrics in plain C, for full runs
 * (DESIGN.md 4.17).
 *
 * THIS IS TEST / MEASUREMENT INFRASTRUCTURE, NOT PRODUCT.  Single-threaded.  Every floating-point statement rounds
 * once: build with -ffp-contract=off and without -ffast-math (oracle/als_implicit_cext.py does).  The loops are
 * reference BLAS / LAPACK's (dspr, daxpy, dpptrf, dpptrs) for the arguments ALS passes them. */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>

#define BLOCKS 10

/* dspr("U", k, alpha, x, ap): returns at once for alpha == 0; column j skipped for x(j) == 0 */
static void dspr(int k, double alpha, const double* x, double* ap) {
  if (alpha == 0.0) return;
  for (int j = 0, kk = 0; j < k; kk += j + 1, ++j) {
    if (x[j] == 0.0) continue;
    const double t = alpha * x[j];
    for (int i = 0; i <= j; ++i) ap[kk + i] = ap[kk + i] + x[i] * t;
  }
}

/* computeYtY over src [n][k] (raw ids ids[n], ascending): block b = the entities with id mod 10 == b, ascending,
 * each summed from zero with dspr(1.0); then out = ((0 + B[order[0]]) + B[order[1]]) + ...  out [k (k + 1) / 2].
 * Returns 0, or -2 when out of memory. */
int32_t srs_oracle_als_yty(const int32_t* ids, int32_t n, const float* src, int32_t k, const int32_t* order,
                           double* out) {
  const int nA = k * (k + 1) / 2;
  double* part = calloc((size_t)BLOCKS * nA, sizeof(double));
  double* x = malloc(sizeof(double) * (k > 0 ? k : 1));
  if (!part || !x) { free(part); free(x); return -2; }
  for (int32_t e = 0; e < n; ++e) {
    for (int i = 0; i < k; ++i) x[i] = (double)src[(size_t)e * k + i];
    dspr(k, 1.0, x, part + (size_t)(ids[e] % BLOCKS) * nA);
  }
  for (int i = 0; i < nA; ++i) out[i] = 0.0;
  for (int b = 0; b < BLOCKS; ++b)
    for (int i = 0; i < nA; ++i) out[i] = out[i] + 1.0 * part[(size_t)order[b] * nA + i];
  free(part); free(x);
  return 0;
}

/* One implicit half-step: entity e's ratings are src[off[e] .. off[e+1]) with ratings r; the source factors srcF
 * [nSrc][k] have raw ids src_ids.  ata = YtY, then per rating (c1 = alpha |r|) dspr(c1) and, for r > 0,
 * daxpy(1 + c1); lambda = reg * (ratings > 0).  dst [nE][k].  Returns -1, the first singular entity, or -2. */
int32_t srs_oracle_als_solve_implicit(const int32_t* off, const int32_t* src, const float* r, int32_t nE,
                                      const float* srcF, const int32_t* src_ids, int32_t nSrc, float* dstF,
                                      int32_t k, double reg, double alpha) {
  static const int32_t order[BLOCKS] = {0, 1, 2, 3, 4, 5, 6, 7, 8, 9};
  const int nA = k * (k + 1) / 2;
  double* yty = malloc(sizeof(double) * nA);
  double* ap = malloc(sizeof(double) * nA);
  double* b = malloc(sizeof(double) * k);
  double* x = malloc(sizeof(double) * k);
  if (!yty || !ap || !b || !x || srs_oracle_als_yty(src_ids, nSrc, srcF, k, order, yty)) {
    free(yty); free(ap); free(b); free(x);
    return -2;
  }
  int32_t bad = -1;
  for (int32_t e = 0; e < nE && bad < 0; ++e) {
    for (int i = 0; i < nA; ++i) ap[i] = 0.0 + 1.0 * yty[i];     /* reset, then merge(YtY) */
    for (int i = 0; i < k; ++i) b[i] = 0.0;
    int32_t n_pos = 0;
    for (int32_t p = off[e]; p < off[e + 1]; ++p) {
      const float* f = srcF + (size_t)src[p] * k;
      for (int i = 0; i < k; ++i) x[i] = (double)f[i];
      const double rv = (double)r[p];
      const double c1 = alpha * fabs(rv);
      if (rv > 0.0) ++n_pos;
      dspr(k, c1, x, ap);
      const double w = rv > 0.0 ? 1.0 + c1 : 0.0;
      if (w != 0.0)                                            /* daxpy(k, 1 + c1, x, b) */
        for (int i = 0; i < k; ++i) b[i] = b[i] + w * x[i];
    }
    const double lambda = (double)n_pos * reg;
    for (int j = 0; j < k; ++j) ap[j * (j + 1) / 2 + j] += lambda;
    for (int j = 0; j < k && bad < 0; ++j) {                   /* dpptrf("U") */
      const int jc = j * (j + 1) / 2;
      for (int jj = 0; jj < j; ++jj) {
        const int kj = jj * (jj + 1) / 2;
        double t = ap[jc + jj];
        for (int i = 0; i < jj; ++i) t = t - ap[kj + i] * ap[jc + i];
        ap[jc + jj] = t / ap[kj + jj];
      }
      double dd = 0.0;
      for (int i = 0; i < j; ++i) dd = dd + ap[jc + i] * ap[jc + i];
      const double ajj = ap[jc + j] - dd;
      if (!(ajj > 0.0)) bad = e;
      else ap[jc + j] = sqrt(ajj);
    }
    if (bad >= 0) break;
    for (int j = 0; j < k; ++j) {                              /* dpptrs("U") */
      const int jc = j * (j + 1) / 2;
      double t = b[j];
      for (int i = 0; i < j; ++i) t = t - ap[jc + i] * b[i];
      b[j] = t / ap[jc + j];
    }
    for (int j = k - 1; j >= 0; --j) {
      const int jc = j * (j + 1) / 2;
      if (b[j] != 0.0) {
        b[j] = b[j] / ap[jc + j];
        const double t = b[j];
        for (int i = j - 1; i >= 0; --i) b[i] = b[i] - t * ap[jc + i];
      }
    }
    for (int i = 0; i < k; ++i) dstF[(size_t)e * k + i] = (float)b[i];
  }
  free(yty); free(ap); free(b); free(x);
  return bad;
}

static int cmp_i32(const void* a, const void* b) {
  const int32_t x = *(const int32_t*)a, y = *(const int32_t*)b;
  return (x > y) - (x < y);
}

static int in_set(const int32_t* s, int n, int32_t v) {
  return bsearch(&v, s, (size_t)n, sizeof(int32_t), cmp_i32) != NULL;
}

/* RankingMetrics per query: out [3][n] = precision@k, NDCG@k, average precision; means [3] StatCounter's mean.
 * Returns 0, or -2 when out of memory. */
int32_t srs_oracle_ranking_metrics(const int32_t* pred, int32_t n, int32_t L, const int32_t* off,
                                   const int32_t* lab, int32_t k, double* out, double* means) {
  int32_t* s = malloc(sizeof(int32_t) * (off[n] > 0 ? off[n] : 1));
  if (!s) return -2;
  for (int32_t q = 0; q < n; ++q) {
    int m = 0;                                                /* the label set, sorted */
    const int cnt0 = off[q + 1] - off[q];
    for (int j = 0; j < cnt0; ++j) s[j] = lab[off[q] + j];
    qsort(s, (size_t)cnt0, sizeof(int32_t), cmp_i32);
    for (int j = 0; j < cnt0; ++j)
      if (j == 0 || s[j] != s[j - 1]) s[m++] = s[j];
    const int32_t* p = pred + (size_t)q * L;
    double prec = 0.0, ndcg = 0.0, ap = 0.0;
    if (m > 0) {
      const int np = L < k ? L : k;
      int cnt = 0;
      for (int i = 0; i < np; ++i) cnt += in_set(s, m, p[i]);
      prec = (double)cnt / (double)k;
      const int nn = (L > m ? L : m) < k ? (L > m ? L : m) : k;
      double dcg = 0.0, max_dcg = 0.0;
      for (int i = 0; i < nn; ++i) {
        const double gain = 1.0 / log((double)(i + 2));
        if (i < L && in_set(s, m, p[i])) dcg += gain;
        if (i < m) max_dcg += gain;
      }
      ndcg = dcg / max_dcg;
      double prec_sum = 0.0;
      cnt = 0;
      for (int i = 0; i < L; ++i)
        if (in_set(s, m, p[i])) {
          ++cnt;
          prec_sum += (double)cnt / (double)(i + 1);
        }
      ap = prec_sum / (double)m;
    }
    out[q] = prec;
    out[n + q] = ndcg;
    out[2 * n + q] = ap;
  }
  for (int v = 0; v < 3; ++v) {
    double mu = 0.0;
    for (int32_t q = 0; q < n; ++q) mu = mu + (out[(size_t)v * n + q] - mu) / (double)(q + 1);
    means[v] = n > 0 ? mu : NAN;
  }
  free(s);
  return 0;
}
