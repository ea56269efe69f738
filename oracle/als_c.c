/* als_c.c - oracle/als.py's ALS in plain C, for full runs (ALS.fit and recommendForAll, DESIGN.md 4.13).
 *
 * THIS IS TEST / MEASUREMENT INFRASTRUCTURE, NOT PRODUCT.  Single-threaded.  Every floating-point statement rounds
 * once: build with -ffp-contract=off and without -ffast-math (oracle/als_cext.py does), so no multiply-add is
 * fused.  The loops are reference BLAS / LAPACK's (dspr, daxpy, dpptrf, dpptrs, snrm2, sdot) for the arguments ALS
 * passes them. */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>

static uint64_t splitmix(uint64_t x, uint64_t i) {
  uint64_t z = x + (i + 1) * 0x9E3779B97F4A7C15ULL;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ULL;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBULL;
  return z ^ (z >> 31);
}

/* out [nU][rank]: user u's factor from nextGaussian's polar method on splitmix(splitmix(seed, id), c) uniforms,
 * each cast to float, times 1.0f / snrm2. */
void srs_oracle_als_init(const int32_t* ids, int32_t n, int32_t rank, uint64_t seed, float* out) {
  for (int32_t u = 0; u < n; ++u) {
    float* f = out + (size_t)u * rank;
    const uint64_t key = splitmix(seed, (uint64_t)(uint32_t)ids[u]);
    uint64_t c = 0;
    for (int d = 0; d < rank; d += 2) {
      double v1, v2, s;
      do {
        v1 = 2 * ((double)(splitmix(key, c++) >> 11) * 0x1p-53) - 1;
        v2 = 2 * ((double)(splitmix(key, c++) >> 11) * 0x1p-53) - 1;
        s = v1 * v1 + v2 * v2;
      } while (s >= 1 || s == 0);
      const double m = sqrt(-2 * log(s) / s);
      f[d] = (float)(v1 * m);
      if (d + 1 < rank) f[d + 1] = (float)(v2 * m);
    }
    float scale = 0.0f, ssq = 1.0f;
    for (int d = 0; d < rank; ++d) {
      if (f[d] == 0.0f) continue;
      const float a = fabsf(f[d]);
      if (scale < a) {
        const float t = scale / a;
        ssq = 1.0f + ssq * (t * t);
        scale = a;
      } else {
        const float t = a / scale;
        ssq = ssq + t * t;
      }
    }
    const float inv = 1.0f / (scale * sqrtf(ssq));
    for (int d = 0; d < rank; ++d) f[d] = f[d] * inv;
  }
}

/* One half-step: entity e's ratings are src[off[e] .. off[e+1]) with ratings r; dst [nE][k] = the solutions.
 * Returns -1, or the first entity (ascending) whose system has a pivot <= 0 or NaN; -2 when out of memory. */
int32_t srs_oracle_als_solve(const int32_t* off, const int32_t* src, const float* r, int32_t nE, const float* srcF,
                             float* dstF, int32_t k, double reg) {
  const int nA = k * (k + 1) / 2;
  double* ap = malloc(sizeof(double) * nA);
  double* b = malloc(sizeof(double) * k);
  double* x = malloc(sizeof(double) * k);
  if (!ap || !b || !x) { free(ap); free(b); free(x); return -2; }
  int32_t bad = -1;
  for (int32_t e = 0; e < nE && bad < 0; ++e) {
    for (int i = 0; i < nA; ++i) ap[i] = 0.0;
    for (int i = 0; i < k; ++i) b[i] = 0.0;
    for (int32_t p = off[e]; p < off[e + 1]; ++p) {
      const float* f = srcF + (size_t)src[p] * k;
      for (int i = 0; i < k; ++i) x[i] = (double)f[i];
      for (int j = 0, kk = 0; j < k; kk += j + 1, ++j) {       /* dspr("U", k, 1.0, x, ap) */
        if (x[j] == 0.0) continue;
        const double t = 1.0 * x[j];
        for (int i = 0; i <= j; ++i) ap[kk + i] = ap[kk + i] + x[i] * t;
      }
      const double rv = (double)r[p];
      if (rv != 0.0)                                          /* daxpy(k, rating, x, b) */
        for (int i = 0; i < k; ++i) b[i] = b[i] + rv * x[i];
    }
    const double lambda = (double)(off[e + 1] - off[e]) * reg;
    for (int j = 0; j < k; ++j) ap[j * (j + 1) / 2 + j] += lambda;
    /* dpptrf("U") */
    for (int j = 0; j < k && bad < 0; ++j) {
      const int jc = j * (j + 1) / 2;
      for (int jj = 0; jj < j; ++jj) {                        /* dtpsv("U", "T", "N", j, ap, ap + jc) */
        const int kj = jj * (jj + 1) / 2;
        double t = ap[jc + jj];
        for (int i = 0; i < jj; ++i) t = t - ap[kj + i] * ap[jc + i];
        ap[jc + jj] = t / ap[kj + jj];
      }
      double dd = 0.0;                                        /* ddot */
      for (int i = 0; i < j; ++i) dd = dd + ap[jc + i] * ap[jc + i];
      const double ajj = ap[jc + j] - dd;
      if (!(ajj > 0.0)) bad = e;
      else ap[jc + j] = sqrt(ajj);
    }
    if (bad >= 0) break;
    /* dpptrs("U"): dtpsv("U", "T", "N") then dtpsv("U", "N", "N") on b */
    for (int j = 0; j < k; ++j) {
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
  free(ap); free(b); free(x);
  return bad;
}

static int better(float sa, int32_t ia, float sb, int32_t ib) {
  const float ka = isnan(sa) ? -INFINITY : sa, kb = isnan(sb) ? -INFINITY : sb;
  return ka > kb || (ka == kb && ia < ib);
}

/* recommendForAll: per source the L best destinations (score desc, then position asc; NaN as -inf), by insertion
 * into a sorted list.  The score is sdot from 0.0f, d ascending. */
void srs_oracle_als_recommend(const float* src, int32_t n_src, const int32_t* dst_ids, const float* dst,
                              int32_t n_dst, int32_t k, int32_t L, int32_t* out_ids, float* out_scores) {
  int32_t* pos = malloc(sizeof(int32_t) * (L > 0 ? L : 1));
  for (int32_t s = 0; s < n_src; ++s) {
    float* sc = out_scores + (size_t)s * L;
    int cnt = 0;
    const float* a = src + (size_t)s * k;
    for (int32_t j = 0; j < n_dst; ++j) {
      const float* bj = dst + (size_t)j * k;
      float dot = 0.0f;
      for (int d = 0; d < k; ++d) dot = dot + a[d] * bj[d];
      if (cnt == L && !better(dot, j, sc[L - 1], pos[L - 1])) continue;
      int at = cnt < L ? cnt : L - 1;
      while (at > 0 && better(dot, j, sc[at - 1], pos[at - 1])) {
        sc[at] = sc[at - 1];
        pos[at] = pos[at - 1];
        --at;
      }
      sc[at] = dot;
      pos[at] = j;
      if (cnt < L) ++cnt;
    }
    for (int e = 0; e < L; ++e) out_ids[(size_t)s * L + e] = dst_ids[pos[e]];
  }
  free(pos);
}
