/* item2vec_c.c - oracle/item2vec.py's training loop in plain C, for full runs (Word2Vec.fit, DESIGN.md 4.12).
 *
 * THIS IS TEST / MEASUREMENT INFRASTRUCTURE, NOT PRODUCT.  Single-threaded; partitions run one after another, each
 * on its own copy of syn0 and syn1.  Every float statement rounds once: build with -ffp-contract=off and without
 * -ffast-math (oracle/item2vec_cext.py does), so no multiply-add is fused. */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define MAX_EXP 6
#define EXP_TABLE_SIZE 1000
#define MAX_CODE 40

static uint64_t splitmix(uint64_t x, uint64_t i) {
  uint64_t z = x + (i + 1) * 0x9E3779B97F4A7C15ULL;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ULL;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBULL;
  return z ^ (z >> 31);
}

/* words [N] vocabulary indices, offs [S + 1]; code [V][40], point [V][40], codelen [V]; exp_table [1000];
 * syn0 [V][D] in: the initial vectors, out: the trained ones.  Returns 0, or -1 when out of memory. */
int srs_oracle_item2vec_train(const int32_t* words, const int64_t* offs, int64_t n_sent, const int8_t* code,
                              const int32_t* point, const int32_t* codelen, const float* exp_table, int32_t V,
                              int32_t D, int32_t window, int32_t iterations, int32_t P, uint64_t seed,
                              int64_t train_words, double lr, float* syn0) {
  const size_t rows = (size_t)V * D;
  float* syn1 = calloc(rows, sizeof(float));
  float* l0 = malloc(rows * P * sizeof(float));
  float* l1 = malloc(rows * P * sizeof(float));
  unsigned char* m0 = malloc((size_t)V * P);
  unsigned char* m1 = malloc((size_t)V * P);
  float* neu1e = malloc(sizeof(float) * D);
  float* x0 = malloc(sizeof(float) * D);
  if (!syn1 || !l0 || !l1 || !m0 || !m1 || !neu1e || !x0) {
    free(syn1); free(l0); free(l1); free(m0); free(m1); free(neu1e); free(x0);
    return -1;
  }
  for (int k = 1; k <= iterations; ++k) {
    const uint64_t kk = splitmix(~seed, (uint64_t)k);
    for (int p = 0; p < P; ++p) {
      float* s0 = l0 + rows * p;
      float* s1 = l1 + rows * p;
      unsigned char* a0 = m0 + (size_t)V * p;
      unsigned char* a1 = m1 + (size_t)V * p;
      memcpy(s0, syn0, rows * sizeof(float));
      memcpy(s1, syn1, rows * sizeof(float));
      memset(a0, 0, V);
      memset(a1, 0, V);
      const uint64_t kp = splitmix(kk, (uint64_t)p);
      double alpha = lr;
      int64_t wc = 0, lwc = 0;
      for (int64_t i = p; i < n_sent; i += P) {
        if (wc - lwc > 10000) {
          lwc = wc;
          alpha = lr * (1 - ((double)P * (double)wc + (double)((int64_t)(k - 1) * train_words)) /
                                (double)((int64_t)iterations * train_words + 1));
          if (alpha < lr * 0.0001) alpha = lr * 0.0001;
        }
        const int64_t lo = offs[i], n = offs[i + 1] - offs[i];
        const int32_t* sent = words + lo;
        wc += n;
        for (int64_t pos = 0; pos < n; ++pos) {
          const int word = sent[pos];
          const int b = (int)((splitmix(kp, (uint64_t)(lo + pos)) >> 32) % (uint64_t)window);
          const int L = codelen[word];
          const int8_t* cd = code + (size_t)word * MAX_CODE;
          const int32_t* pt = point + (size_t)word * MAX_CODE;
          for (int a = b; a < window * 2 + 1 - b; ++a) {
            if (a == window) continue;
            const int64_t c = pos - window + a;
            if (c < 0 || c >= n) continue;
            const int last = sent[c];
            float* r0 = s0 + (size_t)last * D;
            for (int j = 0; j < D; ++j) { x0[j] = r0[j]; neu1e[j] = 0.0f; }
            for (int d = 0; d < L; ++d) {
              float* r1 = s1 + (size_t)pt[d] * D;
              float f = 0.0f;
              for (int j = 0; j < D; ++j) f = f + x0[j] * r1[j];
              if (f > -MAX_EXP && f < MAX_EXP) {
                const int ind = (int)((double)(f + (float)MAX_EXP) * (double)(EXP_TABLE_SIZE / MAX_EXP / 2.0));
                const float g = (float)((double)((float)(1 - cd[d]) - exp_table[ind]) * alpha);
                for (int j = 0; j < D; ++j) neu1e[j] = neu1e[j] + g * r1[j];
                for (int j = 0; j < D; ++j) r1[j] = r1[j] + g * x0[j];
                a1[pt[d]] = 1;
              }
            }
            for (int j = 0; j < D; ++j) r0[j] = r0[j] + neu1e[j];
            a0[last] = 1;
          }
        }
      }
    }
    /* merge: modified rows = their partitions' rows summed in partition order, times 1.0f / count */
    for (int t = 0; t < 2; ++t) {
      float* g = t ? syn1 : syn0;
      const float* loc = t ? l1 : l0;
      const unsigned char* mod = t ? m1 : m0;
      for (int r = 0; r < V; ++r) {
        int cnt = 0;
        for (int p = 0; p < P; ++p) {
          if (!mod[(size_t)V * p + r]) continue;
          const float* src = loc + rows * p + (size_t)r * D;
          if (cnt++ == 0) memcpy(neu1e, src, sizeof(float) * D);
          else for (int j = 0; j < D; ++j) neu1e[j] = neu1e[j] + src[j];
        }
        if (!cnt) continue;
        const float s = 1.0f / (float)cnt;
        for (int j = 0; j < D; ++j) g[(size_t)r * D + j] = neu1e[j] * s;
      }
    }
  }
  free(syn1); free(l0); free(l1); free(m0); free(m1); free(neu1e); free(x0);
  return 0;
}
