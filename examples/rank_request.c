/* rank_request.c - the reference's ranking request over the C ABI, in plain C99.
 *
 * What `RecForYouProcess.getRecList` + `callNeuralCFTFServing` do per request
 * (online/recprocess/RecForYouProcess.java:40-59,113-138: candidates -> scores from the model ->
 * sort -> cut to `size`) as ONE call into libsrs_ctr.so.  This is the body a JNI shim would wrap
 * (INTEGRATION.md section B); it is compiled and linked by tests/test_host_logic.py so that the
 * header stays usable from C, and it runs on a machine with an H100:
 *
 *   gcc -std=c99 -Iinclude examples/rank_request.c -Lsparrowrecsys_b200 -lsrs_ctr \
 *       -Wl,-rpath,$PWD/sparrowrecsys_b200 -o rank_request && ./rank_request
 *
 * The weights here are generated (uniform in +-0.05, the shape of the shipped modeldata/neuralcf
 * export: 1001 movies, 30001 users, E = 10, 20 -> 10 -> 10 -> 1); a server would read them from the
 * export's variables files (sparrowrecsys_b200/bundle.py shows the format).
 */
#include <stdio.h>
#include <stdlib.h>

#include "srs_ctr.h"

enum { N_MOVIES = 1001, N_USERS = 30001, E = 10, N_CAND = 800, SIZE = 10 };

static float* table(size_t n, unsigned* seed) {
  float* p = (float*)malloc(n * sizeof(float));
  size_t i;
  if (!p) return NULL;
  for (i = 0; i < n; ++i) {
    *seed = *seed * 1664525u + 1013904223u;
    p[i] = ((float)(*seed >> 8) / 16777216.0f - 0.5f) * 0.1f;
  }
  return p;
}

int main(void) {
  unsigned seed = 7u;
  srs_spec spec;
  srs_tensor w[8];
  srs_model* model = NULL;
  int32_t movie[N_CAND], user[N_CAND], top_idx[SIZE];
  float top_score[SIZE];
  srs_batch b;
  int i, rc;

  if (srs_abi_version() != SRS_ABI_VERSION) {
    fprintf(stderr, "header / library mismatch: %d vs %d\n", SRS_ABI_VERSION, srs_abi_version());
    return 2;
  }
  /* NeuralCF.py:45-53, 74: embedding size 10, hidden units [10, 10] */
  spec.kind = SRS_NEURALCF; spec.emb_dim = E; spec.n_movies = N_MOVIES; spec.n_users = N_USERS;
  spec.n_genres = 19; spec.hist_len = 5; spec.n_hidden = 2;
  spec.hidden[0] = 10; spec.hidden[1] = 10; spec.hidden[2] = 0; spec.hidden[3] = 0;
  spec.au_hidden = 32; spec.cross_buckets = 10000; spec.proj_dim = 64; spec.final_dense = 1;   /* (not read by this model) */

  /* named float tensors in the reference's own variable shapes (sparrowrecsys_b200/weights.py) */
  {
    static const char* names[8] = {"movieId_embedding", "userId_embedding", "dense_0/kernel", "dense_0/bias",
                                   "dense_1/kernel", "dense_1/bias", "dense_2/kernel", "dense_2/bias"};
    static const int64_t rows[8] = {N_MOVIES, N_USERS, 2 * E, 10, 10, 10, 10, 1};
    static const int64_t cols[8] = {E, E, 10, 1, 10, 1, 1, 1};
    for (i = 0; i < 8; ++i) {
      w[i].name = names[i]; w[i].rows = rows[i]; w[i].cols = cols[i]; w[i].location = SRS_HOST;
      w[i].data = table((size_t)(rows[i] * cols[i]), &seed);
      if (!w[i].data) return 2;
    }
  }
  rc = srs_model_create(&spec, w, 8, /*device=*/0, &model);
  if (rc != SRS_OK) {               /* no GPU, no CPU fallback: the call says so */
    fprintf(stderr, "srs_model_create: %s\n", srs_last_error());
    return 1;
  }

  /* one request: user 10351, the first 800 movies as candidates (RecForYouProcess.java:42-44) */
  for (i = 0; i < N_CAND; ++i) { movie[i] = i + 1; user[i] = 10351; }
  b.B = N_CAND; b.hist_stride = 0; b.movie_id = movie; b.user_id = user;
  b.hist = NULL; b.movie_genre = NULL; b.user_genre = NULL; b.numerics = NULL; b.hist16 = NULL;
  rc = srs_rank_host(model, &b, SIZE, top_idx, top_score);     /* forward + sort + cut on the GPU */
  if (rc != SRS_OK) {
    fprintf(stderr, "srs_rank_host: %s\n", srs_last_error());  /* e.g. SRS_ERR_RANGE for a bad id */
    srs_model_destroy(model);
    return 1;
  }
  printf("kernel %s; top %d of %d candidates:\n", srs_model_kernel_name(model), SIZE, N_CAND);
  for (i = 0; i < SIZE; ++i) printf("  movieId %4d  score %.6f\n", movie[top_idx[i]], top_score[i]);
  srs_model_destroy(model);
  for (i = 0; i < 8; ++i) free((void*)w[i].data);
  return 0;
}
