/*
 * srs_ctr.h - C ABI of the H100-native SparrowRecSys CTR ranking forward path.
 *
 * The reference has no FFI: its hot path is `model.predict(feature_dict)` on a
 * Keras graph (TFRecModel/src/com/sparrowrecsys/offline/tensorflow/<Model>.py) and, at
 * serve time, the same graph behind TF-Serving's REST `:predict`
 * (src/main/java/com/sparrowrecsys/online/recprocess/RecForYouProcess.java:113-138).
 * This header is the boundary a maintainer binds instead (ctypes stub in
 * sparrowrecsys_b200/_lib.py, JNI sketch in INTEGRATION.md).  Each entry point
 * cites the reference interface it replaces.
 *
 * Conventions: plain pointers and sizes only; every function returns SRS_OK (0)
 * or a negative error code and never throws across the ABI; srs_last_error()
 * gives the message of the last failure on the calling thread.  The caller owns
 * all input/output buffers; the library owns its device copy of the weights.
 */
#ifndef SRS_CTR_H_
#define SRS_CTR_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SRS_ABI_VERSION 4

enum srs_status {
  SRS_OK = 0,
  SRS_ERR_INVALID = -1,     /* bad argument / unsupported spec                   */
  SRS_ERR_MISSING = -2,     /* a required weight tensor was not supplied         */
  SRS_ERR_SHAPE = -3,       /* a weight tensor has the wrong shape               */
  SRS_ERR_CUDA = -4,        /* CUDA runtime failure (message has the cudaError)  */
  SRS_ERR_RANGE = -5,       /* an id in the batch is outside its vocabulary:     */
                            /* mirrors TF's assert_less_than_num_buckets         */
  SRS_ERR_NOMEM = -6
};

/* Model families = the reference's model scripts. */
enum srs_model_kind {
  SRS_EMBEDDINGMLP = 0,     /* EmbeddingMLP.py:72-77                             */
  SRS_WIDENDEEP = 1,        /* WideNDeep.py:101-108                              */
  SRS_NEURALCF = 2,         /* NeuralCF.py:45-53  (neural_cf_model_1)            */
  SRS_TWOTOWERS = 3,        /* NeuralCF.py:57-70  (neural_cf_model_2)            */
  SRS_DEEPFM = 4,           /* DeepFM.py:91-113                                  */
  SRS_DEEPFM_V2 = 5,        /* DeepFM_v2.py:98-155                               */
  SRS_DIN = 6,              /* DIN.py:125-167                                    */
  SRS_DIEN = 7              /* DIEN.py:154-256 (y_pred; AUGRU initial state is the  */
                            /* stored tensor "augru_h0", emb_dim <= 32)            */
};

/* Hyper-parameters the reference hard-codes as module constants
 * (DIN.py:30-31,66,132; EmbeddingMLP.py:50-58; NeuralCF.py:74). */
typedef struct srs_spec {
  int32_t kind;             /* enum srs_model_kind                               */
  int32_t emb_dim;          /* E                                                 */
  int32_t n_movies;         /* num_buckets of movieId (valid ids 0..n-1)         */
  int32_t n_users;          /* num_buckets of userId                             */
  int32_t n_genres;         /* 19                                                */
  int32_t hist_len;         /* T (DIN, DIEN); W&D reads history slot 0 only      */
  int32_t n_hidden;         /* entries used in hidden[]                          */
  int32_t hidden[4];        /* MLP widths, model dependent                       */
  int32_t au_hidden;        /* DIN activation-unit / DIEN attention width (32)   */
  int32_t cross_buckets;    /* W&D hash_bucket_size (10000)                      */
  int32_t proj_dim;         /* DeepFM_v2 field projection width (64)             */
  int32_t final_dense;      /* two towers: Dense(1,sigmoid) after the dot        */
} srs_spec;

enum srs_location { SRS_HOST = 0, SRS_DEVICE_BORROWED = 1 };

/* One weight tensor in the reference's own (Keras variable) shape: Dense kernels
 * [in,out], tables [buckets,E], vectors [n] as rows=n, cols=1.  Names are the
 * canonical ones of sparrowrecsys_b200/weights.py (SURVEY.md appendix A).
 * SRS_DEVICE_BORROWED: `data` is a device pointer on the model's device that the
 * library uses in place (no copy; must outlive the model; only for embedding
 * tables whose emb_dim is a multiple of 4) - this is how a 25.6 GB table is
 * handed over without a host round trip. */
typedef struct srs_tensor {
  const char* name;
  const float* data;
  int64_t rows;
  int64_t cols;
  int32_t location;         /* enum srs_location                                 */
} srs_tensor;

/* One batch of ranking instances, structure-of-arrays.  Replaces the feature
 * dict handed to `model.predict` (keys of the Keras `inputs` dicts, e.g.
 * DIN.py:34-59) / the `instances` array of the TF-Serving request
 * (RecForYouProcess.java:118-127).  Genre strings are already vocabulary indices
 * (-1 = missing / out of vocabulary -> zero vector), integer numerics already
 * cast to float32 (what numeric_column does).  Pointers a model does not read may
 * be NULL.  All pointers are host pointers for srs_predict_host* and device
 * pointers (on the model's device) for srs_predict_device.
 * Fast path for host batches: when the arrays lie back to back in memory in the order
 * movie_id, user_id, hist (hist_stride == T), movie_genre, user_genre, numerics (arrays the
 * model does not read left out), srs_predict_host* moves the whole batch with ONE
 * host-to-device copy instead of one per array. */
typedef struct srs_batch {
  int32_t B;                   /* rows                                            */
  int32_t hist_stride;         /* elements between consecutive rows of `hist`     */
  const int32_t* movie_id;     /* [B]                                             */
  const int32_t* user_id;      /* [B]                                             */
  const int32_t* hist;         /* [B, T] userRatedMovie<k> in graph position order */
  const int32_t* movie_genre;  /* [B, 3] movieGenre1..3                           */
  const int32_t* user_genre;   /* [B, 5] userGenre1..5                            */
  const float* numerics;       /* [B, 7] movieAvgRating, movieRatingCount,
                                  movieRatingStddev, releaseYear, userAvgRating,
                                  userRatingCount, userRatingStddev               */
  const uint16_t* hist16;      /* host batches only, optional: the history ids as uint16
                                  [B, T] (same stride and order as `hist`, which is then
                                  ignored) for vocabularies of at most 65536 movies - the
                                  history is most of a DIN batch, so this halves the bytes
                                  that cross PCIe; widened to int32 on the device.  In the
                                  packed layout it takes the place of `hist`, padded to a
                                  multiple of 4 bytes.  NULL otherwise.                 */
} srs_batch;

typedef struct srs_model srs_model;

int srs_abi_version(void);

/* Message of the last error raised on this thread ("" if none). */
const char* srs_last_error(void);

/* Build a model on CUDA device `device`: validates names/shapes against `spec`,
 * copies (and privately re-lays-out) the weights into HBM.  Replaces building
 * the module-level Keras `model` and loading its variables (e.g. DIN.py:169,
 * NeuralCF.py:74 + the SavedModel under webroot/modeldata/). */
int srs_model_create(const srs_spec* spec, const srs_tensor* tensors, int32_t n_tensors,
                     int32_t device, srs_model** out);

/* Same, with kernel-variant options "key=value;key=value": din_impl = tc | cudacore,
 * embmlp_impl / deepfm_impl = tc | cudacore, zero_copy_scores = 0 | 1.  Unknown keys are ignored; a
 * forced variant that does not support the shape makes the call fail.  NULL / "" = the defaults
 * (which srs_model_kernel_name reports).  The environment variables SRS_DIN_IMPL, SRS_EMBMLP_IMPL,
 * SRS_DEEPFM_IMPL, SRS_ZERO_COPY_SCORES are read only for keys the string does not set. */
int srs_model_create_ex(const srs_spec* spec, const srs_tensor* tensors, int32_t n_tensors,
                        int32_t device, const char* options, srs_model** out);

void srs_model_destroy(srs_model* m);

/* Forward pass with everything resident in HBM; asynchronous on `stream`
 * (a cudaStream_t; NULL = the default stream).  `probs` [B] receives the model
 * output (sigmoid probability; raw dot for two towers without final dense);
 * `logits` [B] (may be NULL) receives the pre-sigmoid value.  Replaces the
 * compiled forward that `model.predict` runs per batch (e.g. DIN.py:185).
 * Out-of-range ids are read as id 0 and latch an error flag that
 * srs_model_status() reports. */
int srs_predict_device(srs_model* m, const srs_batch* batch, float* probs, float* logits,
                       void* stream);

/* ---- One ranking call that spans the GPUs of a box (RecForYouProcess.java:56-59,92-94 with the
 * candidate list sharded by rows, SURVEY.md section 8e): every rank needs every rank's scores.
 * Instead of kernel + all-gather, each rank's forward kernel stores its scores into its slice of
 * EVERY rank's gather buffer over NVLink (CUDA IPC peer mappings), followed by one flag word per
 * rank.  One process per GPU; `slice_rows` = rows per rank (the last rank may score fewer).
 *   1. every rank: srs_gather_create, srs_gather_export -> 64-byte handle
 *   2. exchange the handles (torch.distributed / MPI / a pipe), every rank: srs_gather_connect with
 *      the world x 64 bytes in rank order
 *   3. per call: srs_predict_device_gather (asynchronous on `stream`), then srs_gather_wait on the
 *      stream that consumes the scores, then srs_gather_scores for the device pointer of the full
 *      [world * slice_rows] vector (valid until the call after the next one: two buffers alternate).
 * Every rank must make the same sequence of calls.  The step counters live on the device, so a
 * sequence of an EVEN number of predict / wait pairs can be captured in a CUDA graph and replayed
 * (the buffer parity of each pair is fixed at capture). */
typedef struct srs_gather srs_gather;
int srs_gather_create(int32_t device, int32_t world, int32_t rank, int64_t slice_rows, srs_gather** out);
int srs_gather_export(srs_gather* g, void* handle64);
int srs_gather_connect(srs_gather* g, const void* handles /* world * 64 bytes, rank order */);
void srs_gather_destroy(srs_gather* g);
int srs_predict_device_gather(srs_model* m, const srs_batch* batch, srs_gather* g, void* stream);
int srs_gather_wait(srs_gather* g, void* stream);
int srs_gather_scores(srs_gather* g, float** scores, int64_t* rows);
/* copy the gathered vector of the latest call to `dst` (device or host memory), asynchronous on `stream` */
int srs_gather_copy_scores(srs_gather* g, float* dst, int32_t dst_on_host, void* stream);

/* Forward pass from host buffers: H2D of the batch, kernel, D2H of the scores,
 * synchronous.  This is the drop-in for `model.predict(dict) -> float32[B,1]`
 * and for one TF-Serving `:predict` call.  Returns SRS_ERR_RANGE if an id was
 * out of range (outputs are still written). */
int srs_predict_host(srs_model* m, const srs_batch* batch, float* probs, float* logits);

/* A whole dataset in batches, the way `model.predict(dataset)` iterates it (e.g.
 * DIN.py:185 over make_csv_dataset batches): batch i is copied in, scored and copied out
 * on internal slot i % srs_num_slots(), so the PCIe copies of one batch overlap the kernel
 * of another.  Synchronous; probs[i] (and logits[i] if `logits` != NULL) receive batch i.
 * Host buffers should be pinned for the copies to overlap.  Not to be mixed concurrently
 * with srs_predict_host_async on the same model. */
int srs_predict_host_batches(srs_model* m, int32_t n_batches, const srs_batch* batches,
                             float* const* probs, float* const* logits);

/* Pipelined variant: enqueue on one of srs_num_slots() internal slots (each with
 * its own stream and device staging) and return; srs_wait_slot() blocks until that
 * slot's scores are in `probs`.  Host buffers must stay valid (and should be
 * pinned for the copies to overlap) until the wait returns. */
int srs_num_slots(void);
int srs_predict_host_async(srs_model* m, int32_t slot, const srs_batch* batch, float* probs,
                           float* logits);
int srs_wait_slot(srs_model* m, int32_t slot);

/* Synchronises the device and reports SRS_ERR_RANGE if any kernel since the last
 * call saw an out-of-range id, SRS_ERR_CUDA on a sticky CUDA error. */
int srs_model_status(srs_model* m);

/* Algorithmic bytes per inference of this model (SURVEY.md section 8d definition). */
int64_t srs_model_bytes_per_inference(const srs_model* m);

/* Name of the kernel variant srs_predict_* dispatches to for this model.  DIN has two
 * (din_wg_kernel: activation unit - and for emb_dim <= 32 the top MLP - on warpgroup MMAs, the
 * default for 16 < emb_dim <= 64 and hist_len > 8; din_kernel: CUDA cores, every other shape); the
 * choice follows the shape and can be forced with the environment variable SRS_DIN_IMPL = tc | cudacore read by
 * srs_model_create (a forced variant that does not support the shape makes srs_model_create fail).
 * SRS_EMBMLP_IMPL and SRS_DEEPFM_IMPL (tc | cudacore) do the same for EmbeddingMLP / Wide&Deep
 * and DeepFM. */
const char* srs_model_kernel_name(const srs_model* m);

/* Limit the persistent tensor-core kernels of this model (din_wg / embmlp_tc / deepfm_tc) to at most
 * n_sms CTAs per launch (n_sms <= 0: every SM of the device, the default).  A launch then leaves the
 * other SMs to launches of other streams.  Takes effect at the next srs_predict_* call; results
 * do not depend on it. */
int srs_model_set_sm_limit(srs_model* m, int32_t n_sms);

/* Number of kernels this library has launched in this process (all models). */
int64_t srs_launch_count(void);

/* Deterministic counter-based fill of a device float buffer:
 * x[i] = lo + (hi-lo) * u(seed, i), u in [0,1) from a splitmix64 hash of (seed, i).
 * Used to initialise synthetic embedding tables in place (BASELINE cfg 5). */
int srs_fill_uniform(float* device_ptr, int64_t n, uint64_t seed, float lo, float hi,
                     int32_t device, void* stream);

/* Batched cosine similarity of one query embedding against n candidates
 * (online/model/Embedding.java:33-47, used by SimilarMovieProcess.java:121-137
 * and RecForYouProcess.java:93-105).  Device pointers. */
int srs_cosine_scores_device(const float* query, const float* cands, int32_t n, int32_t dim,
                             float* scores, int32_t device, void* stream);

/* Ranking tail of both online rankers: order n candidate scores descending and return the
 * first min(k, n) positions (and, if top_scores != NULL, their scores).  Replaces
 * `candidateScoreMap.entrySet().stream().sorted(comparingByValue(reverseOrder()))` +
 * `subList(0, size)` (RecForYouProcess.java:56-59,92-94; SimilarMovieProcess.java:26-31,
 * 133-135).  Order of Double.compareTo: NaN ranks first, -0.0 after 0.0; equal scores - in
 * HashMap iteration order in the reference, i.e. unspecified - rank by position, lower
 * first.  Device pointers; asynchronous on `stream`. */
int srs_topk_device(const float* scores, int32_t n, int32_t k, int32_t* top_idx,
                    float* top_scores, int32_t device, void* stream);

/* One ranking call from host buffers: H2D of the candidate batch, forward kernel, ranking
 * kernel, D2H of the min(k, B) best positions and scores only.  Replaces
 * RecForYouProcess.ranker (:69-95) with model "nerualcf" followed by getRecList's subList:
 * the score vector never leaves the device.  Synchronous; SRS_ERR_RANGE as srs_predict_host. */
int srs_rank_host(srs_model* m, const srs_batch* batch, int32_t k, int32_t* top_idx,
                  float* top_scores);

/* ---- One ranking request "one user x n candidates" with the movie-side features resident in HBM.
 * The reference defines the serving feature store as Redis hashes `uf:<userId>` / `mf:<movieId>`
 * (FeatureEngForRecModel.scala:130-174,208-259; read at RecForYouProcess.java:46-52 and
 * DataManager.java:127-140).  srs_model_set_movie_features uploads the `mf:` side once: genres
 * [n_movies][3] as vocabulary indices (-1 = missing), numerics [n_movies][4] = movieAvgRating,
 * movieRatingCount, movieRatingStddev, releaseYear (already cast to float32).  A request then ships
 * one srs_user_row and n candidate ids - (9 + T + n) words instead of n full feature rows - and a
 * device kernel expands them into the batch the forward kernel reads (user columns broadcast, movie
 * columns gathered by candidate id).  srs_rank_user_host = that + forward + sort-and-cut
 * (RecForYouProcess.java:56-59), D2H of the best k positions / scores (and all n scores if
 * `probs` != NULL).  Candidate ids outside the table or the model's vocabulary give SRS_ERR_RANGE. */
typedef struct srs_user_row {
  int32_t user_id;
  int32_t user_genre[5];       /* userGenre1..5 vocabulary indices, -1 = missing                        */
  float user_numerics[3];      /* userAvgRating, userRatingCount, userRatingStddev                      */
  int32_t n_hist;              /* entries of `hist` (<= the model's history columns; the rest is id 0)  */
  const int32_t* hist;         /* userRatedMovie1.. in graph position order (most recent first)         */
} srs_user_row;
int srs_model_set_movie_features(srs_model* m, int32_t n_movies, const int32_t* genres,
                                 const float* numerics);
int srs_rank_user_host(srs_model* m, const srs_user_row* user, const int32_t* candidate_movie_ids,
                       int32_t n, int32_t k, int32_t* top_idx, float* top_scores, float* probs);

/* ---- `model.evaluate(dataset)`: the four numbers every CTR script of the reference prints
 * (loss='binary_crossentropy', metrics=['accuracy', AUC(curve='ROC'), AUC(curve='PR')],
 * e.g. DIN.py:171-185, EmbeddingMLP.py:80-91, NeuralCF.py:77-88), with Keras's (TF 2.0) semantics:
 *   loss      mean over rows of the logit-path sigmoid cross-entropy max(x,0) - x*z + log1p(exp(-|x|)),
 *             each row in float32 (for a sigmoid output layer Keras does not clip the probability);
 *   accuracy  binary_accuracy: label == (p > 0.5);
 *   roc_auc, pr_auc   AUC(num_thresholds=200, summation_method='interpolation'): p counts as positive at
 *             threshold t when float32(p) > t; PR by interpolate_pr_auc (Davis & Goadrich).  The
 *             TP/FP/TN/FN counts are exact 64-bit integers (Keras keeps them in float32, which is exact
 *             only up to 2^24 rows).  A single-class input gives an AUC of 0.
 * Labels must be 0 or 1 and probabilities in [0, 1] (Keras asserts this): anything else latches the
 * state's error word and the result call returns SRS_ERR_INVALID. */
typedef struct srs_eval_result {
  int64_t rows, positives, correct;
  double loss, accuracy, roc_auc, pr_auc;
} srs_eval_result;

/* Device-resident metric state on one device: 2 x 201 (label, threshold bin) counts, the correct rows,
 * the loss sum and the error word.  Updates are asynchronous and can be captured in a CUDA graph; the
 * updates of one state must be ordered (one stream, or streams joined by events).  The loss is summed
 * in a fixed order, so it has the same bits on every run over the same batches. */
typedef struct srs_metrics srs_metrics;
int srs_metrics_create(int32_t device, srs_metrics** out);
void srs_metrics_destroy(srs_metrics* mt);
/* zero the state, asynchronous on `stream` */
int srs_metrics_reset(srs_metrics* mt, void* stream);
/* fold n >= 1 rows of device buffers (probs, logits [n] float32, labels [n] int32) into the state,
 * asynchronous on `stream` */
int srs_metrics_update_device(srs_metrics* mt, const float* probs, const float* logits,
                              const int32_t* labels, int32_t n, void* stream);
/* synchronise the device and summarise: AUCs computed on the host in double from the counts.
 * `confusion`: NULL or int64[4][200] = tp, fp, tn, fn per threshold.  SRS_ERR_INVALID if an update saw
 * a bad label or probability (the error stays until srs_metrics_reset) or if no row was folded. */
int srs_metrics_result(srs_metrics* mt, srs_eval_result* out, int64_t* confusion);

/* ---- Keras's sample weights (DESIGN.md section 4.28).  Row i carries a weight w_i >= 0, finite (a negative, NaN
 * or infinite weight gives SRS_ERR_INVALID before any launch).  With weights, srs_eval_result's rows, positives and
 * correct stay integer counts and its four doubles become Keras's weighted metrics:
 *   loss      sum_i w_i l_i / rows (SUM_OVER_BATCH_SIZE: the row count, not the weights' sum), w_i l_i in float32;
 *   accuracy  sum_i w_i [row i correct] / sum_i w_i, 0 when the weights sum to 0;
 *   roc_auc, pr_auc   the same thresholds and formulas, TP/FP/TN/FN the sums of the rows' weights in double.
 * The sums have a fixed order and use no float atomics: the same rows give the same bits on every run and every
 * SM count.  All-ones weights give the unweighted result's bits. */

/* srs_metrics_update_device with weights [n] float32 on the device.  A state folds either weighted or unweighted
 * rows between resets (mixing gives SRS_ERR_INVALID); srs_metrics_result then reports the weighted metrics, and its
 * `confusion` stays the integer counts.  The weights are not range-checked on the device. */
int srs_metrics_update_weighted_device(srs_metrics* mt, const float* probs, const float* logits,
                                       const int32_t* labels, const float* weights, int32_t n, void* stream);

/* `model.evaluate(dataset)` over host batches: each batch is scored and folded into the metrics on the
 * device the way srs_predict_host_batches pipelines it (batch i on slot i % srs_num_slots()); only its
 * labels [B] int32 go in beside the features and no score comes back.  The loss sums of the batches are
 * added in batch order, so the result does not depend on which slot finishes first.  Synchronous.
 * SRS_ERR_RANGE for an out-of-range id, SRS_ERR_INVALID for a bad label or probability, for no rows,
 * and for the models evaluate does not cover - DIEN (its Keras evaluate reports the loss with the auxiliary
 * term and its AUC metrics instead: srs_dien_evaluate_host_batches) and two towers without the final Dense
 * (its output is a raw dot, not a probability).  `out` is written only on success. */
int srs_evaluate_host_batches(srs_model* m, int32_t n_batches, const srs_batch* batches,
                              const int32_t* const* labels, srs_eval_result* out);
/* srs_evaluate_host_batches with sample weights: weights[i] [B] float32 (host) for batch i, each checked before any
 * launch.  weights NULL: srs_evaluate_host_batches exactly.  Each batch's weighted sums are added in batch order. */
int srs_evaluate_weighted_host_batches(srs_model* m, int32_t n_batches, const srs_batch* batches,
                                       const int32_t* const* labels, const float* const* weights,
                                       srs_eval_result* out);

/* ---- DIEN's second output and its Keras evaluate.  The reference's DIEN is a two-output model,
 * `tf.keras.Model(inputs, outputs=[y_pred, auxiliary_loss_value])` (DIEN.py:296): `model.predict(dataset)`
 * (:312) returns both arrays and `model.evaluate(dataset)` (:304) reports the `add_loss` value and the
 * auxiliary layer's AUC metrics.  The second output comes from `auxiliary_loss_layer` (:261-292), which needs
 * the optional weight group aux_pos_dense/kernel [2E,32], aux_pos_dense/bias [32], aux_pos_out/kernel [32,1],
 * aux_pos_out/bias [1] and the same four aux_neg_* (all eight or none at srs_model_create); without it, and
 * for any other model, these calls return SRS_ERR_INVALID.  Per row, with g_t the GRU output and e() a row of
 * the shared movie embedding (1-based positions t = 1..T-1, no mask):
 *   aux = sum_t sigmoid(Dense1_pos(sigmoid(Dense32_pos([g_t | e(hist_{t+1})]))))
 *             + sigmoid(Dense1_neg(sigmoid(Dense32_neg([g_t | e(neg_{t+1})]))))           (:276-285)
 * and per Keras batch (:287), in float32:
 *   final_loss_i = bce_i - 0.5 * mean_{j in batch}(aux_j),  bce_i = max(x,0) - x*y + log1p(exp(-|x|))
 * on the logit x and the 0/1 label y, the batch mean summed in a fixed order.  `neg_hist` holds the ids
 * negtive_userRatedMovie2..T [B][T-1] in graph order (:83-86,123-128): they pass through float32 like the
 * history and an id outside the vocabulary gives SRS_ERR_RANGE (read as row 0).  With T = 1 aux is 0 and
 * neg_hist may be NULL. */
typedef struct srs_dien_eval_result {
  int64_t rows, batches;
  double loss;        /* the Mean of every row's final_loss: sum over all rows / rows                         */
  double auc;         /* the layer's tf.keras.metrics.AUC() over all (label, y_pred): the roc_auc of evaluate  */
  double auc_value;   /* add_metric(auc.result(), aggregation="mean"): the mean over batches k of the ROC AUC   */
                      /* of batches 0..k, so it depends on the batch order; exact counts, AUCs in double       */
} srs_dien_eval_result;

/* One device batch = one Keras batch, asynchronous on `stream`: probs / logits [B] with the bits of
 * srs_predict_device, aux [B], and final_loss [B] from labels [B] int32.  Device pointers, all required when
 * B > 0; neg_hist has neg_stride >= T-1 elements per row.  A label other than 0 / 1 gives a NaN final_loss;
 * an out-of-range id is reported by srs_model_status. */
int srs_dien_outputs_device(srs_model* m, const srs_batch* batch, const int32_t* neg_hist, int32_t neg_stride,
                            const int32_t* labels, float* probs, float* logits, float* aux, float* final_loss,
                            void* stream);

/* `model.predict(dataset)` of the two-output model (DIEN.py:312) over host batches, pipelined over the slots
 * as srs_predict_host_batches: batch i (one Keras batch) with neg_hist[i] [B][T-1] and labels[i] [B] int32
 * gives probs[i] [B] (y_pred) and final_loss[i] [B].  Synchronous.  Labels must be 0 or 1 (SRS_ERR_INVALID,
 * checked before any launch). */
int srs_dien_outputs_host_batches(srs_model* m, int32_t n_batches, const srs_batch* batches,
                                  const int32_t* const* neg_hist, const int32_t* const* labels,
                                  float* const* probs, float* const* final_loss);

/* `model.evaluate(dataset)` of DIEN (DIEN.py:304) with Keras >= 2.3 semantics, over host batches pipelined as
 * srs_dien_outputs_host_batches; no score comes back.  Synchronous; `out` is written only on success. */
int srs_dien_evaluate_host_batches(srs_model* m, int32_t n_batches, const srs_batch* batches,
                                   const int32_t* const* neg_hist, const int32_t* const* labels,
                                   srs_dien_eval_result* out);

/* ---- `model.fit` of NeuralCF (neural_cf_model_1, NeuralCF.py:74-91), DeepFM (DeepFM.py), Wide&Deep
 * (WideNDeep.py:99-117) and DeepFM_v2 (DeepFM_v2.py:158-165): each script compiles
 * with loss='binary_crossentropy', optimizer='adam' and calls `fit(train_dataset, epochs=5)` over make_csv_dataset
 * batches of 12.  A trainer owns fp32 weights and Adam's slots on one device; it never touches an srs_model: a
 * serving model is built from the weights srs_trainer_get_weights exports.  Per step of B_b rows (DESIGN.md
 * sections 4.8, 4.9, 4.18 and 4.19):
 *   loss      the mean over the batch of max(z,0) - z*y + log1p(exp(-|z|)), so dL/dz_i = (sigmoid(z_i) - y_i) / B_b;
 *   gradient  through the Dense layers (relu' = [a > 0]) into the embedding rows of each row (DeepFM: also the four
 *             FM dots, and dz into the 4 one-hot rows of dense_2/kernel a row selects; Wide&Deep: its ten embedding
 *             columns, and dz into the wide row of dense_2/kernel at the row's crossed bucket; DeepFM_v2: out/kernel
 *             gets [first | fm | deep] . dz, dfirst = dz * out/kernel[0] goes to first_cat/bias, first_num/bias,
 *             first_num/kernel (times the raw numerics) and the 4 one-hot rows of first_cat/kernel a row selects,
 *             the FM (no 1/2) gives dF_fc = dz * out/kernel[1 + c] * 2 (sum_f F_fc - F_fc), the deep MLP adds
 *             deep/kernel . delta1, and each field's proj_f/kernel gets x_f (x) dF_f, proj_f/bias dF_f (a row
 *             whose genre is missing included) and its table row proj_f/kernel . dF_f; a missing genre gives no
 *             entry); an id that occurs several times in the batch gets the sum of its rows' gradients, in row
 *             order (TF's _deduplicate_indexed_slices);
 *   Adam      Keras's, t = iterations + 1, alpha = lr * sqrt(1 - beta_2^t) / (1 - beta_1^t) in float32.  Dense
 *             kernels and biases - for DeepFM all 31 040 one-hot rows of dense_2/kernel included, for Wide&Deep all
 *             cross_buckets wide rows, for DeepFM_v2 all fm1_width one-hot rows of first_cat/kernel: m += (g - m)(1 -
 *             beta_1), v += (g^2 - v)(1 - beta_2) (TF's ApplyAdam).  The embedding tables (IndexedSlices gradients,
 *             _resource_apply_sparse): m and v of EVERY row decay, m = beta_1 m + (1 - beta_1) G, v = beta_2 v +
 *             (1 - beta_2) G^2 with G = 0 off the batch, and every row is updated - not "lazy Adam".  All:
 *             w -= alpha m / (sqrt(v) + epsilon).
 * Every sum has a fixed order: the same weights, data and order give the same bits.
 * Supported: emb_dim 1..64; NeuralCF 1..3 hidden layers of width 1..32 (two towers: the same per tower, with
 * final_dense), DeepFM exactly 2 of width 1..64, Wide&Deep
 * exactly 2 of width 1..128 and cross_buckets >= 1, DeepFM_v2 exactly 2 of widths 1..32 and 1..16, proj_dim 64 and
 * n_genres >= 1; any batch size >= 1. */
typedef struct srs_adam {
  float lr, beta_1, beta_2, epsilon;   /* Keras's defaults: 0.001, 0.9, 0.999, 1e-7 */
} srs_adam;
typedef struct srs_trainer srs_trainer;

/* `tensors`: the initial weights in Keras shapes (host, the names and shapes srs_model_create takes for
 * SRS_NEURALCF or SRS_DEEPFM); `hp` NULL = Keras's defaults.  A model kind other than those two, an unsupported
 * shape or bad hyper-parameters give SRS_ERR_INVALID, before any device call. */
int srs_trainer_create(const srs_spec* spec, const srs_tensor* tensors, int32_t n_tensors, int32_t device,
                       const srs_adam* hp, srs_trainer** out);
/* srs_trainer_create for every trainable kind: SRS_NEURALCF, SRS_DEEPFM and SRS_WIDENDEEP (its tensors as
 * srs_model_create takes them).  srs_trainer_create keeps rejecting Wide&Deep, as it always has, for callers that
 * rely on its list. */
int srs_trainer_create_ex(const srs_spec* spec, const srs_tensor* tensors, int32_t n_tensors, int32_t device,
                          const srs_adam* hp, srs_trainer** out);
/* srs_trainer_create for every kind this library can train; the list grows with the library, so a kind it rejects
 * today (SRS_ERR_INVALID) may be accepted by a later version.  Today: SRS_NEURALCF, SRS_TWOTOWERS, SRS_DEEPFM,
 * SRS_WIDENDEEP, SRS_DEEPFM_V2 and SRS_DIEN (its tensors as srs_model_create takes them; DIEN's include the auxiliary
 * head's group of eight, which its objective needs; it accepts emb_dim 1..32, hist_len 1..64, au_hidden 32 and hidden
 * widths up to (128, 64), and trains through srs_trainer_fit_dien_host).  Two towers trains with NeuralCF's shapes
 * (1..3 hidden layers of width 1..32 per tower) and only with final_dense = 1: without the final Dense the output is
 * the raw Dot, on which binary cross-entropy is not defined (SRS_ERR_INVALID).  Callers that rely on a fixed list use
 * srs_trainer_create or srs_trainer_create_ex, whose lists do not change. */
int srs_trainer_create_any(const srs_spec* spec, const srs_tensor* tensors, int32_t n_tensors, int32_t device,
                           const srs_adam* hp, srs_trainer** out);
void srs_trainer_destroy(srs_trainer* tr);

/* `epochs` epochs over the n = batch->B rows of `batch` (host; movie_id, user_id, and for DeepFM and DeepFM_v2
 * movie_genre [n][3]
 * and user_genre [n][5], of which column 0 is read and a negative index is missing, and numerics [n][7]; for
 * Wide&Deep every genre column, numerics and hist, of which column 0 (userRatedMovie1) is read) with
 * labels [n] int32: epoch e
 * takes the rows order[e * n + 0 .. n) (each a permutation of 0..n-1) in batches of `batch_size`, the last one
 * partial.  The dataset is uploaded once and the steps run on the device with no host synchronisation between
 * them.  history (NULL or [epochs]) receives each epoch's loss (mean over its rows), accuracy and ROC / PR AUC, as
 * srs_eval_result, each computed on the step's outputs before that step's update (Keras >= 2.2 `fit` logs).
 * Synchronous.  A label other than 0 / 1, an order row that is not a permutation or a missing model column gives
 * SRS_ERR_INVALID, an id or a genre index outside its vocabulary SRS_ERR_RANGE; all of them are checked before any
 * launch, so a rejected call leaves the trainer as it was. */
int srs_trainer_fit_host(srs_trainer* tr, const srs_batch* batch, const int32_t* labels, const int32_t* order,
                         int32_t batch_size, int32_t epochs, srs_eval_result* history);

/* srs_trainer_fit_host with Keras's `fit(..., validation_data=(x_val, y_val), validation_freq=val_freq)`: at the
 * end of every epoch e with (e + 1) % val_freq == 0, after its last update, `model.evaluate` of the current weights
 * over all val_batch->B rows of `val_batch` (host, the columns `batch` has) with `val_labels` [B] int32, in file
 * order.  val_history (NULL or [epochs]) receives those results as srs_trainer_evaluate_host would report them, and
 * a zeroed entry (rows = 0) for every epoch not validated.  Validation changes no weight, no Adam state and no
 * training history; its rows are uploaded once and each validated epoch adds two launches on the trainer's stream
 * (the forward and one metrics update), with no host synchronisation.  Synchronous.  val_batch NULL: no validation,
 * srs_trainer_fit_host exactly.  The validation rows are checked like the training rows, and val_freq >= 1, before
 * any launch; a validation probability that is NaN or outside [0, 1] gives SRS_ERR_INVALID naming the epoch. */
int srs_trainer_fit_validate_host(srs_trainer* tr, const srs_batch* batch, const int32_t* labels, const int32_t* order,
                                  int32_t batch_size, int32_t epochs, srs_eval_result* history,
                                  const srs_batch* val_batch, const int32_t* val_labels, int32_t val_freq,
                                  srs_eval_result* val_history);

/* `model.evaluate(x)` of the trainer's current weights (srs_evaluate_host_batches' metrics over the n rows as one
 * batch), with no export and no srs_model: the rows (as srs_trainer_fit_host takes them) are uploaded, scored by
 * the serving CUDA-core forward over the trainer's arrays and folded into the metrics on the device.  Synchronous;
 * the checks and errors of srs_trainer_fit_host's rows, before any launch. */
int srs_trainer_evaluate_host(srs_trainer* tr, const srs_batch* batch, const int32_t* labels, srs_eval_result* out);

/* srs_trainer_fit_validate_host with Keras's `fit(..., sample_weight=w)` (DESIGN.md section 4.28): weights [n] and
 * val_weights [val_batch->B] (host float32, each NULL for none).  A step of B rows takes the loss sum_i w_i l_i / B,
 * so dL/dz_i = (w_i (p_i - y_i)) / B; a row of weight 0 contributes no gradient but still counts in B, and every
 * table row still takes Adam's decay.  history and val_history report the weighted metrics (as
 * srs_metrics_update_weighted_device) when their weights are given.  Keras's class_weight is the caller's: it
 * multiplies the training weights only.  The weights are checked with the rows, before any launch; NULL weights and
 * val_weights give srs_trainer_fit_validate_host exactly, and all-ones weights its bits.  No extra launch per step. */
int srs_trainer_fit_weighted_host(srs_trainer* tr, const srs_batch* batch, const int32_t* labels, const float* weights,
                                  const int32_t* order, int32_t batch_size, int32_t epochs, srs_eval_result* history,
                                  const srs_batch* val_batch, const int32_t* val_labels, const float* val_weights,
                                  int32_t val_freq, srs_eval_result* val_history);

/* srs_trainer_evaluate_host with weights [n] (host float32; NULL: srs_trainer_evaluate_host exactly). */
int srs_trainer_evaluate_weighted_host(srs_trainer* tr, const srs_batch* batch, const int32_t* labels,
                                       const float* weights, srs_eval_result* out);

/* `model.fit` of DIEN (DIEN.py:296-304; DESIGN.md section 4.20): `epochs` epochs over the n = batch->B rows of
 * `batch` (host: movie_id, user_id, movie_genre and user_genre (column 0 read), numerics and hist [n][hist_stride
 * >= hist_len]) with their negatives neg_hist [n][neg_stride >= hist_len - 1] (NULL for hist_len 1) and labels [n]
 * int32; epoch e trains rows order[e * n .. e * n + n) (a permutation of 0..n-1; the script's is file order) in
 * batches of batch_size, the last one partial.  The objective of a batch is the SUM over its rows of final_loss_i
 * = bce_i - 0.5 * mean_j aux_j (srs_dien_outputs_device), so dL/dz_i = sigmoid(z_i) - y_i; the GRU consumes the
 * history mask, augru_h0 is not trained, the four tables take Keras's sparse Adam on every row and every other
 * tensor ApplyAdam.  history (NULL or [epochs]) gets each epoch's {rows, batches, loss, auc, auc_value} as
 * srs_dien_evaluate_host_batches reports them, over the steps' outputs before their updates.  Every check (ids,
 * negatives, genres, labels, the order) runs before any launch, so a rejected call leaves the weights as they were;
 * SRS_ERR_INVALID for a trainer of another kind, whose fit is srs_trainer_fit_host (and srs_trainer_fit_host,
 * srs_trainer_fit_validate_host and srs_trainer_evaluate_host reject a DIEN trainer). */
int srs_trainer_fit_dien_host(srs_trainer* tr, const srs_batch* batch, const int32_t* neg_hist, int32_t neg_stride,
                              const int32_t* labels, const int32_t* order, int32_t batch_size, int32_t epochs,
                              srs_dien_eval_result* history);

/* Copy one trained tensor, in its Keras shape, to host memory `dst` (SRS_ERR_MISSING for an unknown name). */
int srs_trainer_get_weights(const srs_trainer* tr, const char* name, float* dst);

/* Adam steps taken so far (Keras's optimizer.iterations). */
int64_t srs_trainer_iterations(const srs_trainer* tr);

/* Known-answer self test of the warpgroup-MMA (wgmma) plumbing the tensor-core kernels are built on:
 * D[128][N] = bf16(A[128][K]) * bf16(B[N][K])^T (inputs truncated to bf16, fp32 accumulate),
 * K = 64 * k_blocks (1..4), N = 16 or 32, A read from shared memory (a_in_regs = 0) or from
 * registers (a_in_regs = 1); N = 8: A read MN-major from shared memory (a_in_regs = 0).  Device
 * pointers; synchronous. */
int srs_selftest_wgmma(const float* A, const float* B, float* D, int32_t N, int32_t k_blocks,
                       int32_t a_in_regs, int32_t device);

/* ---- Sample building: FeatureEngForRecModel.scala:21-130 on the device (DESIGN.md section 4.11) ----
 * Every output column has capacity n_ratings rows (user_rated_movie, user_genre: [n_ratings][5], movie_genre:
 * [n_ratings][3]); the first *n_kept rows are written, in input (file) order.  `row` is each kept row's index in
 * the input, so userId, movieId, rating and timestamp are the caller's own.  Genre columns hold word indices,
 * -1 = none; user_rated_movie 0 = none.  The two-decimal columns hold the float32 nearest format_number's text. */
typedef struct srs_samples {
  int32_t* row;
  int32_t* label;                     /* rating >= 3.5 */
  int32_t* release_year;
  int32_t* movie_genre;               /* [3] movieGenre1..3 */
  int32_t* movie_rating_count;
  float* movie_avg_rating;
  float* movie_rating_stddev;
  int32_t* user_rated_movie;          /* [5] the window's positive movies, most recent first */
  int32_t* user_rating_count;         /* > 1 on every kept row */
  float* user_avg_release_year;       /* integral: the average truncated */
  float* user_release_year_stddev;
  float* user_avg_rating;
  float* user_rating_stddev;
  int32_t* user_genre;                /* [5] by descending count, ties in the reference's hash-map order */
} srs_samples;

/* The samples of n_ratings ratings (host arrays): user_id >= 0, movie_id in [0, n_movie_slots), half = rating in
 * half-stars (1..10), timestamp > 0 (int32 seconds; ordered as its decimal string, as the reference orders it).
 * Per movie id (host, n_movie_slots rows): movie_year (the title rule's year, in -999..9999; 1990 for a movie
 * missing from movies.csv) and movie_genres [n_movie_slots][genres_per_movie], the movie's genre word indices in
 * string order, then -1.  genre_hash [n_genres]: java.lang.String.hashCode of each genre word (the reference's
 * genre counting runs in a Scala hash map, whose order breaks count ties).  Bounds: n_ratings <= 21 000 000,
 * n_movie_slots <= 2^24, genres_per_movie 1..24, n_genres 0..24.  Every input is checked before any device call;
 * a violation gives SRS_ERR_INVALID.  The inputs are uploaded once and the job runs on `device` with no host round
 * trip; synchronous.  The same inputs give the same bits. */
int srs_featureeng_host(const int32_t* user_id, const int32_t* movie_id, const int8_t* half, const int32_t* timestamp,
                        int64_t n_ratings, const int32_t* movie_year, const int32_t* movie_genres,
                        int32_t n_movie_slots, int32_t genres_per_movie, const int32_t* genre_hash, int32_t n_genres,
                        int32_t device, srs_samples* out, int64_t* n_kept);

/* ---- Embeddings: Embedding.scala:27-138 on the device (DESIGN.md section 4.12) ----
 * srs_item2vec_host is Spark MLlib's Word2Vec.fit over each user's positive ratings: a hierarchical-softmax
 * skip-gram trained by SGD, minCount 5, learning rate 0.025, sentences cut at 1000 words.  The ratings are host
 * arrays as srs_featureeng_host takes them: user_id >= 0, movie_id in [0, 2^24), half = rating in half-stars
 * (1..10), timestamp > 0; n_ratings <= 21 000 000.  A sentence is one user's movies rated >= 3.5 (users ascending),
 * ordered by the timestamp's decimal string with ties in input order.  Each of `partitions` partitions trains
 * sentences i = p, p + P, ... on its own copy of the tables; at the end of an iteration each row modified by one or
 * more partitions becomes their rows' sum in partition order times 1.0f / count (partitions = 1: the reference's
 * run).  Random numbers come from a counter-based generator keyed by `seed`.  Every sum has a fixed order and
 * there are no float atomics: the same inputs give the same bits.
 * Output: *vocab_size = V, vocab_ids [V] (movie ids by positive count descending, ties by id ascending) and
 * vectors [V][vector_size]; `capacity` is the room in both, and V is at most the number of distinct movie ids rated
 * >= 3.5.  Every input is checked before any device call (SRS_ERR_INVALID).  A vocabulary that is empty
 * (SRS_ERR_INVALID, as Spark's require), larger than `capacity` (SRS_ERR_RANGE) or with a Huffman code longer
 * than 32 (SRS_ERR_INVALID) is reported after the counting step, with nothing written.  Synchronous. */
typedef struct srs_item2vec_params {
  int32_t vector_size;                /* 1..64 (the reference: 10) */
  int32_t window;                     /* 1..65536 (the reference: 5) */
  int32_t iterations;                 /* 1..100000 (the reference: 10) */
  int32_t partitions;                 /* 1..65536 (the reference: 1) */
  uint64_t seed;
} srs_item2vec_params;
int srs_item2vec_host(const int32_t* user_id, const int32_t* movie_id, const int8_t* half, const int32_t* timestamp,
                      int64_t n_ratings, const srs_item2vec_params* params, int32_t device, int32_t capacity,
                      int32_t* vocab_ids, float* vectors, int32_t* vocab_size);

/* generateUserEmb (Embedding.scala:53-101) as the reference's shipped userEmb.csv was made: per user, the float32
 * sum of the vectors of every movie the user rated (any rating) that has one, taken in reverse input order, with
 * no division; a user with none gets a zero row.  Ratings: user_id >= 0, movie_id in [0, 2^24), n_ratings <=
 * 21 000 000 (host).  Items: n_items distinct ids in [0, 2^24) and vectors [n_items][vector_size] (host),
 * vector_size 1..64.  Output: *n_users = U distinct users, ascending, in user_ids [U] and user_vectors
 * [U][vector_size]; `capacity` is the room in both (U > capacity: SRS_ERR_RANGE, nothing written).  Every input is
 * checked before any device call (SRS_ERR_INVALID).  Synchronous; the same inputs give the same bits. */
int srs_user_embeddings_host(const int32_t* user_id, const int32_t* movie_id, int64_t n_ratings,
                             const int32_t* item_ids, const float* item_vectors, int32_t n_items,
                             int32_t vector_size, int32_t device, int32_t capacity, int32_t* user_ids,
                             float* user_vectors, int32_t* n_users);

/* ---- Graph embedding and LSH: the rest of Embedding.scala on the device (DESIGN.md section 4.14) ----
 * The ratings are host arrays as srs_item2vec_host takes them, with its checks, and its sentences (positive ratings
 * by user, in timestamp-string order).  Every consecutive (a, b) of a sentence is a pair; count(a, b) per distinct
 * pair, out(a) = sum over b, pairTotal = sum of out.  A source is a movie with an outgoing pair.
 * srs_item_transitions_host (generateTransitionMatrix): *n_sources = S sources ascending in sources [S], their out(a)
 * in out_counts [S] and dist(a) = out(a) / pairTotal (a double division) in source_probs [S]; row s's pairs are
 * entries row_offsets[s] .. row_offsets[s + 1] - 1 (row_offsets [S + 1]) of targets / counts / probs [E], targets
 * ascending, probs = count / out(a) in double; *n_edges = E.  S or E beyond its capacity: SRS_ERR_RANGE, nothing
 * written.  Synchronous; the same inputs give the same bits. */
int srs_item_transitions_host(const int32_t* user_id, const int32_t* movie_id, const int8_t* half,
                              const int32_t* timestamp, int64_t n_ratings, int32_t device, int32_t source_capacity,
                              int32_t edge_capacity, int32_t* sources, int32_t* row_offsets, int32_t* out_counts,
                              double* source_probs, int32_t* targets, int32_t* counts, double* probs,
                              int32_t* n_sources, int32_t* n_edges);

/* randomWalk (Embedding.scala:140-184): num_walks walks of at most walk_length items, in walks [num_walks]
 * [walk_length] (-1 past a walk's end) and lengths [num_walks].  Walk w draws u_t = (splitmix(splitmix(splitmix(~seed,
 * 0), w), t) >> 11) / 2^53 at step t; a draw picks the first entry whose cumulative sum (the probabilities added
 * left to right in double, sources and targets ascending) is >= u.  Step 0 draws the first item from dist; each
 * later step stops the walk at an item with no outgoing pair, else draws from its row.  A u past the last sum
 * leaves the current item (it repeats), or at step 0 makes the walk empty.  num_walks, walk_length >= 1 and
 * num_walks * walk_length <= 21 000 000, checked before any device call (SRS_ERR_INVALID).  Synchronous. */
int srs_random_walks_host(const int32_t* user_id, const int32_t* movie_id, const int8_t* half,
                          const int32_t* timestamp, int64_t n_ratings, int32_t num_walks, int32_t walk_length,
                          uint64_t seed, int32_t device, int32_t* walks, int32_t* lengths);

/* graphEmb (Embedding.scala:254-266): srs_random_walks_host's walks with params->seed, each non-empty walk one
 * sentence, trained by srs_item2vec_host's Word2Vec with `params`; outputs, capacity and errors as there. */
int srs_graph_embedding_host(const int32_t* user_id, const int32_t* movie_id, const int8_t* half,
                             const int32_t* timestamp, int64_t n_ratings, const srs_item2vec_params* params,
                             int32_t num_walks, int32_t walk_length, int32_t device, int32_t capacity,
                             int32_t* vocab_ids, float* vectors, int32_t* vocab_size);

/* BucketedRandomProjectionLSHModel.transform: buckets [n][num_tables] (double) = floor(dot(x, v_j) / bucket_length)
 * of the float vectors [n][dim] (host) and the unit vectors [num_tables][dim] (double, host); the dot is summed left
 * to right in double from 0.0, one rounding per operation.  dim 1..1024, num_tables 1..64, bucket_length finite and
 * > 0, every entry finite, n <= 2^31 - 1; checked before any device call (SRS_ERR_INVALID).  Synchronous. */
int srs_lsh_transform_host(const float* vectors, int64_t n, int32_t dim, const double* unit_vectors,
                           int32_t num_tables, double bucket_length, int32_t device, double* buckets);

/* approxNearestNeighbors(dataset, key, k), single probe, for num_keys keys [num_keys][dim] (double) at once: the
 * candidates are the rows sharing the key's bucket in at least one table; the distance is sqrt of the sum of (x - key)^2
 * in double, left to right.  Per key q, out_count[q] = min(k, candidates) rows in out_ids / out_dist [q][k] by
 * distance ascending, ties by id then row ascending; entries past out_count[q] are not written.  k 1..256, keys
 * finite, and srs_lsh_transform_host's checks, before any device call (SRS_ERR_INVALID).  Synchronous. */
int srs_lsh_query_host(const int32_t* ids, const float* vectors, int64_t n, int32_t dim, const double* unit_vectors,
                       int32_t num_tables, double bucket_length, const double* keys, int32_t num_keys, int32_t k,
                       int32_t device, int32_t* out_ids, double* out_dist, int32_t* out_count);

/* approxSimilarityJoin(datasetA, datasetB, threshold): every pair (a of A, b of B) whose bucket ids are equal in at
 * least one table, once however many tables it collides in, with distance sqrt of the sum of (x_a - x_b)^2 in double,
 * left to right, strictly below `threshold` (any double: NaN or <= 0 gives no pair, +inf every candidate).  The pairs
 * are ordered by (id_a, id_b) ascending as signed ints.  A self-join passes the same arrays as A and B.  Each side
 * passes srs_lsh_transform_host's checks, n_a and n_b are 0..2^31-1, ids are unique within each side (the message
 * names the side and the id), capacity >= 0, n_pairs is non-null and the outputs are non-null when capacity > 0; all
 * checked before any device call (SRS_ERR_INVALID).  With an empty side, *n_pairs = 0 and no device call is made.
 * Otherwise *n_pairs = P, the number of pairs, is written after the counting pass, on SRS_OK and on SRS_ERR_RANGE
 * (P > capacity), so that a caller can retry with capacity P; out_ids_a, out_ids_b and out_dist [P] are written only
 * on SRS_OK.  Synchronous; the same inputs give the same bits. */
int srs_lsh_similarity_join_host(const int32_t* ids_a, const float* vectors_a, int64_t n_a,
                                 const int32_t* ids_b, const float* vectors_b, int64_t n_b, int32_t dim,
                                 const double* unit_vectors, int32_t num_tables, double bucket_length,
                                 double threshold, int32_t device, int64_t capacity,
                                 int32_t* out_ids_a, int32_t* out_ids_b, double* out_dist, int64_t* n_pairs);

/* ---- Collaborative filtering: CollaborativeFiltering.scala on the device (DESIGN.md section 4.13) ----
 * srs_als_fit_host is Spark ML's ALS.fit with explicit feedback: `max_iter` times, the movie factors and then the
 * user factors, each entity's from its double-precision normal equations (its ratings in ascending counterpart id,
 * duplicates in input order) plus reg_param * (its rating count) on the diagonal, solved by Cholesky (LAPACK dppsv's
 * loops) and rounded to float.  The users' initial factors come from a Gaussian generator keyed by `seed` and the
 * user id, scaled to unit norm.  Ratings are host arrays: user_id >= 0, movie_id >= 0, rating finite; 1 <=
 * n_ratings <= 21 000 000.  Output: *n_users = U distinct user ids, ascending, in user_ids [U] and user_factors
 * [U][rank]; *n_movies = M, likewise.  Every input is checked before any device call (SRS_ERR_INVALID).  More
 * entities than a capacity give SRS_ERR_RANGE, and a system with a pivot <= 0 or NaN gives SRS_ERR_INVALID naming
 * the user or movie; either way nothing is written.  Synchronous; the same inputs give the same bits. */
typedef struct srs_als_params {
  int32_t rank;                       /* 1..64 (Spark's default: 10) */
  int32_t max_iter;                   /* >= 1 (the reference: 5) */
  double reg_param;                   /* finite, >= 0 (the reference: 0.01) */
  uint64_t seed;
} srs_als_params;
int srs_als_fit_host(const int32_t* user_id, const int32_t* movie_id, const float* rating, int64_t n_ratings,
                     const srs_als_params* params, int32_t device, int32_t user_capacity, int32_t movie_capacity,
                     int32_t* user_ids, float* user_factors, int32_t* n_users, int32_t* movie_ids,
                     float* movie_factors, int32_t* n_movies);

/* ALS.fit with implicitPrefs (DESIGN.md section 4.17): srs_als_fit_host's arguments, layouts, init, order and
 * solve, with `alpha` (finite, >= 0; Spark's default 1.0).  Before each half-step, YtY = the sum of y y^T over every
 * source factor, in double: each of Spark's ten blocks (raw id mod 10, ascending id) summed from zero, then the
 * blocks added in block order.  Each entity's system starts from YtY; each rating r adds c1 y y^T (c1 = alpha |r|)
 * and, when r > 0, (1 + c1) y to the right-hand side; reg_param * (its count of ratings > 0) goes on the diagonal.
 * Checks, errors and outputs as srs_als_fit_host's (alpha's before any device call).  Synchronous; the same inputs
 * give the same bits. */
int srs_als_fit_implicit_host(const int32_t* user_id, const int32_t* movie_id, const float* rating,
                              int64_t n_ratings, const srs_als_params* params, int32_t device, int32_t user_capacity,
                              int32_t movie_capacity, int32_t* user_ids, float* user_factors, int32_t* n_users,
                              int32_t* movie_ids, float* movie_factors, int32_t* n_movies, double alpha);

/* ALS.fit with nonnegative = true (DESIGN.md section 4.21): srs_als_fit_host's arguments, layouts, init, order and
 * normal equations - srs_als_fit_implicit_host's, with `alpha`, when implicit_prefs is 1 - but each entity's factor
 * is Spark's NNLSSolver's: NNLS.solve (projected gradient with conjugate directions, at most max(400, 20 rank)
 * iterations) on the full symmetric matrix with lambda on its diagonal, each x(i) >= 0, rounded to float.  There is
 * no singular system: an all-zero system gives a zero factor.  implicit_prefs 0 or 1; checks, errors and outputs
 * as srs_als_fit_host's, all before any device call.  Synchronous; the same inputs give the same bits. */
int srs_als_fit_nonnegative_host(const int32_t* user_id, const int32_t* movie_id, const float* rating,
                                 int64_t n_ratings, const srs_als_params* params, int32_t device,
                                 int32_t user_capacity, int32_t movie_capacity, int32_t* user_ids, float* user_factors,
                                 int32_t* n_users, int32_t* movie_ids, float* movie_factors, int32_t* n_movies,
                                 int32_t implicit_prefs, double alpha);

/* Many ALS fits over one rating set in one pass (CrossValidator's fold x grid models, DESIGN.md section 4.15).
 * fold [n_ratings] gives each rating a fold in 0..n_folds-1 (2 <= n_folds <= 65536).  Model m of the n_models
 * (1..64) trains on the ratings outside fold models[m].exclude_fold (-1: on all of them) with its own rank,
 * max_iter and reg_param and the shared `seed`; its result is bit for bit what srs_als_fit_host returns on those
 * ratings in input order.  A model's users and movies are those with a training rating in it.  Output of model m,
 * with R_m = the sum of the ranks of models 0..m-1: n_users[m] user ids at user_ids + m * user_capacity and their
 * factors at user_factors + user_capacity * R_m ([n_users[m]][rank]); movies likewise.  The capacities must hold
 * every distinct id of the whole set (else SRS_ERR_RANGE).  Every input is checked before any device call,
 * including that no model's training set is empty (SRS_ERR_INVALID).  A singular system gives SRS_ERR_INVALID
 * naming the lowest failing model and its user or movie, and nothing is written.  Synchronous; the same inputs give
 * the same bits. */
typedef struct srs_als_model {
  int32_t rank;                       /* 1..64 */
  int32_t max_iter;                   /* >= 1 */
  double reg_param;                   /* finite, >= 0 */
  int32_t exclude_fold;               /* -1 or 0..n_folds-1 */
} srs_als_model;
int srs_als_fit_folds_host(const int32_t* user_id, const int32_t* movie_id, const float* rating, const int32_t* fold,
                           int64_t n_ratings, int32_t n_folds, const srs_als_model* models, int32_t n_models,
                           uint64_t seed, int32_t device, int32_t user_capacity, int32_t movie_capacity,
                           int32_t* user_ids, float* user_factors, int32_t* n_users, int32_t* movie_ids,
                           float* movie_factors, int32_t* n_movies);

/* srs_als_fit_folds_host with a solver per model (DESIGN.md section 4.21): nonnegative [n_models], each 0 or 1
 * (checked before any device call, SRS_ERR_INVALID).  A model whose flag is 0 gives srs_als_fit_folds_host's bits,
 * and one whose flag is 1 gives srs_als_fit_nonnegative_host's explicit fit's bits on its training ratings. */
int srs_als_fit_folds_nonnegative_host(const int32_t* user_id, const int32_t* movie_id, const float* rating,
                                       const int32_t* fold, int64_t n_ratings, int32_t n_folds,
                                       const srs_als_model* models, int32_t n_models, uint64_t seed, int32_t device,
                                       int32_t user_capacity, int32_t movie_capacity, int32_t* user_ids,
                                       float* user_factors, int32_t* n_users, int32_t* movie_ids,
                                       float* movie_factors, int32_t* n_movies, const int32_t* nonnegative);

/* ALSModel.recommendForAll: for each of n_src source factors [n_src][rank] (host), the L = min(num, n_dst)
 * destinations of highest score, best first, in out_ids / out_scores [n_src][L].  The score is the float dot
 * sum += src(d) * dst(d) from 0.0f, d ascending, each operation rounded once.  Ties go to the lower destination id
 * (dst_ids must be strictly ascending); a NaN score ranks as -inf.  rank 1..64, num 1..128, factors finite;
 * checked before any device call (SRS_ERR_INVALID).  Synchronous; the same inputs give the same bits. */
int srs_als_recommend_host(const float* src_factors, int32_t n_src, const int32_t* dst_ids, const float* dst_factors,
                           int32_t n_dst, int32_t rank, int32_t num, int32_t device, int32_t* out_ids,
                           float* out_scores);

/* mllib RankingMetrics (Spark 2.4) over n_queries queries: pred_ids [n_queries][pred_len] best first, and query q's
 * relevant ids label_ids[label_off[q] .. label_off[q + 1]) (a set: duplicates count once).  Per query, with
 * |lab| its distinct labels: precision@k = hits in the first min(pred_len, k) / k; NDCG@k = dcg / maxDcg over
 * i < min(max(pred_len, |lab|), k) with gain 1 / ln(i + 2), dcg taking the hits and maxDcg the first |lab|
 * positions; average precision = the sum over every hit of (hits so far) / (i + 1), over |lab|.  An empty label
 * set scores 0.  means [3] = precision@k, NDCG@k, MAP: StatCounter's mu += (x - mu) / n in query order (NaN for no
 * query); per_query [3][n_queries], when not null, the values.  k >= 1, label_off[0] = 0 and non-decreasing;
 * checked before any device call (SRS_ERR_INVALID).  Synchronous; the same inputs give the same bits. */
int srs_ranking_metrics_host(const int32_t* pred_ids, int32_t n_queries, int32_t pred_len, const int32_t* label_off,
                             const int32_t* label_ids, int32_t k, int32_t device, double* per_query, double* means);

/* ---- The FeatureEngineering job and the sample split on the device (DESIGN.md section 4.16) ----
 * Every entry checks its inputs before any device call (SRS_ERR_INVALID) and writes its outputs only on success.
 * Synchronous; the same inputs give the same bits.  Values are never NaN.
 *
 * approxQuantile as Spark 2.4.3's QuantileSummaries answers it with every value in one summary: the n values
 * (1 <= n <= 2^31 - 1) sorted in Double's total order, withHeadBufferInserted, compressImmut with mergeThreshold
 * 2 eps n, then query (targetError = ceil(eps n)) at each probability in [0, 1] (1..65536 of them) -> out.
 * NaN values are rejected (Spark's approxQuantile skips them).  Besides the sort, the compress takes at most
 * min(n, 2 eps n + 4) sequential steps and each query O(log n). */
int srs_approx_quantile_host(const double* values, int64_t n, const double* probabilities, int32_t n_probabilities,
                             double relative_error, int32_t device, double* out);

/* QuantileDiscretizer(num_buckets 2..10000, relative_error 0..1).fit: approxQuantile at the elements of Scala's
 * (0.0 to 1.0 by 1.0 / num_buckets), 0.0 + step * k (num_buckets + 1 of them, or num_buckets when the step's decimal
 * exceeds 1 / num_buckets), the first and last replaced by -inf / +inf, distinct values in order -> splits
 * [<= num_buckets + 1], *n_splits.  `buckets` (or NULL)
 * [n] receives Bucketizer's bucket of each value.  Splits that are not >= 3 strictly increasing values give
 * SRS_ERR_INVALID after the device run. */
int srs_quantile_discretizer_host(const double* values, int64_t n, int32_t num_buckets, double relative_error,
                                  int32_t device, double* splits, int32_t* n_splits, int32_t* buckets);

/* Bucketizer(splits).transform (handleInvalid "error"): 3..10001 strictly increasing splits; every value must lie in
 * [splits[0], splits[n_splits - 1]].  A value on a split goes to the bucket above it; the last bucket includes the
 * last split. */
int srs_bucketize_host(const double* splits, int32_t n_splits, const double* values, int64_t n, int32_t device,
                       int32_t* buckets);

/* MinMaxScaler (min 0, max 1): out[i] = (x - Emin) / (Emax - Emin), 0.5 when Emax == Emin.  Emin / Emax are
 * fit_min_max[0..1] when given, else the values' minimum and maximum in Double's total order; min_max (or NULL)
 * receives the ones used. */
int srs_minmax_scale_host(const double* values, int64_t n, const double* fit_min_max, int32_t device, double* out,
                          double* min_max);

/* groupBy(movieId).agg(count, avg(rating), variance(rating)) over 1..21 000 000 ratings (movie ids 0..2^24 - 1,
 * half-stars 1..10): *n_movies rows, ascending movie id, of the movies with a rating.  avg and var_samp are each
 * one correctly rounded division of exact integer moments; a one-rating movie's variance is NaN (null).  More
 * movies than `capacity` give SRS_ERR_RANGE. */
int srs_rating_features_host(const int32_t* movie_id, const int8_t* half, int64_t n_ratings, int32_t device,
                             int32_t capacity, int32_t* movie_ids, int64_t* counts, double* avg, double* var,
                             int32_t* n_movies);

/* StringIndexer.fit (frequencyDesc) over tokens [n_tokens] (word ids 0..n_words - 1, each word occurring; 1 <=
 * n_words <= 2^20) whose strings have the Java hashCodes word_hash [n_words]: label k is word label_words[k], with
 * label_counts[k] occurrences; by descending count, ties in the iteration order of a Scala 2.11 immutable.HashMap.
 * Two words whose improved hashes are equal are rejected. */
int srs_string_indexer_host(const int32_t* tokens, int64_t n_tokens, const int32_t* word_hash, int32_t n_words,
                            int32_t device, int32_t* label_words, int64_t* label_counts);

/* The multi-hot genre vectors: movie r (distinct ids 0..2^24 - 1) lists the words words[offsets[r] ..
 * offsets[r + 1]) (1..256 distinct words); the labels as srs_string_indexer_host, then per movie in ascending id
 * (out_movie_ids [n_movies]) its label indices ascending, in CSR form: out_offsets [n_movies + 1], out_indices
 * [offsets[n_movies]]. */
int srs_genre_multihot_host(const int32_t* movie_id, const int32_t* offsets, const int32_t* words, int32_t n_movies,
                            const int32_t* word_hash, int32_t n_words, int32_t device, int32_t* label_words,
                            int64_t* label_counts, int32_t* out_movie_ids, int32_t* out_offsets,
                            int32_t* out_indices);

/* sample(fraction) then randomSplit(weights [n_parts], 1..64, finite, >= 0, sum > 0) of rows 0..n - 1: row i is
 * sampled when the top 53 bits of splitmix(splitmix(seed, 0), i) / 2^53 < fraction, and goes to part j when
 * lb_j <= u < ub_j for u from splitmix(splitmix(seed, 1), i), the bounds the running sums of the normalised weights.
 * rows [n] receives part 0's rows, then part 1's, ..., each ascending; part_counts [n_parts] their counts. */
int srs_sample_split_host(int64_t n, uint64_t seed, double fraction, const double* weights, int32_t n_parts,
                          int32_t device, int32_t* rows, int64_t* part_counts);

/* The same sample, then approxQuantile(timestamp, 0.8, relative_error) of the sampled rows (as
 * srs_approx_quantile_host) -> *split_timestamp (NaN when no row is sampled): sampled rows with timestamp <= it
 * are part 0 (training), the rest part 1 (test); rows and part_counts [2] as srs_sample_split_host.  Timestamps
 * within +-2^53. */
int srs_sample_split_by_timestamp_host(const int64_t* timestamp, int64_t n, uint64_t seed, double fraction,
                                       double relative_error, int32_t device, int32_t* rows, int64_t* part_counts,
                                       double* split_timestamp);

/* ---- mllib BinaryClassificationMetrics (Spark 2.4.3; OFF/evaluate/Evaluator.scala; DESIGN.md section 4.22) ----
 * One call takes n (score, label) pairs cut into n_sets score sets: set s is pairs set_off[s] .. set_off[s + 1]
 * (set_off NULL: one set, n_sets 1).  Per set, as mllib with one partition:
 *   a label > 0.5 is a positive (NaN is not); the thresholds are the distinct scores in Double.compare's
 *   descending order, NaN first and 0.0 above -0.0; numBins > 0 with grouping = thresholds / numBins >= 2 merges
 *   runs of `grouping` consecutive thresholds (the last run may be shorter), each keeping its first score; TP / FP
 *   are the exact cumulative counts down the thresholds; precision = TP / (TP + FP) (1 when 0 / 0), recall = TP / P
 *   (0 when P = 0), FPR = FP / N (0 when N = 0), F(beta) = (1 + b^2) * (p * r / (b^2 * p + r)) (0 when p + r = 0);
 *   roc() = (0, 0), (FPR, recall)..., (1, 1); pr() = (0, first precision), (recall, precision)...; each area is the
 *   sum of the trapezoids (x2 - x1) * (y2 + y1) / 2, added in a fixed order (the same inputs give the same bits).
 * 1 <= n <= 2^31 - 1, every set non-empty (set_off[0] = 0, strictly increasing, set_off[n_sets] = n), num_bins >= 0;
 * checked before any device call (SRS_ERR_INVALID).  The handle keeps each point's threshold and counts on
 * `device` (24 bytes a point); a call peaks near 33 bytes a pair on the device (plus 16 for the host path's copy). */
typedef struct srs_binary_metrics srs_binary_metrics;
typedef struct srs_binary_summary {
  int64_t n, positives, negatives, thresholds;   /* thresholds: the points after binning */
  double area_under_roc, area_under_pr;
} srs_binary_summary;
#define SRS_BM_ROC 0          /* double [thresholds + 2][2]: (FPR, recall) */
#define SRS_BM_PR 1           /* double [thresholds + 1][2]: (recall, precision) */
#define SRS_BM_THRESHOLDS 2   /* double [thresholds] */
#define SRS_BM_PRECISION 3    /* double [thresholds][2]: (threshold, value), and so for the next two */
#define SRS_BM_RECALL 4
#define SRS_BM_FMEASURE 5     /* at `beta`; at beta 0 a point with r = 0 < p is 0 / 0, NaN as in Spark */
/* scores and labels [n] float64 on the host.  Synchronous. */
int srs_binary_metrics_create_host(const double* scores, const double* labels, int64_t n, const int64_t* set_off,
                                   int32_t n_sets, int32_t num_bins, int32_t device, srs_binary_metrics** out);
/* scores [n] float32 and labels [n] int32 (positive when > 0) on `device`, e.g. what srs_predict_device wrote;
 * read after the work queued on `stream`.  Returns when the work is done. */
int srs_binary_metrics_create_device(const float* scores, const int32_t* labels, int64_t n, const int64_t* set_off,
                                     int32_t n_sets, int32_t num_bins, int32_t device, void* stream,
                                     srs_binary_metrics** out);
void srs_binary_metrics_destroy(srs_binary_metrics* h);
int srs_binary_metrics_summary(const srs_binary_metrics* h, int32_t set, srs_binary_summary* out);
/* curve `which` (SRS_BM_*) of `set` into host dst, laid out as above; an unknown `which` or set is rejected
 * without touching dst */
int srs_binary_metrics_curve(const srs_binary_metrics* h, int32_t set, int32_t which, double beta, double* dst);
/* the cumulative TP and FP [thresholds] int64 of `set` */
int srs_binary_metrics_confusion(const srs_binary_metrics* h, int32_t set, int64_t* tp, int64_t* fp);

/* ---- Similar movies (ON/recprocess/SimilarMovieProcess.java getRecList; DESIGN.md section 4.23) ----------------
 * A catalogue holds n_movies movies in movies.csv order: distinct ids movie_id [n_movies], and movie m's genres
 * genre[genre_off[m] .. genre_off[m + 1]) (genre_off [n_movies + 1], genre_off[0] = 0), each an index 0 ..
 * n_genres - 1 (n_genres <= 64), distinct within a movie.  The ratings rating_movie / rating_score [n_ratings] (float,
 * as Float.parseFloat reads them) in ratings.csv order give each movie Movie.addRating's running mean in double;
 * ratings of other movies are ignored.  emb [n_emb][dim] are the rows of item2vecEmb.csv, row r the vector of
 * movie emb_id[r] (the last row of an id wins; ids outside the catalogue are ignored).  n_emb 0 is a catalogue
 * without vectors.  Every argument is checked before any device call (SRS_ERR_INVALID).  Synchronous. */
typedef struct srs_similar_catalog srs_similar_catalog;
int srs_similar_catalog_create_host(const int32_t* movie_id, int32_t n_movies, const int32_t* genre_off,
                                    const int32_t* genre, int32_t n_genres, const int32_t* rating_movie,
                                    const float* rating_score, int64_t n_ratings, const int32_t* emb_id,
                                    const float* emb, int32_t n_emb, int32_t dim, int32_t device,
                                    srs_similar_catalog** out);
void srs_similar_catalog_destroy(srs_similar_catalog* catalog);
#define SRS_SIMILAR_DEFAULT 0          /* calculateSimilarScore: 0.7 * genre overlap + 0.3 * averageRating / 5 */
#define SRS_SIMILAR_EMB 1              /* the cosine of the two movies' vectors (-1 for a candidate without one) */
#define SRS_SIMILAR_OK 0
#define SRS_SIMILAR_UNKNOWN_MOVIE 1    /* not in the catalogue: an empty list, as the Java returns */
#define SRS_SIMILAR_NO_EMBEDDING 2     /* model EMB and the query has no vector (the Java throws): an empty list */
/* getRecList(movie_ids[q], size, model) for q < n_queries: the union of the top-100-by-rating lists of the query's
 * genres minus the query, scored by `model`, ordered by score descending (Double.compare; NaN first, 0.0 above
 * -0.0) and ties by movie id ascending, cut to size >= 1.  Host outputs: out_ids [n_queries][size] int32,
 * out_scores [n_queries][size] double, out_count [n_queries] (entries past it are 0), out_status [n_queries]
 * (SRS_SIMILAR_OK / _UNKNOWN_MOVIE / _NO_EMBEDDING).  An unknown id is a status, not an error.  Synchronous; the same
 * inputs give the same bits. */
int srs_similar_movies_host(const srs_similar_catalog* catalog, const int32_t* movie_ids, int32_t n_queries,
                            int32_t size, int32_t model, int32_t* out_ids, double* out_scores, int32_t* out_count,
                            int32_t* out_status);

/* ---- Multi-channel and embedding recall (SimilarMovieProcess.java:56-112; DESIGN.md section 4.24) -------------
 * srs_similar_catalog_create_host with each movie's release_year [n_movies] as well (DataManager.parseReleaseYear:
 * 0 where it fails), which multi-channel recall needs; srs_similar_catalog_create_host is this call with NULL.
 * getMovies(size, sortBy) orders the movies of DataManager.movieMap, a HashMap<Integer, Movie>, whose iteration
 * order (bucket (id ^ id >>> 16) & (capacity - 1) ascending, load order within a bucket) breaks ties.  When the
 * load would treeify a bin (9 or more ids in one bucket of a table of 64 or more), which reorders it, the catalogue
 * is still created but both recalls reject it (SRS_ERR_INVALID) before any device call. */
int srs_similar_catalog_create_ex_host(const int32_t* movie_id, int32_t n_movies, const int32_t* genre_off,
                                       const int32_t* genre, int32_t n_genres, const int32_t* rating_movie,
                                       const float* rating_score, int64_t n_ratings, const int32_t* emb_id,
                                       const float* emb, int32_t n_emb, int32_t dim, const int32_t* release_year,
                                       int32_t device, srs_similar_catalog** out);
#define SRS_SIMILAR_CANDIDATES_GENRE 0     /* candidateGenerator: the query's genres' top 100 by rating */
#define SRS_SIMILAR_CANDIDATES_MULTIPLE 1  /* multipleRetrievalCandidates: the query's genres' top 20 by rating,
                                              getMovies(100, "rating") and getMovies(100, "releaseYear") */
/* srs_similar_movies_host with the candidates of `candidates` (GENRE: exactly srs_similar_movies_host).  MULTIPLE
 * needs a catalogue created with release years; a query movie with no genres still gets the two global lists.
 * The candidates are the union minus the query, ranked as srs_similar_movies_host ranks them. */
int srs_similar_movies_candidates_host(const srs_similar_catalog* catalog, int32_t candidates,
                                       const int32_t* movie_ids, int32_t n_queries, int32_t size, int32_t model,
                                       int32_t* out_ids, double* out_scores, int32_t* out_count, int32_t* out_status);
/* retrievalCandidatesByEmbedding(movie_ids[q], size): every movie of getMovies(10000, "rating"), the query itself
 * included, scored by the emb ranker's cosine (-1 for a movie without a vector, NaN for a zero vector), in
 * ascending Double.compare order (-1s first, NaN last; the Java's Map.Entry.comparingByValue(), so the least similar
 * movies come first), ties by movie id, cut to size >= 1.  Outputs as srs_similar_movies_host's; an unknown id is
 * SRS_SIMILAR_UNKNOWN_MOVIE and a query without a vector SRS_SIMILAR_NO_EMBEDDING (the Java returns null for both),
 * each with an empty list.  Synchronous; the same inputs give the same bits. */
int srs_similar_embedding_recall_host(const srs_similar_catalog* catalog, const int32_t* movie_ids,
                                      int32_t n_queries, int32_t size, int32_t* out_ids, double* out_scores,
                                      int32_t* out_count, int32_t* out_status);

/* ---- Recommended for you (ON/recprocess/RecForYouProcess.java getRecList; DESIGN.md section 4.25) -------------
 * A user table holds DataManager.userMap: every distinct user id of rating_user [n_ratings] (the userId column of
 * ratings.csv's 4-field lines, whether or not the movie is known), and each user's vector from the userEmb.csv rows
 * emb [n_emb][dim], row r the vector of user emb_user[r] (the last row of a user wins; rows of users outside the
 * table are ignored).  n_emb 0 is a table without vectors.  Every argument is checked before any device call
 * (SRS_ERR_INVALID).  Synchronous. */
typedef struct srs_recforyou_users srs_recforyou_users;
int srs_recforyou_users_create_host(const int32_t* rating_user, int64_t n_ratings, const int32_t* emb_user,
                                    const float* emb, int32_t n_emb, int32_t dim, int32_t device,
                                    srs_recforyou_users** out);
void srs_recforyou_users_destroy(srs_recforyou_users* users);
#define SRS_RECFORYOU_DEFAULT 0        /* any other model string: candidates.size() - i for candidate i */
#define SRS_RECFORYOU_EMB 1            /* "emb": the cosine of the user's and the movie's vectors (-1 for a missing
                                          vector or unequal dimensions) */
#define SRS_RECFORYOU_NEURALCF 2       /* "nerualcf" (sic): the served NeuralCF or two-tower model's output on
                                          (userId, movieId), widened to double */
#define SRS_RECFORYOU_OK 0
#define SRS_RECFORYOU_UNKNOWN_USER 1   /* not in the user table: an empty list, as the Java returns */
#define SRS_RECFORYOU_MODEL_RANGE 2    /* NEURALCF and the user, or a candidate, is outside the model's vocabulary
                                          (TF-Serving rejects the request and the Java throws): an empty list */
/* getRecList(user_ids[q], size, ranker) for q < n_users: the candidates are getMovies(800, "rating") of `catalog`
 * (a catalogue whose HashMap order is unknown - see srs_similar_catalog_create_ex_host - is rejected), scored by
 * `ranker`, ordered by score descending (Double.compare; NaN first) and ties by movie id ascending, cut to
 * size >= 1.  `model` is read only by NEURALCF, which needs an SRS_NEURALCF or SRS_TWOTOWERS model; the catalogue, the
 * user table and the model must be on one device.  Host outputs as srs_similar_movies_host's: out_ids
 * [n_users][size] int32, out_scores [n_users][size] double, out_count [n_users] (entries past it are 0), out_status
 * [n_users] (SRS_RECFORYOU_*).  Synchronous; the same inputs give the same bits. */
int srs_recforyou_host(const srs_similar_catalog* catalog, const srs_recforyou_users* users, const srs_model* model,
                       int32_t ranker, const int32_t* user_ids, int32_t n_users, int32_t size, int32_t* out_ids,
                       double* out_scores, int32_t* out_count, int32_t* out_status);
/* ---- Recommended for you with every served CTR model (DESIGN.md section 4.26) ------------------------------------
 * The user side of the serving feature store, the `uf:<userId>` hashes (RecForYouProcess.java:46-52), attached to a
 * user table: row i is user_id[i]'s srs_user_row fields - user_genre [n][5] vocabulary indices (-1 missing; an index
 * >= 19 is SRS_ERR_RANGE), user_numerics [n][3] (userAvgRating, userRatingCount, userRatingStddev) and hist [n][5],
 * userRatedMovie1..5 in key order (the library places them at each model's history positions).  Rows of ids outside
 * the table are ignored and a later row of an id replaces the earlier one; a table user without a row takes an empty
 * hash's values (genres -1, numerics 0, history ids 0).  A second call replaces the whole uf: side.  Every argument
 * is checked before any device call (SRS_ERR_INVALID).  Synchronous. */
int srs_recforyou_users_set_features_host(srs_recforyou_users* users, int32_t n, const int32_t* user_id,
                                          const int32_t* user_genre, const float* user_numerics,
                                          const int32_t* hist);
/* srs_recforyou_host's NEURALCF ranker with a model of any kind.  NeuralCF and two-tower models give
 * srs_recforyou_host's results.  Every other kind scores user u's candidate c as srs_rank_user_host does with u's uf:
 * row and the model's movie table (srs_model_set_movie_features), so it needs both (SRS_ERR_INVALID before any
 * launch).  A user is SRS_RECFORYOU_MODEL_RANGE, with an empty list, when predict would reject one of its rows for
 * range: its userId, a history id the model reads or (for every known user) a candidate outside the model, or a
 * candidate past the movie table; such rows never reach the forward.  The rows of the other users go through the
 * model's own forward kernel in chunks of a fixed byte budget, with the model's lock held.  Outputs as
 * srs_recforyou_host's; the model, the user table and the catalogue must be on one device.  Synchronous; the same
 * inputs give the same bits, wherever the chunks end. */
int srs_recforyou_ctr_host(const srs_similar_catalog* catalog, const srs_recforyou_users* users, srs_model* model,
                           const int32_t* user_ids, int32_t n_users, int32_t size, int32_t* out_ids,
                           double* out_scores, int32_t* out_count, int32_t* out_status);

#ifdef __cplusplus
}
#endif
#endif /* SRS_CTR_H_ */
