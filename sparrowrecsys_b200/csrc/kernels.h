// kernels.h - what model.cu and trainer.cu need of the kernel files: the parameter blocks (device pointers into
// the model's private weight layout) and launch entry points of the fused per-model forward kernels, of the
// training steps, the ranking tail and the metrics.  The offline jobs' shared declarations are in hostcall.h.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include <vector>

#include "common.cuh"

struct srs_eval_result;

namespace srs {

// ---- NeuralCF / two towers (NeuralCF.py:45-70) ------------------------------------
// One thread per row.  All Dense weights live in one small blob that each CTA copies
// to shared memory; offsets are in floats.  Hidden widths are zero-padded to HP.
struct NcfParams {
  const float* movie;      // [n_movies][EP]
  const float* user;       // [n_users][EP]
  const float* blob;       // dense weights, layout below
  int blob_floats;
  int n_movies, n_users;
  int EP, HP;
  int n_layers;            // hidden layers (1..3)
  int two_towers;          // 0: neural_cf_model_1, 1: neural_cf_model_2
  int final_dense;         // two towers only
  // neuralcf:  L0 kernel [2EP][HP] @w_off[0], bias @b_off[0]; Ll kernel [HP][HP] @w_off[l]
  //            out kernel [HP] @out_w, bias @out_b
  // twotowers: item tower @w_off[l]/b_off[l], user tower @w_off[3+l]/b_off[3+l];
  //            out kernel [1] @out_w, bias @out_b
  int w_off[6], b_off[6];
  int out_w, out_b;
};

// ---- NeuralCF's training step (ncf_train.cu; DESIGN.md section 4.8) --------------------------------------------
struct NcfStepArgs {
  const float* tab;        // [n_movies + n_users][EP]: movie rows, then user rows
  const float* blob;       // Dense weights
  const int32_t* movie;    // the dataset [n]
  const int32_t* user;
  const int32_t* label;
  const int32_t* order;    // this step's rows [B]
  int B, n_movies;
  float* probs;            // [B] outputs of the step, before its update
  float* logits;
  int32_t* labels;         // [B] the step's labels, for the metrics
  int32_t* trow;           // [2B] table row of each (movie, user) entry: movie r at r, user r at B + r
  float* gemb;             // [2B][EP] the entries' embedding gradients
  float* part;             // [ctas][blob_floats] per-CTA Dense gradient sums
  const float* weight;     // the dataset's row weights [n] (DESIGN.md section 4.28); null: unweighted
  float* weights;          // [B] the step's weights, for the metrics (written when weight is set)
};
int ncf_train_ctas(int B);
// p: the trainer's NcfParams, for the instantiation <p.EP, p.HP> and the blob layout.  Each step launcher takes a
// null `a` to opt its instantiation into the most dynamic shared memory it asks for, on the current device, instead
// of launching (srs_trainer_create): the opt-in is per device.
cudaError_t launch_ncf_train_step(const NcfStepArgs* a, const NcfParams& p, cudaStream_t s);

// ---- the two-tower model's training step (twotowers_train.cu; DESIGN.md section 4.27) -----------------------
// NeuralCF's arguments and entries: movie r at r, user r at B + r.  p: the trainer's two-tower NcfParams (with its
// final Dense); a null `a` opts the instantiation in, as launch_ncf_train_step.
int twotowers_train_ctas(int B);
cudaError_t launch_twotowers_train_step(const NcfStepArgs* a, const NcfParams& p, cudaStream_t s);

// What the trainer hands each tile model's step (DeepFM, Wide&Deep, DeepFM_v2): the step's rows and where its
// outputs go
struct StepIO {
  BatchView b;             // the step's B rows in order; probs / logits receive its outputs before the update
  const int32_t* label;    // [B]
  int32_t* trow;           // [n_ent B] table row of entry s * B + r (slot s), -1 = none (a missing genre)
  float* gemb;             // [n_ent B][EP] the entries' gradients
  int32_t* frow;           // [n_fent B] one-hot row of entry s * B + r, -1 = none (a missing genre)
  float* fgrad;            // [n_fent B] its gradient
  float* part;             // [ctas][blob floats] per-CTA Dense gradient sums
  const float* weight;     // [B] the step's row weights (DESIGN.md section 4.28); null: unweighted
};

// ---- EmbeddingMLP / Wide&Deep (EmbeddingMLP.py:72-77, WideNDeep.py:101-107) --------
struct EmbMlpParams {
  const float* genre[8];   // movieGenre1..3, userGenre1..5 tables [19][EP]
  const float* movie;      // [n_movies][EP]
  const float* user;       // [n_users][EP]
  const float* W1;         // [KP = 10*EP + 8][128] rows in tile order, zero padded
  const float* b1;         // [128]
  const float* W2;         // [128][128]
  const float* b2;         // [128]
  const float* w3;         // [128] deep rows of dense_2
  const float* b3;         // [1] dense_2/bias, on the device: a trainer's Adam writes it there every step
  const float* wide;       // [cross_buckets] wide rows of dense_2 (nullptr for EmbeddingMLP)
  int n_movies, n_users, n_genres, cross_buckets;
  int EP;
  const uint8_t* image;    // embmlp_tc.cu, EP = 12: W1^T hi / lo, W2^T hi / lo as bf16 SW128 operand tiles (128 KB);
                           //   null: embmlp_kernel runs
  int num_sms;             // embmlp_tc.cu: CTAs per launch at most, one per SM (srs_model_set_sm_limit)
};

// The Dense weights of EmbeddingMLP and Wide&Deep (a model's and a trainer's) as one blob, offsets in floats:
// W1 [10EP + 8][128] in the tile order of embmlp_layers.cuh, b1 [128], W2 [128][128], b2 [128], w3 [128] (the deep
// rows of dense_2/kernel), b3 (dense_2/bias) and 3 floats of padding; hidden widths zero padded to 128, every array
// 16-byte aligned.  Wide&Deep's wide rows of dense_2/kernel live apart (placement.h).
struct EmbMlpBlob {
  int W1, b1, W2, b2, w3, b3, floats;
  __host__ __device__ static EmbMlpBlob of(int EP) {
    EmbMlpBlob l;
    l.W1 = 0;
    l.b1 = (10 * EP + kNumPad) * 128;
    l.W2 = l.b1 + 128;
    l.b2 = l.W2 + 128 * 128;
    l.w3 = l.b2 + 128;
    l.b3 = l.w3 + 128;
    l.floats = l.b3 + 4;
    return l;
  }
};
cudaError_t setup_embmlp_attributes();   // embmlp_kernel's dynamic shared memory opt-in

// ---- Wide&Deep's training step (widendeep_train.cu; DESIGN.md section 4.18) ---------------------------------------
constexpr int kWideDeepTables = 10;   // the kernel's slots: movieGenre1..3, movieId, userGenre1..5, userId
// io: b.hist is userRatedMovie1 (stride 1); 10 table entries per row, and one one-hot entry, the row's wide row
// (crossed bucket) with its dL/dz
struct WideDeepStepArgs {
  EmbMlpParams p;          // the trainer's tables, Dense weights and wide rows
  StepIO io;
  int64_t tab_row0[kWideDeepTables];   // first row of each slot's table in the trainer's table array
};
int widendeep_train_ctas(int B);
cudaError_t launch_widendeep_train_step(int EP, const WideDeepStepArgs* a, cudaStream_t s);

// ---- DeepFM (DeepFM.py:91-113) -----------------------------------------------------
struct DeepFmParams {
  const float* fm_movie;   // [n_movies][EP]
  const float* fm_user;    // [n_users][EP]
  const float* fm_mgenre;  // [19][EP]
  const float* fm_ugenre;  // [19][EP]
  const float* deep_movie; // [n_movies][EP]
  const float* deep_user;  // [n_users][EP]
  const float* blob;       // the Dense weights, DeepFmBlob layout; W1, b1, W2, b2 and wdeep point into it
  const float* W1;         // [KP = 2*EP + 8][64]
  const float* b1;
  const float* W2;         // [64][64]
  const float* b2;
  const float* first;      // [fm1_width] one-hot rows of dense_2 (movieGenre1|movieId|userGenre1|userId)
  const float* wdeep;      // [64]
  float wdot[4];           // dense_2's dot rows and bias, copied from the blob by build_deepfm for deepfm_tc_kernel;
  float bout;              //   deepfm_kernel and the training step load them from the blob (deepfm_load_out)
  int n_movies, n_users, n_genres;
  int EP;
  const uint8_t* image;    // deepfm_tc.cu, EP = 16: W1^T hi / lo, W2^T hi / lo as [128][64] bf16 SW128 tiles (64 KB);
                           //   null: deepfm_kernel runs
  int num_sms;             // deepfm_tc.cu: CTAs per launch at most, two per SM (srs_model_set_sm_limit)
};

// The Dense weights of DeepFM (a model's and a trainer's) as one blob, offsets in floats: W1 [2EP + 8][64] and
// W2 [64][64] in the tile order and padding of deepfm_layers.cuh, b1 [64], b2 [64], wdeep [64] (the deep rows of
// dense_2/kernel), wdot [4] (its dot rows), bout (dense_2/bias) and 3 floats of padding; every array up to wdeep
// starts at a multiple of 64 floats.  The one-hot rows of dense_2/kernel live apart (placement.h).
struct DeepFmBlob {
  int W1, b1, W2, b2, wdeep, wdot, bout, floats;
  __host__ __device__ static DeepFmBlob of(int EP) {
    DeepFmBlob l;
    l.W1 = 0;
    l.b1 = (2 * EP + kNumPad) * 64;
    l.W2 = l.b1 + 64;
    l.b2 = l.W2 + 64 * 64;
    l.wdeep = l.b2 + 64;
    l.wdot = l.wdeep + 64;
    l.bout = l.wdot + 4;
    l.floats = l.bout + 4;
    return l;
  }
};
cudaError_t setup_deepfm_attributes();   // deepfm_kernel's (and deepfm2_kernel's) dynamic shared memory opt-in

// ---- DeepFM's training step (deepfm_train.cu; DESIGN.md section 4.9) ----------------------------
constexpr int kDeepFmTables = 6;   // fm movieId, fm userId, fm movieGenre1, fm userGenre1, deep movieId, deep userId
// io: 6 table entries per row (slot s in kDeepFmTables order), and 4 one-hot entries, rows of dense_2/kernel with
// the row's dL/dz
struct DeepFmStepArgs {
  DeepFmParams p;          // the trainer's tables and Dense weights
  StepIO io;
  int64_t tab_row0[kDeepFmTables];   // first row of each table in the trainer's table array
};
int deepfm_train_ctas(int B);
cudaError_t launch_deepfm_train_step(int EP, const DeepFmStepArgs* a, cudaStream_t s);
struct TrainRows {         // a trainer's dataset on the device, in the srs_batch layout; a column the model does not
  int32_t* movie;          //   read is null.  [n]
  int32_t* user;           // [n]
  int32_t* mgenre;         // [n][3], column 0 read (DeepFM, DeepFM_v2)
  int32_t* ugenre;         // [n][5], column 0 read (DeepFM, DeepFM_v2)
  float* numerics;         // [n][7]
  int32_t* label;          // [n]
  int32_t* rated;          // [n] userRatedMovie1 (Wide&Deep)
  float* weight;           // [n] row weights (DESIGN.md section 4.28); null: unweighted, and not permuted
};
// dst row i = src row order[i], i < n (genres: column 0 only)
cudaError_t launch_deepfm_permute(const TrainRows& src, const TrainRows& dst, const int32_t* order, int n,
                                  cudaStream_t s);
// the same for Wide&Deep: every genre column and userRatedMovie1
cudaError_t launch_widendeep_permute(const TrainRows& src, const TrainRows& dst, const int32_t* order, int n,
                                     cudaStream_t s);

// ---- DeepFM_v2 (DeepFM_v2.py:98-155) -----------------------------------------------
struct DeepFm2Params {
  const float* mgenre;     // [19][EP]
  const float* movie;      // [n_movies][EP]
  const float* ugenre;     // [19][EP]
  const float* user;       // [n_users][EP]
  const float* blob;       // the Dense weights, DeepFm2Blob layout; the pointers below (but `first`) point into it
  const float* first;      // [fm1_width] first_cat kernel
  const float* first_num;  // [8]
  const float* proj[4];    // [EP][64] each, field order movieGenre1, movieId, userGenre1, userId
  const float* proj_b[4];  // [64]
  const float* proj_num;   // [8][64]
  const float* proj_num_b; // [64]
  const float* Wd;         // [320][32]
  const float* bd;         // [32]
  const float* Wd1;        // [32][16]
  const float* bd1;        // [16]
  const float* wout;       // [1 + 64 + 16]
  int n_movies, n_users, n_genres;
  int EP;
};

// The Dense weights of DeepFM_v2 (a model's and a trainer's) as one blob, offsets in floats: the four field
// projections proj [4][EP][64] (rows past E zero), their biases proj_b [4][64], proj_num [8][64] (the 7 numerics'
// rows and a zero row), proj_num_b [64], deep/kernel Wd [320][32], bd [32], deep_1/kernel Wd1 [32][16], bd1 [16]
// (hidden widths zero padded to 32 and 16), out/kernel wout [84] (first | fm 64 | deep 16, zero padded),
// first_num/kernel [8], then first_cat/bias, first_num/bias and out/bias (the forward reads the three biases here:
// a trainer's Adam writes them every step) and one float of padding.  Every array is 16-byte aligned.  The one-hot
// first_cat/kernel lives apart (placement.h).
struct DeepFm2Blob {
  int proj, proj_b, proj_num, proj_num_b, Wd, bd, Wd1, bd1, wout, first_num, first_cat_b, first_num_b, bout, floats;
  __host__ __device__ static DeepFm2Blob of(int EP) {
    DeepFm2Blob l;
    l.proj = 0;
    l.proj_b = 4 * EP * 64;
    l.proj_num = l.proj_b + 4 * 64;
    l.proj_num_b = l.proj_num + kNumPad * 64;
    l.Wd = l.proj_num_b + 64;
    l.bd = l.Wd + 5 * 64 * 32;
    l.Wd1 = l.bd + 32;
    l.bd1 = l.Wd1 + 32 * 16;
    l.wout = l.bd1 + 16;
    l.first_num = l.wout + 84;
    l.first_cat_b = l.first_num + kNumPad;
    l.first_num_b = l.first_cat_b + 1;
    l.bout = l.first_num_b + 1;
    l.floats = l.bout + 2;
    return l;
  }
};

// ---- DeepFM_v2's training step (deepfm2_train.cu; DESIGN.md section 4.19) ----------------------------------------
constexpr int kDeepFm2Tables = 4;   // movieGenre1, movieId, userGenre1, userId: the field order
// io: 4 table entries per row (field s), and 4 one-hot entries, rows of first_cat/kernel with the row's
// dL/dz * out/kernel[0]
struct DeepFm2StepArgs {
  DeepFm2Params p;         // the trainer's tables, Dense weights and one-hot first_cat/kernel
  StepIO io;
  int64_t tab_row0[kDeepFm2Tables];   // first row of each table in the trainer's table array
};
int deepfm2_train_ctas(int B);
cudaError_t launch_deepfm2_train_step(int EP, const DeepFm2StepArgs* a, cudaStream_t s);

// ---- DIN (DIN.py:125-167) ------------------------------------------------------------
struct DinParams {
  const float* movie;      // shared candidate/history table [n_movies][EP]
  const float* user;       // [n_users][EP]
  const float* ugenre;     // [19][EP]
  const float* mgenre;     // [19][EP]
  // the Dense weights point into one DinBlob (below); au_bout and b3 are copies
  // activation unit, algebraically folded (DESIGN.md "DIN activation unit"):
  //   Dense32([h-c, h, c, h*c]) = h.(W_sub+W_h) + (h*c).W_prod + c.(W_c-W_sub) + b
  const float* au_wh;      // [EP][32]  W_sub + W_h
  const float* au_wp;      // [EP][32]  W_prod
  const float* au_wc;      // [EP][32]  W_c - W_sub
  const float* au_b;       // [32]
  const float* au_alpha;   // [T][32]   per-position PReLU
  const float* au_wout;    // [32]
  float au_bout;
  // top MLP, first kernel permuted to the tile order
  //   [userGenre1 | userId | pooled | candidate | movieGenre1] x EP, then 7 numerics + pad
  const float* W1;         // [KP = 5*EP + 8][128]
  const float* b1;         // [128]
  const float* a1;         // [128] PReLU alpha
  const float* W2;         // [128][64]
  const float* b2;         // [64]
  const float* a2;         // [64]
  const float* w3;         // [64]
  float b3;
  int n_movies, n_users, n_genres;
  int T;
  int EP;
  const uint8_t* movie_split;  // din_wg.cu: [n_movies][EP x bf16 hi | EP x bf16 lo] (history rows)
  int max_ctas;                // din_wg.cu: CTAs per launch, 0 = one per 32-row tile (srs_model_set_sm_limit)
  const uint8_t* mlp_image;    // din_wg.cu, EP = 32: W1^T / W2^T bf16 hi / lo images (DinWgLayout<32>::IMG_*)
};

// The Dense weights of DIN as one blob, offsets in floats: au_dense/kernel's four row groups W_sub, W_h, W_c and
// W_prod [EP][32] each (model creation folds them in place into wh = W_sub + W_h and wc = W_c - W_sub: DinParams'
// au_wh and au_wc; wsub is then unused), au_dense/bias [32], au_prelu/alpha [T][32], au_out/kernel [32] and
// au_out/bias; then the top MLP: W1 [5EP + 8][128] in the tile order of din.cu, b1 and a1 (prelu/alpha) [128],
// W2 [128][64], b2, a2 and w3 [64], b3.  Widths past E, hidden widths and padding rows are zero; every array starts
// on a 256-byte line (a multiple of 64 floats).
struct DinBlob {
  int wsub, wh, wc, wp, au_b, au_alpha, au_wout, au_bout, W1, b1, a1, W2, b2, a2, w3, b3, floats;
  static DinBlob of(int EP, int T) {
    DinBlob l;
    l.wsub = 0;
    l.wh = l.wsub + EP * 32;
    l.wc = l.wh + EP * 32;
    l.wp = l.wc + EP * 32;
    l.au_b = l.wp + EP * 32;
    l.au_alpha = l.au_b + 64;
    l.au_wout = l.au_alpha + (T * 32 + 63) / 64 * 64;
    l.au_bout = l.au_wout + 64;
    l.W1 = l.au_bout + 64;
    l.b1 = l.W1 + (5 * EP + kNumPad) * 128;
    l.a1 = l.b1 + 128;
    l.W2 = l.a1 + 128;
    l.b2 = l.W2 + 128 * 64;
    l.a2 = l.b2 + 64;
    l.w3 = l.a2 + 64;
    l.b3 = l.w3 + 64;
    l.floats = l.b3 + 4;
    return l;
  }
};

// ---- DIEN (DIEN.py:154-256), CUDA-core kernel for E <= 32 -------------------------------------
struct DienParams {
  const float* movie;      // shared candidate/history table [n_movies][EP]
  const float* user;       // [n_users][EP]
  const float* ugenre;     // [19][EP]
  const float* mgenre;     // [19][EP]
  const float* seq;        // GRU + attention + AUGRU weights, the sequence part of a DienLayout blob
  // top MLP, first kernel permuted to the tile order
  //   [userGenre1 | userId | augru state | candidate | movieGenre1] x EP, then 7 numerics + pad
  const float* W1;         // [KP = 5*EP + 8][128]
  const float* b1;         // [128]
  const float* a1;         // [128] PReLU alpha
  const float* W2;         // [128][64]
  const float* b2;         // [64]
  const float* a2;         // [64]
  const float* w3;         // [64]
  float b3;
  int n_movies, n_users, n_genres;
  int T;
  int EP;
};

// The Dense weights of DIEN (a model's and a trainer's) as one blob, offsets in floats.  The sequence part
// (DienParams::seq): gru/kernel and gru_recurrent/kernel [EP k][3][EP] (gates z | r | h), att_dense/kernel [EP][32],
// the AUGRU's In, Hid and Act kernels [3 g][EP][EP] (gates r | z | h), the biases of the GRU's input and recurrent
// side, of In and of Act [3][EP] each, augru_h0 [EP], att_dense/bias, att_out/kernel [32] and att_out/bias (+3 pad).
// Then the auxiliary head (DienAuxView::w): aux_pos_dense/kernel and aux_neg_dense/kernel [2EP][32] (g_t rows, then
// the item rows), their biases [32], aux_pos_out/kernel and aux_neg_out/kernel [32], the two output biases (+2
// pad).  Then the top MLP: W1 [5EP + 8][128] in the tile order of dien.cu, b1 and a1 (prelu/alpha) [128], W2
// [128][64], b2, a2 and w3 [64], b3 (+3 pad).  Widths past E, hidden widths and padding rows are zero; every array
// starts at a multiple of 4 floats, the top MLP's at a multiple of 64.  dien_layers.cuh::DienBlob / DienAuxBlob name the same offsets at compile time.
struct DienLayout {
  int GW, GU, AW, IW, HW, SW, BX, BH, BI, BA, H0, AB, AO, ABO, seq;   // the sequence part; seq = its floats
  int aux;                                                             // the auxiliary head's first float, and
  int PW, NW, PB, NB, PO, NO, POB, NOB, aux_floats;                    //   its offsets relative to it
  int W1, b1, a1, W2, b2, a2, w3, b3, floats;
  __host__ __device__ static constexpr DienLayout of(int EP) {
    DienLayout l{};
    const int EE = EP * EP;
    l.GW = 0;
    l.GU = l.GW + 3 * EE;
    l.AW = l.GU + 3 * EE;
    l.IW = l.AW + 32 * EP;
    l.HW = l.IW + 3 * EE;
    l.SW = l.HW + 3 * EE;
    l.BX = l.SW + 3 * EE;
    l.BH = l.BX + 3 * EP;
    l.BI = l.BH + 3 * EP;
    l.BA = l.BI + 3 * EP;
    l.H0 = l.BA + 3 * EP;
    l.AB = l.H0 + EP;
    l.AO = l.AB + 32;
    l.ABO = l.AO + 32;
    l.seq = l.ABO + 4;
    l.aux = l.seq;
    l.PW = 0;
    l.NW = l.PW + 64 * EP;
    l.PB = l.NW + 64 * EP;
    l.NB = l.PB + 32;
    l.PO = l.NB + 32;
    l.NO = l.PO + 32;
    l.POB = l.NO + 32;
    l.NOB = l.POB + 1;
    l.aux_floats = l.POB + 4;
    l.W1 = (l.aux + l.aux_floats + 63) / 64 * 64;    // the top MLP's rows on 256-byte lines, as dense_layer reads them
    l.b1 = l.W1 + (5 * EP + kNumPad) * 128;
    l.a1 = l.b1 + 128;
    l.W2 = l.a1 + 128;
    l.b2 = l.W2 + 128 * 64;
    l.a2 = l.b2 + 64;
    l.w3 = l.a2 + 64;
    l.b3 = l.w3 + 64;
    l.floats = l.b3 + 4;
    return l;
  }
};

// ---- DIEN's training step (dien_train.cu; DESIGN.md section 4.20) ------------------------------------------------
constexpr int kDienMaxT = 64;        // the longest history the step kernel trains (hist_len 1..64)
constexpr int kDienTables = 4;       // embedding, userId_embedding, userGenre1_embedding, movieGenre1_embedding
struct DienStepArgs {
  DienParams p;            // the trainer's tables and Dense weights (DienLayout blob; p.b3 unused: read from blob)
  const float* blob;       // the Dense-weight blob (b3 at DienLayout::b3, the auxiliary head at DienLayout::aux)
  const int32_t* order;    // [B] the step's rows of the dataset
  const int32_t* movie;    // the dataset [n]: movieId, userId, userGenre1 / movieGenre1 (column 0 of [n][5] / [n][3]
  const int32_t* user;     //   after check), numerics [n][7], history [n][T], negatives [n][T - 1], labels [n]
  const int32_t* ugenre;
  const int32_t* mgenre;
  const float* numerics;
  const int32_t* hist;
  const int32_t* neg;
  const int32_t* label;
  int B;
  int64_t tab_row0[kDienTables];   // first row of each table in the trainer's table array
  float* probs;            // [B] outputs of the step, before its update
  float* logits;
  float* aux;              // [B] each row's sum of pos_t + neg_t
  int32_t* labels;         // [B] the step's labels in step order
  int32_t* trow;           // [(2T + 3) B] table row of entry s * B + r, -1 = none (a missing genre)
  float* gemb;             // [(2T + 3) B][EP] the entries' gradients
  float* rec;              // [B][T][kDienRecSlots][32] per (row, position) inputs and deltas of the Dense products
  float* part;             // [ctas][DienLayout::floats] per-CTA Dense gradient sums
};
int dien_train_ctas(int B);
size_t dien_train_rec_floats(int B, int T);   // the floats of DienStepArgs::rec
cudaError_t launch_dien_train_step(int EP, const DienStepArgs* a, cudaStream_t s);

// ---- DIEN's auxiliary head (DIEN.py:261-292), the AUX variant of dien_kernel --------------------------
struct DienAuxView {
  const float* w;          // aux_pos_* / aux_neg_* weights, the auxiliary part of a DienLayout blob
  const int32_t* neg;      // [B][neg_stride] negtive_userRatedMovie2..T in graph order
  int neg_stride;
  float* aux;              // [B] out: sum over t of pos_t + neg_t
};
// the AUX variant of dien_kernel: probs / logits with the bits of launch_dien, plus aux[B]
cudaError_t launch_dien_aux(const DienParams& p, const DienAuxView& a, const BatchView& b, cudaStream_t s);
// final_loss[i] = bce(logits[i], labels[i]) - 0.5 * mean(aux[0..n)) in float32 (DIEN.py:287), the mean summed
// in double in a fixed order; NaN for a label other than 0 / 1.  sum_dst (or null) gets the double sum of
// final_loss[0..n) in a fixed order.  One CTA.
cudaError_t launch_dien_final_loss(const float* logits, const int32_t* labels, const float* aux, int n,
                                   float* final_loss, double* sum_dst, cudaStream_t s);

// launchers (defined next to their kernels); return cudaGetLastError()
cudaError_t launch_din_wg(const DinParams& p, const BatchView& b, cudaStream_t s);
cudaError_t launch_split_table(const float* src, void* dst, int64_t rows, int EP, cudaStream_t s);
cudaError_t launch_ncf(const NcfParams& p, const BatchView& b, cudaStream_t s);
cudaError_t launch_embmlp(const EmbMlpParams& p, const BatchView& b, cudaStream_t s);
cudaError_t launch_embmlp_tc(const EmbMlpParams& p, const BatchView& b, cudaStream_t s);
cudaError_t launch_deepfm(const DeepFmParams& p, const BatchView& b, cudaStream_t s);
cudaError_t launch_deepfm_tc(const DeepFmParams& p, const BatchView& b, cudaStream_t s);
cudaError_t launch_deepfm2(const DeepFm2Params& p, const BatchView& b, cudaStream_t s);
cudaError_t launch_din(const DinParams& p, const BatchView& b, cudaStream_t s);
cudaError_t launch_dien(const DienParams& p, const BatchView& b, cudaStream_t s);
cudaError_t setup_dien_attributes();
cudaError_t launch_fill_uniform(float* x, int64_t n, uint64_t seed, float lo, float hi,
                                cudaStream_t s);
cudaError_t launch_wgmma_selftest(const float* A, const float* B, float* D, int N, int KB,
                                  int a_in_regs, cudaStream_t s);
cudaError_t launch_cosine(const float* q, const float* c, int n, int dim, float* out,
                          cudaStream_t s);
cudaError_t launch_widen_u16(const uint16_t* src, int32_t* dst, int64_t n, cudaStream_t s);
// n_req user records of 9 + hc words x n_cand candidate ids -> n_req * n_cand packed rows, user-major (util.cu)
cudaError_t launch_assemble_request(const int32_t* req, int n_req, const int32_t* cand, int n_cand,
                                    const void* movie_feats, int n_table, int hc, int dense, int32_t* movie_id,
                                    int32_t* user_id, int32_t* hist, int32_t* movie_genre, int32_t* user_genre,
                                    float* numerics, int* err_flag, cudaStream_t s);
// topk.cu: ranking = descending score, ties by position; min(k, n) results
size_t topk_scratch_bytes(int n);
cudaError_t launch_topk(const float* scores, int n, int k, int32_t* top_idx, float* top_scores,
                        void* scratch, cudaStream_t s);
// latency path: the last kernel of the call publishes {seq, error word (cleared)} to a host-mapped record
cudaError_t launch_topk_done(const float* scores, int n, int k, int32_t* top_idx, float* top_scores,
                             void* scratch, int* err_flag, uint32_t* done, uint32_t seq, cudaStream_t s);
cudaError_t launch_finish(int* err_flag, uint32_t* done, uint32_t seq, cudaStream_t s);

// ---- metrics.cu: Keras's evaluate metrics (loss, accuracy, ROC / PR AUC) over labelled batches -----------
constexpr int kMetThresholds = 200;        // Keras AUC num_thresholds
constexpr int kMetBins = kMetThresholds + 1;   // bin k = #{j : p > t_j}, 0..200
constexpr int kMetMaxCtas = 264;           // CTAs of one update launch (fixed by n alone: the loss bits do not
                                           // depend on the SM count or an SM limit)
constexpr int kMetErrLabel = 1;            // MetricsCounters::err bits: a label other than 0 / 1
constexpr int kMetErrProb = 2;             //   a probability that is NaN or outside [0, 1]
struct MetricsCounters {                   // device, zeroed by a reset; integer atomics only
  unsigned long long hist[2 * kMetBins];   // [label 0 | label 1][bin]
  unsigned long long correct;
  int err;
  int pad_;
};
struct MetricsReduce {                     // per stream of updates: the last CTA sums partial[] in CTA order
  unsigned int ticket;
  unsigned int pad_;
  double partial[kMetMaxCtas];
};
struct MetricsState {                      // one history (srs_metrics, an epoch of a fit): counts, loss sum, reduce
  MetricsCounters cnt;
  double loss;
  MetricsReduce red;
};
// Fold n rows into `cnt`; the rows' loss sum goes to *loss_dst (added to it when `accumulate`; not written
// when loss_dst is null).  `own_hist` (zeroed by the caller, or null): the batch's own 2 x 201 (label, bin)
// counts are added to it as well.  Launches sharing one `red` must be stream-ordered.
cudaError_t launch_metrics_update(const float* probs, const float* logits, const int32_t* labels, int n,
                                  MetricsCounters* cnt, MetricsReduce* red, double* loss_dst, int accumulate,
                                  cudaStream_t s, unsigned long long* own_hist = nullptr);
// The weighted sums of Keras's metrics with sample weights w_i (DESIGN.md section 4.28), in double: hist is
// MetricsCounters::hist with each row counted as w_i, correct = sum w_i [row correct], sum = sum w_i.  The loss
// sum of a weighted update is sum w_i l_i, with w_i l_i rounded to float32 as Keras multiplies.
struct MetricsWeighted {
  double hist[2 * kMetBins];
  double correct;
  double sum;
};
constexpr int kMetWSums = 2 * kMetBins + 2;      // the doubles of MetricsWeighted
static_assert(sizeof(MetricsWeighted) == kMetWSums * sizeof(double), "MetricsWeighted is an array of doubles");
// The weighted update's per-CTA partials, summed by the last CTA in CTA order; launches sharing one must be
// stream-ordered.  It needs no reset.
struct MetricsWeightedReduce {
  double partial[kMetMaxCtas][kMetWSums];
};
// launch_metrics_update with row weights w [n]: the integer counts and the error word as launch_metrics_update folds
// them, the loss sum of w_i l_i into *loss_dst, and the weighted sums into *wdst (added to it when `accumulate`).
// No float atomics: each CTA sums its rows' weights per bin in row order and the last CTA adds the CTA partials in
// CTA order, so the result has the same bits on every run and does not depend on the SM count.  One launch.
cudaError_t launch_metrics_update_weighted(const float* probs, const float* logits, const int32_t* labels,
                                           const float* w, int n, MetricsCounters* cnt, MetricsReduce* red,
                                           double* loss_dst, MetricsWeighted* wdst, MetricsWeightedReduce* wred,
                                           int accumulate, cudaStream_t s);
// DIEN's auc_value: `hist` holds K batch histograms [K][2 x 201] in batch order and is turned into their
// prefix sums in place; auc[k] (K doubles) = the ROC AUC of batches 0..k in double, *sum_dst = their sum,
// added in batch order.  Three launches on `s`.
cudaError_t launch_auc_value(unsigned long long* hist, int K, double* auc, double* sum_dst, cudaStream_t s);
// host: the counts -> srs_eval_result (AUCs in double); `confusion` NULL or [4][200] tp, fp, tn, fn
void metrics_summarise(const unsigned long long* hist, unsigned long long correct, double loss_sum,
                       srs_eval_result* out, int64_t* confusion);
// the same with weights: rows, positives and correct from the counts, loss = loss_sum / rows (loss_sum = sum w l),
// accuracy = div_no_nan(w.correct, w.sum) and the AUCs from the weighted bins
void metrics_summarise_weighted(const unsigned long long* hist, unsigned long long correct, const MetricsWeighted& w,
                                double loss_sum, srs_eval_result* out);

extern int64_t g_launch_count;   // kernels launched by this library

}  // namespace srs
