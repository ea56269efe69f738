// placement.h - where the Keras tensors of the serving models (NeuralCF's neural_cf_model_1 and two towers, DeepFM,
// DeepFM_v2, EmbeddingMLP / Wide&Deep, DIN and DIEN) live on the device, written once for the serving builders
// (build_ncf, build_deepfm, build_deepfm2, build_embmlp, build_din, build_dien in model.cu; the tensor-core builders
// derive their operand images from the blobs placed here) and the trainer (srs_trainer_create,
// srs_trainer_get_weights in trainer.cu): the builders and the trainer scatter the caller's host tensors through it,
// and the trainer gathers its weights back through it.  Also the by-name lookup of the caller's tensors that both
// use.  Host code only.
#pragma once

#include <stdint.h>
#include <stdio.h>

#include <map>
#include <string>
#include <vector>

#include "../../include/srs_ctr.h"
#include "hostcall.h"

namespace srs {

// an embedding width padded to the kernels' instantiations
inline int round_ep(int E) {
  if (E <= 12) return 12;
  if (E <= 16) return 16;
  if (E <= 32) return 32;
  return 64;
}

// n rows start, start + 1, ... then padded - n rows of -1
inline std::vector<int> iota_map(int start, int n, int padded) {
  std::vector<int> v(padded, -1);
  for (int i = 0; i < n; ++i) v[i] = start + i;
  return v;
}

inline void append(std::vector<int>& a, const std::vector<int>& b) { a.insert(a.end(), b.begin(), b.end()); }

// The caller's tensors by name (a name given twice: the last one).  A failed lookup sets `status` and the error
// message; every later lookup then returns null and keeps them.
struct TensorLookup {
  std::map<std::string, const srs_tensor*> by_name;
  int status = SRS_OK;

  TensorLookup(const srs_tensor* ts, int n) {
    for (int i = 0; i < n; ++i)
      if (ts[i].name) by_name[ts[i].name] = &ts[i];
  }

  const srs_tensor* need(const char* name, int64_t rows, int64_t cols) {
    if (status != SRS_OK) return nullptr;
    auto it = by_name.find(name);
    if (it == by_name.end()) {
      status = failf(SRS_ERR_MISSING, "missing weight tensor '%s'", name);
      return nullptr;
    }
    const srs_tensor* t = it->second;
    if (t->rows != rows || t->cols != cols) {
      status = failf(SRS_ERR_SHAPE, "weight '%s' has shape [%lld,%lld], expected [%lld,%lld]", name,
                     (long long)t->rows, (long long)t->cols, (long long)rows, (long long)cols);
      return nullptr;
    }
    if (t->data == nullptr) {
      status = failf(SRS_ERR_INVALID, "weight '%s' has a null data pointer", name);
      return nullptr;
    }
    return t;
  }

  // a tensor the caller holds in host memory: its data
  const float* host(const char* name, int64_t rows, int64_t cols) {
    const srs_tensor* t = need(name, rows, cols);
    if (!t) return nullptr;
    if (t->location != SRS_HOST) {
      status = failf(SRS_ERR_INVALID, "weight '%s' must be a host tensor", name);
      return nullptr;
    }
    return t->data;
  }
};

// Rows of a Dense tensor [rows][cols] in one zero-padded block of the Dense-weight blob or of the one-hot array
struct Block {
  bool onehot;                   // false: the blob; true: the one-hot array, the [fm1_width] one-hot rows of DeepFM's
                                 // dense_2/kernel or DeepFM_v2's first_cat/kernel, or the [cross_buckets] wide rows of
                                 // Wide&Deep's dense_2/kernel
  int at;                        // the block's first float
  int width;                     // floats per block row: the tensor's cols, zero padded
  std::vector<int> map;          // block row i holds tensor row map[i]; -1: a zero row
  int col0 = 0, ncols = 0;       // the block holds columns col0 .. col0 + ncols of those rows (ncols 0: all)
};

struct Placed {                  // one Keras tensor [rows][cols]
  std::string name;
  int64_t rows, cols;
  int64_t table_row;             // an embedding table: its first row in a trainer's [sum of rows][EP] array; else -1
  std::vector<Block> blocks;     // a Dense tensor: where its rows go
};

// a model's tensors in the order they are looked up: its tables, then its Dense tensors
using Placement = std::vector<Placed>;

inline void place_table(Placement& pl, const char* name, int64_t rows, int E) {
  const int64_t row = pl.empty() ? 0 : pl.back().table_row + pl.back().rows;
  pl.push_back(Placed{name, rows, E, row, {}});
}

inline void place_dense(Placement& pl, const char* name, int64_t rows, int64_t cols, std::vector<Block> blocks) {
  pl.push_back(Placed{name, rows, cols, -1, std::move(blocks)});
}

// The rows of a trainer's table array: the tables' rows, one table after another
inline int64_t table_rows(const Placement& pl) {
  int64_t n = 0;
  for (const Placed& x : pl)
    if (x.table_row >= 0) n += x.rows;
  return n;
}

// NeuralCF and two towers.  The blob: per hidden layer its kernel [2EP (two towers: EP) or HP][HP] and its bias
// [HP] (two towers: the item tower's layers, then the user tower's), then the output kernel and bias, each block a
// multiple of 4 floats.  Fills p's layout: EP, HP, n_layers, the offsets and blob_floats.  Without dense_out, two
// towers' out_w and out_b are 4 floats each that no tensor fills (build_ncf writes 1 and 0).
inline Placement place_ncf(const srs_spec& s, int EP, int HP, NcfParams* p) {
  const int E = s.emb_dim, L = s.n_hidden;
  const bool two = s.kind == SRS_TWOTOWERS;
  Placement pl;
  place_table(pl, "movieId_embedding", s.n_movies, E);
  place_table(pl, "userId_embedding", s.n_users, E);
  int off = 0;
  auto dense = [&](const char* name, int64_t rows, int64_t cols, std::vector<int> map, int width) {
    const int at = off;
    off += ((int)map.size() * width + 3) / 4 * 4;
    place_dense(pl, name, rows, cols, {Block{false, at, width, std::move(map)}});
    return at;
  };
  char k[48], b[48];
  for (int t = 0; t < (two ? 2 : 1); ++t) {
    int in = two ? E : 2 * E;
    for (int l = 0; l < L; ++l) {
      const int out = s.hidden[l];
      if (two) {
        snprintf(k, sizeof k, "%s_dense_%d/kernel", t ? "user" : "item", l);
        snprintf(b, sizeof b, "%s_dense_%d/bias", t ? "user" : "item", l);
      } else {
        snprintf(k, sizeof k, "dense_%d/kernel", l);
        snprintf(b, sizeof b, "dense_%d/bias", l);
      }
      std::vector<int> map;
      if (l == 0) {                                     // the embedding rows, each side padded to EP
        map = iota_map(0, E, EP);
        if (!two) append(map, iota_map(E, E, EP));
      } else {
        map = iota_map(0, in, HP);
      }
      p->w_off[3 * t + l] = dense(k, in, out, map, HP);
      p->b_off[3 * t + l] = dense(b, out, 1, iota_map(0, out, HP), 1);
      in = out;
    }
    if (!two) {
      snprintf(k, sizeof k, "dense_%d/kernel", L);
      snprintf(b, sizeof b, "dense_%d/bias", L);
      p->out_w = dense(k, in, 1, iota_map(0, in, HP), 1);
      p->out_b = dense(b, 1, 1, iota_map(0, 1, 4), 1);
    }
  }
  if (two && s.final_dense) {
    p->out_w = dense("dense_out/kernel", 1, 1, iota_map(0, 1, 4), 1);
    p->out_b = dense("dense_out/bias", 1, 1, iota_map(0, 1, 4), 1);
  } else if (two) {
    p->out_w = off; off += 4;
    p->out_b = off; off += 4;
  }
  p->blob_floats = off;
  p->n_movies = s.n_movies; p->n_users = s.n_users;
  p->EP = EP; p->HP = HP; p->n_layers = L; p->two_towers = two; p->final_dense = s.final_dense;
  return pl;
}

// DeepFM: the six tables in kDeepFmTables order, the Dense tensors in a DeepFmBlob::of(EP) and the one-hot rows of
// dense_2/kernel in their own [fm1_width] array.  Fills p's sizes and EP.
inline Placement place_deepfm(const srs_spec& s, int EP, DeepFmParams* p) {
  const int E = s.emb_dim, h0 = s.hidden[0], h1 = s.hidden[1];
  const int fm1 = 2 * s.n_genres + s.n_movies + s.n_users;
  const DeepFmBlob ly = DeepFmBlob::of(EP);
  Placement pl;
  place_table(pl, "fm_movieId_embedding", s.n_movies, E);
  place_table(pl, "fm_userId_embedding", s.n_users, E);
  place_table(pl, "fm_movieGenre1_embedding", s.n_genres, E);
  place_table(pl, "fm_userGenre1_embedding", s.n_genres, E);
  place_table(pl, "deep_movieId_embedding", s.n_movies, E);
  place_table(pl, "deep_userId_embedding", s.n_users, E);
  // dense/kernel's rows are DenseFeatures' sorted concat (movieAvgRating | deep movieId | 4 numerics | deep userId |
  // 2 numerics); its tile rows are deep movieId | deep userId | the 7 numerics and one zero row
  std::vector<int> map;
  append(map, iota_map(1, E, EP));
  append(map, iota_map(5 + E, E, EP));
  for (int r : {0, 1 + E, 2 + E, 3 + E, 4 + E, 5 + 2 * E, 6 + 2 * E, -1}) map.push_back(r);
  place_dense(pl, "dense/kernel", 7 + 2 * E, h0, {Block{false, ly.W1, 64, map}});
  place_dense(pl, "dense/bias", h0, 1, {Block{false, ly.b1, 1, iota_map(0, h0, 64)}});
  place_dense(pl, "dense_1/kernel", h0, h1, {Block{false, ly.W2, 64, iota_map(0, h0, 64)}});
  place_dense(pl, "dense_1/bias", h1, 1, {Block{false, ly.b2, 1, iota_map(0, h1, 64)}});
  // dense_2/kernel: the one-hot rows (movieGenre1 | movieId | userGenre1 | userId), the four dot rows, the deep rows
  place_dense(pl, "dense_2/kernel", fm1 + 4 + h1, 1,
              {Block{true, 0, 1, iota_map(0, fm1, fm1)}, Block{false, ly.wdot, 1, iota_map(fm1, 4, 4)},
               Block{false, ly.wdeep, 1, iota_map(fm1 + 4, h1, 64)}});
  place_dense(pl, "dense_2/bias", 1, 1, {Block{false, ly.bout, 1, iota_map(0, 1, 1)}});
  p->n_movies = s.n_movies; p->n_users = s.n_users; p->n_genres = s.n_genres; p->EP = EP;
  return pl;
}

// p's Dense-weight pointers into a DeepFmBlob on the device
inline void point_into_blob(DeepFmParams* p, const float* blob) {
  const DeepFmBlob ly = DeepFmBlob::of(p->EP);
  p->blob = blob;
  p->W1 = blob + ly.W1; p->b1 = blob + ly.b1; p->W2 = blob + ly.W2; p->b2 = blob + ly.b2;
  p->wdeep = blob + ly.wdeep;
}

// DeepFM_v2: the four tables in field order (movieGenre1, movieId, userGenre1, userId: kDeepFm2Tables), the Dense
// tensors in a DeepFm2Blob::of(EP) and first_cat/kernel's one-hot rows in their own [fm1_width] array, looked up in
// the order the builder has always used.  Fills p's sizes and EP.
inline Placement place_deepfm2(const srs_spec& s, int EP, DeepFm2Params* p) {
  const int E = s.emb_dim, h0 = s.hidden[0], h1 = s.hidden[1], P = 64;
  const int fm1 = 2 * s.n_genres + s.n_movies + s.n_users;
  const DeepFm2Blob ly = DeepFm2Blob::of(EP);
  const char* fields[4] = {"movieGenre1", "movieId", "userGenre1", "userId"};
  const int64_t rows[4] = {s.n_genres, s.n_movies, s.n_genres, s.n_users};
  Placement pl;
  char name[64];
  for (int f = 0; f < 4; ++f) {
    snprintf(name, sizeof name, "%s_embedding", fields[f]);
    place_table(pl, name, rows[f], E);
  }
  place_dense(pl, "first_cat/kernel", fm1, 1, {Block{true, 0, 1, iota_map(0, fm1, fm1)}});
  place_dense(pl, "first_cat/bias", 1, 1, {Block{false, ly.first_cat_b, 1, iota_map(0, 1, 1)}});
  place_dense(pl, "first_num/kernel", kNumNumerics, 1, {Block{false, ly.first_num, 1, iota_map(0, 7, kNumPad)}});
  place_dense(pl, "first_num/bias", 1, 1, {Block{false, ly.first_num_b, 1, iota_map(0, 1, 1)}});
  for (int f = 0; f < 4; ++f) {
    snprintf(name, sizeof name, "proj_%s/kernel", fields[f]);
    place_dense(pl, name, E, P, {Block{false, ly.proj + f * EP * P, P, iota_map(0, E, EP)}});
    snprintf(name, sizeof name, "proj_%s/bias", fields[f]);
    place_dense(pl, name, P, 1, {Block{false, ly.proj_b + f * P, 1, iota_map(0, P, P)}});
  }
  place_dense(pl, "proj_num/kernel", kNumNumerics, P, {Block{false, ly.proj_num, P, iota_map(0, 7, kNumPad)}});
  place_dense(pl, "proj_num/bias", P, 1, {Block{false, ly.proj_num_b, 1, iota_map(0, P, P)}});
  place_dense(pl, "deep/kernel", 5 * P, h0, {Block{false, ly.Wd, 32, iota_map(0, 5 * P, 5 * P)}});
  place_dense(pl, "deep/bias", h0, 1, {Block{false, ly.bd, 1, iota_map(0, h0, 32)}});
  place_dense(pl, "deep_1/kernel", h0, h1, {Block{false, ly.Wd1, 16, iota_map(0, h0, 32)}});
  place_dense(pl, "deep_1/bias", h1, 1, {Block{false, ly.bd1, 1, iota_map(0, h1, 16)}});
  // out/kernel: first | fm (64) | deep (h1), the deep rows padded to 16
  place_dense(pl, "out/kernel", 1 + P + h1, 1, {Block{false, ly.wout, 1, iota_map(0, 1 + P + h1, 84)}});
  place_dense(pl, "out/bias", 1, 1, {Block{false, ly.bout, 1, iota_map(0, 1, 1)}});
  p->n_movies = s.n_movies; p->n_users = s.n_users; p->n_genres = s.n_genres; p->EP = EP;
  return pl;
}

// p's tables (tables[k]: the k-th table of place_deepfm2's order) and Dense-weight pointers into a DeepFm2Blob on
// the device
inline void point_into_blob(DeepFm2Params* p, const float* const* tables, const float* blob) {
  const DeepFm2Blob ly = DeepFm2Blob::of(p->EP);
  p->mgenre = tables[0]; p->movie = tables[1]; p->ugenre = tables[2]; p->user = tables[3];
  p->blob = blob;
  p->first_num = blob + ly.first_num;
  for (int f = 0; f < 4; ++f) {
    p->proj[f] = blob + ly.proj + f * p->EP * 64;
    p->proj_b[f] = blob + ly.proj_b + f * 64;
  }
  p->proj_num = blob + ly.proj_num; p->proj_num_b = blob + ly.proj_num_b;
  p->Wd = blob + ly.Wd; p->bd = blob + ly.bd; p->Wd1 = blob + ly.Wd1; p->bd1 = blob + ly.bd1;
  p->wout = blob + ly.wout;
}

// EmbeddingMLP and Wide&Deep: the ten tables (movieGenre1..3, userGenre1..5, movieId, userId: the order the
// builder has always looked them up in; EmbMlpSlotTable maps a kernel slot to it), the Dense tensors in an
// EmbMlpBlob::of(EP) and, for Wide&Deep, the wide rows of dense_2/kernel in their own [cross_buckets] one-hot array.
// Fills p's sizes and EP.
constexpr int kEmbMlpSlotTable[10] = {0, 1, 2, 8, 3, 4, 5, 6, 7, 9};   // kernel slot -> placement index

inline Placement place_embmlp(const srs_spec& s, int EP, EmbMlpParams* p) {
  const int E = s.emb_dim, h0 = s.hidden[0], h1 = s.hidden[1];
  const bool wide = s.kind == SRS_WIDENDEEP;
  const EmbMlpBlob ly = EmbMlpBlob::of(EP);
  Placement pl;
  char name[48];
  for (int k = 1; k <= 3; ++k) {
    snprintf(name, sizeof name, "movieGenre%d_embedding", k);
    place_table(pl, name, s.n_genres, E);
  }
  for (int k = 1; k <= 5; ++k) {
    snprintf(name, sizeof name, "userGenre%d_embedding", k);
    place_table(pl, name, s.n_genres, E);
  }
  place_table(pl, "movieId_embedding", s.n_movies, E);
  place_table(pl, "userId_embedding", s.n_users, E);
  // dense/kernel's rows are DenseFeatures' sorted concat (movieAvgRating | movieGenre1..3 | movieId | 4 numerics |
  // userGenre1..5 | userId | 2 numerics); its tile rows are the ten slots, then the 7 numerics and one zero row
  std::vector<int> map;
  for (int k = 0; k < 3; ++k) append(map, iota_map(1 + k * E, E, EP));         // movieGenre1..3
  append(map, iota_map(1 + 3 * E, E, EP));                                        // movieId
  for (int k = 0; k < 5; ++k) append(map, iota_map(5 + 4 * E + k * E, E, EP));   // userGenre1..5
  append(map, iota_map(5 + 9 * E, E, EP));                                        // userId
  for (int r : {0, 1 + 4 * E, 2 + 4 * E, 3 + 4 * E, 4 + 4 * E, 5 + 10 * E, 6 + 10 * E, -1}) map.push_back(r);
  place_dense(pl, "dense/kernel", 7 + 10 * E, h0, {Block{false, ly.W1, 128, map}});
  place_dense(pl, "dense/bias", h0, 1, {Block{false, ly.b1, 1, iota_map(0, h0, 128)}});
  place_dense(pl, "dense_1/kernel", h0, h1, {Block{false, ly.W2, 128, iota_map(0, h0, 128)}});
  place_dense(pl, "dense_1/bias", h1, 1, {Block{false, ly.b2, 1, iota_map(0, h1, 128)}});
  // dense_2/kernel: the deep rows, then (Wide&Deep) the wide rows
  std::vector<Block> k3 = {Block{false, ly.w3, 1, iota_map(0, h1, 128)}};
  if (wide) k3.push_back(Block{true, 0, 1, iota_map(h1, s.cross_buckets, s.cross_buckets)});
  place_dense(pl, "dense_2/kernel", h1 + (wide ? s.cross_buckets : 0), 1, std::move(k3));
  place_dense(pl, "dense_2/bias", 1, 1, {Block{false, ly.b3, 1, iota_map(0, 1, 1)}});
  p->n_movies = s.n_movies; p->n_users = s.n_users; p->n_genres = s.n_genres;
  p->cross_buckets = s.cross_buckets; p->EP = EP;
  return pl;
}

// p's tables (tables[k]: the k-th table of place_embmlp's order) and Dense-weight pointers into an EmbMlpBlob on the
// device
inline void point_into_blob(EmbMlpParams* p, const float* const* tables, const float* blob) {
  const EmbMlpBlob ly = EmbMlpBlob::of(p->EP);
  for (int k = 0; k < 8; ++k) p->genre[k] = tables[k];
  p->movie = tables[8];
  p->user = tables[9];
  p->W1 = blob + ly.W1; p->b1 = blob + ly.b1; p->W2 = blob + ly.W2; p->b2 = blob + ly.b2;
  p->w3 = blob + ly.w3; p->b3 = blob + ly.b3;
}

// The top MLP of DIN and DIEN (dense/kernel .. dense_2/bias with the PReLU alphas) at ly's offsets W1 .. b3.
// dense/kernel's rows are the concat of the sequence output (DIN's pooled behaviours, DIEN's AUGRU state), the
// candidate embedding and the user_profile and context DenseFeatures layers, each layer sorted by column name
// inside; up, seq, cand and ctx are the first rows of the four.  Its tile rows are userGenre1 | userId | sequence |
// candidate | movieGenre1, then the 7 numerics and one zero row.
template <class Layout>
inline void place_top_mlp(Placement& pl, const srs_spec& s, int EP, const Layout& ly, int up, int seq, int cand,
                          int ctx) {
  const int E = s.emb_dim, h0 = s.hidden[0], h1 = s.hidden[1];
  std::vector<int> map;
  append(map, iota_map(up + 1, E, EP));
  append(map, iota_map(up + 1 + E, E, EP));
  append(map, iota_map(seq, E, EP));
  append(map, iota_map(cand, E, EP));
  append(map, iota_map(ctx + 1, E, EP));
  for (int r : {ctx, ctx + 1 + E, ctx + 2 + E, ctx + 3 + E, up, up + 1 + 2 * E, up + 2 + 2 * E, -1}) map.push_back(r);
  place_dense(pl, "dense/kernel", 5 * E + 7, h0, {Block{false, ly.W1, 128, map}});
  place_dense(pl, "dense/bias", h0, 1, {Block{false, ly.b1, 1, iota_map(0, h0, 128)}});
  place_dense(pl, "prelu/alpha", h0, 1, {Block{false, ly.a1, 1, iota_map(0, h0, 128)}});
  place_dense(pl, "dense_1/kernel", h0, h1, {Block{false, ly.W2, 64, iota_map(0, h0, 128)}});
  place_dense(pl, "dense_1/bias", h1, 1, {Block{false, ly.b2, 1, iota_map(0, h1, 64)}});
  place_dense(pl, "prelu_1/alpha", h1, 1, {Block{false, ly.a2, 1, iota_map(0, h1, 64)}});
  place_dense(pl, "dense_2/kernel", h1, 1, {Block{false, ly.w3, 1, iota_map(0, h1, 64)}});
  place_dense(pl, "dense_2/bias", 1, 1, {Block{false, ly.b3, 1, iota_map(0, 1, 1)}});
}

// DIN: the four tables (embedding, userId_embedding, userGenre1_embedding, movieGenre1_embedding) and the Dense
// tensors in one DinBlob::of(EP, T), looked up in the order the builder has always used.  au_dense/kernel's four
// E-row groups go unfolded into the blob's W_sub, W_h, W_c and W_prod blocks (build_din folds them).  Fills p's
// sizes, T and EP.
inline Placement place_din(const srs_spec& s, int EP, DinParams* p) {
  const int E = s.emb_dim, T = s.hist_len, A = 32;
  const DinBlob ly = DinBlob::of(EP, T);
  Placement pl;
  place_table(pl, "embedding", s.n_movies, E);
  place_table(pl, "userId_embedding", s.n_users, E);
  place_table(pl, "userGenre1_embedding", s.n_genres, E);
  place_table(pl, "movieGenre1_embedding", s.n_genres, E);
  // au_dense/kernel's rows are [h - c | h | c | h * c], E each (DIN.py:146-149)
  const int au[4] = {ly.wsub, ly.wh, ly.wc, ly.wp};
  std::vector<Block> aub;
  for (int g = 0; g < 4; ++g) aub.push_back(Block{false, au[g], A, iota_map(g * E, E, EP)});
  place_dense(pl, "au_dense/kernel", 4 * E, A, std::move(aub));
  place_dense(pl, "au_dense/bias", A, 1, {Block{false, ly.au_b, 1, iota_map(0, A, A)}});
  place_dense(pl, "au_prelu/alpha", T, A, {Block{false, ly.au_alpha, A, iota_map(0, T, T)}});
  place_dense(pl, "au_out/kernel", A, 1, {Block{false, ly.au_wout, 1, iota_map(0, A, A)}});
  place_dense(pl, "au_out/bias", 1, 1, {Block{false, ly.au_bout, 1, iota_map(0, 1, 1)}});
  // dense/kernel's rows are [user_profile | pooled | candidate | context] (DIN.py:161-162)
  place_top_mlp(pl, s, EP, ly, 0, 3 + 2 * E, 3 + 3 * E, 3 + 4 * E);
  p->n_movies = s.n_movies; p->n_users = s.n_users; p->n_genres = s.n_genres;
  p->T = T; p->EP = EP;
  return pl;
}

// p's tables (tables[k]: the k-th table of place_din's order) and Dense-weight pointers into a folded DinBlob on
// the device; p->au_bout and p->b3 from the host copy of the blob
inline void point_into_blob(DinParams* p, const float* const* tables, const float* blob, const float* host_blob) {
  const DinBlob ly = DinBlob::of(p->EP, p->T);
  p->movie = tables[0]; p->user = tables[1]; p->ugenre = tables[2]; p->mgenre = tables[3];
  p->au_wh = blob + ly.wh; p->au_wp = blob + ly.wp; p->au_wc = blob + ly.wc; p->au_b = blob + ly.au_b;
  p->au_alpha = blob + ly.au_alpha; p->au_wout = blob + ly.au_wout;
  p->au_bout = host_blob[ly.au_bout];
  p->W1 = blob + ly.W1; p->b1 = blob + ly.b1; p->a1 = blob + ly.a1;
  p->W2 = blob + ly.W2; p->b2 = blob + ly.b2; p->a2 = blob + ly.a2;
  p->w3 = blob + ly.w3;
  p->b3 = host_blob[ly.b3];
}

// DIEN: the four tables (embedding, userId_embedding, userGenre1_embedding, movieGenre1_embedding: kDienTables
// order) and the Dense tensors in one DienLayout::of(EP) blob, looked up in the order the builder has always used;
// `aux`: with the auxiliary head's group of eight (else its part of the blob stays zero).  The GRU's kernels and
// biases keep Keras's z | r | h column blocks, each padded to EP.  Fills p's sizes, T and EP.
inline Placement place_dien(const srs_spec& s, int EP, bool aux, DienParams* p) {
  const int E = s.emb_dim, A = 32, EE = EP * EP;
  const DienLayout ly = DienLayout::of(EP);
  Placement pl;
  place_table(pl, "embedding", s.n_movies, E);
  place_table(pl, "userId_embedding", s.n_users, E);
  place_table(pl, "userGenre1_embedding", s.n_genres, E);
  place_table(pl, "movieGenre1_embedding", s.n_genres, E);
  auto gates = [&](int at, int stride, std::vector<int> map) {   // a [.][3E] tensor's z | r | h blocks
    std::vector<Block> b;
    for (int g = 0; g < 3; ++g) b.push_back(Block{false, at + g * EP, stride, map, g * E, E});
    return b;
  };
  place_dense(pl, "gru/kernel", E, 3 * E, gates(ly.GW, 3 * EP, iota_map(0, E, E)));
  place_dense(pl, "gru_recurrent/kernel", E, 3 * E, gates(ly.GU, 3 * EP, iota_map(0, E, E)));
  std::vector<Block> gb = gates(ly.BX, EP, {0}), gbh = gates(ly.BH, EP, {1});
  gb.insert(gb.end(), gbh.begin(), gbh.end());
  place_dense(pl, "gru/bias", 2, 3 * E, gb);
  place_dense(pl, "att_dense/kernel", E, A, {Block{false, ly.AW, 32, iota_map(0, E, E)}});
  place_dense(pl, "att_dense/bias", A, 1, {Block{false, ly.AB, 1, iota_map(0, A, A)}});
  place_dense(pl, "att_out/kernel", A, 1, {Block{false, ly.AO, 1, iota_map(0, A, A)}});
  place_dense(pl, "att_out/bias", 1, 1, {Block{false, ly.ABO, 1, iota_map(0, 1, 1)}});
  const char* gate[3] = {"r", "z", "h"};
  char name[64];
  for (int g = 0; g < 3; ++g) {
    snprintf(name, sizeof name, "augru_%s_input/kernel", gate[g]);
    place_dense(pl, name, E, E, {Block{false, ly.IW + g * EE, EP, iota_map(0, E, E)}});
    snprintf(name, sizeof name, "augru_%s_input/bias", gate[g]);
    place_dense(pl, name, E, 1, {Block{false, ly.BI + g * EP, 1, iota_map(0, E, E)}});
    snprintf(name, sizeof name, "augru_%s_hidden/kernel", gate[g]);
    place_dense(pl, name, E, E, {Block{false, ly.HW + g * EE, EP, iota_map(0, E, E)}});
    snprintf(name, sizeof name, "augru_%s_act/kernel", gate[g]);
    place_dense(pl, name, E, E, {Block{false, ly.SW + g * EE, EP, iota_map(0, E, E)}});
    snprintf(name, sizeof name, "augru_%s_act/bias", gate[g]);
    place_dense(pl, name, E, 1, {Block{false, ly.BA + g * EP, 1, iota_map(0, E, E)}});
  }
  place_dense(pl, "augru_h0", 1, E, {Block{false, ly.H0, EP, {0}}});
  // dense/kernel's rows are [augru | candidate | user_profile | context] (DIEN.py:250)
  place_top_mlp(pl, s, EP, ly, 2 * E, 0, E, 4 * E + 3);
  if (aux) {                                   // [g_t | e] rows: E hidden-state rows, then E item rows
    std::vector<int> amap = iota_map(0, E, EP);
    append(amap, iota_map(E, E, EP));
    for (int side = 0; side < 2; ++side) {
      const char* sd = side ? "neg" : "pos";
      snprintf(name, sizeof name, "aux_%s_dense/kernel", sd);
      place_dense(pl, name, 2 * E, A, {Block{false, ly.aux + (side ? ly.NW : ly.PW), 32, amap}});
      snprintf(name, sizeof name, "aux_%s_dense/bias", sd);
      place_dense(pl, name, A, 1, {Block{false, ly.aux + (side ? ly.NB : ly.PB), 1, iota_map(0, A, A)}});
      snprintf(name, sizeof name, "aux_%s_out/kernel", sd);
      place_dense(pl, name, A, 1, {Block{false, ly.aux + (side ? ly.NO : ly.PO), 1, iota_map(0, A, A)}});
      snprintf(name, sizeof name, "aux_%s_out/bias", sd);
      place_dense(pl, name, 1, 1, {Block{false, ly.aux + (side ? ly.NOB : ly.POB), 1, iota_map(0, 1, 1)}});
    }
  }
  p->n_movies = s.n_movies; p->n_users = s.n_users; p->n_genres = s.n_genres;
  p->T = s.hist_len; p->EP = EP;
  return pl;
}

// p's tables (tables[k]: the k-th table of place_dien's order) and Dense-weight pointers into a DienLayout blob on
// the device; p->b3 from the host copy of the blob
inline void point_into_blob(DienParams* p, const float* const* tables, const float* blob, const float* host_blob) {
  const DienLayout ly = DienLayout::of(p->EP);
  p->movie = tables[0]; p->user = tables[1]; p->ugenre = tables[2]; p->mgenre = tables[3];
  p->seq = blob;
  p->W1 = blob + ly.W1; p->b1 = blob + ly.b1; p->a1 = blob + ly.a1;
  p->W2 = blob + ly.W2; p->b2 = blob + ly.b2; p->a2 = blob + ly.a2;
  p->w3 = blob + ly.w3;
  p->b3 = host_blob[ly.b3];
}

// a Dense tensor's data [rows][cols] into its blocks; what no block row takes stays as it was (zero)
inline void scatter(const Placed& x, const float* src, float* blob, float* onehot) {
  for (const Block& k : x.blocks) {
    float* dst = (k.onehot ? onehot : blob) + k.at;
    const int64_t n = k.ncols ? k.ncols : x.cols;
    for (size_t i = 0; i < k.map.size(); ++i)
      if (k.map[i] >= 0)
        for (int64_t j = 0; j < n; ++j) dst[i * k.width + j] = src[(size_t)k.map[i] * x.cols + k.col0 + j];
  }
}

// the inverse: a Dense tensor's data [rows][cols] from its blocks
inline void gather(const Placed& x, const float* blob, const float* onehot, float* dst) {
  for (const Block& k : x.blocks) {
    const float* src = (k.onehot ? onehot : blob) + k.at;
    const int64_t n = k.ncols ? k.ncols : x.cols;
    for (size_t i = 0; i < k.map.size(); ++i)
      if (k.map[i] >= 0)
        for (int64_t j = 0; j < n; ++j) dst[(size_t)k.map[i] * x.cols + k.col0 + j] = src[i * k.width + j];
  }
}

}  // namespace srs
