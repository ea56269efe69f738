// model.cu - the C ABI (include/srs_ctr.h): model construction (validation + the private
// device re-layout of the reference's weights), and the predict entry points.
#include <cuda_runtime.h>

#include <cfloat>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <atomic>
#include <map>
#include <mutex>
#include <string>
#include <vector>

#include "../../include/srs_ctr.h"
#include "hostcall.h"
#include "placement.h"

namespace srs {
cudaError_t setup_embmlp_attributes();
cudaError_t setup_din_attributes();
cudaError_t setup_din_wg_attributes();
#ifdef SRS_DIN_PHASES
cudaError_t din_take_phases(unsigned long long* out);
cudaError_t din_wg_take_phases(unsigned long long* out);
#endif
cudaError_t setup_embmlp_tc_attributes();
cudaError_t setup_deepfm_tc_attributes();
// gather.cu
struct PeerGather;
cudaError_t gather_create(int device, int world, int rank, int64_t slice_rows, PeerGather** out);
cudaError_t gather_export(PeerGather* g, void* handle64);
cudaError_t gather_connect(PeerGather* g, const void* handles);
void gather_destroy(PeerGather* g);
bool gather_connected(const PeerGather* g);
int gather_begin_step(PeerGather* g, BatchView& v, bool in_kernel_signal);
cudaError_t gather_signal(PeerGather* g, cudaStream_t s);
cudaError_t gather_wait(PeerGather* g, cudaStream_t s);
float* gather_buffer(PeerGather* g, int parity);
int gather_parity(const PeerGather* g);
int64_t gather_rows(const PeerGather* g);
int gather_device(const PeerGather* g);
int64_t gather_slice_rows(const PeerGather* g);
}  // namespace srs

using namespace srs;

namespace {
thread_local std::string g_err;
}  // namespace

int srs::failf(int code, const char* fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  g_err = buf;
  return code;
}

int srs::check_device(int device) {
  int ndev = 0;
  const cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess || ndev == 0)
    return failf(SRS_ERR_CUDA, "no CUDA device available (%s); this library has no CPU path", cudaGetErrorString(e));
  if (device < 0 || device >= ndev) return failf(SRS_ERR_INVALID, "device %d out of range", device);
  return SRS_OK;
}

namespace {

constexpr auto fail = failf;        // this file's name for it

// Kernel-variant options of the model being created: "key=value;key=value" handed to
// srs_model_create_ex (keys: din_impl, embmlp_impl, deepfm_impl, zero_copy_scores).  The environment variables SRS_<KEY> remain as a tuning override of last resort.
thread_local std::string g_create_opts;
const char* opt(const char* key, const char* env_name) {
  static thread_local std::string val;
  const std::string& o = g_create_opts;
  const std::string k = std::string(key) + "=";
  size_t pos = 0;
  while (pos < o.size()) {
    size_t end = o.find(';', pos);
    if (end == std::string::npos) end = o.size();
    if (o.compare(pos, k.size(), k) == 0) {
      val = o.substr(pos + k.size(), end - pos - k.size());
      return val.c_str();
    }
    pos = end + 1;
  }
  return getenv(env_name);
}

constexpr int kSlots = 4;           // public pipelining slots; slot kSlots is private to
                                    // the synchronous srs_predict_host
constexpr int kErrWords = kSlots + 2;

// The single owner of one device (cudaMalloc) or pinned host (cudaMallocHost) buffer and its capacity in
// rows.  grow(n, first, bytes) makes room for n rows: when it holds fewer it frees, then allocates
// max(n, first) rows of bytes(rows) bytes; a failed allocation leaves it empty ({nullptr, 0}).
template <class T, bool Pinned = false>
struct Buffer {
  T* p = nullptr;
  int cap = 0;
  Buffer() = default;
  Buffer(const Buffer&) = delete;
  Buffer& operator=(const Buffer&) = delete;
  ~Buffer() { release(); }
  template <class F>
  cudaError_t grow(int n, int first, F bytes) {
    if (n <= cap) return cudaSuccess;
    release();
    const int c = std::max(n, first);
    void* q = nullptr;
    const cudaError_t e = Pinned ? cudaMallocHost(&q, bytes(c)) : cudaMalloc(&q, bytes(c));
    if (e == cudaSuccess) { p = static_cast<T*>(q); cap = c; }
    return e;
  }

 private:
  void release() {
    if (p) { if (Pinned) cudaFreeHost(p); else cudaFree(p); }
    p = nullptr; cap = 0;
  }
};
template <class T> using PinnedBuffer = Buffer<T, true>;

inline size_t word_bytes(int rows) { return (size_t)rows * 4; }     // one 4-byte word per row

struct Slot {
  cudaStream_t stream = nullptr;
  int capacity = 0;                 // rows d_block, d_probs, d_logits and d_hist32 all hold
  Buffer<uint8_t> d_block;          // one allocation: [movie|user|hist|movie_genre|user_genre|numerics]
  Buffer<float> d_probs;
  Buffer<float> d_logits;
  Buffer<int32_t> d_hist32;         // widened history ids when the batch came with hist16
  Buffer<uint8_t> d_rank;           // ranking only: [top_idx cap | top_scores cap | sort scratch]
  PinnedBuffer<int> h_err;          // pinned mirror of the device error flag
  // latency path (synchronous single calls): the last kernel of the call writes {sequence number, error
  // word} into a pinned record the caller spins on - no device-to-host copy, no stream synchronise
  PinnedBuffer<uint32_t> h_done;    // [4]
  uint32_t seq = 0;
  PinnedBuffer<int32_t> h_res;      // top positions [cap] | top scores [cap]
  Buffer<int32_t> d_req;            // srs_rank_user_host only: [user row | history | candidate ids]
  PinnedBuffer<int32_t> h_req;      //   and its pinned copy
  Buffer<int32_t> d_labels;         // srs_evaluate_host_batches only (ensure_labels)
  Buffer<MetricsReduce> d_mred;     // the metrics kernel's CTA partials and ticket for this slot's stream
  Buffer<float> d_weights;          // srs_evaluate_weighted_host_batches only (ensure_weights): the batch's weights
  Buffer<MetricsWeightedReduce> d_wred;   //   and the weighted metrics' CTA partials for this slot's stream
  Buffer<int32_t> d_neg;            // srs_dien_*_host_batches only (ensure_dien): negative ids [B][T-1],
  Buffer<float> d_aux;              //   the auxiliary head's per-row sums [B]
  Buffer<float> d_final;            //   and final_loss [B]
};

}  // namespace

struct srs_model {
  srs_spec spec{};
  int device = 0;
  int EP = 0;
  int hist_cols = 0;                // history columns the model reads (T for DIN, 1 for W&D)
  std::vector<void*> owned;
  int* err_flag = nullptr;          // kErrWords device words: [0] srs_predict_device, [1 + i] host slot i.  One word
                                    // per slot: a flag shared by every slot could be copied by slot A, set by
                                    // slot B's kernel and cleared by A's wait before B ever read it
  NcfParams ncf{};
  EmbMlpParams emb{};
  DeepFmParams fm{};
  DeepFm2Params fm2{};
  DinParams din{};
  DienParams dien{};
  DienAuxView dien_aux{};            // DIEN's auxiliary-head weights (w == nullptr: built without them)
  const char* kernel_name = "";
  int zero_copy_scores = -1;         // the zero_copy_scores option: 0 switches the latency path of srs_predict_host
                                     // off; 1 (experimental): kernels write the scores of every host batch
                                     // straight into the caller's pinned buffer; anything else: the default
  void* movie_feats = nullptr;       // srs_model_set_movie_features: [n][8 words] movie-side features in HBM
  int movie_feats_rows = 0;
  int device_sms = 132;
  int64_t bytes_per_inf = 0;
  Slot slots[kSlots + 1];
  Buffer<MetricsCounters> eval_cnt;  // srs_evaluate_host_batches (ensure_eval): counts shared by the slots
  Buffer<double> eval_loss;          //   and one loss sum per batch, added in batch order on the host
  Buffer<MetricsWeighted> eval_w;    //   and, weighted, one set of weighted sums per batch, added likewise
  Buffer<unsigned long long> eval_bhist;   // srs_dien_evaluate_host_batches (ensure_dien_eval): each batch's
  Buffer<double> eval_auc;                 //   own histogram, the prefix AUCs and (last entry) their sum
  std::mutex mu;
};

srs::ModelView srs::model_view(const srs_model* m) {
  return {m->spec.kind, m->device, &m->ncf, m->hist_cols, m->spec.n_users, m->spec.n_movies, m->movie_feats,
          m->movie_feats_rows};
}
std::mutex& srs::model_mutex(srs_model* m) { return m->mu; }

// srs_metrics_*: one allocation on the device
struct srs_metrics {
  int device = 0;
  MetricsState* d = nullptr;
  MetricsWeighted* w = nullptr;        // the weighted sums (srs_metrics_update_weighted_device)
  MetricsWeightedReduce* wred = nullptr;
  int weighted = -1;                   // -1: nothing folded since the reset, 0: unweighted rows, 1: weighted rows
};

namespace {
inline int* slot_err(srs_model* m, const Slot& s) { return m->err_flag + 1 + (&s - m->slots); }
// build_din_wg has given din the pre-split history table that din_wg_kernel gathers from (else din_kernel runs)
inline bool runs_din_wg(const srs_model* m) { return m->din.movie_split != nullptr; }
}  // namespace

namespace {

struct Builder : TensorLookup {
  srs_model* m;
  std::vector<float> blob;    // the host copy of the Dense-weight blob build_embmlp, build_deepfm or build_din
                              // uploaded, which the tensor-core builders make their operand images from

  Builder(srs_model* m, const srs_tensor* ts, int n) : TensorLookup(ts, n), m(m) {}

  // host weights, or a tensor-core operand image (write_sw128 tiles) -> a device copy the model owns
  template <class T>
  T* upload(const std::vector<T>& v) {
    if (status != SRS_OK) return nullptr;
    T* d = nullptr;
    size_t bytes = (v.size() ? v.size() : 1) * sizeof(T);
    cudaError_t e = cudaMalloc(&d, bytes);
    if (e != cudaSuccess) {
      status = fail(SRS_ERR_NOMEM, "cudaMalloc(%zu) failed: %s", bytes, cudaGetErrorString(e));
      return nullptr;
    }
    m->owned.push_back(d);
    if (!v.empty()) {
      e = cudaMemcpy(d, v.data(), v.size() * sizeof(T), cudaMemcpyHostToDevice);
      if (e != cudaSuccess) {
        status = fail(SRS_ERR_CUDA, "cudaMemcpy H2D failed: %s", cudaGetErrorString(e));
        return nullptr;
      }
    }
    return d;
  }

  // embedding table [V][E] -> device [V][EP] (zero padded rows), chunked upload
  const float* table(const char* name, int64_t V, int E) {
    const srs_tensor* t = need(name, V, E);
    if (!t) return nullptr;
    const int EP = m->EP;
    if (t->location == SRS_DEVICE_BORROWED) {
      if (E != EP) {
        status = fail(SRS_ERR_INVALID,
                      "borrowed device table '%s' needs emb_dim == padded dim (%d != %d)", name, E, EP);
        return nullptr;
      }
      return t->data;
    }
    float* d = nullptr;
    size_t bytes = (size_t)V * EP * sizeof(float);
    cudaError_t e = cudaMalloc(&d, bytes);
    if (e != cudaSuccess) {
      status = fail(SRS_ERR_NOMEM, "cudaMalloc(%zu) for '%s' failed: %s", bytes, name,
                    cudaGetErrorString(e));
      return nullptr;
    }
    m->owned.push_back(d);
    if (E == EP) {
      e = cudaMemcpy(d, t->data, bytes, cudaMemcpyHostToDevice);
    } else {
      const int64_t chunk = 1 << 16;
      std::vector<float> buf((size_t)std::min<int64_t>(chunk, V) * EP);
      e = cudaSuccess;
      for (int64_t v0 = 0; v0 < V && e == cudaSuccess; v0 += chunk) {
        const int64_t nv = std::min<int64_t>(chunk, V - v0);
        std::fill(buf.begin(), buf.end(), 0.f);
        for (int64_t v = 0; v < nv; ++v)
          memcpy(&buf[(size_t)v * EP], t->data + (size_t)(v0 + v) * E, (size_t)E * sizeof(float));
        e = cudaMemcpy(d + (size_t)v0 * EP, buf.data(), (size_t)nv * EP * sizeof(float),
                       cudaMemcpyHostToDevice);
      }
    }
    if (e != cudaSuccess) {
      status = fail(SRS_ERR_CUDA, "table upload '%s' failed: %s", name, cudaGetErrorString(e));
      return nullptr;
    }
    return d;
  }
};

// The tensors of a trainable model through its placement (placement.h): the Dense tensors scattered into the host
// blob and one-hot arrays; the tables uploaded as the model's own arrays, tables[k] the k-th in placement order
void place_host(Builder& B, const Placement& pl, const float** tables, float* blob, float* onehot) {
  int k = 0;
  for (const Placed& x : pl) {
    if (x.table_row >= 0) {
      tables[k++] = B.table(x.name.c_str(), x.rows, (int)x.cols);
    } else if (const float* src = B.host(x.name.c_str(), x.rows, x.cols)) {
      scatter(x, src, blob, onehot);
    }
  }
}

// ------------------------------------------------------------------------------------
int build_ncf(Builder& B) {
  srs_model* m = B.m;
  const srs_spec& s = m->spec;
  const bool two = s.kind == SRS_TWOTOWERS;
  if (s.n_hidden < 1 || s.n_hidden > 3) return fail(SRS_ERR_INVALID, "1..3 hidden layers supported");
  int hmax = 0;
  for (int i = 0; i < s.n_hidden; ++i) hmax = std::max(hmax, s.hidden[i]);
  if (hmax > 32 || hmax < 1) return fail(SRS_ERR_INVALID, "hidden widths must be in 1..32");
  NcfParams& p = m->ncf;
  const Placement pl = place_ncf(s, m->EP, hmax <= 16 ? 16 : 32, &p);
  std::vector<float> blob(p.blob_floats, 0.f);
  if (two && !s.final_dense) std::fill_n(blob.begin() + p.out_w, 4, 1.f);   // no dense_out: z = 1 * dot + 0
  const float* tables[2];
  place_host(B, pl, tables, blob.data(), nullptr);
  if (B.status != SRS_OK) return B.status;
  p.movie = tables[0];
  p.user = tables[1];
  p.blob = B.upload(blob);
  m->kernel_name = two ? "ncf_kernel<two_towers>" : "ncf_kernel<neural_cf_model_1>";
  return B.status;
}

int build_embmlp(Builder& B) {
  srs_model* m = B.m;
  const srs_spec& s = m->spec;
  const bool wide = s.kind == SRS_WIDENDEEP;
  if (s.n_hidden != 2 || s.hidden[0] > 128 || s.hidden[1] > 128 || s.hidden[0] < 1 || s.hidden[1] < 1)
    return fail(SRS_ERR_INVALID, "EmbeddingMLP/W&D need two hidden layers of width <= 128");
  EmbMlpParams& p = m->emb;
  const Placement pl = place_embmlp(s, m->EP, &p);
  B.blob.assign(EmbMlpBlob::of(m->EP).floats, 0.f);
  std::vector<float> wide_rows(wide ? s.cross_buckets : 0, 0.f);
  const float* tables[kWideDeepTables];
  place_host(B, pl, tables, B.blob.data(), wide_rows.data());
  if (B.status != SRS_OK) return B.status;
  point_into_blob(&p, tables, B.upload(B.blob));
  p.wide = wide ? B.upload(wide_rows) : nullptr;
  m->kernel_name = wide ? "embmlp_kernel<wide&deep>" : "embmlp_kernel";
  return B.status;
}

int build_deepfm(Builder& B) {
  srs_model* m = B.m;
  const srs_spec& s = m->spec;
  if (s.n_hidden != 2 || s.hidden[0] > 64 || s.hidden[1] > 64 || s.hidden[0] < 1 || s.hidden[1] < 1)
    return fail(SRS_ERR_INVALID, "DeepFM needs two hidden layers of width <= 64");
  DeepFmParams& p = m->fm;
  const Placement pl = place_deepfm(s, m->EP, &p);
  const DeepFmBlob ly = DeepFmBlob::of(m->EP);
  B.blob.assign(ly.floats, 0.f);
  std::vector<float> first((size_t)2 * s.n_genres + s.n_movies + s.n_users, 0.f);
  const float* tables[kDeepFmTables];
  place_host(B, pl, tables, B.blob.data(), first.data());
  if (B.status != SRS_OK) return B.status;
  p.fm_movie = tables[0]; p.fm_user = tables[1]; p.fm_mgenre = tables[2]; p.fm_ugenre = tables[3];
  p.deep_movie = tables[4]; p.deep_user = tables[5];
  point_into_blob(&p, B.upload(B.blob));
  p.first = B.upload(first);
  for (int d = 0; d < 4; ++d) p.wdot[d] = B.blob[ly.wdot + d];
  p.bout = B.blob[ly.bout];
  m->kernel_name = "deepfm_kernel";
  return B.status;
}

int build_deepfm2(Builder& B) {
  srs_model* m = B.m;
  const srs_spec& s = m->spec;
  const int EP = m->EP;
  if (s.proj_dim != 64) return fail(SRS_ERR_INVALID, "DeepFM_v2 projection width must be 64");
  if (s.n_hidden != 2 || s.hidden[0] > 32 || s.hidden[1] > 16 || s.hidden[0] < 1 || s.hidden[1] < 1)
    return fail(SRS_ERR_INVALID, "DeepFM_v2 needs hidden widths <= (32, 16)");
  DeepFm2Params& p = m->fm2;
  const Placement pl = place_deepfm2(s, EP, &p);
  std::vector<float> blob(DeepFm2Blob::of(EP).floats, 0.f), first((size_t)2 * s.n_genres + s.n_movies + s.n_users, 0.f);
  const float* tables[kDeepFm2Tables];
  place_host(B, pl, tables, blob.data(), first.data());
  if (B.status != SRS_OK) return B.status;
  point_into_blob(&p, tables, B.upload(blob));
  p.first = B.upload(first);
  m->kernel_name = "deepfm2_kernel";
  return B.status;
}

int build_din(Builder& B) {
  srs_model* m = B.m;
  const srs_spec& s = m->spec;
  const int EP = m->EP, T = s.hist_len;
  if (s.au_hidden != 32) return fail(SRS_ERR_INVALID, "DIN activation-unit width must be 32");
  if (s.n_hidden != 2 || s.hidden[0] > 128 || s.hidden[1] > 64 || s.hidden[0] < 1 || s.hidden[1] < 1)
    return fail(SRS_ERR_INVALID, "DIN needs hidden widths <= (128, 64)");
  if (T < 1) return fail(SRS_ERR_INVALID, "hist_len must be >= 1");
  DinParams& p = m->din;
  const Placement pl = place_din(s, EP, &p);
  const DinBlob ly = DinBlob::of(EP, T);
  B.blob.assign(ly.floats, 0.f);
  const float* tables[4];
  place_host(B, pl, tables, B.blob.data(), nullptr);
  if (B.status != SRS_OK) return B.status;
  // the activation-unit fold (DESIGN.md "DIN activation unit"): W_sub + W_h and W_c - W_sub
  float* w = B.blob.data();
  for (int i = 0; i < EP * 32; ++i) {
    w[ly.wh + i] += w[ly.wsub + i];
    w[ly.wc + i] -= w[ly.wsub + i];
  }
  point_into_blob(&p, tables, B.upload(B.blob), B.blob.data());
  m->kernel_name = "din_kernel";
  return B.status;
}

// ---- DIEN (DIEN.py:154-292): one blob in the layout of kernels.h::DienLayout (placement.h::place_dien); the
// auxiliary head's group of eight tensors is optional, all or none ----------------------------------------------
const char* const kDienAuxNames[8] = {"aux_pos_dense/kernel", "aux_pos_dense/bias", "aux_pos_out/kernel",
                                      "aux_pos_out/bias",     "aux_neg_dense/kernel", "aux_neg_dense/bias",
                                      "aux_neg_out/kernel",   "aux_neg_out/bias"};

int build_dien(Builder& B) {
  srs_model* m = B.m;
  const srs_spec& s = m->spec;
  const int E = s.emb_dim, EP = m->EP, T = s.hist_len;
  if (E > 32) return fail(SRS_ERR_INVALID, "DIEN supports emb_dim <= 32");
  if (s.au_hidden != 32) return fail(SRS_ERR_INVALID, "DIEN attention width must be 32");
  if (s.n_hidden != 2 || s.hidden[0] > 128 || s.hidden[1] > 64 || s.hidden[0] < 1 || s.hidden[1] < 1)
    return fail(SRS_ERR_INVALID, "DIEN needs hidden widths <= (128, 64)");
  if (T < 1) return fail(SRS_ERR_INVALID, "hist_len must be >= 1");
  bool aux = false;
  for (const char* n : kDienAuxNames) aux = aux || B.by_name.count(n);
  DienParams& p = m->dien;
  const Placement pl = place_dien(s, EP, aux, &p);
  std::vector<float> blob(DienLayout::of(EP).floats, 0.f);
  const float* tables[kDienTables];
  place_host(B, pl, tables, blob.data(), nullptr);
  if (B.status != SRS_OK) return B.status;
  const float* d = B.upload(blob);
  point_into_blob(&p, tables, d, blob.data());
  m->dien_aux.w = aux && d ? d + DienLayout::of(EP).aux : nullptr;
  m->kernel_name = "dien_kernel";
  return B.status;
}

// ---- tensor-core DIN: shared-memory image ------------------------------------------------
inline uint32_t f2u(float x) { uint32_t u; memcpy(&u, &x, 4); return u; }
inline float u2f(uint32_t u) { float x; memcpy(&x, &u, 4); return x; }
inline uint16_t bf16_rn_bits(float x) {
  const uint32_t u = f2u(x);
  return (uint16_t)((u + 0x7FFFu + ((u >> 16) & 1u)) >> 16);
}
inline uint32_t sw128_off(uint32_t row, uint32_t chunk) { return row * 128u + ((chunk ^ (row & 7u)) << 4); }

// Write logical matrix M[rows][k0 + 64*kblocks] (via getter) from column k0 on as K-major SW128 bf16
// tiles; `part` selects the hi half (x rounded to bf16) or the lo half (x - hi rounded to bf16).  With
// `chunks` < 8 only that many 16-byte chunks (8 k each) of every 128-byte row are written, from chunk
// `chunk0` on: a 32-wide K tail at bytes 0..63 or 64..127 of a K block.
template <class F>
void write_sw128(uint8_t* dst, int rows, int kblocks, bool lo_part, F get, int k0 = 0, int chunk0 = 0,
                 int chunks = 8) {
  for (int kb = 0; kb < kblocks; ++kb)
    for (int r = 0; r < rows; ++r)
      for (int c = 0; c < chunks; ++c)
        for (int i = 0; i < 8; ++i) {
          const float x = get(r, k0 + kb * 64 + c * 8 + i);
          const uint16_t hb = bf16_rn_bits(x);
          const uint16_t v = lo_part ? bf16_rn_bits(x - u2f((uint32_t)hb << 16)) : hb;
          memcpy(dst + (size_t)kb * rows * 128 + sw128_off(r, chunk0 + c) + i * 2, &v, 2);
        }
}

// The hi and lo halves of W^T (see write_sw128) for W, a [kn][ld] block of a placed host blob: image row u (of
// `units`), column k (kblocks K blocks of 64 from k0) holds W[k][u], zero for u >= ld or k >= kn.  `chunks` and
// `lo_chunk0` as write_sw128's `chunks` and the lo half's `chunk0`: a 32-wide K tail can hold both halves.
void write_wt(uint8_t* hi, uint8_t* lo, const float* w, int kn, int ld, int units, int kblocks, int k0 = 0,
              int chunks = 8, int lo_chunk0 = 0) {
  auto get = [&](int u, int k) -> float { return u < ld && k < kn ? w[(size_t)k * ld + u] : 0.f; };
  write_sw128(hi, units, kblocks, false, get, k0, 0, chunks);
  write_sw128(lo, units, kblocks, true, get, k0, lo_chunk0, chunks);
}

// Tensor-core DIN kernel (din_wg.cu): the movie table pre-split into bf16 hi / lo rows and, for EP = 32,
// the top MLP's operand images; every other tensor is the one build_din uploaded.
int build_din_wg(Builder& B) {
  srs_model* m = B.m;
  DinParams& p = m->din;
  if (m->EP == 32) {
    // W1^T over the 160 embedding columns of the tile: K blocks 0..63 and 64..127 as a hi and a lo image, then
    // one tail block whose rows are [hi k 128..159 | lo k 128..159]; W2^T as a hi and a lo image.  Offsets:
    // din_wg.cu::DinWgLayout::IMG_*
    const DinBlob ly = DinBlob::of(32, m->spec.hist_len);
    const float* w1 = B.blob.data() + ly.W1;
    const float* w2 = B.blob.data() + ly.W2;
    std::vector<uint8_t> img(114688, 0);
    write_wt(img.data() + 0, img.data() + 32768, w1, 5 * 32, 128, 128, 2);
    write_wt(img.data() + 65536, img.data() + 65536, w1, 5 * 32, 128, 128, 1, 128, 4, 4);
    write_wt(img.data() + 81920, img.data() + 98304, w2, 128, 64, 64, 2);
    p.mlp_image = B.upload(img);
    if (B.status != SRS_OK) return B.status;
  }
  void* d_split = nullptr;
  const size_t split_bytes = (size_t)m->spec.n_movies * m->EP * 4;
  cudaError_t e = cudaMalloc(&d_split, split_bytes);
  if (e != cudaSuccess) return fail(SRS_ERR_NOMEM, "cudaMalloc(%zu) failed: %s", split_bytes, cudaGetErrorString(e));
  m->owned.push_back(d_split);
  e = launch_split_table(p.movie, d_split, m->spec.n_movies, m->EP, nullptr);
  if (e != cudaSuccess) return fail(SRS_ERR_CUDA, "table split failed: %s", cudaGetErrorString(e));
  p.movie_split = static_cast<const uint8_t*>(d_split);
  m->kernel_name = "din_wg_kernel";
  return B.status;
}

// Tensor-core EmbeddingMLP / W&D (E <= 12): operand images from the blob build_embmlp placed.
int build_embmlp_tc(Builder& B) {
  srs_model* m = B.m;
  const EmbMlpBlob ly = EmbMlpBlob::of(12);
  // W1^T over K = slot * 12 + e (the ten slots; the numerics' rows stay out of the MMA), W2^T
  std::vector<uint8_t> img(131072, 0);
  write_wt(img.data() + 0, img.data() + 32768, B.blob.data() + ly.W1, 10 * 12, 128, 128, 2);
  write_wt(img.data() + 65536, img.data() + 98304, B.blob.data() + ly.W2, 128, 128, 128, 2);
  m->emb.image = B.upload(img);
  m->emb.num_sms = m->device_sms;
  m->kernel_name = m->spec.kind == SRS_WIDENDEEP ? "embmlp_tc_kernel<wide&deep>" : "embmlp_tc_kernel";
  return B.status;
}

// Tensor-core DeepFM (emb_dim 13..16): operand images from the blob build_deepfm placed.
int build_deepfm_tc(Builder& B) {
  srs_model* m = B.m;
  const DeepFmBlob ly = DeepFmBlob::of(16);
  // W1^T over K = [deep movieId emb (16) | deep userId emb (16) | 0] (the numerics' rows stay out of the MMA), W2^T;
  // units 64..127 are zero
  std::vector<uint8_t> img(65536, 0);
  write_wt(img.data() + 0, img.data() + 16384, B.blob.data() + ly.W1, 2 * 16, 64, 128, 1);
  write_wt(img.data() + 32768, img.data() + 49152, B.blob.data() + ly.W2, 64, 64, 128, 1);
  m->fm.image = B.upload(img);
  m->fm.num_sms = m->device_sms;
  m->kernel_name = "deepfm_tc_kernel";
  return B.status;
}

// Kernel variant of a model kind whose CUDA-core kernel build_* has built: the tensor-core one (its builder
// `build_tc`) when the shape `fits` it and `by_default`.  The option `key` (environment variable `env`)
// overrides: cudacore keeps the CUDA-core kernel; tc builds the tensor-core one, or fails loudly on a shape that
// does not fit.
int choose_kernel(Builder& B, const char* key, const char* env, bool fits, bool by_default, const char* fit_rule,
                  int (*build_tc)(Builder&)) {
  const char* impl = opt(key, env);
  bool tc = fits && by_default;
  if (impl && !strcmp(impl, "cudacore")) tc = false;
  if (impl && !strcmp(impl, "tc")) {
    if (!fits) return fail(SRS_ERR_INVALID, "%s=%s needs %s", env, impl, fit_rule);
    tc = true;
  }
  return tc ? build_tc(B) : SRS_OK;
}

int64_t bytes_per_inference(const srs_spec& s) {
  const int64_t E = s.emb_dim, T = s.hist_len;
  switch (s.kind) {
    case SRS_EMBEDDINGMLP: return 10 * 4 * E + 10 * 4 + 7 * 4 + 4;
    case SRS_WIDENDEEP: return 10 * 4 * E + 11 * 4 + 7 * 4 + 4 + 4;
    case SRS_NEURALCF:
    case SRS_TWOTOWERS: return 2 * 4 * E + 2 * 4 + 4;
    case SRS_DEEPFM: return 6 * 4 * E + 4 * 4 + 4 * 4 + 7 * 4 + 4;
    case SRS_DEEPFM_V2: return 4 * 4 * E + 4 * 4 + 4 * 4 + 7 * 4 + 4;
    case SRS_DIN:
    case SRS_DIEN: return (T + 1) * 4 * E + 3 * 4 * E + 28 + 4 * (T + 4) + 4;
  }
  return 0;
}

int check_batch(const srs_model* m, const srs_batch* b) {
  if (!m || !b) return fail(SRS_ERR_INVALID, "null model or batch");
  if (b->B < 0) return fail(SRS_ERR_INVALID, "negative batch size");
  if (b->B == 0) return SRS_OK;
  if (!b->movie_id || !b->user_id) return fail(SRS_ERR_INVALID, "movie_id / user_id are required");
  const int k = m->spec.kind;
  const bool dense_feats = !(k == SRS_NEURALCF || k == SRS_TWOTOWERS);
  if (dense_feats && (!b->movie_genre || !b->user_genre || !b->numerics))
    return fail(SRS_ERR_INVALID, "movie_genre / user_genre / numerics are required for this model");
  if (m->hist_cols > 0) {
    if (!b->hist && !b->hist16) return fail(SRS_ERR_INVALID, "hist is required for this model");
    if (b->hist16 && m->spec.n_movies > 65536)
      return fail(SRS_ERR_INVALID, "hist16 needs a movie vocabulary of at most 65536 ids");
    if (b->hist_stride < m->hist_cols)
      return fail(SRS_ERR_INVALID, "hist_stride %d < history columns %d", b->hist_stride, m->hist_cols);
  }
  return SRS_OK;
}

// The batches of a multi-batch call, all checked before its first launch: a call that failed on an argument
// after launching would leave that launch's error word behind for the next call.  `out[i]` (batch i's probs
// or labels, named `what`) must be non-null when the batch has rows.
template <class T>
int check_batches(const srs_model* m, int n, const srs_batch* batches, T* const* out, const char* what) {
  for (int i = 0; i < n; ++i) {
    const int rc = check_batch(m, &batches[i]);
    if (rc != SRS_OK) return rc;
    if (batches[i].B > 0 && !out[i]) return fail(SRS_ERR_INVALID, "%s of batch %d are null", what, i);
  }
  return SRS_OK;
}

// The BatchView of a caller's device batch (srs_predict_device, srs_predict_device_gather)
int device_view(const srs_model* m, const srs_batch* b, float* probs, float* logits, BatchView* v) {
  if (m->hist_cols > 0 && !b->hist)
    return fail(SRS_ERR_INVALID, "device batches carry int32 history ids (hist16 is for host batches)");
  *v = BatchView{};
  v->B = b->B; v->hist_stride = b->hist_stride;
  v->movie_id = b->movie_id; v->user_id = b->user_id; v->hist = b->hist;
  v->movie_genre = b->movie_genre; v->user_genre = b->user_genre; v->numerics = b->numerics;
  v->probs = probs; v->logits = logits; v->err_flag = m->err_flag;
  return SRS_OK;
}

int launch(srs_model* m, const BatchView& v, cudaStream_t stream) {
  cudaError_t e = cudaSuccess;
  switch (m->spec.kind) {
    case SRS_NEURALCF:
    case SRS_TWOTOWERS: e = launch_ncf(m->ncf, v, stream); break;
    case SRS_EMBEDDINGMLP:
    case SRS_WIDENDEEP:
      e = m->emb.image ? launch_embmlp_tc(m->emb, v, stream) : launch_embmlp(m->emb, v, stream);
      break;
    case SRS_DEEPFM:
      e = m->fm.image ? launch_deepfm_tc(m->fm, v, stream) : launch_deepfm(m->fm, v, stream);
      break;
    case SRS_DEEPFM_V2: e = launch_deepfm2(m->fm2, v, stream); break;
    case SRS_DIN:
      e = runs_din_wg(m) ? launch_din_wg(m->din, v, stream) : launch_din(m->din, v, stream);
      break;
    case SRS_DIEN: e = launch_dien(m->dien, v, stream); break;
    default: return fail(SRS_ERR_INVALID, "unknown model kind");
  }
  if (e != cudaSuccess) return fail(SRS_ERR_CUDA, "kernel launch failed: %s", cudaGetErrorString(e));
  return SRS_OK;
}

// Device staging of one batch is a single block in the canonical packed order
//   [movie_id B | user_id B | hist B*hc | movie_genre B*3 | user_genre B*5 | numerics B*7] x 4 bytes;
// a host batch laid out the same way (arrays back to back) goes over PCIe as ONE copy.
struct PackedLayout {
  size_t movie, user, hist, mg, ug, num, total;
};
PackedLayout packed_layout(const srs_model* m, size_t B, bool narrow_hist = false) {
  const int k = m->spec.kind;
  const bool dense_feats = !(k == SRS_NEURALCF || k == SRS_TWOTOWERS);
  PackedLayout L{};
  size_t off = 0;
  L.movie = off; off += B * 4;
  L.user = off; off += B * 4;
  L.hist = off;
  off += narrow_hist ? ((B * (size_t)m->hist_cols * 2 + 3) & ~(size_t)3) : B * (size_t)m->hist_cols * 4;
  L.mg = off; off += dense_feats ? B * 3 * 4 : 0;
  L.ug = off; off += dense_feats ? B * 5 * 4 : 0;
  L.num = off; off += dense_feats ? B * 7 * 4 : 0;
  L.total = off;
  return L;
}

int ensure_slot(srs_model* m, Slot& s, int B) {
  if (!s.stream) CUDA_TRY(cudaStreamCreateWithFlags(&s.stream, cudaStreamNonBlocking));
  if (!s.h_err.p) {
    CUDA_TRY(s.h_err.grow(1, 1, [](int) { return sizeof(int); }));
    *s.h_err.p = 0;
  }
  if (B <= s.capacity) return SRS_OK;
  const int cap = std::max(B, 1024);
  s.capacity = 0;
  CUDA_TRY(s.d_block.grow(cap, cap, [&](int c) { return packed_layout(m, (size_t)c).total + 256; }));
  CUDA_TRY(s.d_probs.grow(cap, cap, word_bytes));
  CUDA_TRY(s.d_logits.grow(cap, cap, word_bytes));
  if (m->hist_cols > 0 && m->spec.n_movies <= 65536)
    CUDA_TRY(s.d_hist32.grow(cap, cap, [&](int c) { return (size_t)c * m->hist_cols * 4; }));
  s.capacity = cap;
  return SRS_OK;
}

// The BatchView of n rows staged in the slot's block in the packed order; the scores go to the slot's buffer.
BatchView staged_view(srs_model* m, Slot& s, size_t n, const PackedLayout& L) {
  const uint8_t* d = s.d_block.p;
  BatchView v{};
  v.B = (int)n; v.hist_stride = m->hist_cols;
  v.movie_id = reinterpret_cast<const int32_t*>(d + L.movie);
  v.user_id = reinterpret_cast<const int32_t*>(d + L.user);
  v.hist = reinterpret_cast<const int32_t*>(d + L.hist);
  v.movie_genre = reinterpret_cast<const int32_t*>(d + L.mg);
  v.user_genre = reinterpret_cast<const int32_t*>(d + L.ug);
  v.numerics = reinterpret_cast<const float*>(d + L.num);
  v.probs = s.d_probs.p; v.logits = nullptr; v.err_flag = slot_err(m, s);
  return v;
}

// H2D of the batch into the slot's staging, on the slot's stream; *v is the view of the staged rows (left
// as it is for an empty batch), its scores going to s.d_probs.
int stage(srs_model* m, Slot& s, const srs_batch* b, BatchView* v) {
  int rc = check_batch(m, b);
  if (rc != SRS_OK) return rc;
  CUDA_TRY(cudaSetDevice(m->device));
  rc = ensure_slot(m, s, b->B);
  if (rc != SRS_OK) return rc;
  if (b->B == 0) return SRS_OK;
  const size_t B = (size_t)b->B;
  const int k = m->spec.kind;
  const bool dense_feats = !(k == SRS_NEURALCF || k == SRS_TWOTOWERS);
  const bool narrow = m->hist_cols > 0 && b->hist16 != nullptr;
  const PackedLayout L = packed_layout(m, B, narrow);
  uint8_t* d = s.d_block.p;
  const uint8_t* h0 = reinterpret_cast<const uint8_t*>(b->movie_id);
  bool packed = reinterpret_cast<const uint8_t*>(b->user_id) == h0 + L.user;
  if (m->hist_cols > 0)
    packed = packed && b->hist_stride == m->hist_cols &&
             (narrow ? reinterpret_cast<const uint8_t*>(b->hist16)
                     : reinterpret_cast<const uint8_t*>(b->hist)) == h0 + L.hist;
  if (dense_feats)
    packed = packed && reinterpret_cast<const uint8_t*>(b->movie_genre) == h0 + L.mg &&
             reinterpret_cast<const uint8_t*>(b->user_genre) == h0 + L.ug &&
             reinterpret_cast<const uint8_t*>(b->numerics) == h0 + L.num;
  if (packed) {
    CUDA_TRY(cudaMemcpyAsync(d, h0, L.total, cudaMemcpyHostToDevice, s.stream));
  } else {
    CUDA_TRY(cudaMemcpyAsync(d + L.movie, b->movie_id, B * 4, cudaMemcpyHostToDevice, s.stream));
    CUDA_TRY(cudaMemcpyAsync(d + L.user, b->user_id, B * 4, cudaMemcpyHostToDevice, s.stream));
    if (m->hist_cols > 0) {
      const size_t es = narrow ? 2 : 4;                       // bytes per history id on the host
      const void* hsrc = narrow ? static_cast<const void*>(b->hist16) : static_cast<const void*>(b->hist);
      if (b->hist_stride == m->hist_cols) {
        CUDA_TRY(cudaMemcpyAsync(d + L.hist, hsrc, B * m->hist_cols * es, cudaMemcpyHostToDevice, s.stream));
      } else {
        CUDA_TRY(cudaMemcpy2DAsync(d + L.hist, (size_t)m->hist_cols * es, hsrc, (size_t)b->hist_stride * es,
                                   (size_t)m->hist_cols * es, B, cudaMemcpyHostToDevice, s.stream));
      }
    }
    if (dense_feats) {
      CUDA_TRY(cudaMemcpyAsync(d + L.mg, b->movie_genre, B * 3 * 4, cudaMemcpyHostToDevice, s.stream));
      CUDA_TRY(cudaMemcpyAsync(d + L.ug, b->user_genre, B * 5 * 4, cudaMemcpyHostToDevice, s.stream));
      CUDA_TRY(cudaMemcpyAsync(d + L.num, b->numerics, B * 7 * 4, cudaMemcpyHostToDevice, s.stream));
    }
  }
  *v = staged_view(m, s, B, L);
  if (narrow) {
    CUDA_TRY(launch_widen_u16(reinterpret_cast<const uint16_t*>(d + L.hist), s.d_hist32.p,
                              (int64_t)B * m->hist_cols, s.stream));
    v->hist = s.d_hist32.p;
  }
  return SRS_OK;
}

// stage() and the forward kernel, on the slot's stream; the scores are left in s.d_probs (and s.d_logits).
// `probs_out`: where the kernel writes the scores (default: the slot's device buffer).
int stage_and_launch(srs_model* m, Slot& s, const srs_batch* b, bool want_logits,
                     float* probs_out = nullptr, float* logits_out = nullptr) {
  BatchView v;
  const int rc = stage(m, s, b, &v);
  if (rc != SRS_OK || b->B == 0) return rc;
  if (probs_out) v.probs = probs_out;
  if (want_logits) v.logits = logits_out ? logits_out : s.d_logits.p;
  return launch(m, v, s.stream);
}

// device-visible alias of a host pointer if it is pinned (page-locked) memory, else nullptr
float* pinned_alias(float* p) {
  if (!p) return nullptr;
  cudaPointerAttributes at{};
  if (cudaPointerGetAttributes(&at, p) == cudaSuccess && at.type == cudaMemoryTypeHost && at.devicePointer)
    return static_cast<float*>(at.devicePointer);
  cudaGetLastError();                                   // pageable memory: not an error
  return nullptr;
}

int enqueue_host(srs_model* m, Slot& s, const srs_batch* b, float* probs, float* logits,
                 bool copy_err = true) {
  if (!probs) return fail(SRS_ERR_INVALID, "probs is null");
  // Experimental (zero_copy_scores=1): a pinned output buffer is device-addressable under
  // unified addressing, so the kernel can write the 4 B per row over PCIe itself and the
  // device-to-host copy - one driver call and one copy-engine operation per batch - goes away.
  float* direct = m->zero_copy_scores == 1 && b && b->B > 0 ? pinned_alias(probs) : nullptr;
  int rc = stage_and_launch(m, s, b, logits != nullptr, direct);
  if (rc != SRS_OK) return rc;
  if (b->B == 0) return SRS_OK;
  const size_t B = (size_t)b->B;
  if (!direct) CUDA_TRY(cudaMemcpyAsync(probs, s.d_probs.p, B * 4, cudaMemcpyDeviceToHost, s.stream));
  if (logits) CUDA_TRY(cudaMemcpyAsync(logits, s.d_logits.p, B * 4, cudaMemcpyDeviceToHost, s.stream));
  if (copy_err)
    CUDA_TRY(cudaMemcpyAsync(s.h_err.p, slot_err(m, s), sizeof(int), cudaMemcpyDeviceToHost, s.stream));
  return SRS_OK;
}

int wait_slot(srs_model* m, Slot& s) {
  if (!s.stream) return SRS_OK;
  CUDA_TRY(cudaSetDevice(m->device));
  CUDA_TRY(cudaStreamSynchronize(s.stream));
  if (s.h_err.p && *s.h_err.p) {
    *s.h_err.p = 0;
    CUDA_TRY(cudaMemsetAsync(slot_err(m, s), 0, sizeof(int), s.stream));
    CUDA_TRY(cudaStreamSynchronize(s.stream));
    return fail(SRS_ERR_RANGE, "an id in the batch is outside its vocabulary");
  }
  return SRS_OK;
}

// The completion record of the latency path and room for k ranking results (positions | scores).
int ensure_done(Slot& s, int k) {
  if (!s.h_done.p) {
    CUDA_TRY(s.h_done.grow(1, 1, [](int) { return 4 * sizeof(uint32_t); }));
    memset(s.h_done.p, 0, 4 * sizeof(uint32_t));
  }
  CUDA_TRY(s.h_res.grow(k, std::max(k, 1024), [](int c) { return (size_t)c * 8; }));
  return SRS_OK;
}

// Spin until the call's last kernel has published sequence number `s.seq` (the stream is polled now
// and then so that a failed launch or a faulting kernel ends the wait with an error, not a hang).
int wait_done(Slot& s) {
  volatile uint32_t* d = s.h_done.p;
  uint64_t spins = 0;
  while (d[0] != s.seq) {
    if ((++spins & 0x1FFF) == 0) {
      const cudaError_t q = cudaStreamQuery(s.stream);
      if (q == cudaSuccess) {
        if (d[0] == s.seq) break;
        return fail(SRS_ERR_CUDA, "the stream drained without the completion record being written");
      }
      if (q != cudaErrorNotReady) return fail(SRS_ERR_CUDA, "kernel failed: %s", cudaGetErrorString(q));
    }
#if defined(__x86_64__) || defined(__i386__)
    __builtin_ia32_pause();
#endif
  }
  std::atomic_thread_fence(std::memory_order_acquire);
  if (d[1]) return fail(SRS_ERR_RANGE, "an id in the batch is outside its vocabulary");
  return SRS_OK;
}

// The ranking tail of srs_rank_host / srs_rank_user_host: the k best of the n scores in s.d_probs.  The ranking
// kernel writes the k positions / scores into pinned host memory and then the completion record the caller
// spins on: no device-to-host copy, no stream synchronise.
int rank_and_wait(srs_model* m, Slot& s, int n, int k, int32_t* top_idx, float* top_scores) {
  int rc = ensure_done(s, k);
  if (rc != SRS_OK) return rc;
  if (k > 0)
    CUDA_TRY(s.d_rank.grow(n, s.capacity, [](int c) { return (size_t)c * 8 + topk_scratch_bytes(c) + 256; }));
  int32_t* r_idx = s.h_res.p;
  float* r_top = reinterpret_cast<float*>(s.h_res.p + s.h_res.cap);
  void* scratch = s.d_rank.p ? s.d_rank.p + (size_t)s.d_rank.cap * 8 : nullptr;
  s.seq += 1;
  CUDA_TRY(launch_topk_done(s.d_probs.p, n, k, r_idx, r_top, scratch, slot_err(m, s), s.h_done.p, s.seq, s.stream));
  rc = wait_done(s);
  if (k > 0) {
    memcpy(top_idx, r_idx, (size_t)k * 4);
    if (top_scores) memcpy(top_scores, r_top, (size_t)k * 4);
  }
  return rc;
}

// srs_evaluate_host_batches: the slot's label staging and metrics-reduction scratch
int ensure_labels(Slot& s, int B) {
  if (!s.d_mred.p) {
    CUDA_TRY(s.d_mred.grow(1, 1, [](int) { return sizeof(MetricsReduce); }));
    CUDA_TRY(cudaMemsetAsync(s.d_mred.p, 0, sizeof(MetricsReduce), s.stream));
  }
  CUDA_TRY(s.d_labels.grow(B, 1024, word_bytes));
  return SRS_OK;
}

// srs_evaluate_host_batches: the model's shared counts and per-batch loss sums (weighted: and weighted sums) for n
// batches
int ensure_eval(srs_model* m, int n, bool weighted) {
  CUDA_TRY(m->eval_cnt.grow(1, 1, [](int) { return sizeof(MetricsCounters); }));
  CUDA_TRY(m->eval_loss.grow(n, 64, [](int c) { return (size_t)c * sizeof(double); }));
  if (weighted) CUDA_TRY(m->eval_w.grow(n, 64, [](int c) { return (size_t)c * sizeof(MetricsWeighted); }));
  return SRS_OK;
}

// srs_evaluate_weighted_host_batches: the slot's weight staging and weighted-metrics scratch
int ensure_weights(Slot& s, int B) {
  CUDA_TRY(s.d_wred.grow(1, 1, [](int) { return sizeof(MetricsWeightedReduce); }));
  CUDA_TRY(s.d_weights.grow(B, 1024, word_bytes));
  return SRS_OK;
}

// Sample weights of a weighted evaluate or metrics update: finite and >= 0 (checked before any launch)
int check_weights(const float* w, int B, int batch) {
  for (int r = 0; r < B; ++r)
    if (!(w[r] >= 0.f && w[r] <= FLT_MAX))
      return fail(SRS_ERR_INVALID, "sample weight %g (batch %d, row %d) is not finite and >= 0", (double)w[r], batch, r);
  return SRS_OK;
}

// Reads the error words [first, first + n), and clears them when one is set.
int read_error_words(int* first, int n) {
  int flags[kErrWords] = {0};
  CUDA_TRY(cudaMemcpy(flags, first, n * sizeof(int), cudaMemcpyDeviceToHost));
  for (int k = 0; k < n; ++k)
    if (flags[k]) {
      CUDA_TRY(cudaMemset(first, 0, n * sizeof(int)));
      return fail(SRS_ERR_RANGE, "an id in a batch was outside its vocabulary");
    }
  return SRS_OK;
}

// Runs step(slot, i) for the batches i = 0..n-1 round-robin over the public slots, each slot taking its next
// batch once its previous one is done.  Then every slot is synchronised, the first failure is kept, and - when
// there is none - the slots' error words are read.
template <class Step>
int run_pipelined(srs_model* m, int n, Step step) {
  int rc = SRS_OK;
  for (int i = 0; i < n && rc == SRS_OK; ++i) {
    Slot& s = m->slots[i % kSlots];
    if (i >= kSlots && s.stream) CUDA_TRY(cudaStreamSynchronize(s.stream));     // slot's previous batch is done
    rc = step(s, i);
  }
  for (int k = 0; k < kSlots; ++k)
    if (m->slots[k].stream) {
      cudaError_t e = cudaStreamSynchronize(m->slots[k].stream);
      if (e != cudaSuccess && rc == SRS_OK)
        rc = fail(SRS_ERR_CUDA, "stream synchronize failed: %s", cudaGetErrorString(e));
    }
  if (rc != SRS_OK) return rc;
  return read_error_words(m->err_flag + 1, kSlots);
}

// the model kinds whose output is a probability Keras's evaluate metrics apply to
int check_evaluable(const srs_model* m) {
  if (m->spec.kind == SRS_DIEN)
    return fail(SRS_ERR_INVALID, "evaluate does not cover DIEN: its Keras evaluate reports the loss with the "
                                 "auxiliary negative-sample term and its AUC metrics, not these four numbers; "
                                 "use srs_dien_evaluate_host_batches");
  if (m->spec.kind == SRS_TWOTOWERS && !m->spec.final_dense)
    return fail(SRS_ERR_INVALID, "evaluate needs a probability: two towers without the final Dense output a raw dot");
  return SRS_OK;
}

// srs_dien_*: a DIEN model built with the auxiliary-head group
int check_dien_aux(const srs_model* m) {
  if (m->spec.kind != SRS_DIEN)
    return fail(SRS_ERR_INVALID, "the auxiliary-loss output belongs to DIEN (DIEN.py:261-296); this model is not DIEN");
  if (!m->dien_aux.w)
    return fail(SRS_ERR_INVALID, "this DIEN model was built without the auxiliary-head weights "
                                 "(aux_pos_dense/kernel ... aux_neg_out/bias)");
  return SRS_OK;
}

// The negatives and labels of a srs_dien_*_host_batches call, all checked before its first launch; labels must be
// 0 or 1 (Keras's evaluate asserts the same).
int check_dien_batches(const srs_model* m, int n, const srs_batch* batches, const int32_t* const* neg_hist,
                       const int32_t* const* labels) {
  for (int i = 0; i < n; ++i) {
    const int B = batches[i].B;
    if (B == 0) continue;
    if (!labels[i]) return fail(SRS_ERR_INVALID, "labels of batch %d are null", i);
    if (m->hist_cols > 1 && !neg_hist[i]) return fail(SRS_ERR_INVALID, "neg_hist of batch %d is null", i);
    for (int r = 0; r < B; ++r)
      if (labels[i][r] != 0 && labels[i][r] != 1)
        return fail(SRS_ERR_INVALID, "a label is not 0 or 1 (batch %d, row %d)", i, r);
  }
  return SRS_OK;
}

// srs_dien_*_host_batches: the slot's staging of negatives and labels and its aux / final_loss outputs
int ensure_dien(const srs_model* m, Slot& s, int B) {
  const size_t cols = (size_t)std::max(m->hist_cols - 1, 1);
  CUDA_TRY(s.d_neg.grow(B, 1024, [&](int c) { return (size_t)c * cols * 4; }));
  CUDA_TRY(s.d_aux.grow(B, 1024, word_bytes));
  CUDA_TRY(s.d_final.grow(B, 1024, word_bytes));
  return ensure_labels(s, B);
}

// srs_dien_evaluate_host_batches: K batch histograms, K prefix AUCs and their sum
int ensure_dien_eval(srs_model* m, int K) {
  CUDA_TRY(m->eval_bhist.grow(K, 64, [](int c) { return (size_t)c * 2 * kMetBins * sizeof(unsigned long long); }));
  CUDA_TRY(m->eval_auc.grow(K + 1, 65, [](int c) { return (size_t)c * sizeof(double); }));
  return SRS_OK;
}

// One Keras batch of a srs_dien_*_host_batches call on slot s: the batch, its negatives and its labels go in; the
// AUX kernel leaves probs / logits / aux in the slot and the final-loss kernel final_loss in s.d_final (and its
// sum in *loss_sum when that is not null).
int dien_stage_and_launch(srs_model* m, Slot& s, const srs_batch* b, const int32_t* neg, const int32_t* labels,
                          double* loss_sum) {
  BatchView v;
  int rc = stage(m, s, b, &v);
  if (rc == SRS_OK) rc = ensure_dien(m, s, b->B);
  if (rc != SRS_OK) return rc;
  const size_t B = (size_t)b->B;
  const int cols = m->hist_cols - 1;
  if (cols > 0) CUDA_TRY(cudaMemcpyAsync(s.d_neg.p, neg, B * cols * 4, cudaMemcpyHostToDevice, s.stream));
  CUDA_TRY(cudaMemcpyAsync(s.d_labels.p, labels, B * 4, cudaMemcpyHostToDevice, s.stream));
  v.logits = s.d_logits.p;
  DienAuxView a = m->dien_aux;
  a.neg = s.d_neg.p; a.neg_stride = cols; a.aux = s.d_aux.p;
  CUDA_TRY(launch_dien_aux(m->dien, a, v, s.stream));
  CUDA_TRY(launch_dien_final_loss(s.d_logits.p, s.d_labels.p, s.d_aux.p, (int)B, s.d_final.p, loss_sum, s.stream));
  return SRS_OK;
}

}  // namespace

// ---- what recforyou.cu's CTR page runs of a model (hostcall.h) ------------------------
size_t srs::model_batch_bytes(const srs_model* m, size_t B) { return packed_layout(m, B).total; }

BatchView srs::model_batch_view(const srs_model* m, uint8_t* block, size_t B, float* probs, int* err_flag) {
  const PackedLayout L = packed_layout(m, B);
  BatchView v{};
  v.B = (int)B; v.hist_stride = m->hist_cols;
  v.movie_id = reinterpret_cast<const int32_t*>(block + L.movie);
  v.user_id = reinterpret_cast<const int32_t*>(block + L.user);
  v.hist = reinterpret_cast<const int32_t*>(block + L.hist);
  v.movie_genre = reinterpret_cast<const int32_t*>(block + L.mg);
  v.user_genre = reinterpret_cast<const int32_t*>(block + L.ug);
  v.numerics = reinterpret_cast<const float*>(block + L.num);
  v.probs = probs; v.logits = nullptr; v.err_flag = err_flag;
  return v;
}

int srs::model_launch(srs_model* m, const BatchView& v, cudaStream_t s) { return launch(m, v, s); }

// ======================================================================================
extern "C" {

int srs_abi_version(void) { return SRS_ABI_VERSION; }

const char* srs_last_error(void) { return g_err.c_str(); }

int srs_model_create(const srs_spec* spec, const srs_tensor* tensors, int32_t n_tensors,
                     int32_t device, srs_model** out) {
  if (!spec || !out || (n_tensors > 0 && !tensors)) return fail(SRS_ERR_INVALID, "null argument");
  *out = nullptr;
  if (spec->kind < SRS_EMBEDDINGMLP || spec->kind > SRS_DIEN)
    return fail(SRS_ERR_INVALID, "unknown model kind %d", spec->kind);
  if (spec->emb_dim < 1 || spec->emb_dim > 64) return fail(SRS_ERR_INVALID, "emb_dim must be in 1..64");
  if (spec->n_movies < 1 || spec->n_users < 1 || spec->n_genres < 1)
    return fail(SRS_ERR_INVALID, "vocabulary sizes must be positive");
  if (spec->n_hidden < 0 || spec->n_hidden > 4) return fail(SRS_ERR_INVALID, "n_hidden must be in 0..4");
  int rc = check_device(device);
  if (rc != SRS_OK) return rc;
  CUDA_TRY(cudaSetDevice(device));
  CUDA_TRY(setup_embmlp_attributes());
  CUDA_TRY(setup_deepfm_attributes());
  CUDA_TRY(setup_din_attributes());
  CUDA_TRY(setup_dien_attributes());
  CUDA_TRY(setup_din_wg_attributes());
  CUDA_TRY(setup_embmlp_tc_attributes());
  CUDA_TRY(setup_deepfm_tc_attributes());

  srs_model* m = new srs_model();
  m->spec = *spec;
  m->device = device;
  if (const char* zc = opt("zero_copy_scores", "SRS_ZERO_COPY_SCORES")) m->zero_copy_scores = atoi(zc);
  int sms = 0;
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device);
  m->device_sms = sms > 0 ? sms : 132;
  m->EP = round_ep(spec->emb_dim);
  m->hist_cols = (spec->kind == SRS_DIN || spec->kind == SRS_DIEN) ? spec->hist_len
                 : spec->kind == SRS_WIDENDEEP ? 1 : 0;
  m->bytes_per_inf = bytes_per_inference(*spec);
  Builder B(m, tensors, n_tensors);
  switch (spec->kind) {
    case SRS_NEURALCF:
    case SRS_TWOTOWERS: rc = build_ncf(B); break;
    case SRS_EMBEDDINGMLP:
    case SRS_WIDENDEEP:
      // tensor cores for the reference shape (E <= 12)
      rc = build_embmlp(B);
      if (rc == SRS_OK)
        rc = choose_kernel(B, "embmlp_impl", "SRS_EMBMLP_IMPL", m->EP == 12, true, "emb_dim <= 12", build_embmlp_tc);
      break;
    case SRS_DEEPFM:
      // tensor-core deep MLP when emb_dim pads to 16
      rc = build_deepfm(B);
      if (rc == SRS_OK)
        rc = choose_kernel(B, "deepfm_impl", "SRS_DEEPFM_IMPL", m->EP == 16, true, "12 < emb_dim <= 16",
                           build_deepfm_tc);
      break;
    case SRS_DEEPFM_V2: rc = build_deepfm2(B); break;
    case SRS_DIEN: rc = build_dien(B); break;
    default:
      // the activation unit on warpgroup MMAs (din_wg.cu) for E padded to 32 or 64; the default for T > 8,
      // where it measured faster on the H100 (DESIGN.md section 6): BASELINE cfg 5 (E padded to 64) and
      // cfg 3 (E = 32, where the top MLP runs on wgmma too).  cudacore stays the only kernel for E <= 16.
      rc = build_din(B);
      if (rc == SRS_OK)
        rc = choose_kernel(B, "din_impl", "SRS_DIN_IMPL", m->EP == 32 || m->EP == 64, spec->hist_len > 8,
                           "16 < emb_dim <= 64", build_din_wg);
      break;
  }
  cudaError_t e = cudaSuccess;
  if (rc == SRS_OK) {
    e = cudaMalloc(&m->err_flag, kErrWords * sizeof(int));
    if (e == cudaSuccess) e = cudaMemset(m->err_flag, 0, kErrWords * sizeof(int));
    if (e != cudaSuccess) rc = fail(SRS_ERR_CUDA, "error-flag allocation failed: %s", cudaGetErrorString(e));
  }
  if (rc == SRS_OK) {
    e = cudaDeviceSynchronize();
    if (e != cudaSuccess) rc = fail(SRS_ERR_CUDA, "weight upload failed: %s", cudaGetErrorString(e));
  }
  if (rc != SRS_OK) {
    std::string keep = g_err;
    srs_model_destroy(m);
    g_err = keep;
    return rc;
  }
  *out = m;
  return SRS_OK;
}

int srs_model_create_ex(const srs_spec* spec, const srs_tensor* tensors, int32_t n_tensors, int32_t device,
                        const char* options, srs_model** out) {
  g_create_opts = options ? options : "";
  const int rc = srs_model_create(spec, tensors, n_tensors, device, out);
  g_create_opts.clear();
  return rc;
}

void srs_model_destroy(srs_model* m) {
  if (!m) return;
  cudaSetDevice(m->device);
  for (Slot& s : m->slots)
    if (s.stream) { cudaStreamSynchronize(s.stream); cudaStreamDestroy(s.stream); }
  for (void* p : m->owned) cudaFree(p);
  if (m->err_flag) cudaFree(m->err_flag);
  cudaFree(m->movie_feats);
  delete m;                                             // the slot and evaluate buffers free themselves
}

int srs_predict_device(srs_model* m, const srs_batch* b, float* probs, float* logits, void* stream) {
  int rc = check_batch(m, b);
  if (rc != SRS_OK) return rc;
  if (!probs) return fail(SRS_ERR_INVALID, "probs is null");
  if (b->B == 0) return SRS_OK;
  BatchView v;
  rc = device_view(m, b, probs, logits, &v);
  if (rc != SRS_OK) return rc;
  CUDA_TRY(cudaSetDevice(m->device));
  return launch(m, v, static_cast<cudaStream_t>(stream));
}

// ---- score exchange over peer memory (gather.cu) -------------------------------------------------
int srs_gather_create(int32_t device, int32_t world, int32_t rank, int64_t slice_rows, srs_gather** out) {
  if (!out) return fail(SRS_ERR_INVALID, "null argument");
  PeerGather* g = nullptr;
  cudaError_t e = gather_create(device, world, rank, slice_rows, &g);
  if (e == cudaErrorInvalidValue) return fail(SRS_ERR_INVALID, "need 1 <= world <= 8, 0 <= rank < world, slice_rows >= 1");
  if (e != cudaSuccess) return fail(SRS_ERR_CUDA, "gather buffer allocation failed: %s", cudaGetErrorString(e));
  *out = reinterpret_cast<srs_gather*>(g);
  return SRS_OK;
}

int srs_gather_export(srs_gather* g, void* handle64) {
  if (!g || !handle64) return fail(SRS_ERR_INVALID, "null argument");
  CUDA_TRY(gather_export(reinterpret_cast<PeerGather*>(g), handle64));
  return SRS_OK;
}

int srs_gather_connect(srs_gather* g, const void* handles) {
  if (!g || !handles) return fail(SRS_ERR_INVALID, "null argument");
  CUDA_TRY(gather_connect(reinterpret_cast<PeerGather*>(g), handles));
  return SRS_OK;
}

void srs_gather_destroy(srs_gather* g) { gather_destroy(reinterpret_cast<PeerGather*>(g)); }

int srs_predict_device_gather(srs_model* m, const srs_batch* b, srs_gather* gg, void* stream) {
  int rc = check_batch(m, b);
  if (rc != SRS_OK) return rc;
  PeerGather* g = reinterpret_cast<PeerGather*>(gg);
  if (!g) return fail(SRS_ERR_INVALID, "null gather object");
  if (!gather_connected(g)) return fail(SRS_ERR_INVALID, "srs_gather_connect has not been called");
  if (gather_device(g) != m->device) return fail(SRS_ERR_INVALID, "gather object lives on another device");
  if (b->B < 1 || b->B > gather_slice_rows(g)) return fail(SRS_ERR_INVALID, "batch rows must be in 1..slice_rows");
  BatchView v;
  rc = device_view(m, b, nullptr, nullptr, &v);          // gather_begin_step points the scores at the exchange
  if (rc != SRS_OK) return rc;
  CUDA_TRY(cudaSetDevice(m->device));
  const bool in_kernel = m->spec.kind == SRS_DIN && runs_din_wg(m);   // kernels ending in gather_signal_tail()
  gather_begin_step(g, v, in_kernel);
  rc = launch(m, v, static_cast<cudaStream_t>(stream));
  if (rc != SRS_OK) return rc;
  if (!in_kernel) CUDA_TRY(gather_signal(g, static_cast<cudaStream_t>(stream)));
  return SRS_OK;
}

int srs_gather_wait(srs_gather* g, void* stream) {
  if (!g) return fail(SRS_ERR_INVALID, "null gather object");
  CUDA_TRY(cudaSetDevice(gather_device(reinterpret_cast<PeerGather*>(g))));
  CUDA_TRY(gather_wait(reinterpret_cast<PeerGather*>(g), static_cast<cudaStream_t>(stream)));
  return SRS_OK;
}

int srs_gather_scores(srs_gather* gg, float** scores, int64_t* rows) {
  PeerGather* g = reinterpret_cast<PeerGather*>(gg);
  if (!g || !scores) return fail(SRS_ERR_INVALID, "null argument");
  *scores = gather_buffer(g, gather_parity(g));
  if (rows) *rows = gather_rows(g);
  return SRS_OK;
}

int srs_gather_copy_scores(srs_gather* gg, float* dst, int32_t dst_on_host, void* stream) {
  PeerGather* g = reinterpret_cast<PeerGather*>(gg);
  if (!g || !dst) return fail(SRS_ERR_INVALID, "null argument");
  CUDA_TRY(cudaSetDevice(gather_device(g)));
  CUDA_TRY(cudaMemcpyAsync(dst, gather_buffer(g, gather_parity(g)), (size_t)gather_rows(g) * 4,
                           dst_on_host ? cudaMemcpyDeviceToHost : cudaMemcpyDeviceToDevice,
                           static_cast<cudaStream_t>(stream)));
  return SRS_OK;
}

int srs_predict_host(srs_model* m, const srs_batch* b, float* probs, float* logits) {
  if (!m) return fail(SRS_ERR_INVALID, "null model");
  std::lock_guard<std::mutex> lock(m->mu);
  Slot& s = m->slots[kSlots];
  // Latency path: when the caller's output buffers are pinned, the kernel writes the scores (4 B per row)
  // straight into them over PCIe and a one-warp kernel publishes the completion record: two copy-engine
  // operations, two driver calls and the stream synchronise of the general path go away.
  if (probs && b && b->B > 0 && m->zero_copy_scores != 0) {
    float* dp = pinned_alias(probs);
    float* dl = logits ? pinned_alias(logits) : nullptr;
    if (dp && (!logits || dl)) {
      int rc = ensure_slot(m, s, b->B);
      if (rc == SRS_OK) rc = ensure_done(s, 0);
      if (rc != SRS_OK) return rc;
      rc = stage_and_launch(m, s, b, logits != nullptr, dp, dl);
      if (rc != SRS_OK) return rc;
      s.seq += 1;
      CUDA_TRY(launch_finish(slot_err(m, s), s.h_done.p, s.seq, s.stream));
      return wait_done(s);
    }
  }
  int rc = enqueue_host(m, s, b, probs, logits);
  if (rc != SRS_OK) return rc;
  return wait_slot(m, s);
}

int srs_predict_host_batches(srs_model* m, int32_t n, const srs_batch* batches,
                             float* const* probs, float* const* logits) {
  if (!m) return fail(SRS_ERR_INVALID, "null model");
  if (n < 0 || (n > 0 && (!batches || !probs))) return fail(SRS_ERR_INVALID, "null argument");
  int rc = check_batches(m, n, batches, probs, "probs");
  if (rc != SRS_OK) return rc;
  std::lock_guard<std::mutex> lock(m->mu);
  CUDA_TRY(cudaSetDevice(m->device));
  return run_pipelined(m, n, [&](Slot& s, int i) -> int {
    if (batches[i].B == 0) return SRS_OK;                // nothing to stage, and its probs may be null
    return enqueue_host(m, s, &batches[i], probs[i], logits ? logits[i] : nullptr, false);
  });
}

int srs_num_slots(void) { return kSlots; }

int srs_predict_host_async(srs_model* m, int32_t slot, const srs_batch* b, float* probs,
                           float* logits) {
  if (!m) return fail(SRS_ERR_INVALID, "null model");
  if (slot < 0 || slot >= kSlots) return fail(SRS_ERR_INVALID, "slot %d out of range", slot);
  return enqueue_host(m, m->slots[slot], b, probs, logits);
}

int srs_wait_slot(srs_model* m, int32_t slot) {
  if (!m) return fail(SRS_ERR_INVALID, "null model");
  if (slot < 0 || slot >= kSlots) return fail(SRS_ERR_INVALID, "slot %d out of range", slot);
  return wait_slot(m, m->slots[slot]);
}

int srs_model_status(srs_model* m) {
  if (!m) return fail(SRS_ERR_INVALID, "null model");
  CUDA_TRY(cudaSetDevice(m->device));
  CUDA_TRY(cudaDeviceSynchronize());
  return read_error_words(m->err_flag, kErrWords);
}

int64_t srs_model_bytes_per_inference(const srs_model* m) { return m ? m->bytes_per_inf : 0; }

const char* srs_model_kernel_name(const srs_model* m) { return m ? m->kernel_name : ""; }

int srs_model_set_sm_limit(srs_model* m, int32_t n_sms) {
  if (!m) return fail(SRS_ERR_INVALID, "null model");
  const int n = (n_sms <= 0 || n_sms > m->device_sms) ? m->device_sms : n_sms;
  std::lock_guard<std::mutex> lock(m->mu);
  m->emb.num_sms = n;
  m->fm.num_sms = n;
  m->din.max_ctas = n < m->device_sms ? n : 0;
  return SRS_OK;
}

int64_t srs_launch_count(void) { return g_launch_count; }

int srs_fill_uniform(float* device_ptr, int64_t n, uint64_t seed, float lo, float hi,
                     int32_t device, void* stream) {
  if (!device_ptr && n > 0) return fail(SRS_ERR_INVALID, "null pointer");
  CUDA_TRY(cudaSetDevice(device));
  CUDA_TRY(launch_fill_uniform(device_ptr, n, seed, lo, hi, static_cast<cudaStream_t>(stream)));
  return SRS_OK;
}

int srs_cosine_scores_device(const float* query, const float* cands, int32_t n, int32_t dim,
                             float* scores, int32_t device, void* stream) {
  if ((!query || !cands || !scores) && n > 0) return fail(SRS_ERR_INVALID, "null pointer");
  if (dim < 1) return fail(SRS_ERR_INVALID, "dim must be positive");
  CUDA_TRY(cudaSetDevice(device));
  CUDA_TRY(launch_cosine(query, cands, n, dim, scores, static_cast<cudaStream_t>(stream)));
  return SRS_OK;
}

int srs_topk_device(const float* scores, int32_t n, int32_t k, int32_t* top_idx,
                    float* top_scores, int32_t device, void* stream) {
  if (n < 0 || k < 0) return fail(SRS_ERR_INVALID, "negative n or k");
  if (n == 0 || k == 0) return SRS_OK;
  if (!scores || !top_idx) return fail(SRS_ERR_INVALID, "null pointer");
  if (n > (1 << 30)) return fail(SRS_ERR_INVALID, "at most 2^30 scores");
  CUDA_TRY(cudaSetDevice(device));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  void* scratch = nullptr;
  const size_t need = topk_scratch_bytes(n);
  if (need) CUDA_TRY(cudaMallocAsync(&scratch, need, s));
  cudaError_t e = launch_topk(scores, n, k, top_idx, top_scores, scratch, s);
  if (scratch) cudaFreeAsync(scratch, s);
  CUDA_TRY(e);
  return SRS_OK;
}

int srs_rank_host(srs_model* m, const srs_batch* b, int32_t k, int32_t* top_idx,
                  float* top_scores) {
  if (!m) return fail(SRS_ERR_INVALID, "null model");
  if (k < 0) return fail(SRS_ERR_INVALID, "negative k");
  if (b && std::min(k, b->B) > 0 && !top_idx) return fail(SRS_ERR_INVALID, "top_idx is null");
  std::lock_guard<std::mutex> lock(m->mu);
  Slot& s = m->slots[kSlots];
  const int rc = stage_and_launch(m, s, b, false);
  if (rc != SRS_OK) return rc;
  const int n = b->B;
  if (n == 0) return SRS_OK;
  return rank_and_wait(m, s, n, std::min(k, n), top_idx, top_scores);
}

int srs_model_set_movie_features(srs_model* m, int32_t n_movies, const int32_t* genres, const float* numerics) {
  if (!m) return fail(SRS_ERR_INVALID, "null model");
  if (n_movies < 1 || !genres || !numerics) return fail(SRS_ERR_INVALID, "null or empty movie feature table");
  std::lock_guard<std::mutex> lock(m->mu);
  CUDA_TRY(cudaSetDevice(m->device));
  std::vector<int32_t> packed((size_t)n_movies * 8, 0);
  for (int i = 0; i < n_movies; ++i) {
    for (int g = 0; g < 3; ++g) {
      const int32_t v = genres[(size_t)i * 3 + g];
      if (v >= m->spec.n_genres) return fail(SRS_ERR_RANGE, "movie %d: genre index %d outside the vocabulary", i, v);
      packed[(size_t)i * 8 + g] = v < 0 ? -1 : v;
    }
    memcpy(&packed[(size_t)i * 8 + 3], numerics + (size_t)i * 4, 16);
  }
  cudaFree(m->movie_feats);
  m->movie_feats = nullptr; m->movie_feats_rows = 0;
  CUDA_TRY(cudaMalloc(&m->movie_feats, packed.size() * 4));
  CUDA_TRY(cudaMemcpy(m->movie_feats, packed.data(), packed.size() * 4, cudaMemcpyHostToDevice));
  m->movie_feats_rows = n_movies;
  return SRS_OK;
}

int srs_rank_user_host(srs_model* m, const srs_user_row* user, const int32_t* cand, int32_t n, int32_t k,
                       int32_t* top_idx, float* top_scores, float* probs) {
  if (!m) return fail(SRS_ERR_INVALID, "null model");
  if (!user || (n > 0 && !cand) || n < 0 || k < 0) return fail(SRS_ERR_INVALID, "bad argument");
  const int kind = m->spec.kind;
  const bool dense_feats = !(kind == SRS_NEURALCF || kind == SRS_TWOTOWERS);
  if (dense_feats && !m->movie_feats)
    return fail(SRS_ERR_INVALID, "this model reads movie features: call srs_model_set_movie_features first");
  const int hc = m->hist_cols;
  if (user->n_hist < 0 || user->n_hist > hc || (user->n_hist > 0 && !user->hist))
    return fail(SRS_ERR_INVALID, "n_hist must be in 0..%d", hc);
  if (std::min(k, n) > 0 && !top_idx) return fail(SRS_ERR_INVALID, "top_idx is null");
  std::lock_guard<std::mutex> lock(m->mu);
  Slot& s = m->slots[kSlots];
  CUDA_TRY(cudaSetDevice(m->device));
  int rc = ensure_slot(m, s, n);
  if (rc != SRS_OK) return rc;
  if (n == 0) return SRS_OK;
  auto req_bytes = [&](int c) { return (16 + (size_t)hc + (size_t)c) * 4; };
  CUDA_TRY(s.d_req.grow(n, s.capacity, req_bytes));
  CUDA_TRY(s.h_req.grow(n, s.capacity, req_bytes));
  // request block: [userId | userGenre1..5 | 3 user numerics | hist[hc] | candidate ids[n]]
  int32_t* h = s.h_req.p;
  h[0] = user->user_id;
  for (int g = 0; g < 5; ++g) h[1 + g] = user->user_genre[g] < 0 ? -1 : user->user_genre[g];
  memcpy(h + 6, user->user_numerics, 12);
  for (int t = 0; t < hc; ++t) h[9 + t] = t < user->n_hist ? user->hist[t] : 0;     // 0 = the padding id
  memcpy(h + 9 + hc, cand, (size_t)n * 4);
  // one small copy: (9 + T + n) words instead of n full feature rows.  (Letting the assemble kernel read the
  // pinned block over PCIe itself was measured slower: every row re-reads the user part from host memory.)
  CUDA_TRY(cudaMemcpyAsync(s.d_req.p, h, (9 + (size_t)hc + (size_t)n) * 4, cudaMemcpyHostToDevice, s.stream));
  const PackedLayout L = packed_layout(m, (size_t)n);
  uint8_t* d = s.d_block.p;
  CUDA_TRY(launch_assemble_request(s.d_req.p, 1, s.d_req.p + 9 + hc, n, m->movie_feats, m->movie_feats_rows, hc,
                                   dense_feats ? 1 : 0, reinterpret_cast<int32_t*>(d + L.movie),
                                   reinterpret_cast<int32_t*>(d + L.user), reinterpret_cast<int32_t*>(d + L.hist),
                                   reinterpret_cast<int32_t*>(d + L.mg),
                                   reinterpret_cast<int32_t*>(d + L.ug), reinterpret_cast<float*>(d + L.num),
                                   slot_err(m, s), s.stream));
  rc = launch(m, staged_view(m, s, (size_t)n, L), s.stream);
  if (rc != SRS_OK) return rc;
  if (probs) CUDA_TRY(cudaMemcpyAsync(probs, s.d_probs.p, (size_t)n * 4, cudaMemcpyDeviceToHost, s.stream));
  return rank_and_wait(m, s, n, std::min(k, n), top_idx, top_scores);
}

// ---- evaluate: Keras's loss / accuracy / ROC AUC / PR AUC (metrics.cu) ----------------------------------
int srs_metrics_create(int32_t device, srs_metrics** out) {
  if (!out) return fail(SRS_ERR_INVALID, "null argument");
  *out = nullptr;
  const int rc = check_device(device);
  if (rc != SRS_OK) return rc;
  CUDA_TRY(cudaSetDevice(device));
  srs_metrics* mt = new srs_metrics();
  mt->device = device;
  cudaError_t e = cudaMalloc(&mt->d, sizeof(MetricsState));
  if (e == cudaSuccess) e = cudaMalloc(&mt->w, sizeof(MetricsWeighted));
  if (e == cudaSuccess) e = cudaMalloc(&mt->wred, sizeof(MetricsWeightedReduce));
  if (e == cudaSuccess) e = cudaMemset(mt->d, 0, sizeof(MetricsState));
  if (e == cudaSuccess) e = cudaMemset(mt->w, 0, sizeof(MetricsWeighted));
  if (e == cudaSuccess) e = cudaDeviceSynchronize();
  if (e != cudaSuccess) {
    cudaFree(mt->d);
    cudaFree(mt->w);
    cudaFree(mt->wred);
    delete mt;
    return fail(SRS_ERR_CUDA, "metrics state allocation failed: %s", cudaGetErrorString(e));
  }
  *out = mt;
  return SRS_OK;
}

void srs_metrics_destroy(srs_metrics* mt) {
  if (!mt) return;
  cudaSetDevice(mt->device);
  cudaFree(mt->d);
  cudaFree(mt->w);
  cudaFree(mt->wred);
  delete mt;
}

int srs_metrics_reset(srs_metrics* mt, void* stream) {
  if (!mt) return fail(SRS_ERR_INVALID, "null metrics state");
  CUDA_TRY(cudaSetDevice(mt->device));
  CUDA_TRY(cudaMemsetAsync(mt->d, 0, sizeof(MetricsState), static_cast<cudaStream_t>(stream)));
  CUDA_TRY(cudaMemsetAsync(mt->w, 0, sizeof(MetricsWeighted), static_cast<cudaStream_t>(stream)));
  mt->weighted = -1;
  return SRS_OK;
}

int srs_metrics_update_device(srs_metrics* mt, const float* probs, const float* logits, const int32_t* labels,
                              int32_t n, void* stream) {
  return srs_metrics_update_weighted_device(mt, probs, logits, labels, nullptr, n, stream);
}

int srs_metrics_update_weighted_device(srs_metrics* mt, const float* probs, const float* logits,
                                       const int32_t* labels, const float* weights, int32_t n, void* stream) {
  if (!mt) return fail(SRS_ERR_INVALID, "null metrics state");
  if (n < 1) return fail(SRS_ERR_INVALID, "n must be at least 1");
  if (!probs || !logits || !labels) return fail(SRS_ERR_INVALID, "probs, logits and labels are required");
  const int weighted = weights != nullptr;
  if (mt->weighted >= 0 && mt->weighted != weighted)
    return fail(SRS_ERR_INVALID, "a metrics state folds either weighted or unweighted rows between resets");
  CUDA_TRY(cudaSetDevice(mt->device));
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (weighted)
    CUDA_TRY(launch_metrics_update_weighted(probs, logits, labels, weights, n, &mt->d->cnt, &mt->d->red,
                                            &mt->d->loss, mt->w, mt->wred, 1, s));
  else
    CUDA_TRY(launch_metrics_update(probs, logits, labels, n, &mt->d->cnt, &mt->d->red, &mt->d->loss, 1, s));
  mt->weighted = weighted;
  return SRS_OK;
}

int srs_metrics_result(srs_metrics* mt, srs_eval_result* out, int64_t* confusion) {
  if (!mt || !out) return fail(SRS_ERR_INVALID, "null argument");
  CUDA_TRY(cudaSetDevice(mt->device));
  CUDA_TRY(cudaDeviceSynchronize());
  MetricsCounters c;
  double loss = 0.0;
  CUDA_TRY(cudaMemcpy(&c, &mt->d->cnt, sizeof(c), cudaMemcpyDeviceToHost));
  CUDA_TRY(cudaMemcpy(&loss, &mt->d->loss, sizeof(loss), cudaMemcpyDeviceToHost));
  if (c.err & kMetErrLabel) return fail(SRS_ERR_INVALID, "a label is not 0 or 1");
  if (c.err & kMetErrProb) return fail(SRS_ERR_INVALID, "a probability is NaN or outside [0, 1]");
  srs_eval_result r{};
  metrics_summarise(c.hist, c.correct, loss, &r, confusion);
  if (mt->weighted == 1) {                              // confusion stays the integer counts
    MetricsWeighted w;
    CUDA_TRY(cudaMemcpy(&w, mt->w, sizeof(w), cudaMemcpyDeviceToHost));
    metrics_summarise_weighted(c.hist, c.correct, w, loss, &r);
  }
  if (r.rows == 0) return fail(SRS_ERR_INVALID, "no rows have been folded into the metrics");
  *out = r;
  return SRS_OK;
}

int srs_evaluate_host_batches(srs_model* m, int32_t n, const srs_batch* batches, const int32_t* const* labels,
                              srs_eval_result* out) {
  return srs_evaluate_weighted_host_batches(m, n, batches, labels, nullptr, out);
}

int srs_evaluate_weighted_host_batches(srs_model* m, int32_t n, const srs_batch* batches,
                                       const int32_t* const* labels, const float* const* weights,
                                       srs_eval_result* out) {
  if (!m) return fail(SRS_ERR_INVALID, "null model");
  if (n < 0 || (n > 0 && (!batches || !labels)) || !out) return fail(SRS_ERR_INVALID, "null argument");
  int rc = check_evaluable(m);
  if (rc != SRS_OK) return rc;
  rc = check_batches(m, n, batches, labels, "labels");
  if (rc != SRS_OK) return rc;
  for (int i = 0; weights && i < n; ++i) {
    if (batches[i].B > 0 && !weights[i]) return fail(SRS_ERR_INVALID, "weights of batch %d are null", i);
    rc = check_weights(weights[i], batches[i].B, i);
    if (rc != SRS_OK) return rc;
  }
  int64_t rows = 0;
  for (int i = 0; i < n; ++i) rows += batches[i].B;
  if (rows == 0) return fail(SRS_ERR_INVALID, "evaluate needs at least one row");
  std::lock_guard<std::mutex> lock(m->mu);
  CUDA_TRY(cudaSetDevice(m->device));
  rc = ensure_eval(m, n, weights != nullptr);
  if (rc != SRS_OK) return rc;
  {
    Slot& s0 = m->slots[0];
    rc = ensure_slot(m, s0, 0);
    if (rc != SRS_OK) return rc;
    CUDA_TRY(cudaMemsetAsync(m->eval_cnt.p, 0, sizeof(MetricsCounters), s0.stream));
    CUDA_TRY(cudaStreamSynchronize(s0.stream));               // before any slot folds into the counts
  }
  rc = run_pipelined(m, n, [&](Slot& s, int i) -> int {
    const srs_batch* b = &batches[i];
    if (b->B == 0) return SRS_OK;
    int r = stage_and_launch(m, s, b, true);
    if (r == SRS_OK) r = ensure_labels(s, b->B);
    if (r != SRS_OK) return r;
    CUDA_TRY(cudaMemcpyAsync(s.d_labels.p, labels[i], (size_t)b->B * sizeof(int32_t), cudaMemcpyHostToDevice,
                             s.stream));
    // the batch's loss sum (and weighted sums) go to its own entry: the batch order, not the slot completion order,
    // fixes the sums
    if (!weights) {
      CUDA_TRY(launch_metrics_update(s.d_probs.p, s.d_logits.p, s.d_labels.p, b->B, m->eval_cnt.p, s.d_mred.p,
                                     m->eval_loss.p + i, 0, s.stream));
      return SRS_OK;
    }
    r = ensure_weights(s, b->B);
    if (r != SRS_OK) return r;
    CUDA_TRY(cudaMemcpyAsync(s.d_weights.p, weights[i], (size_t)b->B * sizeof(float), cudaMemcpyHostToDevice,
                             s.stream));
    CUDA_TRY(launch_metrics_update_weighted(s.d_probs.p, s.d_logits.p, s.d_labels.p, s.d_weights.p, b->B,
                                            m->eval_cnt.p, s.d_mred.p, m->eval_loss.p + i, m->eval_w.p + i,
                                            s.d_wred.p, 0, s.stream));
    return SRS_OK;
  });
  if (rc != SRS_OK) return rc;
  MetricsCounters c;
  std::vector<double> batch_loss((size_t)n);
  std::vector<MetricsWeighted> batch_w(weights ? (size_t)n : 0);
  CUDA_TRY(cudaMemcpy(&c, m->eval_cnt.p, sizeof(c), cudaMemcpyDeviceToHost));
  CUDA_TRY(cudaMemcpy(batch_loss.data(), m->eval_loss.p, (size_t)n * sizeof(double), cudaMemcpyDeviceToHost));
  if (weights)
    CUDA_TRY(cudaMemcpy(batch_w.data(), m->eval_w.p, (size_t)n * sizeof(MetricsWeighted), cudaMemcpyDeviceToHost));
  if (c.err & kMetErrLabel) return fail(SRS_ERR_INVALID, "a label is not 0 or 1");
  if (c.err & kMetErrProb) return fail(SRS_ERR_INVALID, "a probability is NaN or outside [0, 1]");
  double loss = 0.0;
  MetricsWeighted w{};
  for (int i = 0; i < n; ++i) {
    if (batches[i].B == 0) continue;
    loss += batch_loss[(size_t)i];
    if (!weights) continue;
    const double* src = reinterpret_cast<const double*>(&batch_w[(size_t)i]);
    double* dst = reinterpret_cast<double*>(&w);
    for (int q = 0; q < kMetWSums; ++q) dst[q] += src[q];
  }
  if (weights)
    metrics_summarise_weighted(c.hist, c.correct, w, loss, out);
  else
    metrics_summarise(c.hist, c.correct, loss, out, nullptr);
  return SRS_OK;
}

// ---- DIEN's second output and its Keras evaluate (DIEN.py:261-304) ---------------------------------------
int srs_dien_outputs_device(srs_model* m, const srs_batch* b, const int32_t* neg_hist, int32_t neg_stride,
                            const int32_t* labels, float* probs, float* logits, float* aux, float* final_loss,
                            void* stream) {
  int rc = check_batch(m, b);
  if (rc == SRS_OK) rc = check_dien_aux(m);
  if (rc != SRS_OK) return rc;
  if (b->B == 0) return SRS_OK;
  if (!labels || !probs || !logits || !aux || !final_loss)
    return fail(SRS_ERR_INVALID, "labels, probs, logits, aux and final_loss are required");
  const int cols = m->hist_cols - 1;
  if (cols > 0 && (!neg_hist || neg_stride < cols))
    return fail(SRS_ERR_INVALID, "neg_hist [B][neg_stride >= %d] is required", cols);
  BatchView v;
  rc = device_view(m, b, probs, logits, &v);
  if (rc != SRS_OK) return rc;
  CUDA_TRY(cudaSetDevice(m->device));
  DienAuxView a = m->dien_aux;
  a.neg = neg_hist; a.neg_stride = neg_stride; a.aux = aux;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  CUDA_TRY(launch_dien_aux(m->dien, a, v, st));
  CUDA_TRY(launch_dien_final_loss(logits, labels, aux, b->B, final_loss, nullptr, st));
  return SRS_OK;
}

int srs_dien_outputs_host_batches(srs_model* m, int32_t n, const srs_batch* batches, const int32_t* const* neg_hist,
                                  const int32_t* const* labels, float* const* probs, float* const* final_loss) {
  if (!m) return fail(SRS_ERR_INVALID, "null model");
  if (n < 0 || (n > 0 && (!batches || !labels || !probs || !final_loss || (m->hist_cols > 1 && !neg_hist))))
    return fail(SRS_ERR_INVALID, "null argument");
  int rc = check_dien_aux(m);
  if (rc == SRS_OK) rc = check_batches(m, n, batches, probs, "probs");
  if (rc == SRS_OK) rc = check_batches(m, n, batches, final_loss, "final_loss");
  if (rc == SRS_OK) rc = check_dien_batches(m, n, batches, neg_hist, labels);
  if (rc != SRS_OK) return rc;
  std::lock_guard<std::mutex> lock(m->mu);
  CUDA_TRY(cudaSetDevice(m->device));
  return run_pipelined(m, n, [&](Slot& s, int i) -> int {
    const srs_batch* b = &batches[i];
    if (b->B == 0) return SRS_OK;
    const int r = dien_stage_and_launch(m, s, b, neg_hist ? neg_hist[i] : nullptr, labels[i], nullptr);
    if (r != SRS_OK) return r;
    CUDA_TRY(cudaMemcpyAsync(probs[i], s.d_probs.p, (size_t)b->B * 4, cudaMemcpyDeviceToHost, s.stream));
    CUDA_TRY(cudaMemcpyAsync(final_loss[i], s.d_final.p, (size_t)b->B * 4, cudaMemcpyDeviceToHost, s.stream));
    return SRS_OK;
  });
}

int srs_dien_evaluate_host_batches(srs_model* m, int32_t n, const srs_batch* batches, const int32_t* const* neg_hist,
                                   const int32_t* const* labels, srs_dien_eval_result* out) {
  if (!m) return fail(SRS_ERR_INVALID, "null model");
  if (n < 0 || (n > 0 && (!batches || !labels || (m->hist_cols > 1 && !neg_hist))) || !out)
    return fail(SRS_ERR_INVALID, "null argument");
  int rc = check_dien_aux(m);
  if (rc == SRS_OK) rc = check_batches(m, n, batches, labels, "labels");
  if (rc == SRS_OK) rc = check_dien_batches(m, n, batches, neg_hist, labels);
  if (rc != SRS_OK) return rc;
  int64_t rows = 0;
  std::vector<int> nth((size_t)n, -1);                  // position of batch i among the batches with rows
  int K = 0;
  for (int i = 0; i < n; ++i) {
    rows += batches[i].B;
    if (batches[i].B > 0) nth[(size_t)i] = K++;
  }
  if (rows == 0) return fail(SRS_ERR_INVALID, "evaluate needs at least one row");
  std::lock_guard<std::mutex> lock(m->mu);
  CUDA_TRY(cudaSetDevice(m->device));
  rc = ensure_eval(m, n, false);
  if (rc == SRS_OK) rc = ensure_dien_eval(m, K);
  if (rc != SRS_OK) return rc;
  Slot& s0 = m->slots[0];
  rc = ensure_slot(m, s0, 0);
  if (rc != SRS_OK) return rc;
  CUDA_TRY(cudaMemsetAsync(m->eval_cnt.p, 0, sizeof(MetricsCounters), s0.stream));
  CUDA_TRY(cudaMemsetAsync(m->eval_bhist.p, 0, (size_t)K * 2 * kMetBins * sizeof(unsigned long long), s0.stream));
  CUDA_TRY(cudaStreamSynchronize(s0.stream));               // before any slot folds into the counts
  rc = run_pipelined(m, n, [&](Slot& s, int i) -> int {
    const srs_batch* b = &batches[i];
    if (b->B == 0) return SRS_OK;
    // each batch's final_loss sum and histogram go to its own entry: batch order, not slot completion, fixes them
    const int r = dien_stage_and_launch(m, s, b, neg_hist ? neg_hist[i] : nullptr, labels[i], m->eval_loss.p + i);
    if (r != SRS_OK) return r;
    CUDA_TRY(launch_metrics_update(s.d_probs.p, s.d_logits.p, s.d_labels.p, b->B, m->eval_cnt.p, s.d_mred.p, nullptr,
                                   0, s.stream, m->eval_bhist.p + (size_t)nth[(size_t)i] * 2 * kMetBins));
    return SRS_OK;
  });
  if (rc != SRS_OK) return rc;
  CUDA_TRY(launch_auc_value(m->eval_bhist.p, K, m->eval_auc.p, m->eval_auc.p + K, s0.stream));
  CUDA_TRY(cudaStreamSynchronize(s0.stream));
  MetricsCounters c;
  std::vector<double> batch_loss((size_t)n);
  double auc_sum = 0.0;
  CUDA_TRY(cudaMemcpy(&c, m->eval_cnt.p, sizeof(c), cudaMemcpyDeviceToHost));
  CUDA_TRY(cudaMemcpy(batch_loss.data(), m->eval_loss.p, (size_t)n * sizeof(double), cudaMemcpyDeviceToHost));
  CUDA_TRY(cudaMemcpy(&auc_sum, m->eval_auc.p + K, sizeof(double), cudaMemcpyDeviceToHost));
  if (c.err & kMetErrLabel) return fail(SRS_ERR_INVALID, "a label is not 0 or 1");
  if (c.err & kMetErrProb) return fail(SRS_ERR_INVALID, "a probability is NaN or outside [0, 1]");
  double loss = 0.0;
  for (int i = 0; i < n; ++i)
    if (batches[i].B > 0) loss += batch_loss[(size_t)i];
  srs_eval_result r{};
  metrics_summarise(c.hist, c.correct, loss, &r, nullptr);
  out->rows = rows;
  out->batches = K;
  out->loss = r.loss;
  out->auc = r.roc_auc;
  out->auc_value = auc_sum / (double)K;
  return SRS_OK;
}

int srs_selftest_wgmma(const float* A, const float* B, float* D, int32_t N, int32_t k_blocks,
                       int32_t a_in_regs, int32_t device) {
  if (!A || !B || !D) return fail(SRS_ERR_INVALID, "null pointer");
  CUDA_TRY(cudaSetDevice(device));
  CUDA_TRY(launch_wgmma_selftest(A, B, D, N, k_blocks, a_in_regs, nullptr));
  CUDA_TRY(cudaDeviceSynchronize());
  return SRS_OK;
}

#ifdef SRS_DIN_PHASES
// Phase-timing builds only (tools/din_phases.py): the cycles the DIN kernel of this model spent in each
// srs::DinPhase since the previous call, summed over timing units; the counters are cleared.
int srs_debug_din_phases(const srs_model* m, uint64_t* out, int32_t n) {
  if (!m || !out || n < kDinPhases) return fail(SRS_ERR_INVALID, "need %d counters", (int)kDinPhases);
  CUDA_TRY(cudaSetDevice(m->device));
  CUDA_TRY(cudaDeviceSynchronize());
  unsigned long long c[kDinPhases];
  CUDA_TRY(runs_din_wg(m) ? din_wg_take_phases(c) : din_take_phases(c));
  for (int i = 0; i < kDinPhases; ++i) out[i] = c[i];
  return SRS_OK;
}
#endif

}  // extern "C"
