// dien_train.cu - the forward / backward step of DIEN's `model.fit` (DIEN.py:296-304: compile(optimizer="adam"),
// fit over batches of 12 in file order); the trainer that drives it (dedupe, Adam, metrics) is srs_trainer in
// trainer.cu.  DESIGN.md section 4.20.
//
// dien_train_step_kernel<EP>: one 32-row tile per CTA, 256 threads, one warp per row and lane e on element e of
// every state vector, as dien_kernel.  The objective is the sum over the batch of final_loss_i = bce_i - 0.5 *
// mean_j(aux_j) (tape.gradient of a non-scalar target), so dL/dz_i = sigmoid(z_i) - y_i and every pos_t / neg_t of
// every row gets -0.5.
//   forward   dien_layers.cuh's GRU, attention, AUGRU and auxiliary head, the sequence of each row in one warp;
//             the states h_{t-1}, u_{t-1} of every position go to the row's records.  Then the top MLP on the tile,
//             keeping the pre-activations PReLU's gradient needs.  probs / logits / aux have the bits of
//             dien_kernel<EP, true> on the same rows.
//   top       dz -> delta2, delta1 (PReLU: up * ([x > 0] + alpha [x < 0]), dalpha = up * min(x, 0)) -> the tile
//             input's gradient (augru state, candidate, the three side rows)
//   sequence  per row, t = T-1 .. 0: the position's forward is recomputed from its stored states, then AUGRU,
//             attention, GRU (a masked position passes dh through and adds nothing) and, for t >= 1, the
//             auxiliary head are differentiated.  Each Dense product's input and output delta go to the record of
//             (row, t); the embedding gradients to the entry list.
//   partials  thread q sums Dense parameter q's gradient over the CTA's rows (and positions) in order.  augru_h0
//             gets none: it is not a variable in the reference (a fresh draw inside `call`), so Adam leaves it as
//             it was.
// Entries of row r (table_grad_kernel dedupes them in entry order): s * B + r with s = 0 userGenre1, 1 userId, 2
// movieGenre1 (a missing genre: none), 3 the candidate, 4 + t history position t (the GRU's input gradient plus,
// t >= 1, the auxiliary head's), 4 + T + t - 1 the negative of position t >= 1.  No float atomics.
#include "dien_layers.cuh"

namespace srs {

namespace {

// 32-float slots of one (row, position) record, indexed by lane
enum DienRec {
  RX, RHP, RHT, RPC, RUP, RUZ, RPR, RPZ, RPH, RXN, RAA, RSP, RSN,                        // inputs
  RDXZ, RDXR, RDXH, RDRH, RDPR, RDPZ, RDPH, RDAR, RDAZ, RDAH, RDAT, RDAP, RDAN,          // output deltas
  RSC,                       // scalars: [0] att_out's pre-activation delta, [1] aux_pos_out's, [2] aux_neg_out's
  kDienRecSlots
};

constexpr int kLDH1 = 128 + 4, kLDH2 = 64 + 4;

template <int EP>
constexpr int step_smem_floats() {
  constexpr int LDX = 5 * EP + kNumPad + 4;
  return kDienRows * (LDX + 4 * kLDH1 + 4 * kLDH2 + 1) + DienBlob<EP>::TOTAL + DienAuxBlob<EP>::TOTAL;
}
static_assert(step_smem_floats<32>() * 4 <= 227 * 1024, "the EP = 32 step tile must fit in shared memory");

// sum_e w[le * ld + e] * d_e over e < EP (d held by lane e): row le of a matrix against a delta; 0 on lanes >= EP
template <int EP>
__device__ __forceinline__ float row_dot_lanes(const float* w, int ld, int le, float d, bool on) {
  float s = 0.f;
#pragma unroll
  for (int e = 0; e < EP; ++e) s = fmaf(w[le * ld + e], __shfl_sync(0xffffffffu, d, e), s);
  return on ? s : 0.f;
}

// the same over the 32 units of a Dense32 layer
template <int EP>
__device__ __forceinline__ float row_dot32(const float* w, int le, float d, bool on) {
  float s = 0.f;
#pragma unroll
  for (int j = 0; j < 32; ++j) s = fmaf(w[le * 32 + j], __shfl_sync(0xffffffffu, d, j), s);
  return on ? s : 0.f;
}

template <int EP>
__global__ void __launch_bounds__(kThreads) dien_train_step_kernel(DienStepArgs a) {
  static_assert(EP <= 32, "one lane per state element");
  using L = DienBlob<EP>;
  using A = DienAuxBlob<EP>;
  constexpr int R = kDienRows;
  constexpr int KP = 5 * EP + kNumPad;
  constexpr int LDX = KP + 4;
  constexpr int OFF_UG = 0, OFF_U = EP, OFF_ST = 2 * EP, OFF_C = 3 * EP, OFF_MG = 4 * EP, OFF_NUM = 5 * EP;
  constexpr int NS = kDienRecSlots * 32;
  extern __shared__ __align__(16) float smem[];
  float* Xs = smem;                        // [R][LDX] the tile input; later its gradient
  float* P1 = Xs + R * LDX;                // [R][kLDH1] pre-activations, PReLU outputs, upstream, deltas
  float* H1 = P1 + R * kLDH1;
  float* U1 = H1 + R * kLDH1;
  float* D1 = U1 + R * kLDH1;
  float* P2 = D1 + R * kLDH1;              // [R][kLDH2]
  float* H2 = P2 + R * kLDH2;
  float* U2 = H2 + R * kLDH2;
  float* D2 = U2 + R * kLDH2;
  float* dzs = D2 + R * kLDH2;             // [R]
  float* Sq = dzs + R;                     // the sequence weights
  float* Sa = Sq + L::TOTAL;               // the auxiliary head's weights
  const DienParams& p = a.p;
  const DienLayout ly = DienLayout::of(EP);
  const int T = p.T, B = a.B;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int row0 = blockIdx.x * R;
  const int nv = min(R, B - row0);

  stage_weights(Sq, p.seq, L::TOTAL);
  stage_weights(Sa, a.blob + ly.aux, A::TOTAL);
  // ---- side features through the order: userGenre1, userId, movieGenre1 rows, numerics -------------------------
  constexpr int Q = EP / 4;
  for (int i = tid; i < R * 3 * Q; i += kThreads) {
    const int q = i % Q, slot = (i / Q) % 3, r = i / Q / 3;
    int id = -1;
    const float* table = p.user;
    if (r < nv) {
      const int row = __ldg(a.order + row0 + r);
      if (slot == 1) {
        id = __ldg(a.user + row);
      } else {
        id = slot == 0 ? __ldg(a.ugenre + row) : __ldg(a.mgenre + row);
        if (id < 0) id = -1;
        table = slot == 0 ? p.ugenre : p.mgenre;
      }
    }
    gather_row<EP>(Xs + r * LDX + (slot == 0 ? OFF_UG : slot == 1 ? OFF_U : OFF_MG), table, id, q);
  }
  for (int i = tid; i < R * kNumPad; i += kThreads) {
    const int r = i / kNumPad, j = i % kNumPad;
    float v = 0.f;
    if (j < kNumNumerics && r < nv) v = __ldg(a.numerics + (size_t)__ldg(a.order + row0 + r) * kNumNumerics + j);
    Xs[r * LDX + OFF_NUM + j] = v;
  }
  stage_wait();
  __syncthreads();

  // ---- sequence forward: dien_kernel<EP, true>'s row loop, the states of every position kept -----------------------
  const int le = lane < EP ? lane : EP - 1;
  const bool on = lane < EP;
  const float att_b = Sq[L::AB + lane], att_wo = Sq[L::AO + lane], att_bo = Sq[L::ABO];
  for (int r = warp; r < R; r += kThreads / 32) {
    float* xrow = Xs + r * LDX;
    if (r >= nv) {
      if (lane < EP) { xrow[OFF_C + lane] = 0.f; xrow[OFF_ST + lane] = 0.f; }
      continue;
    }
    const int row = __ldg(a.order + row0 + r);
    const int cid = dien_id(__ldg(a.movie + row));
    const float c = lane < EP ? __ldg(p.movie + (size_t)cid * EP + lane) : 0.f;
    const int32_t* hrow = a.hist + (size_t)row * T;
    const int32_t* nrow = a.neg + (size_t)row * (T - 1);
    float h = 0.f, u = Sq[L::H0 + le], aux_row = 0.f;
    for (int t = 0; t < T; ++t) {
      float* rec = a.rec + ((size_t)(row0 + r) * T + t) * NS;
      rec[RHP * 32 + lane] = h;
      rec[RUP * 32 + lane] = u;
      const int hid = dien_id(__ldg(hrow + t));
      const bool valid = hid != 0;
      const float x = lane < EP ? __ldg(p.movie + (size_t)hid * EP + lane) : 0.f;
      float g_prev = 0.f, xn = 0.f;
      if (t > 0) {
        g_prev = h;
        const int nid = dien_id(__ldg(nrow + t - 1));
        xn = lane < EP ? __ldg(p.movie + (size_t)nid * EP + lane) : 0.f;
      }
      float gz, gr, ghh, grh;
      const float hn = dien_gru_step<EP>(Sq, le, x, h, &gz, &gr, &ghh, &grh);
      if (valid) h = hn;
      float sp, sn, pos, neg;
      if (t > 0) aux_row += dien_aux_step<EP>(Sa, g_prev, x, xn, lane, &sp, &sn, &pos, &neg);
      float at;
      const float s = dien_attention<EP>(Sq, lane, h * c, att_b, att_wo, att_bo, &at);
      DienAugruStep st;
      u = dien_augru_step<EP>(Sq, le, h, u, s, &st);
    }
    if (lane < EP) { xrow[OFF_C + lane] = c; xrow[OFF_ST + lane] = u; }
    if (lane == 0) a.aux[row0 + r] = aux_row;
  }
  __syncthreads();

  // ---- top MLP forward, pre-activations kept (PReLU applied as dense_layer applies it) ------------------------
  dense_layer<R, 128, 2, 8>(Xs, LDX, KP, p.W1, p.b1, ACT_NONE, nullptr, P1, kLDH1);
  __syncthreads();
  for (int i = tid; i < R * 128; i += kThreads) {
    const int r = i >> 7, j = i & 127;
    const float v = P1[r * kLDH1 + j];
    H1[r * kLDH1 + j] = v > 0.f ? v : __ldg(p.a1 + j) * v;
  }
  __syncthreads();
  dense_layer<R, 64, 1, 8>(H1, kLDH1, 128, p.W2, p.b2, ACT_NONE, nullptr, P2, kLDH2);
  __syncthreads();
  for (int i = tid; i < R * 64; i += kThreads) {
    const int r = i >> 6, j = i & 63;
    const float v = P2[r * kLDH2 + j];
    H2[r * kLDH2 + j] = v > 0.f ? v : __ldg(p.a2 + j) * v;
  }
  __syncthreads();
  const float b3 = __ldg(a.blob + ly.b3);
  row_dot<R>(H2, kLDH2, 64, p.w3, [&](int r, float s) {
    if (r >= nv) { dzs[r] = 0.f; return; }
    const int row = __ldg(a.order + row0 + r);
    const float z = s + b3;
    const float pr = sigmoidf_acc(z);
    const int y = __ldg(a.label + row);
    a.probs[row0 + r] = pr;
    a.logits[row0 + r] = z;
    a.labels[row0 + r] = y;
    dzs[r] = pr - (float)y;
  });
  __syncthreads();

  // ---- top MLP backward -------------------------------------------------------------------------------------
  for (int i = tid; i < R * 64; i += kThreads) {
    const int r = i >> 6, j = i & 63;
    const float up = dzs[r] * __ldg(p.w3 + j), x = P2[r * kLDH2 + j];
    U2[r * kLDH2 + j] = up;
    D2[r * kLDH2 + j] = x > 0.f ? up : x < 0.f ? up * __ldg(p.a2 + j) : 0.f;
  }
  __syncthreads();
  for (int i = tid; i < R * 128; i += kThreads) {
    const int r = i >> 7, k = i & 127;
    float up = 0.f;
    for (int j = 0; j < 64; ++j) up = fmaf(__ldg(p.W2 + k * 64 + j), D2[r * kLDH2 + j], up);
    const float x = P1[r * kLDH1 + k];
    U1[r * kLDH1 + k] = up;
    D1[r * kLDH1 + k] = x > 0.f ? up : x < 0.f ? up * __ldg(p.a1 + k) : 0.f;
  }
  __syncthreads();
  // the top MLP's Dense gradients of this CTA's rows, in row order
  for (int q = ly.W1 + tid; q < ly.floats; q += kThreads) {
    const float* in = nullptr;               // null: the constant 1 (a bias)
    const float* dl = nullptr;               // null: no gradient (padding)
    const float* pre = nullptr;              // a PReLU alpha: sum of up * min(pre, 0)
    int ldi = 0, ldd = 0;
    if (q < ly.b1) {
      in = Xs + (q - ly.W1) / 128; ldi = LDX; dl = D1 + (q - ly.W1) % 128; ldd = kLDH1;
    } else if (q < ly.a1) {
      dl = D1 + (q - ly.b1); ldd = kLDH1;
    } else if (q < ly.W2) {
      dl = U1 + (q - ly.a1); pre = P1 + (q - ly.a1); ldd = kLDH1;
    } else if (q < ly.b2) {
      in = H1 + (q - ly.W2) / 64; ldi = kLDH1; dl = D2 + (q - ly.W2) % 64; ldd = kLDH2;
    } else if (q < ly.a2) {
      dl = D2 + (q - ly.b2); ldd = kLDH2;
    } else if (q < ly.w3) {
      dl = U2 + (q - ly.a2); pre = P2 + (q - ly.a2); ldd = kLDH2;
    } else if (q < ly.b3) {
      in = H2 + (q - ly.w3); ldi = kLDH2; dl = dzs; ldd = 1;
    } else if (q == ly.b3) {
      dl = dzs; ldd = 1;
    }
    float s = 0.f;
    if (pre) {
      for (int r = 0; r < nv; ++r) s = fmaf(dl[r * ldd], fminf(pre[r * ldd], 0.f), s);
    } else if (dl && in) {
      for (int r = 0; r < nv; ++r) s = fmaf(in[r * ldi], dl[r * ldd], s);
    } else if (dl) {
      for (int r = 0; r < nv; ++r) s += dl[r * ldd];
    }
    a.part[(size_t)blockIdx.x * ly.floats + q] = s;
  }
  __syncthreads();
  // the tile input's gradient: dX[r][k] = W1[k] . delta1[r], over the 5 EP embedding columns (into Xs)
  for (int i = tid; i < R * 5 * EP; i += kThreads) {
    const int r = i / (5 * EP), k = i % (5 * EP);
    float s = 0.f;
    for (int j = 0; j < 128; ++j) s = fmaf(__ldg(p.W1 + k * 128 + j), D1[r * kLDH1 + j], s);
    Xs[r * LDX + k] = s;
  }
  __syncthreads();

  // ---- the three side rows' entries ---------------------------------------------------------------------------
  for (int i = tid; i < nv * 3 * EP; i += kThreads) {
    const int r = i / (3 * EP), s = (i / EP) % 3, k = i % EP;
    const int row = __ldg(a.order + row0 + r);
    const int id = s == 0 ? __ldg(a.ugenre + row) : s == 1 ? __ldg(a.user + row) : __ldg(a.mgenre + row);
    const int tab = s == 0 ? 2 : s == 1 ? 1 : 3;
    const size_t e = (size_t)s * B + row0 + r;
    if (k == 0) a.trow[e] = id < 0 ? -1 : (int32_t)(a.tab_row0[tab] + id);
    a.gemb[e * EP + k] = Xs[r * LDX + (s == 0 ? OFF_UG : s == 1 ? OFF_U : OFF_MG) + k];
  }

  // ---- sequence backward, one warp per row ----------------------------------------------------------------------
  for (int r = warp; r < nv; r += kThreads / 32) {
    const int row = __ldg(a.order + row0 + r);
    const int cid = dien_id(__ldg(a.movie + row));
    const float c = on ? __ldg(p.movie + (size_t)cid * EP + lane) : 0.f;
    const int32_t* hrow = a.hist + (size_t)row * T;
    const int32_t* nrow = a.neg + (size_t)row * (T - 1);
    float du = on ? Xs[r * LDX + OFF_ST + lane] : 0.f;     // dL/du_t
    float dc = on ? Xs[r * LDX + OFF_C + lane] : 0.f;      // dL/dc
    float dh = 0.f;                                        // dL/dg_t from later positions
    for (int t = T - 1; t >= 0; --t) {
      float* rec = a.rec + ((size_t)(row0 + r) * T + t) * NS;
      const float hp = rec[RHP * 32 + lane], up = rec[RUP * 32 + lane];
      // the position's forward again
      const int hid = dien_id(__ldg(hrow + t));
      const bool valid = hid != 0;
      const float x = on ? __ldg(p.movie + (size_t)hid * EP + lane) : 0.f;
      int nid = 0;
      float xn = 0.f;
      if (t > 0) {
        nid = dien_id(__ldg(nrow + t - 1));
        xn = on ? __ldg(p.movie + (size_t)nid * EP + lane) : 0.f;
      }
      float gz, gr, ghh, grh;
      const float hn = dien_gru_step<EP>(Sq, le, x, hp, &gz, &gr, &ghh, &grh);
      const float ht = valid ? hn : hp;
      float sp = 0.f, sn = 0.f, pos = 0.f, neg = 0.f;
      if (t > 0) dien_aux_step<EP>(Sa, hp, x, xn, lane, &sp, &sn, &pos, &neg);
      float at;
      const float pc = ht * c;
      const float s = dien_attention<EP>(Sq, lane, pc, att_b, att_wo, att_bo, &at);
      DienAugruStep st;
      dien_augru_step<EP>(Sq, le, ht, up, s, &st);
      // AUGRU: u_t = (1 - ra) u + ra hn, ra = s r
      const float d_ra = du * (st.hn - up);
      const float d_hn = du * st.ra;
      float du_p = du * (1.f - st.ra);
      const float d_s = warp_sum(d_ra * st.rg);
      const float d_rg = d_ra * s;
      const float d_ah = d_hn * (1.f - st.hn * st.hn);
      const float d_ph = row_dot_lanes<EP>(Sq + L::SW + 2 * EP * EP, EP, le, d_ah, on);
      const float d_uz = row_dot_lanes<EP>(Sq + L::HW + 2 * EP * EP, EP, le, d_ph, on);
      du_p += d_uz * st.zg;
      const float d_zg = d_uz * up;
      const float d_ar = d_rg * st.rg * (1.f - st.rg);
      const float d_az = d_zg * st.zg * (1.f - st.zg);
      const float d_pr = row_dot_lanes<EP>(Sq + L::SW, EP, le, d_ar, on);
      const float d_pz = row_dot_lanes<EP>(Sq + L::SW + EP * EP, EP, le, d_az, on);
      du_p += row_dot_lanes<EP>(Sq + L::HW, EP, le, d_pr, on);
      du_p += row_dot_lanes<EP>(Sq + L::HW + EP * EP, EP, le, d_pz, on);
      float d_ht = row_dot_lanes<EP>(Sq + L::IW, EP, le, d_pr, on);
      d_ht += row_dot_lanes<EP>(Sq + L::IW + EP * EP, EP, le, d_pz, on);
      d_ht += row_dot_lanes<EP>(Sq + L::IW + 2 * EP * EP, EP, le, d_ph, on);
      // attention: s = sigmoid(a . wo + bo), a = sigmoid(pc . AW + ab)
      const float d_sz = d_s * s * (1.f - s);
      const float d_at = d_sz * att_wo * at * (1.f - at);
      const float d_pc = row_dot32<EP>(Sq + L::AW, le, d_at, on);
      d_ht += d_pc * c;
      dc += d_pc * ht;
      // GRU: a masked position carries the state, so its gradient passes through
      dh += d_ht;
      float dxz = 0.f, dxr = 0.f, dxh = 0.f, drh = 0.f, dx = 0.f, dh_p = dh;
      if (valid) {
        const float d_z = dh * (hp - ghh);
        const float d_hh = dh * (1.f - gz);
        dxh = d_hh * (1.f - ghh * ghh);
        drh = dxh * gr;
        const float d_r = dxh * grh;
        dxz = d_z * gz * (1.f - gz);
        dxr = d_r * gr * (1.f - gr);
        dh_p = dh * gz;
        dx = row_dot_lanes<EP>(Sq + L::GW, 3 * EP, le, dxz, on);
        dx += row_dot_lanes<EP>(Sq + L::GW + EP, 3 * EP, le, dxr, on);
        dx += row_dot_lanes<EP>(Sq + L::GW + 2 * EP, 3 * EP, le, dxh, on);
        dh_p += row_dot_lanes<EP>(Sq + L::GU, 3 * EP, le, dxz, on);
        dh_p += row_dot_lanes<EP>(Sq + L::GU + EP, 3 * EP, le, dxr, on);
        dh_p += row_dot_lanes<EP>(Sq + L::GU + 2 * EP, 3 * EP, le, drh, on);
      }
      // the auxiliary head of position t >= 1: every pos_t and neg_t gets -0.5
      float d_posz = 0.f, d_negz = 0.f, d_ap = 0.f, d_an = 0.f;
      if (t > 0) {
        d_posz = -0.5f * pos * (1.f - pos);
        d_negz = -0.5f * neg * (1.f - neg);
        d_ap = d_posz * Sa[A::PO + lane] * sp * (1.f - sp);
        d_an = d_negz * Sa[A::NO + lane] * sn * (1.f - sn);
        dh_p += row_dot32<EP>(Sa + A::PW, le, d_ap, on);
        dh_p += row_dot32<EP>(Sa + A::NW, le, d_an, on);
        dx += row_dot32<EP>(Sa + A::PW + EP * 32, le, d_ap, on);
        const float dn = row_dot32<EP>(Sa + A::NW + EP * 32, le, d_an, on);
        const size_t en = (size_t)(4 + T + t - 1) * B + row0 + r;
        if (lane == 0) a.trow[en] = (int32_t)(a.tab_row0[0] + nid);
        if (on) a.gemb[en * EP + lane] = dn;
      }
      const size_t eh = (size_t)(4 + t) * B + row0 + r;
      if (lane == 0) a.trow[eh] = (int32_t)(a.tab_row0[0] + hid);
      if (on) a.gemb[eh * EP + lane] = dx;
      // the record: inputs, then deltas
      rec[RX * 32 + lane] = x;
      rec[RHT * 32 + lane] = ht;
      rec[RPC * 32 + lane] = pc;
      rec[RUZ * 32 + lane] = st.uz;
      rec[RPR * 32 + lane] = st.pr;
      rec[RPZ * 32 + lane] = st.pz;
      rec[RPH * 32 + lane] = st.ph;
      rec[RXN * 32 + lane] = xn;
      rec[RAA * 32 + lane] = at;
      rec[RSP * 32 + lane] = sp;
      rec[RSN * 32 + lane] = sn;
      rec[RDXZ * 32 + lane] = on ? dxz : 0.f;
      rec[RDXR * 32 + lane] = on ? dxr : 0.f;
      rec[RDXH * 32 + lane] = on ? dxh : 0.f;
      rec[RDRH * 32 + lane] = on ? drh : 0.f;
      rec[RDPR * 32 + lane] = d_pr;
      rec[RDPZ * 32 + lane] = d_pz;
      rec[RDPH * 32 + lane] = d_ph;
      rec[RDAR * 32 + lane] = on ? d_ar : 0.f;
      rec[RDAZ * 32 + lane] = on ? d_az : 0.f;
      rec[RDAH * 32 + lane] = on ? d_ah : 0.f;
      rec[RDAT * 32 + lane] = d_at;
      rec[RDAP * 32 + lane] = d_ap;
      rec[RDAN * 32 + lane] = d_an;
      rec[RSC * 32 + lane] = lane == 0 ? d_sz : lane == 1 ? d_posz : lane == 2 ? d_negz : 0.f;
      dh = dh_p;
      du = du_p;
    }
    const size_t ec = (size_t)3 * B + row0 + r;           // the candidate
    if (lane == 0) a.trow[ec] = (int32_t)(a.tab_row0[0] + cid);
    if (on) a.gemb[ec * EP + lane] = dc;
  }
  __syncthreads();

  // ---- the sequence part's and the auxiliary head's Dense gradients: rows in order, positions in order ----------
  const float* rec0 = a.rec + (size_t)row0 * T * NS;
  const int n_rec = nv * T;
  for (int q = tid; q < ly.W1; q += kThreads) {
    int in = -1, dl = -1;                  // record float offsets; in -1: the constant 1; dl -1: no gradient
    if (q < L::AW) {                       // gru/kernel, gru_recurrent/kernel [k][g][e]
      const int qq = q < L::GU ? q : q - L::GU, k = qq / (3 * EP), g = (qq / EP) % 3, e = qq % EP;
      in = (q < L::GU ? RX : RHP) * 32 + k;
      dl = (g == 0 ? RDXZ : g == 1 ? RDXR : (q < L::GU ? RDXH : RDRH)) * 32 + e;
    } else if (q < L::IW) {                // att_dense/kernel [k][j]
      in = RPC * 32 + (q - L::AW) / 32; dl = RDAT * 32 + (q - L::AW) % 32;
    } else if (q < L::BX) {                // the AUGRU's In, Hid, Act kernels [g][k][e]
      const int m = (q - L::IW) / (3 * EP * EP), qq = (q - L::IW) % (3 * EP * EP);
      const int g = qq / (EP * EP), k = (qq / EP) % EP, e = qq % EP;
      const int din = g == 0 ? RDPR : g == 1 ? RDPZ : RDPH;
      if (m == 0) { in = RHT * 32 + k; dl = din * 32 + e; }
      else if (m == 1) { in = (g < 2 ? RUP : RUZ) * 32 + k; dl = din * 32 + e; }
      else { in = (g == 0 ? RPR : g == 1 ? RPZ : RPH) * 32 + k; dl = (g == 0 ? RDAR : g == 1 ? RDAZ : RDAH) * 32 + e; }
    } else if (q < L::H0) {                // the biases [3][EP]
      const int m = (q - L::BX) / (3 * EP), g = ((q - L::BX) / EP) % 3, e = (q - L::BX) % EP;
      const int gx[4][3] = {{RDXZ, RDXR, RDXH}, {RDXZ, RDXR, RDRH}, {RDPR, RDPZ, RDPH}, {RDAR, RDAZ, RDAH}};
      dl = gx[m][g] * 32 + e;
    } else if (q < L::AB) {                // augru_h0: not trained
    } else if (q < L::AO) {
      dl = RDAT * 32 + (q - L::AB);
    } else if (q < L::ABO) {
      in = RAA * 32 + (q - L::AO); dl = RSC * 32;
    } else if (q == L::ABO) {
      dl = RSC * 32;
    } else if (q >= ly.aux) {              // the auxiliary head
      const int qa = q - ly.aux;
      if (qa < A::PB) {                    // aux_{pos,neg}_dense/kernel [2EP k][j]
        const bool ng = qa >= A::NW;
        const int k = (qa - (ng ? A::NW : A::PW)) / 32, j = qa % 32;
        in = (k < EP ? RHP * 32 + k : (ng ? RXN : RX) * 32 + k - EP);
        dl = (ng ? RDAN : RDAP) * 32 + j;
      } else if (qa < A::NB) {
        dl = RDAP * 32 + (qa - A::PB);
      } else if (qa < A::PO) {
        dl = RDAN * 32 + (qa - A::NB);
      } else if (qa < A::NO) {
        in = RSP * 32 + (qa - A::PO); dl = RSC * 32 + 1;
      } else if (qa < A::POB) {
        in = RSN * 32 + (qa - A::NO); dl = RSC * 32 + 2;
      } else if (qa == A::POB) {
        dl = RSC * 32 + 1;
      } else if (qa == A::NOB) {
        dl = RSC * 32 + 2;
      }
    }
    float s = 0.f;
    if (dl >= 0 && in >= 0) {
      for (int i = 0; i < n_rec; ++i) s = fmaf(rec0[(size_t)i * NS + in], rec0[(size_t)i * NS + dl], s);
    } else if (dl >= 0) {
      for (int i = 0; i < n_rec; ++i) s += rec0[(size_t)i * NS + dl];
    }
    a.part[(size_t)blockIdx.x * ly.floats + q] = s;
  }
}

template <int EP>
cudaError_t launch_step_t(const DienStepArgs* a, cudaStream_t s) {
  constexpr int smem = step_smem_floats<EP>() * (int)sizeof(float);
  if (!a)                                             // the opt-in on the current device, no launch
    return cudaFuncSetAttribute(dien_train_step_kernel<EP>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  dien_train_step_kernel<EP><<<dien_train_ctas(a->B), kThreads, smem, s>>>(*a);
  ++g_launch_count;
  return cudaGetLastError();
}

}  // namespace

int dien_train_ctas(int B) { return (B + kDienRows - 1) / kDienRows; }

size_t dien_train_rec_floats(int B, int T) { return (size_t)B * T * kDienRecSlots * 32; }

cudaError_t launch_dien_train_step(int EP, const DienStepArgs* a, cudaStream_t s) {
  if (a && a->B <= 0) return cudaSuccess;
#define SRS_DIEN_STEP_CASE(E_) \
  if (EP == E_) return launch_step_t<E_>(a, s);
  SRS_DIEN_STEP_CASE(12) SRS_DIEN_STEP_CASE(16) SRS_DIEN_STEP_CASE(32)
#undef SRS_DIEN_STEP_CASE
  return cudaErrorInvalidValue;
}

}  // namespace srs
