// dien_layers.cuh - DIEN's per-row sequence arithmetic (DIEN.py:154-292), shared by the serving kernel (dien.cu) and
// the training step (dien_train.cu), so that both compute every value of a row with the same instructions.
//
// One warp owns a row and lane e owns element e of every state vector (E <= EP <= 32; lanes >= EP mirror lane EP - 1
// and are never read).  A matrix-vector product is EP shuffle-broadcasts against weight rows in shared memory, in
// the layouts below.  The functions return the values a backward pass needs beside their result; a caller that
// does not read them leaves them to the compiler to drop.
#pragma once

#include <cmath>

#include "kernels.h"

namespace srs {

constexpr int kDienRows = 32;     // rows per CTA tile

// DienLayout's offsets (kernels.h) as compile-time constants of one padded width
template <int EP>
struct DienBlob {                 // float offsets inside DienParams::seq
  static constexpr DienLayout l = DienLayout::of(EP);
  static constexpr int GW = l.GW, GU = l.GU, AW = l.AW, IW = l.IW, HW = l.HW, SW = l.SW, BX = l.BX, BH = l.BH,
                       BI = l.BI, BA = l.BA, H0 = l.H0, AB = l.AB, AO = l.AO, ABO = l.ABO, TOTAL = l.seq;
};

template <int EP>
struct DienAuxBlob {              // float offsets inside DienAuxView::w
  static constexpr DienLayout l = DienLayout::of(EP);
  static constexpr int PW = l.PW, NW = l.NW, PB = l.PB, NB = l.NB, PO = l.PO, NO = l.NO, POB = l.POB, NOB = l.NOB,
                       TOTAL = l.aux_floats;
};

// the auxiliary head at one position: g = g_t, e = e(h_{t+1}), n = e(n_{t+1}), lane k holding element k.  Returns
// pos_t + neg_t; sp / sn get lane j's sigmoid(Dense32) unit of each side, pos / neg the two outputs.
template <int EP>
__device__ __forceinline__ float dien_aux_step(const float* Sa, float g, float e, float n, int lane, float* sp,
                                               float* sn, float* pos_out, float* neg_out) {
  using A = DienAuxBlob<EP>;
  float ap = Sa[A::PB + lane], an = Sa[A::NB + lane];
#pragma unroll
  for (int k = 0; k < EP; ++k) {
    const float gk = __shfl_sync(0xffffffffu, g, k);
    const float ek = __shfl_sync(0xffffffffu, e, k);
    const float nk = __shfl_sync(0xffffffffu, n, k);
    ap = fmaf(gk, Sa[A::PW + k * 32 + lane], ap);
    an = fmaf(gk, Sa[A::NW + k * 32 + lane], an);
    ap = fmaf(ek, Sa[A::PW + (EP + k) * 32 + lane], ap);
    an = fmaf(nk, Sa[A::NW + (EP + k) * 32 + lane], an);
  }
  *sp = sigmoidf_acc(ap);
  const float pos = sigmoidf_acc(warp_sum(*sp * Sa[A::PO + lane]) + Sa[A::POB]);
  *sn = sigmoidf_acc(an);
  const float neg = sigmoidf_acc(warp_sum(*sn * Sa[A::NO + lane]) + Sa[A::NOB]);
  *pos_out = pos;
  *neg_out = neg;
  return pos + neg;
}

// One Keras GRU step (z | r | h, reset_after) on input x and state h; le = min(lane, EP - 1).  Returns the new
// state hn (the caller applies the mask); z, r, hh and rh (the recurrent h-gate product before the reset gate) are
// what the backward needs.
template <int EP>
__device__ __forceinline__ float dien_gru_step(const float* Sq, int le, float x, float h, float* z_out, float* r_out,
                                               float* hh_out, float* rh_out) {
  using L = DienBlob<EP>;
  const float* gw = Sq + L::GW + le;
  const float* gu = Sq + L::GU + le;
  float xz = Sq[L::BX + le], xr = Sq[L::BX + EP + le], xh = Sq[L::BX + 2 * EP + le];
  float rz = Sq[L::BH + le], rr = Sq[L::BH + EP + le], rh = Sq[L::BH + 2 * EP + le];
#pragma unroll
  for (int k = 0; k < EP; ++k) {
    const float xk = __shfl_sync(0xffffffffu, x, k);
    const float hk = __shfl_sync(0xffffffffu, h, k);
    xz = fmaf(xk, gw[k * 3 * EP], xz);
    xr = fmaf(xk, gw[k * 3 * EP + EP], xr);
    xh = fmaf(xk, gw[k * 3 * EP + 2 * EP], xh);
    rz = fmaf(hk, gu[k * 3 * EP], rz);
    rr = fmaf(hk, gu[k * 3 * EP + EP], rr);
    rh = fmaf(hk, gu[k * 3 * EP + 2 * EP], rh);
  }
  const float z = sigmoidf_acc(xz + rz);
  const float rg = sigmoidf_acc(xr + rr);
  const float hh = tanhf(xh + rg * rh);
  *z_out = z; *r_out = rg; *hh_out = hh; *rh_out = rh;
  return z * h + (1.f - z) * hh;
}

// The attention score of one position: s = sigmoid(Dense1(sigmoid(Dense32(pc)))), pc = g_t * c; lane j owns unit
// j of Dense32 and gets its output in *a_out.
template <int EP>
__device__ __forceinline__ float dien_attention(const float* Sq, int lane, float pc, float att_b, float att_wo,
                                                float att_bo, float* a_out) {
  using L = DienBlob<EP>;
  const float* aw = Sq + L::AW + lane;
  float a = att_b;
#pragma unroll
  for (int k = 0; k < EP; ++k) a = fmaf(__shfl_sync(0xffffffffu, pc, k), aw[k * 32], a);
  a = sigmoidf_acc(a);
  *a_out = a;
  return sigmoidf_acc(warp_sum(a * att_wo) + att_bo);
}

// What one AUGRU step leaves for the backward: the three act-layer inputs, the two gates, u * z, the candidate
// state and the attention-scaled update gate
struct DienAugruStep { float pr, pz, ph, rg, zg, uz, hn, ra; };

// One AUGRU step (DIEN.py:204-245): input h = g_t, state u, attention score s.  Returns the new state.
template <int EP>
__device__ __forceinline__ float dien_augru_step(const float* Sq, int le, float h, float u, float s,
                                                 DienAugruStep* o) {
  using L = DienBlob<EP>;
  const float* iw = Sq + L::IW + le;
  const float* hw = Sq + L::HW + le;
  const float* sw = Sq + L::SW + le;
  float pr = Sq[L::BI + le], pz = Sq[L::BI + EP + le], ph = Sq[L::BI + 2 * EP + le];
#pragma unroll
  for (int k = 0; k < EP; ++k) {
    const float hk = __shfl_sync(0xffffffffu, h, k);
    const float uk = __shfl_sync(0xffffffffu, u, k);
    pr = fmaf(hk, iw[k * EP], pr);
    pz = fmaf(hk, iw[EP * EP + k * EP], pz);
    ph = fmaf(hk, iw[2 * EP * EP + k * EP], ph);
    pr = fmaf(uk, hw[k * EP], pr);
    pz = fmaf(uk, hw[EP * EP + k * EP], pz);
  }
  float ar = Sq[L::BA + le], az = Sq[L::BA + EP + le];
#pragma unroll
  for (int k = 0; k < EP; ++k) {
    ar = fmaf(__shfl_sync(0xffffffffu, pr, k), sw[k * EP], ar);
    az = fmaf(__shfl_sync(0xffffffffu, pz, k), sw[EP * EP + k * EP], az);
  }
  const float rg = sigmoidf_acc(ar), zg = sigmoidf_acc(az);
  const float uz = u * zg;
#pragma unroll
  for (int k = 0; k < EP; ++k)
    ph = fmaf(__shfl_sync(0xffffffffu, uz, k), hw[2 * EP * EP + k * EP], ph);
  float ah = Sq[L::BA + 2 * EP + le];
#pragma unroll
  for (int k = 0; k < EP; ++k)
    ah = fmaf(__shfl_sync(0xffffffffu, ph, k), sw[2 * EP * EP + k * EP], ah);
  const float hn = tanhf(ah);
  const float ra = s * rg;
  o->pr = pr; o->pz = pz; o->ph = ph; o->rg = rg; o->zg = zg; o->uz = uz; o->hn = hn; o->ra = ra;
  return (1.f - ra) * u + ra * hn;
}

// a history or negative id as the Embedding layer sees it: through a float32 numeric column (DIEN.py:96-105)
__device__ __forceinline__ int dien_id(int raw) { return __float2int_rz(__int2float_rn(raw)); }

}  // namespace srs
