// The per-item arithmetic of the EIG assembly of the full scoring pass (gain.cu: k_eig_assemble_g8, k_gain_eig),
// restated operation for operation for the sampled pass (sample.cu), so that an item scored by either gets the same
// bits (tests/test_prefilter_sample.py).  gain.cu keeps its own copy: routed through these helpers its kernels
// compiled to differently scheduled SASS.
//
//   s = sum_c U[n][c],   e = sum_c U[n][c] * g0[c] + sum_entries U[n][c_e] * (gain_e - g0[c_e]),   eig = e / max(s, 1e-12)
//
// g0[c] is the gain of class c's empty-set template row; one entry per distinct predicted class of the item.
#pragma once
#include "common.cuh"

// coda.py:230 clamp, coda.py:278
__device__ __forceinline__ float eig_value(float e, float s) { return e / fmaxf(s, 1e-12f); }

// 8-lane group g of an item (C <= 128, <= 32 entries): classes g + 8 k, then entries g + 8 j (er < 0: none), then
// the sums over the group's 8 lanes.  Every lane of the group ends with the item's s and e.
template <int KC8>
__device__ __forceinline__ void g8_item_sums(const float (&u)[KC8], const int (&er)[4], const int (&ec)[4],
                                             const float (&eu)[4], const float (&eg)[4], const float* g0, int C, int g,
                                             float& s, float& e) {
  s = 0.f;
  e = 0.f;
#pragma unroll
  for (int k = 0; k < KC8; ++k) {
    const int c = g + 8 * k;
    s += u[k];
    if (c < C) e = fmaf(u[k], g0[c], e);
  }
#pragma unroll
  for (int j = 0; j < 4; ++j)
    if (er[j] >= 0) e = fmaf(eu[j], eg[j] - g0[ec[j]], e);
#pragma unroll
  for (int o = 4; o > 0; o >>= 1) {
    s += __shfl_xor_sync(CODA_FULL, s, o);
    e += __shfl_xor_sync(CODA_FULL, e, o);
  }
}

// One warp, one item, any C and any number of entries: the entries [e0, e1) in chunks of 32 lanes, then the classes
// c = lane + 32 k, then the warp sums.  KC > 0: the U row is passed in u (C <= 32 KC); KC = 0: it is read from urow.
// gain_at(r): the gain of row r.
template <int KC, typename GainAt>
__device__ __forceinline__ void warp_item_sums(const float* urow, const float (&u)[KC > 0 ? KC : 1], int C, int e0,
                                               int e1, const int32_t* __restrict__ ent_row,
                                               const uint16_t* __restrict__ ent_cls, const float* g0, GainAt gain_at,
                                               int lane, float& s_out, float& e_out) {
  constexpr int KR = KC > 0 ? KC : 1;
  float s = 0.f, e = 0.f;
  for (int eb = e0; eb < e1; eb += 32) {       // one trip unless an item has > 32 distinct predicted classes
    int r = -1, c = 0;
    if (eb + lane < e1) {
      r = __ldg(ent_row + eb + lane);
      c = __ldg(ent_cls + eb + lane);
    }
    const float myg = r >= 0 ? gain_at(r) : 0.f;
    // correction of this chunk's entries: xi_c * (gain - gain of the empty-set template)
    float ucls = 0.f;
    if (KC > 0) {
#pragma unroll
      for (int k = 0; k < KR; ++k) {
        const float t = __shfl_sync(CODA_FULL, u[k], c & 31);
        if ((c >> 5) == k) ucls = t;
      }
    } else if (r >= 0) {
      ucls = __ldg(urow + c);
    }
    if (r >= 0) e = fmaf(ucls, myg - g0[c], e);
  }
  if (KC > 0) {
#pragma unroll
    for (int k = 0; k < KR; ++k) {
      const int c = lane + 32 * k;
      s += u[k];
      if (c < C) e = fmaf(u[k], g0[c], e);
    }
  } else {
    for (int c = lane; c < C; c += 32) {
      const float v = __ldg(urow + c);
      s += v;
      e = fmaf(v, g0[c], e);
    }
  }
  s_out = warp_sum(s);
  e_out = warp_sum(e);
}
