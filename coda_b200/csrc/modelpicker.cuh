// ModelPicker pieces shared by the selector's kernels (baselines.cu: k_mp_entropy, k_bl_draw, k_bl_step) and the
// batched epsilon search (eps_search.cu: k_mp_runs).  Both must round alike step for step: a run of the search is
// pinned bit for bit to ModelPicker.run_steps on the same pool, so the arithmetic of an item's entropy and of the
// Philox tie draws lives here once.
#pragma once
#include "common.cuh"

#include <curand_philox4x32_x.h>
#include <limits.h>

__device__ __forceinline__ int warp_min_int(int v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = min(v, __shfl_xor_sync(CODA_FULL, v, o));
  return v;
}

// Walks the groups of models that predict the same class for one item, in the order of each group's lowest model
// index (a relabelling of the classes keeps the groups and therefore the order and every rounding step).  `row` is the
// item's hard row in shared memory; for each group `fn(c, lane_bits)` is called on every lane, lane_bits = the slots
// (h = slot * 32 + lane) of this lane that belong to the group.
template <typename Fn>
__device__ __forceinline__ void for_each_group(const uint16_t* row, int H, int lane, Fn fn) {
  const int nslots = (H + 31) >> 5;
  unsigned rem = 0;
  for (int s = 0; s < nslots; ++s)
    if (s * 32 + lane < H) rem |= 1u << s;
  while (true) {
    const int hl = rem ? (__ffs(rem) - 1) * 32 + lane : INT_MAX;
    const int hmin = warp_min_int(hl);
    if (hmin == INT_MAX) break;
    const uint16_t c = row[hmin];
    unsigned mine = 0;
    for (unsigned r = rem; r; r &= r - 1) {
      const int s = __ffs(r) - 1;
      if (row[s * 32 + lane] == c) mine |= 1u << s;
    }
    rem &= ~mine;
    fn(c, mine);
  }
}

// ---------------------------------------------------------------------------------------------------------------
// ModelPicker acquisition (modelpicker.py:58-86) in closed form over the groups Z_c of an item (DESIGN.md §5b).
// sp[h] = p_h and spl[h] = p_h log2 p_h (0 log 0 = 0) in shared memory; S = sum p_h and B = sum p_h log2 p_h.
// ---------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void mp_post_terms(float post_h, double& p, double& pl) {
  p = (double)post_h;
  pl = p > 0.0 ? p * log2(p) : 0.0;
}

// S and B of one warp: lane partials over h = lane, lane + 32, ..., then warp_sum (every lane gets the same bits)
__device__ __forceinline__ void mp_sums(const double* sp, const double* spl, int H, int lane, double& S, double& B) {
  S = 0.0;
  B = 0.0;
  for (int h = lane; h < H; h += 32) { S += sp[h]; B += spl[h]; }
  S = warp_sum(S);
  B = warp_sum(B);
}

// the entropy of a class no model predicts (the posterior is unchanged)
__device__ __forceinline__ double mp_h_none(double S, double B) { return log2(S) - B / S; }

// one group's term of the item's acc: a = sum of p_h and q = sum of p_h log2 p_h over the group (lane partials in slot
// order, then warp_sum), gm1 = gamma - 1, glg = gamma log2 gamma
__device__ __forceinline__ double mp_group_term(const double* sp, const double* spl, unsigned mine, int lane, double S,
                                                double B, double gm1, double glg) {
  double a = 0.0, q = 0.0;
  for (unsigned r = mine; r; r &= r - 1) {
    const int h = (__ffs(r) - 1) * 32 + lane;
    a += sp[h];
    q += spl[h];
  }
  a = warp_sum(a);
  q = warp_sum(q);
  const double norm = S + gm1 * a;
  return log2(norm) - (B + gm1 * q + glg * a) / norm;
}

// the item's expected posterior entropy from acc (the sum of its K group terms, in group order)
__device__ __forceinline__ float mp_item_entropy(double acc, int K, int C, double h_none) {
  return (float)((acc + (double)(C - K) * h_none) / (double)C);
}

// ---------------------------------------------------------------------------------------------------------------
// Tie draws of the host-free loops (include/coda_b200.h)
// ---------------------------------------------------------------------------------------------------------------
// r.x of Philox4x32-10 at key = the 64-bit seed, counter = {label count, purpose, 0, 0}
__device__ __forceinline__ unsigned bl_philox(long long seed, long long count, unsigned purpose) {
  const unsigned long long k = (unsigned long long)seed;
  return curand_Philox4x32_10(make_uint4((unsigned)count, purpose, 0u, 0u), make_uint2((unsigned)k, (unsigned)(k >> 32))).x;
}
// (r * cnt) >> 32 in 96-bit arithmetic: the tie j in [0, cnt) in ascending index order
__device__ __forceinline__ long long bl_tie_pick(unsigned r, long long cnt) {
  const unsigned long long c = (unsigned long long)cnt, lo = (unsigned long long)r * (c & 0xffffffffull);
  return (long long)(((unsigned long long)r * (c >> 32)) + (lo >> 32));
}

// One model's LURE risk from the loop's running sums after m labels of Ng items: (s1 + (Ng - m) s2) / m, the product
// and the sum as one explicit fused multiply-add.  k_bl_step and k_bl_best_ref both decide the best model's exact ties
// on it, so they see the same bits whatever the compiler would contract (tests/test_selector_kernels.py models it as
// fl(fma(Ng - m, s2, s1) / m)).  At m = Ng it is s1 / m, the plain mean loss.
__device__ __forceinline__ double bl_lure_risk(double s1, double s2, double Ng, double m) {
  return __fma_rn(Ng - m, s2, s1) / m;
}
