// The competing selectors of the paper's comparison (reference coda/baselines/*.py): per-item scores and the
// selection primitives they share.  Everything here reads the products of one slab scan (hard [N][H] u16,
// disagree [N], ens [N][C]); nothing touches the slab itself.
#include "common.cuh"

#include <limits.h>

#define BL_THREADS 256
#define BL_IPT 16                              // items per thread of a selection chunk (contiguous)
#define BL_CHUNK (BL_THREADS * BL_IPT)         // items per block of the selection kernels

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
// ModelPicker acquisition (modelpicker.py:58-86) in closed form over the groups Z_c of an item (see the header).
// Block prologue: p_h and p_h log2 p_h (0 log 0 = 0) in shared memory, S and B by every warp in the same order.
// ---------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(BL_THREADS) k_mp_entropy(const uint16_t* __restrict__ hard, const float* __restrict__ post,
                                                           int H, long long N, int C, double gamma,
                                                           const uint8_t* __restrict__ labeled,
                                                           const uint8_t* __restrict__ disagree, int mask_agreeing,
                                                           float* __restrict__ ent) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  double* sp = reinterpret_cast<double*>(smem_raw);
  double* spl = sp + H;
  const int Hp = (H + 31) & ~31;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  uint16_t* row = reinterpret_cast<uint16_t*>(spl + H) + (size_t)warp * Hp;
  for (int h = threadIdx.x; h < H; h += blockDim.x) {
    const double p = (double)post[h];
    sp[h] = p;
    spl[h] = p > 0.0 ? p * log2(p) : 0.0;
  }
  __syncthreads();
  double S = 0.0, B = 0.0;
  for (int h = lane; h < H; h += 32) { S += sp[h]; B += spl[h]; }
  S = warp_sum(S);
  B = warp_sum(B);
  const double gm1 = gamma - 1.0, glg = gamma * log2(gamma);
  const double h_none = log2(S) - B / S;               // a class no model predicts: the posterior is unchanged
  const long long nw = (long long)gridDim.x * (blockDim.x >> 5);
  for (long long n = (long long)blockIdx.x * (blockDim.x >> 5) + warp; n < N; n += nw) {
    if (labeled[n] || (mask_agreeing && !disagree[n])) {   // warp-uniform
      if (lane == 0) ent[n] = INFINITY;
      continue;
    }
    const uint16_t* src = hard + (size_t)n * H;
    for (int h = lane; h < H; h += 32) row[h] = src[h];
    __syncwarp();
    double acc = 0.0;
    int K = 0;
    for_each_group(row, H, lane, [&](uint16_t, unsigned mine) {
      double a = 0.0, q = 0.0;
      for (unsigned r = mine; r; r &= r - 1) {
        const int h = (__ffs(r) - 1) * 32 + lane;
        a += sp[h];
        q += spl[h];
      }
      a = warp_sum(a);
      q = warp_sum(q);
      const double norm = S + gm1 * a;
      acc += log2(norm) - (B + gm1 * q + glg * a) / norm;
      ++K;
    });
    if (lane == 0) ent[n] = (float)((acc + (double)(C - K) * h_none) / (double)C);
    __syncwarp();
  }
}

extern "C" int coda_b200_mp_entropy(const uint16_t* hard, const float* posterior, int H, int64_t N, int C, double gamma,
                                    const uint8_t* labeled, const uint8_t* disagree, int mask_agreeing, float* ent,
                                    coda_stream_t stream) {
  CODA_CHECK_ARG(hard && posterior && labeled && disagree && ent, "mp_entropy: null pointer");
  CODA_CHECK_ARG(H >= 1 && H <= 1024 && N >= 1 && C >= 1, "mp_entropy: bad shape H=%d N=%lld C=%d", H, (long long)N, C);
  CODA_CHECK_ARG(gamma > 0.0, "mp_entropy: gamma must be > 0");
  const int Hp = (H + 31) & ~31;
  const size_t smem = (size_t)2 * H * sizeof(double) + (size_t)(BL_THREADS / 32) * Hp * sizeof(uint16_t);
  long long grid = (N + BL_THREADS / 32 - 1) / (BL_THREADS / 32);
  grid = min(grid, (long long)coda_sm_count() * 8);
  k_mp_entropy<<<(unsigned)grid, BL_THREADS, smem, as_stream(stream)>>>(hard, posterior, H, N, C, gamma, labeled,
                                                                         disagree, mask_agreeing, ent);
  CODA_LAUNCH_OK("k_mp_entropy");
  return CODA_B200_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// ActiveTesting and VMA scores (activetesting.py:33-44, vma.py:18-41) over the distinct predicted classes.
// ---------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(BL_THREADS) k_static_scores(const uint16_t* __restrict__ hard, const float* __restrict__ ens,
                                                              int H, long long N, int C, float* __restrict__ at_score,
                                                              float* __restrict__ vma_score) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int Hp = (H + 31) & ~31;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float* lk = reinterpret_cast<float*>(smem_raw) + (size_t)warp * Hp;                     // loss of group k
  int* mk = reinterpret_cast<int*>(smem_raw) + (size_t)(BL_THREADS / 32) * Hp + (size_t)warp * Hp;   // its size
  uint16_t* row = reinterpret_cast<uint16_t*>(reinterpret_cast<int*>(smem_raw) + (size_t)2 * (BL_THREADS / 32) * Hp) +
                  (size_t)warp * Hp;
  const float fH = (float)H;
  const long long nw = (long long)gridDim.x * (blockDim.x >> 5);
  for (long long n = (long long)blockIdx.x * (blockDim.x >> 5) + warp; n < N; n += nw) {
    const uint16_t* src = hard + (size_t)n * H;
    for (int h = lane; h < H; h += 32) row[h] = src[h];
    __syncwarp();
    const float* e = ens + (size_t)n * C;
    int K = 0;
    double at = 0.0;
    for_each_group(row, H, lane, [&](uint16_t c, unsigned mine) {
      const int m = warp_sum((int)__popc(mine));
      const float l = 1.0f - __fdiv_rn(e[c], fH);       // 1 - mean_h preds[h][n][c]
      if (lane == 0) { lk[K] = l; mk[K] = m; }
      at += (double)m * (double)l;
      ++K;
    });
    __syncwarp();
    double v = 0.0;
    for (int i = lane; i < K; i += 32) {
      const double li = lk[i], mi = mk[i];
      for (int j = i + 1; j < K; ++j) v += mi * (double)mk[j] * fabs(li - (double)lk[j]);
    }
    v = warp_sum(v);
    if (lane == 0) {
      if (at_score) at_score[n] = (float)at;
      if (vma_score) vma_score[n] = (float)v;
    }
    __syncwarp();
  }
}

extern "C" int coda_b200_static_scores(const uint16_t* hard, const float* ens, int H, int64_t N, int C, float* at_score,
                                       float* vma_score, coda_stream_t stream) {
  CODA_CHECK_ARG(hard && ens && (at_score || vma_score), "static_scores: null pointer");
  CODA_CHECK_ARG(H >= 1 && H <= 1024 && N >= 1 && C >= 1, "static_scores: bad shape H=%d N=%lld C=%d", H, (long long)N, C);
  const int Hp = (H + 31) & ~31;
  const size_t smem = (size_t)(BL_THREADS / 32) * Hp * (sizeof(float) + sizeof(int) + sizeof(uint16_t));
  if (smem > 48 * 1024)
    CODA_CUDA_OK(cudaFuncSetAttribute(k_static_scores, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  long long grid = (N + BL_THREADS / 32 - 1) / (BL_THREADS / 32);
  grid = min(grid, (long long)coda_sm_count() * 8);
  k_static_scores<<<(unsigned)grid, BL_THREADS, smem, as_stream(stream)>>>(hard, ens, H, N, C, at_score, vma_score);
  CODA_LAUNCH_OK("k_static_scores");
  return CODA_B200_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// Selection over the unlabeled items.  Block b owns items [b * BL_CHUNK, (b + 1) * BL_CHUNK); thread t of a block owns
// BL_IPT consecutive items of it, so per-block partials and the in-block scan see the items in index order.
// ---------------------------------------------------------------------------------------------------------------
template <typename T>
__device__ __forceinline__ T warp_incl_scan(T x, int lane) {
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const T y = __shfl_up_sync(CODA_FULL, x, o);
    if (lane >= o) x += y;
  }
  return x;
}

// Exclusive prefix of x over the block's threads (thread order) and the block total.  sh: >= BL_THREADS / 32 slots.
template <typename T>
__device__ __forceinline__ T block_excl_scan(T x, T* sh, T& total) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarp = blockDim.x >> 5;
  const T incl = warp_incl_scan(x, lane);
  if (lane == 31) sh[warp] = incl;
  __syncthreads();
  if (warp == 0) {
    const T w = lane < nwarp ? sh[lane] : T(0);
    const T wi = warp_incl_scan(w, lane);
    __syncwarp();
    if (lane < nwarp) sh[lane] = wi;
  }
  __syncthreads();
  T before = __shfl_up_sync(CODA_FULL, incl, 1);
  if (lane == 0) before = T(0);
  const T out = (warp > 0 ? sh[warp - 1] : T(0)) + before;
  total = sh[nwarp - 1];
  __syncthreads();
  return out;
}

__device__ __forceinline__ long long chunk_lo(long long N) {
  return min(N, (long long)blockIdx.x * BL_CHUNK + (long long)threadIdx.x * BL_IPT);
}

// -- weighted draw (random.choices, activetesting.py:45-48 / vma.py:44-60) ---------------------------------------
// partials [nblocks][2] double: {sum of the block's weights, number of unlabeled items in it}.
template <bool NORMALISED>
__global__ void __launch_bounds__(BL_THREADS) k_wsum_blocks(const float* __restrict__ w, const uint8_t* __restrict__ labeled,
                                                           long long N, const double* __restrict__ total,
                                                           double* __restrict__ partials) {
  __shared__ double shs[BL_THREADS / 32];
  __shared__ int shc[BL_THREADS / 32];
  const long long lo = chunk_lo(N), hi = min(N, lo + BL_IPT);
  const float tf = NORMALISED ? (float)total[0] : 1.0f;
  double s = 0.0;
  int cnt = 0;
  for (long long i = lo; i < hi; ++i)
    if (!labeled[i]) {
      s += (double)(NORMALISED ? __fdiv_rn(w[i], tf) : w[i]);
      ++cnt;
    }
  double st;
  int ct;
  block_excl_scan(s, shs, st);
  block_excl_scan(cnt, shc, ct);
  if (threadIdx.x == 0) {
    partials[2 * blockIdx.x] = st;
    partials[2 * blockIdx.x + 1] = (double)ct;
  }
}

__global__ void k_wsum_final(const double* __restrict__ partials, int nblocks, double* __restrict__ total) {
  double s = 0.0, c = 0.0;
  for (int b = 0; b < nblocks; ++b) { s += partials[2 * b]; c += partials[2 * b + 1]; }
  total[0] = s;
  total[1] = c;
}

// One block: cum = running sum of the normalised weights in index order; the pick is the first unlabeled item with
// cum > u * cum_total (bisect_right), the last one when rounding leaves none.  out = {position among the unlabeled
// items, item, float bits of its normalised weight}.
__global__ void __launch_bounds__(BL_THREADS) k_wdraw_pick(const float* __restrict__ w, const uint8_t* __restrict__ labeled,
                                                          long long N, const double* __restrict__ total,
                                                          const double* __restrict__ partials, int nblocks, double u,
                                                          long long* __restrict__ out) {
  __shared__ double shs[BL_THREADS / 32];
  __shared__ int shc[BL_THREADS / 32];
  __shared__ double s_base, s_target;
  __shared__ long long s_pos0;
  __shared__ int s_blk;
  __shared__ unsigned long long s_first;
  const float tf = (float)total[0];
  if (threadIdx.x == 0) {
    double grand = 0.0;
    for (int b = 0; b < nblocks; ++b) grand += partials[2 * b];
    const double target = u * grand;
    double base = 0.0, pos = 0.0;
    int blk = -1, last = -1;
    for (int b = 0; b < nblocks; ++b) {
      if (partials[2 * b + 1] == 0.0) continue;
      last = b;
      if (base + partials[2 * b] > target) { blk = b; break; }
      base += partials[2 * b];
      pos += partials[2 * b + 1];
    }
    if (blk < 0 && last >= 0) {                        // target at or beyond the total: the last unlabeled item
      blk = last;
      base -= partials[2 * last];
      pos -= partials[2 * last + 1];
    }
    s_blk = blk;
    s_base = base;
    s_target = target;
    s_pos0 = (long long)pos;
    s_first = ~0ull;
  }
  __syncthreads();
  const int blk = s_blk;
  if (blk < 0) {
    if (threadIdx.x == 0) { out[0] = -1; out[1] = -1; out[2] = 0; }
    return;
  }
  const long long lo = min(N, (long long)blk * BL_CHUNK + (long long)threadIdx.x * BL_IPT), hi = min(N, lo + BL_IPT);
  double s = 0.0;
  int cnt = 0;
  for (long long i = lo; i < hi; ++i)
    if (!labeled[i]) { s += (double)__fdiv_rn(w[i], tf); ++cnt; }
  double st;
  int ct;
  const double before = block_excl_scan(s, shs, st);
  const int cbefore = block_excl_scan(cnt, shc, ct);
  // the same per-thread sums as k_wsum_blocks, so the running sum of the chunk ends at base + its partial
  double cum = s_base + before;
  long long pos = s_pos0 + cbefore;
  long long last_i = -1, last_pos = -1;
  for (long long i = lo; i < hi; ++i) {
    if (labeled[i]) continue;
    cum += (double)__fdiv_rn(w[i], tf);
    if (cum > s_target) {
      atomicMin(&s_first, ((unsigned long long)pos << 16) | (unsigned long long)(i - (long long)blk * BL_CHUNK));
      break;
    }
    last_i = i;
    last_pos = pos;
    ++pos;
  }
  __syncthreads();
  if (s_first == ~0ull && last_i >= 0 && last_pos == s_pos0 + ct - 1) {   // the owner of the chunk's last unlabeled item
    s_first = ((unsigned long long)last_pos << 16) | (unsigned long long)(last_i - (long long)blk * BL_CHUNK);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    const long long i = (long long)blk * BL_CHUNK + (long long)(s_first & 0xffffull);
    out[0] = (long long)(s_first >> 16);
    out[1] = i;
    out[2] = (long long)__float_as_uint(__fdiv_rn(w[i], tf));
  }
}

extern "C" int coda_b200_select_blocks(int64_t N) { return (int)((N + BL_CHUNK - 1) / BL_CHUNK); }

extern "C" int coda_b200_weighted_total(const float* w, const uint8_t* labeled, int64_t N, double* partials,
                                        double* total, coda_stream_t stream) {
  CODA_CHECK_ARG(w && labeled && partials && total, "weighted_total: null pointer");
  CODA_CHECK_ARG(N >= 1 && N < (1LL << 40), "weighted_total: bad N=%lld", (long long)N);
  const int nb = coda_b200_select_blocks(N);
  k_wsum_blocks<false><<<nb, BL_THREADS, 0, as_stream(stream)>>>(w, labeled, N, nullptr, partials);
  CODA_LAUNCH_OK("k_wsum_blocks");
  k_wsum_final<<<1, 1, 0, as_stream(stream)>>>(partials, nb, total);
  CODA_LAUNCH_OK("k_wsum_final");
  return CODA_B200_OK;
}

extern "C" int coda_b200_weighted_draw(const float* w, const uint8_t* labeled, int64_t N, const double* total, double u,
                                       double* partials, int64_t* out, coda_stream_t stream) {
  CODA_CHECK_ARG(w && labeled && total && partials && out, "weighted_draw: null pointer");
  CODA_CHECK_ARG(N >= 1 && N < (1LL << 40), "weighted_draw: bad N=%lld", (long long)N);
  CODA_CHECK_ARG(u >= 0.0 && u < 1.0, "weighted_draw: u must be in [0, 1)");
  const int nb = coda_b200_select_blocks(N);
  k_wsum_blocks<true><<<nb, BL_THREADS, 0, as_stream(stream)>>>(w, labeled, N, total, partials);
  CODA_LAUNCH_OK("k_wsum_blocks");
  k_wdraw_pick<<<1, BL_THREADS, 0, as_stream(stream)>>>(w, labeled, N, total, partials, nb, u, (long long*)out);
  CODA_LAUNCH_OK("k_wdraw_pick");
  return CODA_B200_OK;
}

// -- extreme value with exact ties (modelpicker.py:68-70 min, uncertainty.py:37-42 max) ---------------------------
// {value, count} partials merge associatively: the better value wins, equal values add their counts.
struct ValCnt {
  float v;
  long long n;
};
__device__ __forceinline__ void vc_merge(ValCnt& a, const ValCnt& b, bool want_max) {
  if (b.n == 0) return;
  if (a.n == 0 || (want_max ? b.v > a.v : b.v < a.v)) { a = b; return; }
  if (b.v == a.v) a.n += b.n;
}

__global__ void __launch_bounds__(BL_THREADS) k_extreme_blocks(const float* __restrict__ v, const uint8_t* __restrict__ labeled,
                                                              long long N, int want_max, long long* __restrict__ partials) {
  __shared__ float shv[BL_THREADS / 32];
  __shared__ long long shn[BL_THREADS / 32];
  const long long lo = chunk_lo(N), hi = min(N, lo + BL_IPT);
  ValCnt a{0.f, 0};
  for (long long i = lo; i < hi; ++i)
    if (!labeled[i]) vc_merge(a, ValCnt{v[i], 1}, want_max);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    ValCnt b{__shfl_xor_sync(CODA_FULL, a.v, o), __shfl_xor_sync(CODA_FULL, a.n, o)};
    vc_merge(a, b, want_max);
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) { shv[warp] = a.v; shn[warp] = a.n; }
  __syncthreads();
  if (threadIdx.x == 0) {
    ValCnt t{0.f, 0};
    for (int k = 0; k < BL_THREADS / 32; ++k) vc_merge(t, ValCnt{shv[k], shn[k]}, want_max);
    partials[2 * blockIdx.x] = (long long)__float_as_uint(t.v);
    partials[2 * blockIdx.x + 1] = t.n;
  }
}

__global__ void k_extreme_final(const long long* __restrict__ partials, int nblocks, int want_max, long long* __restrict__ out) {
  ValCnt t{0.f, 0};
  for (int b = 0; b < nblocks; ++b) vc_merge(t, ValCnt{__uint_as_float((unsigned)partials[2 * b]), partials[2 * b + 1]}, want_max);
  out[0] = (long long)__float_as_uint(t.v);
  out[1] = t.n;
}

// One block: the k-th (ascending index) unlabeled item whose value equals best[0].  Only blocks whose partial value is
// the best hold such items, so the partials locate the chunk without another pass over the vector.
__global__ void __launch_bounds__(BL_THREADS) k_select_kth(const float* __restrict__ v, const uint8_t* __restrict__ labeled,
                                                          long long N, const long long* __restrict__ partials, int nblocks,
                                                          const long long* __restrict__ best, long long k,
                                                          long long* __restrict__ out) {
  __shared__ long long shc[BL_THREADS / 32];
  __shared__ int s_blk;
  __shared__ long long s_k;
  const float bv = __uint_as_float((unsigned)best[0]);
  if (threadIdx.x == 0) {
    int blk = -1;
    long long kk = k;
    for (int b = 0; b < nblocks && blk < 0; ++b) {
      const long long n = partials[2 * b + 1];
      if (n == 0 || __uint_as_float((unsigned)partials[2 * b]) != bv) continue;
      if (kk < n) blk = b;
      else kk -= n;
    }
    s_blk = blk;
    s_k = kk;
  }
  __syncthreads();
  const int blk = s_blk;
  if (blk < 0) {
    if (threadIdx.x == 0) out[0] = -1;
    return;
  }
  const long long lo = min(N, (long long)blk * BL_CHUNK + (long long)threadIdx.x * BL_IPT), hi = min(N, lo + BL_IPT);
  long long cnt = 0;
  for (long long i = lo; i < hi; ++i) cnt += (!labeled[i] && v[i] == bv);
  long long tot;
  long long r = s_k - block_excl_scan(cnt, shc, tot);
  if (r >= 0 && r < cnt) {
    for (long long i = lo; i < hi; ++i)
      if (!labeled[i] && v[i] == bv && r-- == 0) { out[0] = i; break; }
  }
}

extern "C" int coda_b200_select_extreme(const float* v, const uint8_t* labeled, int64_t N, int want_max,
                                        int64_t* partials, int64_t* out, coda_stream_t stream) {
  CODA_CHECK_ARG(v && labeled && partials && out, "select_extreme: null pointer");
  CODA_CHECK_ARG(N >= 1 && N < (1LL << 40), "select_extreme: bad N=%lld", (long long)N);
  const int nb = coda_b200_select_blocks(N);
  k_extreme_blocks<<<nb, BL_THREADS, 0, as_stream(stream)>>>(v, labeled, N, want_max, (long long*)partials);
  CODA_LAUNCH_OK("k_extreme_blocks");
  k_extreme_final<<<1, 1, 0, as_stream(stream)>>>((const long long*)partials, nb, want_max, (long long*)out);
  CODA_LAUNCH_OK("k_extreme_final");
  return CODA_B200_OK;
}

extern "C" int coda_b200_select_kth(const float* v, const uint8_t* labeled, int64_t N, const int64_t* partials,
                                    const int64_t* best, int64_t k, int64_t* out_idx, coda_stream_t stream) {
  CODA_CHECK_ARG(v && labeled && partials && best && out_idx, "select_kth: null pointer");
  CODA_CHECK_ARG(N >= 1 && N < (1LL << 40) && k >= 0, "select_kth: bad N=%lld k=%lld", (long long)N, (long long)k);
  k_select_kth<<<1, BL_THREADS, 0, as_stream(stream)>>>(v, labeled, N, (const long long*)partials,
                                                        coda_b200_select_blocks(N), (const long long*)best, k,
                                                        (long long*)out_idx);
  CODA_LAUNCH_OK("k_select_kth");
  return CODA_B200_OK;
}
