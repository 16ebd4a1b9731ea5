// The competing selectors of the paper's comparison (reference coda/baselines/*.py): per-item scores and the
// selection primitives they share.  Everything here reads the products of one slab scan (hard [N][H] u16,
// disagree [N], ens [N][C]); nothing touches the slab itself.  N-range shards exchange their selection records through
// the mailboxes of xchg.cuh (record channel), so every shard ends a selection call with the same global answer.
#include "xchg.cuh"
#include "modelpicker.cuh"
#include "pyrandom.cuh"

#define BL_THREADS 256
#define BL_IPT 16                              // items per thread of a selection chunk (contiguous)
#define BL_CHUNK (BL_THREADS * BL_IPT)         // items per block of the selection kernels

// ---------------------------------------------------------------------------------------------------------------
// ModelPicker acquisition (modelpicker.py:58-86) in closed form over the groups Z_c of an item (modelpicker.cuh).
// Block prologue: p_h and p_h log2 p_h (0 log 0 = 0) in shared memory, S and B by every warp in the same order.
// ---------------------------------------------------------------------------------------------------------------
// DEV: the mask switch is *mask_dev > 0 (device loop) instead of mask_agreeing
template <bool DEV>
__global__ void __launch_bounds__(BL_THREADS) k_mp_entropy(const uint16_t* __restrict__ hard, const float* __restrict__ post,
                                                           int H, long long N, int C, double gamma,
                                                           const uint8_t* __restrict__ labeled,
                                                           const uint8_t* __restrict__ disagree, int mask_agreeing,
                                                           const long long* __restrict__ mask_dev,
                                                           float* __restrict__ ent) {
  if (DEV) mask_agreeing = *mask_dev > 0;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  double* sp = reinterpret_cast<double*>(smem_raw);
  double* spl = sp + H;
  const int Hp = (H + 31) & ~31;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  uint16_t* row = reinterpret_cast<uint16_t*>(spl + H) + (size_t)warp * Hp;
  for (int h = threadIdx.x; h < H; h += blockDim.x) mp_post_terms(post[h], sp[h], spl[h]);
  __syncthreads();
  double S, B;
  mp_sums(sp, spl, H, lane, S, B);
  const double gm1 = gamma - 1.0, glg = gamma * log2(gamma);
  const double h_none = mp_h_none(S, B);
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
      acc += mp_group_term(sp, spl, mine, lane, S, B, gm1, glg);
      ++K;
    });
    if (lane == 0) ent[n] = mp_item_entropy(acc, K, C, h_none);
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
  k_mp_entropy<false><<<(unsigned)grid, BL_THREADS, smem, as_stream(stream)>>>(hard, posterior, H, N, C, gamma, labeled,
                                                                                disagree, mask_agreeing, nullptr, ent);
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

// Every thread of one block: cum = base0 + running sum of the normalised weights in index order over this vector's
// chunks; the pick is the first unlabeled item with cum > target (bisect_right), the last one when rounding leaves
// none.  base0, pos0 (the weight and the number of unlabeled items before this vector) and target are read from
// thread 0.  res (thread 0) = {position among the unlabeled items, item, float bits of its normalised weight}, or
// {-1, -1, 0} when no item is unlabeled.
__device__ void wdraw_in_chunks(const float* __restrict__ w, const uint8_t* __restrict__ labeled, long long N, float tf,
                                const double* __restrict__ partials, int nblocks, double base0, double pos0,
                                double target, long long* res) {
  __shared__ double shs[BL_THREADS / 32];
  __shared__ int shc[BL_THREADS / 32];
  __shared__ double s_base, s_target;
  __shared__ long long s_pos0;
  __shared__ int s_blk;
  __shared__ unsigned long long s_first;
  if (threadIdx.x == 0) {
    double base = base0, pos = pos0;
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
    if (threadIdx.x == 0) { res[0] = -1; res[1] = -1; res[2] = 0; }
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
    res[0] = (long long)(s_first >> 16);
    res[1] = i;
    res[2] = (long long)__float_as_uint(__fdiv_rn(w[i], tf));
  }
}

extern "C" int coda_b200_select_blocks(int64_t N) { return (int)((N + BL_CHUNK - 1) / BL_CHUNK); }

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

// One block: the k-th (ascending index) item i with in(i).  Only blocks whose partial is {bv, count > 0} hold such
// items, so the partials locate the chunk without another pass over the vector.
// Every thread of the block calls it; returns the item (to every thread), -1 if there is none.
template <class Pred>
__device__ long long kth_in_chunks_if(const Pred& in, long long N, const long long* __restrict__ partials, int nblocks,
                                      float bv, long long k) {
  __shared__ long long shc[BL_THREADS / 32];
  __shared__ int s_blk;
  __shared__ long long s_k, s_out;
  if (threadIdx.x == 0) {
    s_out = -1;
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
  if (blk >= 0) {                                            // block-uniform
    const long long lo = min(N, (long long)blk * BL_CHUNK + (long long)threadIdx.x * BL_IPT), hi = min(N, lo + BL_IPT);
    long long cnt = 0;
    for (long long i = lo; i < hi; ++i) cnt += in(i);
    long long tot;
    long long r = s_k - block_excl_scan(cnt, shc, tot);
    if (r >= 0 && r < cnt) {
      for (long long i = lo; i < hi; ++i)
        if (in(i) && r-- == 0) { s_out = i; break; }
    }
  }
  __syncthreads();
  return s_out;
}
// the unlabeled items whose value equals bv: the chunks of k_extreme_blocks
struct EqualTo {
  const float* __restrict__ v;
  const uint8_t* __restrict__ labeled;
  float bv;
  __device__ __forceinline__ bool operator()(long long i) const { return !labeled[i] && v[i] == bv; }
};
__device__ __forceinline__ long long kth_in_chunks(const float* __restrict__ v, const uint8_t* __restrict__ labeled,
                                                   long long N, const long long* __restrict__ partials, int nblocks,
                                                   float bv, long long k) {
  return kth_in_chunks_if(EqualTo{v, labeled, bv}, N, partials, nblocks, bv, k);
}

// ---------------------------------------------------------------------------------------------------------------
// The selection calls.  Each runs the shard-local pass, then ONE single-CTA kernel that stores this shard's
// record into every peer's mailbox (record channel of xchg.cuh), waits for every peer's record and merges them in rank
// order, so every shard leaves with the same global answer.  Selection merges are exact integer / compare operations;
// the weighted draw adds per-shard fp64 sums in rank order (DESIGN.md §6 (ix)).  With world 1 (x NULL) the kernels
// touch no mailbox and merge their own record only.  A peer that never arrives sets CODA_B200_FLAG_XCHG_TIMEOUT in
// `flags`.
// ---------------------------------------------------------------------------------------------------------------
// the epoch of this kernel's (first) exchange; without peers there is no mailbox and no epoch counter to read (the
// view's epoch pointer is NULL), and the epoch is never used
__device__ __forceinline__ unsigned long long bl_epoch(const XchgView& x) {
  return x.world > 1 ? xch_epoch(x, XCH_REC) : 0ull;
}
// src of rank s at epoch ep: its slot in the local mailbox, or this shard's own stage when there is no exchange
__device__ __forceinline__ const void* bl_rec(const XchgView& x, unsigned long long ep, int s, const void* stage) {
  return x.world > 1 ? (const void*)xch_data(x, XCH_REC, ep, s) : stage;
}
// all threads: stage (16-byte aligned, `bytes` a multiple of 16) to every peer, then wait for theirs -> epoch
__device__ __forceinline__ unsigned long long bl_exchange(const XchgView& x, unsigned long long ep, const void* stage,
                                                          uint32_t bytes, uint32_t* flags) {
  if (x.world <= 1) return ep;
  xch_push(x, XCH_REC, ep, stage, bytes);
  const bool ok = xch_wait(x, XCH_REC, ep);
  if (!ok && threadIdx.x == 0) atomicOr(flags, CODA_B200_FLAG_XCHG_TIMEOUT);
  return ep;
}
// all threads, after every read of epoch ep's records
__device__ __forceinline__ void bl_exchange_done(const XchgView& x, unsigned long long ep) {
  __syncthreads();
  if (x.world > 1) xch_done(x, XCH_REC, ep);
}

// out = {float bits of the global extreme, global count of items equal to it, such items on lower ranks, on this rank}
__global__ void __launch_bounds__(BL_THREADS) k_extreme_xchg(const long long* __restrict__ partials, int nblocks,
                                                            int want_max, XchgView x, long long* __restrict__ out,
                                                            uint32_t* __restrict__ flags) {
  __shared__ __align__(16) long long stage[2];
  if (threadIdx.x == 0) {
    ValCnt t{0.f, 0};
    for (int b = 0; b < nblocks; ++b) vc_merge(t, ValCnt{__uint_as_float((unsigned)partials[2 * b]), partials[2 * b + 1]}, want_max);
    stage[0] = (long long)__float_as_uint(t.v);
    stage[1] = t.n;
  }
  __syncthreads();
  const unsigned long long ep = bl_exchange(x, bl_epoch(x), stage, 16, flags);
  if (threadIdx.x == 0) {
    ValCnt g{0.f, 0};
    for (int s = 0; s < x.world; ++s) {
      const long long* r = reinterpret_cast<const long long*>(bl_rec(x, ep, s, stage));
      vc_merge(g, ValCnt{__uint_as_float((unsigned)r[0]), r[1]}, want_max);
    }
    long long lower = 0, mine = 0;
    for (int s = 0; s <= x.rank; ++s) {
      const long long* r = reinterpret_cast<const long long*>(bl_rec(x, ep, s, stage));
      const long long n = (g.n > 0 && r[1] > 0 && __uint_as_float((unsigned)r[0]) == g.v) ? r[1] : 0;
      if (s < x.rank) lower += n;
      else mine = n;
    }
    out[0] = (long long)__float_as_uint(g.v);
    out[1] = g.n;
    out[2] = lower;
    out[3] = mine;
  }
  bl_exchange_done(x, ep);
}

// the k-th tied item over all shards: the shard whose ties cover k picks its local (k - lower)-th, all get n_offset + it
__device__ __forceinline__ void kth_xchg_body(const float* __restrict__ v, const uint8_t* __restrict__ labeled,
                                              long long N, const long long* __restrict__ partials, int nblocks,
                                              const long long* __restrict__ best, long long k, long long n_offset,
                                              const XchgView& x, long long* __restrict__ out, uint32_t* __restrict__ flags) {
  __shared__ __align__(16) long long stage[2];
  const long long kk = k - best[2];
  long long i = -1;
  if (kk >= 0 && kk < best[3])                                // block-uniform
    i = kth_in_chunks(v, labeled, N, partials, nblocks, __uint_as_float((unsigned)best[0]), kk);
  if (threadIdx.x == 0) {
    stage[0] = i >= 0 ? n_offset + i : -1;
    stage[1] = 0;
  }
  __syncthreads();
  const unsigned long long ep = bl_exchange(x, bl_epoch(x), stage, 16, flags);
  if (threadIdx.x == 0) {
    long long g = -1;
    for (int s = 0; s < x.world; ++s) {
      const long long r = reinterpret_cast<const long long*>(bl_rec(x, ep, s, stage))[0];
      if (r >= 0) g = r;
    }
    out[0] = g;
  }
  bl_exchange_done(x, ep);
}
__global__ void __launch_bounds__(BL_THREADS) k_select_kth_xchg(const float* __restrict__ v, const uint8_t* __restrict__ labeled,
                                                               long long N, const long long* __restrict__ partials,
                                                               int nblocks, const long long* __restrict__ best, long long k,
                                                               long long n_offset, XchgView x, long long* __restrict__ out,
                                                               uint32_t* __restrict__ flags) {
  kth_xchg_body(v, labeled, N, partials, nblocks, best, k, n_offset, x, out, flags);
}
// device loop: k and the stop word from device memory (the stop word is the same on every shard: no exchange is skipped
// on one shard only)
__global__ void __launch_bounds__(BL_THREADS) k_select_kth_dev(const float* __restrict__ v, const uint8_t* __restrict__ labeled,
                                                              long long N, const long long* __restrict__ partials,
                                                              int nblocks, const long long* __restrict__ best,
                                                              const long long* __restrict__ k, const long long* __restrict__ stop,
                                                              long long n_offset, XchgView x, long long* __restrict__ out,
                                                              uint32_t* __restrict__ flags) {
  if (*stop) return;
  kth_xchg_body(v, labeled, N, partials, nblocks, best, *k, n_offset, x, out, flags);
}

// total = {fp64 sum over the shards (rank order) of each shard's block-ordered sum, number of unlabeled items}
__global__ void __launch_bounds__(BL_THREADS) k_wsum_xchg(const double* __restrict__ partials, int nblocks, XchgView x,
                                                         double* __restrict__ total, uint32_t* __restrict__ flags) {
  __shared__ __align__(16) double stage[2];
  if (threadIdx.x == 0) {
    double s = 0.0, c = 0.0;
    for (int b = 0; b < nblocks; ++b) { s += partials[2 * b]; c += partials[2 * b + 1]; }
    stage[0] = s;
    stage[1] = c;
  }
  __syncthreads();
  const unsigned long long ep = bl_exchange(x, bl_epoch(x), stage, 16, flags);
  if (threadIdx.x == 0) {
    double s = 0.0, c = 0.0;
    for (int r = 0; r < x.world; ++r) {
      const double* d = reinterpret_cast<const double*>(bl_rec(x, ep, r, stage));
      s += d[0];
      c += d[1];
    }
    total[0] = s;
    total[1] = c;
  }
  bl_exchange_done(x, ep);
}

// Exchange 1: every shard's {sum of its normalised weights (block order), unlabeled count}; every shard forms the grand
// total in rank order, target = u * grand, and the owner shard (the first one whose running sum passes target, the
// last non-empty one when rounding leaves none).  The owner draws inside its chunks from the lower ranks' running sum
// and position.  Exchange 2: {owner?, position, global item, q bits} -> out on every shard.
__device__ __forceinline__ void wdraw_xchg_body(const float* __restrict__ w, const uint8_t* __restrict__ labeled,
                                                long long N, const double* __restrict__ total,
                                                const double* __restrict__ partials, int nblocks, double u,
                                                long long n_offset, const XchgView& x, long long* __restrict__ out,
                                                uint32_t* __restrict__ flags) {
  __shared__ __align__(16) double stage[2];
  __shared__ __align__(16) long long pick[4];
  __shared__ int s_own;
  __shared__ double s_base, s_pos, s_target;
  if (threadIdx.x == 0) {
    double s = 0.0, c = 0.0;
    for (int b = 0; b < nblocks; ++b) { s += partials[2 * b]; c += partials[2 * b + 1]; }
    stage[0] = s;
    stage[1] = c;
  }
  __syncthreads();
  const unsigned long long ep = bl_exchange(x, bl_epoch(x), stage, 16, flags);
  if (threadIdx.x == 0) {
    double grand = 0.0;
    for (int r = 0; r < x.world; ++r) grand += reinterpret_cast<const double*>(bl_rec(x, ep, r, stage))[0];
    const double target = u * grand;
    double base = 0.0, pos = 0.0;
    int owner = -1, last = -1;
    for (int r = 0; r < x.world; ++r) {
      const double* d = reinterpret_cast<const double*>(bl_rec(x, ep, r, stage));
      if (d[1] == 0.0) continue;
      last = r;
      if (base + d[0] > target) { owner = r; break; }
      base += d[0];
      pos += d[1];
    }
    if (owner < 0 && last >= 0) {                      // target at or beyond the total: the last unlabeled item
      const double* d = reinterpret_cast<const double*>(bl_rec(x, ep, last, stage));
      owner = last;
      base -= d[0];
      pos -= d[1];
    }
    s_own = owner == x.rank;
    s_base = base;
    s_pos = pos;
    s_target = target;
  }
  bl_exchange_done(x, ep);
  long long res[3] = {-1, -1, 0};
  if (s_own) wdraw_in_chunks(w, labeled, N, (float)total[0], partials, nblocks, s_base, s_pos, s_target, res);
  if (threadIdx.x == 0) {
    const bool own = s_own && res[1] >= 0;
    pick[0] = own ? 1 : 0;
    pick[1] = own ? res[0] : -1;
    pick[2] = own ? n_offset + res[1] : -1;
    pick[3] = own ? res[2] : 0;
  }
  __syncthreads();
  const unsigned long long ep2 = bl_exchange(x, ep + 1, pick, 32, flags);
  if (threadIdx.x == 0) {
    out[0] = -1; out[1] = -1; out[2] = 0;
    for (int r = 0; r < x.world; ++r) {
      const long long* p = reinterpret_cast<const long long*>(bl_rec(x, ep2, r, pick));
      if (p[0] == 1) { out[0] = p[1]; out[1] = p[2]; out[2] = p[3]; }
    }
  }
  bl_exchange_done(x, ep2);
}
__global__ void __launch_bounds__(BL_THREADS) k_wdraw_xchg(const float* __restrict__ w, const uint8_t* __restrict__ labeled,
                                                          long long N, const double* __restrict__ total,
                                                          const double* __restrict__ partials, int nblocks, double u,
                                                          long long n_offset, XchgView x, long long* __restrict__ out,
                                                          uint32_t* __restrict__ flags) {
  wdraw_xchg_body(w, labeled, N, total, partials, nblocks, u, n_offset, x, out, flags);
}
__global__ void __launch_bounds__(BL_THREADS) k_wdraw_dev(const float* __restrict__ w, const uint8_t* __restrict__ labeled,
                                                         long long N, const double* __restrict__ total,
                                                         const double* __restrict__ partials, int nblocks,
                                                         const double* __restrict__ u, const long long* __restrict__ stop,
                                                         long long n_offset, XchgView x, long long* __restrict__ out,
                                                         uint32_t* __restrict__ flags) {
  if (*stop) return;
  wdraw_xchg_body(w, labeled, N, total, partials, nblocks, *u, n_offset, x, out, flags);
}

// The owner's `bytes` from src -> dst on every shard (header {owner?, 0, 0, 0} + payload; the others send the header).
__global__ void __launch_bounds__(BL_THREADS) k_owner_share(const unsigned char* __restrict__ src, int bytes, int own,
                                                           unsigned char* __restrict__ dst, XchgView x,
                                                           uint32_t* __restrict__ flags) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  int* hdr = reinterpret_cast<int*>(smem_raw);
  unsigned char* pay = smem_raw + 16;
  const int padded = (int)xch_align16((uint32_t)bytes);
  __shared__ int s_src;
  if (threadIdx.x < 4) hdr[threadIdx.x] = (threadIdx.x == 0 && own) ? 1 : 0;
  for (int i = threadIdx.x; i < padded; i += blockDim.x) pay[i] = (own && i < bytes) ? src[i] : (unsigned char)0;
  __syncthreads();
  const unsigned long long ep = bl_exchange(x, bl_epoch(x), smem_raw, own ? 16u + (uint32_t)padded : 16u, flags);
  if (threadIdx.x == 0) {
    int from = -1;
    for (int s = 0; s < x.world; ++s)
      if (reinterpret_cast<const int*>(bl_rec(x, ep, s, smem_raw))[0] == 1) from = s;
    s_src = from;
  }
  __syncthreads();
  if (s_src >= 0) {
    const unsigned char* p = reinterpret_cast<const unsigned char*>(bl_rec(x, ep, s_src, smem_raw)) + 16;
    for (int i = threadIdx.x; i < bytes; i += blockDim.x) dst[i] = p[i];
  }
  bl_exchange_done(x, ep);
}

static int bl_view(const coda_xchg_t* x, XchgView* v, uint32_t need, const char* what) {
  if (int rc = xchg_view_from(x, v)) return rc;
  CODA_CHECK_ARG(v->world == 1 || need <= v->slot_bytes[XCH_REC], "%s: %u-byte record larger than the mailbox slot", what, need);
  return CODA_B200_OK;
}

extern "C" int coda_b200_select_extreme_xchg(const float* v, const uint8_t* labeled, int64_t N, int want_max,
                                             int64_t* partials, int64_t* out, const coda_xchg_t* x, uint32_t* flags,
                                             coda_stream_t stream) {
  CODA_CHECK_ARG(v && labeled && partials && out && flags, "select_extreme_xchg: null pointer");
  CODA_CHECK_ARG(N >= 1 && N < (1LL << 40), "select_extreme_xchg: bad N=%lld", (long long)N);
  XchgView xv;
  if (int rc = bl_view(x, &xv, 16, "select_extreme_xchg")) return rc;
  const int nb = coda_b200_select_blocks(N);
  k_extreme_blocks<<<nb, BL_THREADS, 0, as_stream(stream)>>>(v, labeled, N, want_max, (long long*)partials);
  CODA_LAUNCH_OK("k_extreme_blocks");
  k_extreme_xchg<<<1, BL_THREADS, 0, as_stream(stream)>>>((const long long*)partials, nb, want_max, xv, (long long*)out,
                                                          flags);
  CODA_LAUNCH_OK("k_extreme_xchg");
  return CODA_B200_OK;
}

extern "C" int coda_b200_select_kth_xchg(const float* v, const uint8_t* labeled, int64_t N, const int64_t* partials,
                                         const int64_t* best, int64_t k, int64_t n_offset, int64_t* out_idx,
                                         const coda_xchg_t* x, uint32_t* flags, coda_stream_t stream) {
  CODA_CHECK_ARG(v && labeled && partials && best && out_idx && flags, "select_kth_xchg: null pointer");
  CODA_CHECK_ARG(N >= 1 && N < (1LL << 40) && k >= 0 && n_offset >= 0, "select_kth_xchg: bad N=%lld k=%lld",
                 (long long)N, (long long)k);
  XchgView xv;
  if (int rc = bl_view(x, &xv, 16, "select_kth_xchg")) return rc;
  k_select_kth_xchg<<<1, BL_THREADS, 0, as_stream(stream)>>>(v, labeled, N, (const long long*)partials,
                                                             coda_b200_select_blocks(N), (const long long*)best, k,
                                                             n_offset, xv, (long long*)out_idx, flags);
  CODA_LAUNCH_OK("k_select_kth_xchg");
  return CODA_B200_OK;
}

extern "C" int coda_b200_weighted_total_xchg(const float* w, const uint8_t* labeled, int64_t N, double* partials,
                                             double* total, const coda_xchg_t* x, uint32_t* flags,
                                             coda_stream_t stream) {
  CODA_CHECK_ARG(w && labeled && partials && total && flags, "weighted_total_xchg: null pointer");
  CODA_CHECK_ARG(N >= 1 && N < (1LL << 40), "weighted_total_xchg: bad N=%lld", (long long)N);
  XchgView xv;
  if (int rc = bl_view(x, &xv, 16, "weighted_total_xchg")) return rc;
  const int nb = coda_b200_select_blocks(N);
  k_wsum_blocks<false><<<nb, BL_THREADS, 0, as_stream(stream)>>>(w, labeled, N, nullptr, partials);
  CODA_LAUNCH_OK("k_wsum_blocks");
  k_wsum_xchg<<<1, BL_THREADS, 0, as_stream(stream)>>>(partials, nb, xv, total, flags);
  CODA_LAUNCH_OK("k_wsum_xchg");
  return CODA_B200_OK;
}

extern "C" int coda_b200_weighted_draw_xchg(const float* w, const uint8_t* labeled, int64_t N, const double* total,
                                            double u, int64_t n_offset, double* partials, int64_t* out,
                                            const coda_xchg_t* x, uint32_t* flags, coda_stream_t stream) {
  CODA_CHECK_ARG(w && labeled && total && partials && out && flags, "weighted_draw_xchg: null pointer");
  CODA_CHECK_ARG(N >= 1 && N < (1LL << 40) && n_offset >= 0, "weighted_draw_xchg: bad N=%lld", (long long)N);
  CODA_CHECK_ARG(u >= 0.0 && u < 1.0, "weighted_draw_xchg: u must be in [0, 1)");
  XchgView xv;
  if (int rc = bl_view(x, &xv, 32, "weighted_draw_xchg")) return rc;
  const int nb = coda_b200_select_blocks(N);
  k_wsum_blocks<true><<<nb, BL_THREADS, 0, as_stream(stream)>>>(w, labeled, N, total, partials);
  CODA_LAUNCH_OK("k_wsum_blocks");
  k_wdraw_xchg<<<1, BL_THREADS, 0, as_stream(stream)>>>(w, labeled, N, total, partials, nb, u, n_offset, xv,
                                                        (long long*)out, flags);
  CODA_LAUNCH_OK("k_wdraw_xchg");
  return CODA_B200_OK;
}

extern "C" int coda_b200_owner_share(const void* src, int bytes, int own, void* dst, const coda_xchg_t* x,
                                     uint32_t* flags, coda_stream_t stream) {
  CODA_CHECK_ARG(dst && flags && (src || !own), "owner_share: null pointer");
  CODA_CHECK_ARG(bytes >= 1 && bytes <= 8192, "owner_share: bad size %d", bytes);
  XchgView xv;
  if (int rc = bl_view(x, &xv, 16u + xch_align16((uint32_t)bytes), "owner_share")) return rc;
  const size_t smem = 16 + xch_align16((uint32_t)bytes);
  k_owner_share<<<1, BL_THREADS, smem, as_stream(stream)>>>((const unsigned char*)src, bytes, own, (unsigned char*)dst,
                                                            xv, flags);
  CODA_LAUNCH_OK("k_owner_share");
  return CODA_B200_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// Host-free loop of the competing selectors (include/coda_b200.h, coda_bl_loop_t).  Per step and shard: the
// selection pass of the method, bl_draw (k or u of the step), the *_dev selection kernel, bl_step.  Every per-step
// scalar is read from the loop words, so one captured graph serves every step.
// ---------------------------------------------------------------------------------------------------------------
extern "C" int coda_b200_select_kth_xchg_dev(const float* v, const uint8_t* labeled, int64_t N, const int64_t* partials,
                                             const int64_t* best, const int64_t* k, const int64_t* stop,
                                             int64_t n_offset, int64_t* out_idx, const coda_xchg_t* x, uint32_t* flags,
                                             coda_stream_t stream) {
  CODA_CHECK_ARG(v && labeled && partials && best && k && stop && out_idx && flags, "select_kth_xchg_dev: null pointer");
  CODA_CHECK_ARG(N >= 1 && N < (1LL << 40) && n_offset >= 0, "select_kth_xchg_dev: bad N=%lld", (long long)N);
  XchgView xv;
  if (int rc = bl_view(x, &xv, 16, "select_kth_xchg_dev")) return rc;
  k_select_kth_dev<<<1, BL_THREADS, 0, as_stream(stream)>>>(v, labeled, N, (const long long*)partials,
                                                            coda_b200_select_blocks(N), (const long long*)best,
                                                            (const long long*)k, (const long long*)stop, n_offset, xv,
                                                            (long long*)out_idx, flags);
  CODA_LAUNCH_OK("k_select_kth_dev");
  return CODA_B200_OK;
}

extern "C" int coda_b200_weighted_draw_xchg_dev(const float* w, const uint8_t* labeled, int64_t N, const double* total,
                                                const double* u, const int64_t* stop, int64_t n_offset, double* partials,
                                                int64_t* out, const coda_xchg_t* x, uint32_t* flags,
                                                coda_stream_t stream) {
  CODA_CHECK_ARG(w && labeled && total && u && stop && partials && out && flags, "weighted_draw_xchg_dev: null pointer");
  CODA_CHECK_ARG(N >= 1 && N < (1LL << 40) && n_offset >= 0, "weighted_draw_xchg_dev: bad N=%lld", (long long)N);
  XchgView xv;
  if (int rc = bl_view(x, &xv, 32, "weighted_draw_xchg_dev")) return rc;
  const int nb = coda_b200_select_blocks(N);
  k_wsum_blocks<true><<<nb, BL_THREADS, 0, as_stream(stream)>>>(w, labeled, N, total, partials);
  CODA_LAUNCH_OK("k_wsum_blocks");
  k_wdraw_dev<<<1, BL_THREADS, 0, as_stream(stream)>>>(w, labeled, N, total, partials, nb, u, (const long long*)stop,
                                                       n_offset, xv, (long long*)out, flags);
  CODA_LAUNCH_OK("k_wdraw_dev");
  return CODA_B200_OK;
}

extern "C" int coda_b200_mp_entropy_dev(const uint16_t* hard, const float* posterior, int H, int64_t N, int C,
                                        double gamma, const uint8_t* labeled, const uint8_t* disagree,
                                        const int64_t* n_disagree, float* ent, coda_stream_t stream) {
  CODA_CHECK_ARG(hard && posterior && labeled && disagree && n_disagree && ent, "mp_entropy_dev: null pointer");
  CODA_CHECK_ARG(H >= 1 && H <= 1024 && N >= 1 && C >= 1, "mp_entropy_dev: bad shape H=%d N=%lld C=%d", H, (long long)N, C);
  CODA_CHECK_ARG(gamma > 0.0, "mp_entropy_dev: gamma must be > 0");
  const int Hp = (H + 31) & ~31;
  const size_t smem = (size_t)2 * H * sizeof(double) + (size_t)(BL_THREADS / 32) * Hp * sizeof(uint16_t);
  long long grid = (N + BL_THREADS / 32 - 1) / (BL_THREADS / 32);
  grid = min(grid, (long long)coda_sm_count() * 8);
  k_mp_entropy<true><<<(unsigned)grid, BL_THREADS, smem, as_stream(stream)>>>(hard, posterior, H, N, C, gamma, labeled,
                                                                               disagree, 0, (const long long*)n_disagree,
                                                                               ent);
  CODA_LAUNCH_OK("k_mp_entropy");
  return CODA_B200_OK;
}

#define BL_STOP_VMA_UNIFORM 1
#define BL_STOP_AT_TOTAL 2
#define BL_STOP_NO_ITEM 3

__global__ void k_bl_draw(const coda_bl_loop_t a) {
  long long* ls = reinterpret_cast<long long*>(a.ls);
  if (ls[2]) return;
  const long long s = ls[1];
  switch (a.method) {
    case CODA_B200_BL_IID:
      ls[3] = (long long)a.pre[s];
      ls[4] = 0;
      break;
    case CODA_B200_BL_UNCERTAINTY:
    case CODA_B200_BL_MODELPICKER: {
      const long long cnt = a.best[1];
      if (cnt < 1) { ls[2] = BL_STOP_NO_ITEM; return; }
      ls[3] = cnt > 1 ? bl_tie_pick(bl_philox(ls[6], ls[0], 0u), cnt) : 0;
      ls[4] = cnt > 1;
      break;
    }
    default: {                                        // ActiveTesting, VMA: the API's checks on the fp32 total
      const float t = (float)a.total[0];
      if (a.method == CODA_B200_BL_VMA ? t < 1e-12f : !(t > 0.f)) {
        ls[2] = a.method == CODA_B200_BL_VMA ? BL_STOP_VMA_UNIFORM : BL_STOP_AT_TOTAL;
        return;
      }
      reinterpret_cast<double*>(ls)[8] = a.pre[s];
      ls[4] = 0;
    }
  }
}

__global__ void __launch_bounds__(BL_THREADS) k_bl_step(const coda_bl_loop_t a, XchgView x) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int H = a.H, nwords = (H + 31) >> 5;
  const uint32_t hrow = xch_align16((uint32_t)H * 2);
  unsigned char* stage = smem_raw;                                   // {owner?, disagree bit, 0, 0} + hard row
  uint16_t* row = reinterpret_cast<uint16_t*>(smem_raw + 16 + hrow);
  double* rv = reinterpret_cast<double*>(smem_raw + 16 + 2 * hrow);  // the value the best model minimises
  __shared__ unsigned tie_w[32];
  __shared__ double s_red[BL_THREADS / 32];
  __shared__ long long s_idx, s_lab;
  __shared__ double s_q, s_min, s_sum;
  __shared__ int s_stop, s_src, s_dis;
  long long* ls = reinterpret_cast<long long*>(a.ls);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const bool lure = a.method == CODA_B200_BL_ACTIVETESTING || a.method == CODA_B200_BL_VMA;
  if (threadIdx.x == 0) {
    s_stop = ls[2] != 0;
    if (!s_stop) {
      const long long idx = lure ? a.pick[1] : a.pick[0];
      if (idx < 0 || idx >= a.n_global) {             // every shard holds the same global pick: all stop together
        ls[2] = BL_STOP_NO_ITEM;
        s_stop = 1;
      } else {
        s_idx = idx;
        s_lab = a.labels[idx];
        s_q = lure ? (double)__uint_as_float((unsigned)a.pick[2])
                   : (a.method == CODA_B200_BL_UNCERTAINTY ? (double)__uint_as_float((unsigned)a.best[0])
                                                           : 1.0 / (double)(a.n_global - ls[0]));
      }
    }
  }
  __syncthreads();
  if (s_stop) return;
  // the owner's hard row (and disagree bit) to every shard
  const long long idx = s_idx, loc = idx - a.n_offset;
  const bool own = loc >= 0 && loc < a.N;
  int* hdr = reinterpret_cast<int*>(stage);
  uint16_t* srow = reinterpret_cast<uint16_t*>(stage + 16);
  if (threadIdx.x < 4)
    hdr[threadIdx.x] = threadIdx.x == 0 ? (int)own : (threadIdx.x == 1 && own && a.disagree ? (int)a.disagree[loc] : 0);
  for (int i = threadIdx.x; i < (int)(hrow >> 1); i += blockDim.x) srow[i] = (own && i < H) ? a.hard[(size_t)loc * H + i] : 0;
  if (own && threadIdx.x == 0) a.labeled[loc] = 1;
  __syncthreads();
  const unsigned long long ep = bl_exchange(x, bl_epoch(x), stage, own ? 16u + hrow : 16u, a.flags);
  if (threadIdx.x == 0) {
    int from = -1;
    for (int s = 0; s < x.world; ++s)
      if (reinterpret_cast<const int*>(bl_rec(x, ep, s, stage))[0] == 1) from = s;
    s_src = from;
    s_dis = from >= 0 ? reinterpret_cast<const int*>(bl_rec(x, ep, from, stage))[1] : 0;
  }
  __syncthreads();
  {
    const uint16_t* src = s_src >= 0 ? reinterpret_cast<const uint16_t*>(
                                           reinterpret_cast<const unsigned char*>(bl_rec(x, ep, s_src, stage)) + 16)
                                     : nullptr;                       // a peer timed out (flag set): no row
    for (int h = threadIdx.x; h < H; h += blockDim.x) row[h] = src ? src[h] : (uint16_t)0xFFFF;
  }
  bl_exchange_done(x, ep);
  // the method's sums
  const long long lab = s_lab, M = ls[0] + 1, slot = ls[5] % a.hist_cap;
  if (lure) {
    // LURE (activetesting.py:61-90) from running fp64 sums: sum_m v_m L_m = S1 + (N - M) S2, with
    // S2 = sum_m L_m a_m / (N - m) and a_m = 1 / ((N - m + 1) q_m) - 1
    const double Ng = (double)a.n_global, m = (double)M;
    const double am = 1.0 / ((Ng - m + 1.0) * s_q) - 1.0;
    const double t = Ng - m > 0.0 ? am / (Ng - m) : 0.0;
    for (int h = threadIdx.x; h < H; h += blockDim.x) {
      const bool L = (long long)row[h] != lab;
      const double s1 = a.s1[h] + (L ? 1.0 : 0.0), s2 = a.s2[h] + (L ? t : 0.0);
      a.s1[h] = s1;
      a.s2[h] = s2;
      if (a.hist_loss) a.hist_loss[(size_t)slot * H + h] = L;
      rv[h] = bl_lure_risk(s1, s2, Ng, m);
    }
  } else if (a.method == CODA_B200_BL_MODELPICKER) {
    // modelpicker.py:89-95: post * gamma^agree / sum (fp32 products, the sum in fp64 in a fixed order, rounded once)
    double part = 0.0;
    for (int h = threadIdx.x; h < H; h += blockDim.x) {
      const bool agree = (long long)row[h] == lab;
      const int c = a.counts[h] + (agree ? 1 : 0);
      a.counts[h] = c;
      const float p = agree ? __fmul_rn(a.post[h], a.gamma) : a.post[h];
      rv[h] = (double)p;
      part += (double)p;
    }
    part = warp_sum(part);
    if (lane == 0) s_red[warp] = part;
    __syncthreads();
    if (threadIdx.x == 0) {
      double t = 0.0;
      for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t += s_red[w];
      s_sum = t;
    }
    __syncthreads();
    const float sf = (float)s_sum;
    for (int h = threadIdx.x; h < H; h += blockDim.x) {
      a.post[h] = __fdiv_rn((float)rv[h], sf);
      rv[h] = -(double)a.counts[h];                        // most correct labels
    }
  } else {                                                 // IID, Uncertainty: the mean loss is count / M
    for (int h = threadIdx.x; h < H; h += blockDim.x) {
      const int c = a.counts[h] + ((long long)row[h] != lab ? 1 : 0);
      a.counts[h] = c;
      rv[h] = (double)c;
    }
  }
  __syncthreads();
  // the best model: the lowest rv, a Philox draw among exact ties
  double mn = INFINITY;
  for (int h = threadIdx.x; h < H; h += blockDim.x) mn = fmin(mn, rv[h]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mn = fmin(mn, __shfl_xor_sync(CODA_FULL, mn, o));
  if (lane == 0) s_red[warp] = mn;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = INFINITY;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t = fmin(t, s_red[w]);
    s_min = t;
  }
  __syncthreads();
  for (int base = 0; base < H; base += blockDim.x) {       // block-uniform trip count
    const int h = base + threadIdx.x;
    const unsigned b = __ballot_sync(CODA_FULL, h < H && rv[h] == s_min);
    if (lane == 0 && (base >> 5) + warp < nwords) tie_w[(base >> 5) + warp] = b;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    int cnt = 0;
    for (int w = 0; w < nwords; ++w) cnt += __popc(tie_w[w]);
    long long j = cnt > 1 ? bl_tie_pick(bl_philox(ls[6], M, 1u), cnt) : 0;
    int best = -1;
    for (int w = 0; w < nwords && best < 0; ++w) {
      unsigned b = tie_w[w];
      const int c = __popc(b);
      if (j < c) {
        for (; j > 0; --j) b &= b - 1;
        best = w * 32 + __ffs(b) - 1;
      } else {
        j -= c;
      }
    }
    a.hist_idx[slot] = idx;
    a.hist_q[slot] = s_q;
    a.hist_tie[slot] = (int)ls[4];
    a.hist_best[slot] = best;
    a.hist_best_tie[slot] = cnt > 1;
    if (a.method == CODA_B200_BL_MODELPICKER && s_dis) ls[7] -= 1;
    ls[0] = M;
    ls[1] += 1;
    ls[5] += 1;
  }
}

static int bl_loop_ok(const coda_bl_loop_t* a, const char* what) {
  CODA_CHECK_ARG(a && a->ls && a->flags, "%s: null pointer", what);
  CODA_CHECK_ARG(a->method >= CODA_B200_BL_IID && a->method <= CODA_B200_BL_MODELPICKER, "%s: bad method %d", what,
                 a->method);
  CODA_CHECK_ARG(a->H >= 1 && a->H <= 1024 && a->N >= 1 && a->n_global >= a->N && a->n_offset >= 0,
                 "%s: bad shape H=%d N=%lld", what, a->H, (long long)a->N);
  return CODA_B200_OK;
}

extern "C" int coda_b200_bl_draw(const coda_bl_loop_t* a, coda_stream_t stream) {
  if (int rc = bl_loop_ok(a, "bl_draw")) return rc;
  const bool lure = a->method == CODA_B200_BL_ACTIVETESTING || a->method == CODA_B200_BL_VMA;
  CODA_CHECK_ARG((a->method == CODA_B200_BL_UNCERTAINTY || a->method == CODA_B200_BL_MODELPICKER || a->pre) &&
                 (!lure || a->total) && (lure || a->best), "bl_draw: null pointer");
  k_bl_draw<<<1, 1, 0, as_stream(stream)>>>(*a);
  CODA_LAUNCH_OK("k_bl_draw");
  return CODA_B200_OK;
}

extern "C" int coda_b200_bl_step(const coda_bl_loop_t* a, const coda_xchg_t* x, coda_stream_t stream) {
  if (int rc = bl_loop_ok(a, "bl_step")) return rc;
  const bool lure = a->method == CODA_B200_BL_ACTIVETESTING || a->method == CODA_B200_BL_VMA;
  const bool mp = a->method == CODA_B200_BL_MODELPICKER;
  CODA_CHECK_ARG(a->hard && a->labeled && a->labels && a->pick && a->best && a->hist_idx && a->hist_q && a->hist_tie &&
                 a->hist_best && a->hist_best_tie && (lure ? (a->s1 && a->s2) : a->counts != nullptr) &&
                 (!mp || (a->post && a->disagree)), "bl_step: null pointer");
  CODA_CHECK_ARG(a->hist_cap >= 1, "bl_step: bad hist_cap");
  const uint32_t hrow = xch_align16((uint32_t)a->H * 2);
  XchgView xv;
  if (int rc = bl_view(x, &xv, 16u + hrow, "bl_step")) return rc;
  const size_t smem = 16 + 2 * (size_t)hrow + (size_t)a->H * sizeof(double);
  k_bl_step<<<1, BL_THREADS, smem, as_stream(stream)>>>(*a, xv);
  CODA_LAUNCH_OK("k_bl_step");
  return CODA_B200_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// CODA's other acquisitions in its host-free loop (include/coda_b200.h, "CODA ablations"): q='uncertainty' and
// q='iid' (coda.py:287-295) and the --prefilter-n subsample (coda.py:215-224).  The candidates are the unlabeled
// items some model disagrees on, all unlabeled items when there are none (coda.py:239): the exact maximum ties of the
// disagreement bits as floats (`cand`) under select_extreme_xchg(want_max = 1).  `pre` holds the host's pre-draws,
// one row of `width` words per step: {n_s the host predicted, then the iid k or the prefilter's sample positions};
// lw[0] is this step's row.
// ---------------------------------------------------------------------------------------------------------------
#define AB_KEY_SHIFT 40                                    // prefilter record key: sample position << 40 | global item

// per-block CODA records from a static score vector, in the layout of the EIG assembly's block records
__global__ void __launch_bounds__(BL_THREADS) k_static_records(const float* __restrict__ score,
                                                              const uint8_t* __restrict__ labeled,
                                                              const uint8_t* __restrict__ disagree, long long N,
                                                              long long n_offset, long long* __restrict__ partials) {
  __shared__ float sv[2][BL_THREADS / 32], sv2[2][BL_THREADS / 32];
  __shared__ long long si[2][BL_THREADS / 32], sc[BL_THREADS / 32];
  Best2 A = best2_empty(), B = best2_empty();
  long long cn = 0;
  for (long long n = (long long)blockIdx.x * BL_THREADS + threadIdx.x; n < N; n += (long long)gridDim.x * BL_THREADS) {
    if (labeled[n]) continue;
    const float v = score[n];
    best2_add(B, v, n_offset + n);
    if (disagree[n]) {
      best2_add(A, v, n_offset + n);
      ++cn;
    }
  }
  best2_warp(A);
  best2_warp(B);
  cn = warp_sum(cn);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) {
    sv[0][warp] = A.v; si[0][warp] = A.i; sv2[0][warp] = A.v2;
    sv[1][warp] = B.v; si[1][warp] = B.i; sv2[1][warp] = B.v2;
    sc[warp] = cn;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    Best2 fa = best2_empty(), fb = best2_empty();
    long long c = 0;
    for (int w = 0; w < BL_THREADS / 32; ++w) {
      best2_merge(fa, Best2{sv[0][w], si[0][w], sv2[0][w]});
      best2_merge(fb, Best2{sv[1][w], si[1][w], sv2[1][w]});
      c += sc[w];
    }
    rec_store(partials + (size_t)blockIdx.x * REC_W, fa, c, fb);
  }
}

// the step's pick -> sel, the history slots and the counters (what step_select writes after its arg-max)
__device__ void abl_commit(const coda_step_t& a, long long g, float q, int tie, long long* lw) {
  const long long k = *a.step_ctr;
  long long loc = -1;
  int t = 0;
  if (g >= 0 && g < (1LL << AB_KEY_SHIFT)) {
    t = (int)a.labels_global[g];                                       // oracle(idx), coda/oracle.py:23-24
    if (t < 0 || t >= a.C) t = 0;
    loc = g - a.n_offset;
    if (loc < 0 || loc >= a.N) loc = -1;
  } else {
    g = -1;
    atomicOr(a.flags, CODA_B200_FLAG_NO_CANDIDATE);
  }
  a.sel[0] = loc;
  a.sel[1] = t;
  if (a.hist_idx && a.hist_cap > 0) {
    const long long slot = k % a.hist_cap;
    a.hist_idx[slot] = g;
    if (a.hist_q) a.hist_q[slot] = q;
    if (a.hist_tie) a.hist_tie[slot] = tie;
  }
  *a.step_ctr = k + 1;
  lw[0] += 1;
}

__global__ void k_abl_draw(const long long* __restrict__ pre, int width, long long* __restrict__ lw) {
  lw[1] = pre[lw[0] * width + 1];
}

// iid: the pick is the k-th candidate (random.choice over the ascending list), q = fp32(1 / n_s)
__global__ void k_abl_commit(const coda_step_t a, const long long* __restrict__ best, const long long* __restrict__ pick,
                             const long long* __restrict__ pre, int width, long long* __restrict__ lw) {
  const long long n = best[1];
  if (n != pre[lw[0] * width]) atomicOr(a.flags, CODA_B200_FLAG_PREDRAW_MISMATCH);
  abl_commit(a, n > 0 ? pick[0] : -1, n > 0 ? (float)(1.0 / (double)n) : 0.f, n > 1 ? 1 : 0, lw);
}

// one warp: the item (local index) of sample position j if this shard holds it, else -1 (warp-uniform)
__device__ __forceinline__ long long pf_item(const float* __restrict__ cand, const uint8_t* __restrict__ labeled,
                                             long long N, const long long* __restrict__ xp, int nxb,
                                             const long long* __restrict__ best, const long long* __restrict__ pre,
                                             int width, int m, const long long* __restrict__ lw, long long j, int lane) {
  const float bv = __uint_as_float((unsigned)best[0]);
  const long long p = j < m ? pre[lw[0] * width + 1 + j] - best[2] : -1;
  long long item = -1;
  if (p >= 0 && p < best[3]) {                                         // warp-uniform
    long long base = 0;
    int blk = -1;
    for (int b0 = 0; b0 < nxb && blk < 0; b0 += 32) {
      const int bb = b0 + lane;
      long long n = 0;
      if (bb < nxb && xp[2 * bb + 1] > 0 && __uint_as_float((unsigned)xp[2 * bb]) == bv) n = xp[2 * bb + 1];
      const long long incl = warp_incl_scan(n, lane);
      const unsigned hit = __ballot_sync(CODA_FULL, base + incl > p);
      if (hit) {
        const int l = __ffs(hit) - 1;
        blk = b0 + l;
        base += __shfl_sync(CODA_FULL, incl - n, l);
      } else {
        base += __shfl_sync(CODA_FULL, incl, 31);
      }
    }
    long long r = p - base;
    if (blk >= 0) {
      const long long lo = (long long)blk * BL_CHUNK, hi = min(N, lo + BL_CHUNK);
      for (long long i0 = lo; i0 < hi; i0 += 32) {
        const long long i = i0 + lane;
        const unsigned bal = __ballot_sync(CODA_FULL, i < hi && !labeled[i] && cand[i] == bv);
        const int pc = __popc(bal);
        if (r < pc) {
          unsigned w = bal;
          for (long long t = 0; t < r; ++t) w &= w - 1;
          item = i0 + __ffs(w) - 1;
          break;
        }
        r -= pc;
      }
    }
  }
  return item;
}

// prefilter: one warp per sample position j.  The position counts the candidates of all shards in ascending index
// order; the shard whose candidates cover it finds the selection chunk from the select_extreme_xchg partials (as
// kth_in_chunks does), then the item inside the chunk with ballots.  Block record {bits(v), key, bits(v2), 0} over
// the block's samples, key = j << 40 | global item: equal values go to the earliest sample position.
__global__ void __launch_bounds__(BL_THREADS) k_prefilter_pick(const float* __restrict__ eig, const float* __restrict__ cand,
                                                              const uint8_t* __restrict__ labeled, long long N,
                                                              long long n_offset, const long long* __restrict__ xp,
                                                              int nxb, const long long* __restrict__ best,
                                                              const long long* __restrict__ pre, int width, int m,
                                                              const long long* __restrict__ lw,
                                                              long long* __restrict__ recs) {
  __shared__ float sv[BL_THREADS / 32], sv2[BL_THREADS / 32];
  __shared__ long long si[BL_THREADS / 32];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long j = (long long)blockIdx.x * (BL_THREADS / 32) + warp;
  Best2 b = best2_empty();
  const long long item = pf_item(cand, labeled, N, xp, nxb, best, pre, width, m, lw, j, lane);
  if (item >= 0) best2_add(b, eig[item], (j << AB_KEY_SHIFT) | (n_offset + item));
  if (lane == 0) { sv[warp] = b.v; si[warp] = b.i; sv2[warp] = b.v2; }
  __syncthreads();
  if (threadIdx.x == 0) {
    Best2 f = best2_empty();
    for (int w = 0; w < BL_THREADS / 32; ++w) best2_merge(f, Best2{sv[w], si[w], sv2[w]});
    long long* r = recs + (size_t)blockIdx.x * 4;
    r[0] = (long long)__float_as_int(f.v); r[1] = f.i; r[2] = (long long)__float_as_int(f.v2); r[3] = 0;
  }
}

// prefilter with sample scoring: one warp per sample position, its local item on this shard (or -1), resolved as
// k_prefilter_pick resolves it
__global__ void __launch_bounds__(BL_THREADS) k_pf_resolve(const float* __restrict__ cand,
                                                          const uint8_t* __restrict__ labeled, long long N,
                                                          const long long* __restrict__ xp, int nxb,
                                                          const long long* __restrict__ best,
                                                          const long long* __restrict__ pre, int width, int m,
                                                          const long long* __restrict__ lw, int32_t* __restrict__ items) {
  const int lane = threadIdx.x & 31;
  const long long j = (long long)blockIdx.x * (BL_THREADS / 32) + (threadIdx.x >> 5);
  const long long item = pf_item(cand, labeled, N, xp, nxb, best, pre, width, m, lw, j, lane);
  if (lane == 0 && j < m) items[j] = (int32_t)item;
}

// one CTA: merge the block records, exchange them (record channel), the global winner -> abl_commit.  The isclose test
// of coda.py:307 over the sample needs only the runner-up value v2.
// DEFER (tie_rule="reference"): a winner with an isclose runner-up is not committed; *pending = 1 and lw[4] = bits(v)
// instead (pf_band / pf_tie_draw finish the step); otherwise *pending = 0.
template <bool DEFER>
__global__ void __launch_bounds__(BL_THREADS) k_prefilter_commit(const coda_step_t a, const long long* __restrict__ recs,
                                                                int nrec, const long long* __restrict__ best,
                                                                const long long* __restrict__ pre, int width,
                                                                long long* __restrict__ lw, XchgView x,
                                                                long long* __restrict__ pending) {
  __shared__ __align__(16) long long stage[4];
  if (threadIdx.x == 0) {
    Best2 f = best2_empty();
    for (int r = 0; r < nrec; ++r)
      best2_merge(f, Best2{__int_as_float((int)recs[4 * r]), recs[4 * r + 1], __int_as_float((int)recs[4 * r + 2])});
    stage[0] = (long long)__float_as_int(f.v); stage[1] = f.i; stage[2] = (long long)__float_as_int(f.v2); stage[3] = 0;
  }
  __syncthreads();
  const unsigned long long ep = bl_exchange(x, bl_epoch(x), stage, 32, a.flags);
  if (threadIdx.x == 0) {
    Best2 g = best2_empty();
    for (int s = 0; s < x.world; ++s) {
      const long long* r = reinterpret_cast<const long long*>(bl_rec(x, ep, s, stage));
      best2_merge(g, Best2{__int_as_float((int)r[0]), r[1], __int_as_float((int)r[2])});
    }
    if (best[1] != pre[lw[0] * width]) atomicOr(a.flags, CODA_B200_FLAG_PREDRAW_MISMATCH);
    const bool valid = g.i != IDX_NONE;
    const int tie = (valid && isclose_best(g.v2, g.v)) ? 1 : 0;
    if constexpr (DEFER) {
      *pending = tie;
      lw[4] = (long long)__float_as_int(g.v);
    }
    if (!DEFER || !tie) abl_commit(a, valid ? (g.i & ((1LL << AB_KEY_SHIFT) - 1)) : -1, valid ? g.v : 0.f, tie, lw);
  }
  bl_exchange_done(x, ep);
}

static int abl_step_ok(const coda_step_t* st, const char* what) {
  CODA_CHECK_ARG(st && st->flags && st->sel && st->step_ctr && st->labels_global && st->N >= 1 && st->C >= 1,
                 "%s: bad step struct", what);
  return CODA_B200_OK;
}

extern "C" int coda_b200_static_records(const float* score, const uint8_t* labeled, const uint8_t* disagree, int64_t N,
                                        int64_t n_offset, int nblocks, int64_t* partials, coda_stream_t stream) {
  CODA_CHECK_ARG(score && labeled && disagree && partials, "static_records: null pointer");
  CODA_CHECK_ARG(N >= 1 && N < (1LL << AB_KEY_SHIFT) && n_offset >= 0 && nblocks >= 1, "static_records: bad N=%lld",
                 (long long)N);
  k_static_records<<<nblocks, BL_THREADS, 0, as_stream(stream)>>>(score, labeled, disagree, N, n_offset,
                                                                  (long long*)partials);
  CODA_LAUNCH_OK("k_static_records");
  return CODA_B200_OK;
}

extern "C" int coda_b200_abl_draw(const int64_t* pre, int width, int64_t* lw, coda_stream_t stream) {
  CODA_CHECK_ARG(pre && lw && width >= 2, "abl_draw: bad arguments");
  k_abl_draw<<<1, 1, 0, as_stream(stream)>>>((const long long*)pre, width, (long long*)lw);
  CODA_LAUNCH_OK("k_abl_draw");
  return CODA_B200_OK;
}

extern "C" int coda_b200_abl_commit(const coda_step_t* st, const int64_t* best, const int64_t* pick, const int64_t* pre,
                                    int width, int64_t* lw, coda_stream_t stream) {
  if (int rc = abl_step_ok(st, "abl_commit")) return rc;
  CODA_CHECK_ARG(best && pick && pre && lw && width >= 1, "abl_commit: bad arguments");
  k_abl_commit<<<1, 1, 0, as_stream(stream)>>>(*st, (const long long*)best, (const long long*)pick,
                                               (const long long*)pre, width, (long long*)lw);
  CODA_LAUNCH_OK("k_abl_commit");
  return CODA_B200_OK;
}

extern "C" int coda_b200_prefilter_blocks(int m) { return (m + BL_THREADS / 32 - 1) / (BL_THREADS / 32); }

extern "C" int coda_b200_prefilter_pick(const float* eig, const float* cand, const uint8_t* labeled, int64_t N,
                                        int64_t n_offset, const int64_t* partials, const int64_t* best,
                                        const int64_t* pre, int width, int m, const int64_t* lw, int64_t* recs,
                                        coda_stream_t stream) {
  CODA_CHECK_ARG(eig && cand && labeled && partials && best && pre && lw && recs, "prefilter_pick: null pointer");
  CODA_CHECK_ARG(N >= 1 && N < (1LL << AB_KEY_SHIFT) && n_offset >= 0 && m >= 1 && m < (1 << 23) && width == m + 1,
                 "prefilter_pick: bad N=%lld m=%d width=%d", (long long)N, m, width);
  k_prefilter_pick<<<coda_b200_prefilter_blocks(m), BL_THREADS, 0, as_stream(stream)>>>(
      eig, cand, labeled, N, n_offset, (const long long*)partials, coda_b200_select_blocks(N), (const long long*)best,
      (const long long*)pre, width, m, (const long long*)lw, (long long*)recs);
  CODA_LAUNCH_OK("k_prefilter_pick");
  return CODA_B200_OK;
}

extern "C" int coda_b200_pf_resolve(const float* cand, const uint8_t* labeled, int64_t N, const int64_t* partials,
                                    const int64_t* best, const int64_t* pre, int width, int m, const int64_t* lw,
                                    int32_t* items, coda_stream_t stream) {
  CODA_CHECK_ARG(cand && labeled && partials && best && pre && lw && items, "pf_resolve: null pointer");
  CODA_CHECK_ARG(N >= 1 && N < (1LL << 31) && m >= 1 && m < (1 << 23) && width == m + 1,
                 "pf_resolve: bad N=%lld m=%d width=%d", (long long)N, m, width);
  k_pf_resolve<<<coda_b200_prefilter_blocks(m), BL_THREADS, 0, as_stream(stream)>>>(
      cand, labeled, N, (const long long*)partials, coda_b200_select_blocks(N), (const long long*)best,
      (const long long*)pre, width, m, (const long long*)lw, items);
  CODA_LAUNCH_OK("k_pf_resolve");
  return CODA_B200_OK;
}

extern "C" int coda_b200_prefilter_commit(const coda_step_t* st, const int64_t* recs, int nrec, const int64_t* best,
                                          const int64_t* pre, int width, int64_t* lw, const coda_xchg_t* x,
                                          coda_stream_t stream) {
  if (int rc = abl_step_ok(st, "prefilter_commit")) return rc;
  CODA_CHECK_ARG(recs && nrec >= 1 && best && pre && lw && width >= 2, "prefilter_commit: bad arguments");
  XchgView xv;
  if (int rc = bl_view(x, &xv, 32, "prefilter_commit")) return rc;
  k_prefilter_commit<false><<<1, BL_THREADS, 0, as_stream(stream)>>>(*st, (const long long*)recs, nrec,
                                                                     (const long long*)best, (const long long*)pre,
                                                                     width, (long long*)lw, xv, nullptr);
  CODA_LAUNCH_OK("k_prefilter_commit");
  return CODA_B200_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// tie_rule="reference" (include/coda_b200.h, "isclose ties from Python's random"): where the reference breaks an
// isclose tie with random.choice (coda.py:306-311), the loop draws the same _randbelow from a device replica of the
// Python generator (pyrandom.cuh) and takes that item.  The deferring select / prefilter commit leave such a step
// pending (lw[3] for the prefilter, any word for the select); the kernels below exit at once on every other step.
// ---------------------------------------------------------------------------------------------------------------
// the isclose band of the global winner among the candidates (the predicate and `useA` fallback of k_ties)
struct TieBand {
  const float* __restrict__ v;
  const uint8_t* __restrict__ labeled;
  const uint8_t* __restrict__ disagree;
  bool useA;
  float bv;
  __device__ __forceinline__ bool operator()(long long i) const {
    return !labeled[i] && (!useA || disagree[i]) && isclose_best(v[i], bv);
  }
};
__device__ __forceinline__ TieBand tie_band_of(const float* v, const uint8_t* labeled, const uint8_t* disagree,
                                               const long long* bestrec) {
  const bool useA = bestrec[2] > 0;                                   // coda.py:239 `or` fallback
  return TieBand{v, labeled, disagree, useA, __int_as_float((int)(useA ? bestrec[0] : bestrec[3]))};
}

// per selection chunk {bits(bv), band items in it}: the partial layout of select_extreme_xchg
__global__ void __launch_bounds__(BL_THREADS) k_tie_band(const float* __restrict__ v, const uint8_t* __restrict__ labeled,
                                                        const uint8_t* __restrict__ disagree, long long N,
                                                        const long long* __restrict__ bestrec,
                                                        const long long* __restrict__ pending,
                                                        long long* __restrict__ partials) {
  if (!*pending) return;
  __shared__ long long sh[BL_THREADS / 32];
  const TieBand in = tie_band_of(v, labeled, disagree, bestrec);
  const long long lo = chunk_lo(N), hi = min(N, lo + BL_IPT);
  long long c = 0;
  for (long long i = lo; i < hi; ++i) c += in(i);
  c = warp_sum(c);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = c;
  __syncthreads();
  if (threadIdx.x == 0) {
    long long t = 0;
    for (int w = 0; w < BL_THREADS / 32; ++w) t += sh[w];
    partials[2 * blockIdx.x] = (long long)__float_as_uint(in.bv);
    partials[2 * blockIdx.x + 1] = t;
  }
}

// one CTA: the shards' band counts (record channel) -> n; r = _randbelow(n) on every replica; the shard holding the
// r-th band item in ascending global order finds it (kth_in_chunks_if); its index and value (second exchange) ->
// abl_commit with hist_tie = 1
__global__ void __launch_bounds__(BL_THREADS) k_tie_draw(const coda_step_t a, const float* __restrict__ v,
                                                        const uint8_t* __restrict__ disagree,
                                                        const long long* __restrict__ partials, int nblocks,
                                                        const long long* __restrict__ pending, uint32_t* __restrict__ rng,
                                                        long long* __restrict__ lw, XchgView x) {
  if (!*pending) return;
  __shared__ __align__(16) long long stage[2];
  __shared__ long long sh[BL_THREADS / 32];
  __shared__ uint32_t mt[PR_N];
  __shared__ long long s_n, s_lower, s_r;
  const TieBand in = tie_band_of(v, a.labeled, disagree, (const long long*)a.bestrec);
  long long c = 0;
  for (int b = threadIdx.x; b < nblocks; b += BL_THREADS) c += partials[2 * b + 1];
  long long mine;
  block_excl_scan(c, sh, mine);
  if (threadIdx.x == 0) { stage[0] = mine; stage[1] = 0; }
  __syncthreads();
  const unsigned long long ep = bl_exchange(x, bl_epoch(x), stage, 16, a.flags);
  if (threadIdx.x == 0) {
    long long n = 0, lower = 0;
    for (int s = 0; s < x.world; ++s) {
      const long long r = reinterpret_cast<const long long*>(bl_rec(x, ep, s, stage))[0];
      if (s < x.rank) lower += r;
      n += r;
    }
    s_n = n;
    s_lower = lower;
  }
  bl_exchange_done(x, ep);
  const int pos = pr_load(rng, mt);
  if (threadIdx.x < 32) {
    PyRand g{mt, pos};
    const long long r = s_n > 0 ? pr_randbelow(g, s_n) : -1;
    if (threadIdx.x == 0) s_r = r;
    pr_store(g, rng);
  }
  __syncthreads();
  const long long k = s_r - s_lower;
  long long i = -1;
  if (s_r >= 0 && k >= 0 && k < mine) i = kth_in_chunks_if(in, a.N, partials, nblocks, in.bv, k);   // block-uniform
  if (threadIdx.x == 0) {
    stage[0] = i >= 0 ? a.n_offset + i : -1;
    stage[1] = i >= 0 ? (long long)__float_as_int(v[i]) : 0;
  }
  __syncthreads();
  const unsigned long long ep2 = bl_exchange(x, ep + 1, stage, 16, a.flags);
  if (threadIdx.x == 0) {
    long long g = -1;
    float q = 0.f;
    for (int s = 0; s < x.world; ++s) {
      const long long* r = reinterpret_cast<const long long*>(bl_rec(x, ep2, s, stage));
      if (r[0] >= 0) { g = r[0]; q = __int_as_float((int)r[1]); }
    }
    abl_commit(a, g, q, 1, lw);
  }
  bl_exchange_done(x, ep2);
}

// prefilter: this step's sample row {n_s, random.sample(range(n_s), m)} into pre row 0, lw[0] = 0 (then prefilter_pick
// as with the host's rows).  n_s <= m means the host predicted a sampled step the device does not see: flagged.
__global__ void __launch_bounds__(32) k_pf_sample(const long long* __restrict__ best, long long* __restrict__ pre, int m,
                                                 long long setsize, uint32_t* __restrict__ rng, int* __restrict__ pool,
                                                 uint32_t* __restrict__ seen, long long* __restrict__ lw,
                                                 uint32_t* __restrict__ flags) {
  __shared__ uint32_t mt[PR_N];
  const long long n = best[1];
  if (threadIdx.x == 0) { pre[0] = n; lw[0] = 0; }
  if (n <= m) {
    if (threadIdx.x == 0) atomicOr(flags, CODA_B200_FLAG_PREDRAW_MISMATCH);
    return;
  }
  PyRand g{mt, pr_load(rng, mt)};
  pr_sample(g, n, m, setsize, pre + 1, pool, seen);
  pr_store(g, rng);
}

// prefilter with sample scoring, a step with n_s <= m candidates (the reference takes them all, coda.py:221-223, and
// draws nothing): pre row 0 = {n_s, 0, 1, ..., n_s - 1, -1, ...} (every candidate, ascending), lw[0] = 0.  No word of
// the generator is used.  n_s > m sets CODA_B200_FLAG_PREDRAW_MISMATCH (the host predicted a step without a sample).
__global__ void __launch_bounds__(BL_THREADS) k_pf_identity(const long long* __restrict__ best, long long* __restrict__ pre,
                                                           int m, long long* __restrict__ lw, uint32_t* __restrict__ flags) {
  const long long n = best[1];
  if (threadIdx.x == 0) {
    pre[0] = n;
    lw[0] = 0;
    if (n > m) atomicOr(flags, CODA_B200_FLAG_PREDRAW_MISMATCH);
  }
  for (int j = threadIdx.x; j < m; j += BL_THREADS) pre[1 + j] = j < n ? j : -1;
}

// prefilter, pending step: band_item[j] = the global item of sample position j if this shard holds it and its EIG is
// isclose to the winner's (lw[4]), else -1
__global__ void __launch_bounds__(BL_THREADS) k_pf_band(const float* __restrict__ eig, const float* __restrict__ cand,
                                                       const uint8_t* __restrict__ labeled, long long N, long long n_offset,
                                                       const long long* __restrict__ xp, int nxb,
                                                       const long long* __restrict__ best,
                                                       const long long* __restrict__ pre, int width, int m,
                                                       const long long* __restrict__ lw,
                                                       const long long* __restrict__ pending,
                                                       long long* __restrict__ band_item) {
  if (!*pending) return;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long j = (long long)blockIdx.x * (BL_THREADS / 32) + warp;
  const long long item = pf_item(cand, labeled, N, xp, nxb, best, pre, width, m, lw, j, lane);
  if (j < m && lane == 0)
    band_item[j] = (item >= 0 && isclose_best(eig[item], __int_as_float((int)lw[4]))) ? n_offset + item : -1;
}

// prefilter, pending step, one CTA: the band as a bitmap over the sample positions, OR-ed over the shards (record
// channel, one slot: m <= 8 * slot bytes), r = _randbelow(band size), the r-th band position in SAMPLE order (the
// reference walks the sample, coda.py:306-311); its holder sends the item and its EIG -> abl_commit, hist_tie = 1
__global__ void __launch_bounds__(BL_THREADS) k_pf_tie_draw(const coda_step_t a, const long long* __restrict__ band_item,
                                                           int m, const long long* __restrict__ pending,
                                                           uint32_t* __restrict__ rng, uint32_t* __restrict__ bits,
                                                           long long* __restrict__ lw, XchgView x) {
  if (!*pending) return;
  __shared__ __align__(16) long long stage[2];
  __shared__ long long sh[BL_THREADS / 32];
  __shared__ uint32_t mt[PR_N];
  __shared__ long long s_r, s_p;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int words = (m + 31) / 32;
  for (int w = warp; w < words; w += BL_THREADS / 32) {
    const int j = w * 32 + lane;
    const unsigned bal = __ballot_sync(CODA_FULL, j < m && band_item[j] >= 0);
    if (lane == 0) bits[w] = bal;
  }
  __syncthreads();
  const unsigned long long ep = bl_epoch(x);
  if (x.world > 1) {
    bl_exchange(x, ep, bits, xch_align16((uint32_t)words * 4u), a.flags);
    for (int w = threadIdx.x; w < words; w += BL_THREADS) {
      uint32_t u = 0;
      for (int s = 0; s < x.world; ++s) u |= reinterpret_cast<const uint32_t*>(xch_data(x, XCH_REC, ep, s))[w];
      bits[w] = u;
    }
    bl_exchange_done(x, ep);
  }
  const int per = (words + BL_THREADS - 1) / BL_THREADS;
  const int w0 = min(words, (int)threadIdx.x * per), w1 = min(words, w0 + per);
  long long c = 0;
  for (int w = w0; w < w1; ++w) c += __popc(bits[w]);
  long long n;
  const long long before = block_excl_scan(c, sh, n);
  const int pos = pr_load(rng, mt);
  if (threadIdx.x < 32) {
    PyRand g{mt, pos};
    const long long r = n > 0 ? pr_randbelow(g, n) : -1;
    if (threadIdx.x == 0) { s_r = r; s_p = -1; }
    pr_store(g, rng);
  }
  __syncthreads();
  long long r = s_r - before;
  if (s_r >= 0 && r >= 0 && r < c) {
    for (int w = w0; w < w1; ++w) {
      unsigned u = bits[w];
      const int pc = __popc(u);
      if (r < pc) {
        for (long long t = 0; t < r; ++t) u &= u - 1;
        s_p = (long long)w * 32 + __ffs(u) - 1;
        break;
      }
      r -= pc;
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    const long long g = s_p >= 0 ? band_item[s_p] : -1;
    stage[0] = g;
    stage[1] = g >= 0 ? (long long)__float_as_int(a.eig[g - a.n_offset]) : 0;
  }
  __syncthreads();
  const unsigned long long ep2 = x.world > 1 ? ep + 1 : 0;
  bl_exchange(x, ep2, stage, 16, a.flags);
  if (threadIdx.x == 0) {
    long long g = -1;
    float q = 0.f;
    for (int s = 0; s < x.world; ++s) {
      const long long* rr = reinterpret_cast<const long long*>(bl_rec(x, ep2, s, stage));
      if (rr[0] >= 0) { g = rr[0]; q = __int_as_float((int)rr[1]); }
    }
    abl_commit(a, g, q, 1, lw);
  }
  bl_exchange_done(x, ep2);
}

// the kernel-level check of pyrandom.cuh: ops [nops][4] = {0, n, -, -}: _randbelow(n) -> 1 output;
// {1, n, m, setsize}: random.sample(range(n), m) -> m outputs; outputs back to back
__global__ void __launch_bounds__(32) k_pyrandom_run(uint32_t* __restrict__ state, const long long* __restrict__ ops,
                                                    int nops, long long* __restrict__ out, int* __restrict__ pool,
                                                    uint32_t* __restrict__ seen) {
  __shared__ uint32_t mt[PR_N];
  PyRand g{mt, pr_load(state, mt)};
  long long o = 0;
  for (int k = 0; k < nops; ++k) {
    const long long* op = ops + 4 * k;
    if (op[0] == 0) {
      const long long r = pr_randbelow(g, op[1]);
      if (threadIdx.x == 0) out[o] = r;
      ++o;
    } else {
      pr_sample(g, op[1], (int)op[2], op[3], out + o, pool, seen);
      o += op[2];
    }
  }
  pr_store(g, state);
}

static int ref_step_ok(const coda_step_t* st, const char* what) {
  if (int rc = abl_step_ok(st, what)) return rc;
  CODA_CHECK_ARG(st->labeled && st->bestrec && st->eig && st->N < (1LL << AB_KEY_SHIFT), "%s: bad step struct", what);
  return CODA_B200_OK;
}

extern "C" int coda_b200_tie_band(const float* v, const uint8_t* labeled, const uint8_t* disagree, int64_t N,
                                  const int64_t* bestrec, const int64_t* pending, int64_t* partials,
                                  coda_stream_t stream) {
  CODA_CHECK_ARG(v && labeled && disagree && bestrec && pending && partials, "tie_band: null pointer");
  CODA_CHECK_ARG(N >= 1 && N < (1LL << AB_KEY_SHIFT), "tie_band: bad N=%lld", (long long)N);
  k_tie_band<<<coda_b200_select_blocks(N), BL_THREADS, 0, as_stream(stream)>>>(
      v, labeled, disagree, N, (const long long*)bestrec, (const long long*)pending, (long long*)partials);
  CODA_LAUNCH_OK("k_tie_band");
  return CODA_B200_OK;
}

extern "C" int coda_b200_tie_draw(const coda_step_t* st, const float* v, const uint8_t* disagree,
                                  const int64_t* partials, const int64_t* pending, uint32_t* rng, int64_t* lw,
                                  const coda_xchg_t* x, coda_stream_t stream) {
  if (int rc = ref_step_ok(st, "tie_draw")) return rc;
  CODA_CHECK_ARG(v && disagree && partials && pending && rng && lw, "tie_draw: null pointer");
  XchgView xv;
  if (int rc = bl_view(x, &xv, 16, "tie_draw")) return rc;
  k_tie_draw<<<1, BL_THREADS, 0, as_stream(stream)>>>(*st, v, disagree, (const long long*)partials,
                                                      coda_b200_select_blocks(st->N), (const long long*)pending, rng,
                                                      (long long*)lw, xv);
  CODA_LAUNCH_OK("k_tie_draw");
  return CODA_B200_OK;
}

extern "C" int coda_b200_pf_sample(const int64_t* best, int64_t* pre, int m, int64_t setsize, uint32_t* rng,
                                   int32_t* pool, uint32_t* seen, int64_t* lw, uint32_t* flags, coda_stream_t stream) {
  CODA_CHECK_ARG(best && pre && rng && pool && seen && lw && flags, "pf_sample: null pointer");
  CODA_CHECK_ARG(m >= 1 && m < (1 << 23) && setsize >= 21, "pf_sample: bad m=%d setsize=%lld", m, (long long)setsize);
  k_pf_sample<<<1, 32, 0, as_stream(stream)>>>((const long long*)best, (long long*)pre, m, setsize, rng, pool, seen,
                                                (long long*)lw, flags);
  CODA_LAUNCH_OK("k_pf_sample");
  return CODA_B200_OK;
}

extern "C" int coda_b200_pf_identity(const int64_t* best, int64_t* pre, int m, int64_t* lw, uint32_t* flags,
                                     coda_stream_t stream) {
  CODA_CHECK_ARG(best && pre && lw && flags && m >= 1, "pf_identity: bad arguments");
  k_pf_identity<<<1, BL_THREADS, 0, as_stream(stream)>>>((const long long*)best, (long long*)pre, m, (long long*)lw,
                                                         flags);
  CODA_LAUNCH_OK("k_pf_identity");
  return CODA_B200_OK;
}

extern "C" int coda_b200_prefilter_commit_defer(const coda_step_t* st, const int64_t* recs, int nrec,
                                                const int64_t* best, const int64_t* pre, int width, int64_t* lw,
                                                int64_t* pending, const coda_xchg_t* x, coda_stream_t stream) {
  if (int rc = abl_step_ok(st, "prefilter_commit_defer")) return rc;
  CODA_CHECK_ARG(recs && nrec >= 1 && best && pre && lw && pending && width >= 2, "prefilter_commit_defer: bad arguments");
  XchgView xv;
  if (int rc = bl_view(x, &xv, 32, "prefilter_commit_defer")) return rc;
  k_prefilter_commit<true><<<1, BL_THREADS, 0, as_stream(stream)>>>(*st, (const long long*)recs, nrec,
                                                                    (const long long*)best, (const long long*)pre,
                                                                    width, (long long*)lw, xv, (long long*)pending);
  CODA_LAUNCH_OK("k_prefilter_commit_defer");
  return CODA_B200_OK;
}

extern "C" int coda_b200_pf_band(const float* eig, const float* cand, const uint8_t* labeled, int64_t N,
                                 int64_t n_offset, const int64_t* partials, const int64_t* best, const int64_t* pre,
                                 int width, int m, const int64_t* lw, const int64_t* pending, int64_t* band_item,
                                 coda_stream_t stream) {
  CODA_CHECK_ARG(eig && cand && labeled && partials && best && pre && lw && pending && band_item, "pf_band: null pointer");
  CODA_CHECK_ARG(N >= 1 && N < (1LL << AB_KEY_SHIFT) && n_offset >= 0 && m >= 1 && m < (1 << 23) && width == m + 1,
                 "pf_band: bad N=%lld m=%d width=%d", (long long)N, m, width);
  k_pf_band<<<coda_b200_prefilter_blocks(m), BL_THREADS, 0, as_stream(stream)>>>(
      eig, cand, labeled, N, n_offset, (const long long*)partials, coda_b200_select_blocks(N), (const long long*)best,
      (const long long*)pre, width, m, (const long long*)lw, (const long long*)pending, (long long*)band_item);
  CODA_LAUNCH_OK("k_pf_band");
  return CODA_B200_OK;
}

extern "C" int coda_b200_pf_tie_max_m(int H) {
  return 8 * (64 + 2 * (int)xch_align16((uint32_t)H * 2));   // the record slot (xchg_layout) as a bitmap
}

extern "C" int coda_b200_pf_tie_draw(const coda_step_t* st, const int64_t* band_item, int m, const int64_t* pending,
                                     uint32_t* rng, uint32_t* bits, int64_t* lw, const coda_xchg_t* x,
                                     coda_stream_t stream) {
  if (int rc = ref_step_ok(st, "pf_tie_draw")) return rc;
  CODA_CHECK_ARG(band_item && pending && rng && bits && lw && m >= 1 && m < (1 << 23), "pf_tie_draw: bad arguments");
  CODA_CHECK_ARG((reinterpret_cast<uintptr_t>(bits) & 15) == 0, "pf_tie_draw: bits must be 16-byte aligned");
  XchgView xv;
  if (int rc = bl_view(x, &xv, 16, "pf_tie_draw")) return rc;
  CODA_CHECK_ARG(xv.world == 1 || m <= coda_b200_pf_tie_max_m(st->H),
                 "pf_tie_draw: prefilter_n=%d above %d, the bitmap one record slot holds at H=%d", m,
                 coda_b200_pf_tie_max_m(st->H), st->H);
  k_pf_tie_draw<<<1, BL_THREADS, 0, as_stream(stream)>>>(*st, (const long long*)band_item, m, (const long long*)pending,
                                                         rng, bits, (long long*)lw, xv);
  CODA_LAUNCH_OK("k_pf_tie_draw");
  return CODA_B200_OK;
}

extern "C" int coda_b200_pyrandom_run(uint32_t* state, const int64_t* ops, int nops, int64_t* out, int32_t* pool,
                                      uint32_t* seen, coda_stream_t stream) {
  CODA_CHECK_ARG(state && ops && out && pool && seen && nops >= 0, "pyrandom_run: bad arguments");
  k_pyrandom_run<<<1, 32, 0, as_stream(stream)>>>(state, (const long long*)ops, nops, (long long*)out, pool, seen);
  CODA_LAUNCH_OK("k_pyrandom_run");
  return CODA_B200_OK;
}

CODA_MODULE_ANCHOR(baselines, k_static_scores)
