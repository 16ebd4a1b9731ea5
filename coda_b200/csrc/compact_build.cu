// Compaction of a dense score slab into the compact top-K form of compact.cu, on the device, and the true losses of a
// compact slab.
//
// compact_build: for every (h, n) row of C scores (fp32 / fp16 / bf16, widened exactly to fp32 at the load) the K
// highest scores in descending order, equal scores by ascending class -- so ids[0] is torch.argmax's first-index
// maximum of the dense row, which is what the dense scan calls the hard prediction.  A group of CB_G = 8 lanes takes a
// row (a warp works on 4 rows at once): the lanes read the row with coalesced loads (class c on lane c % 8 of the
// group), each lane keeps its own K+1 best (score, class) pairs sorted in registers, then K+1 arg-max rounds over the
// group's heads pick the row's K+1 best in order.  The (K+1)-th is the best score the compaction drops.  Eight lanes
// rather than 32 because the rounds, not the loads, bounded a warp-per-row kernel at C <= 1000 (K+1 rounds of 5
// shuffle levels for every row).  Per model two diagnostics are accumulated (one atomic per CTA each):
//   dropped_max[h]   max over the rows of the (K+1)-th score, as the int32 bits of the float (exact for scores >= 0;
//                    the caller starts it at +0.0)
//   flat_rows[h]     rows whose uniform remainder rest = (1 - sum_j probs) * fp32(1 / (C - K)) (compact_rest's fp32
//                    arithmetic) is >= probs[0]: there the densified row's arg-max can be a remainder class
// Input checks are the dense scan's (slab.cu): a non-finite score sets FLAG_NONFINITE_INPUT, one < 0 or > 1.0001 sets
// FLAG_RANGE_INPUT.
#include "common.cuh"

#include <limits.h>

#define CB_THREADS 256
#define CB_G 8                                                   // lanes per row, >= the largest K
#define CB_PASSES 4                                              // row passes per warp
#define CB_ROWS (CB_THREADS / CB_G * CB_PASSES)
#define CB_UNROLL 4

// descending score, then ascending class; -0.0 == 0.0
__device__ __forceinline__ bool cb_better(float v, int c, float bv, int bc) { return v > bv || (v == bv && c < bc); }

template <typename T, int K>
__global__ void __launch_bounds__(CB_THREADS) k_compact_build(const T* __restrict__ src, long long ldh, long long N, int C,
                                                              uint16_t* __restrict__ ids, float* __restrict__ probs,
                                                              long long out_ldh, int* __restrict__ dropped_bits,
                                                              unsigned long long* __restrict__ flat_rows,
                                                              uint32_t* __restrict__ flags) {
  static_assert(K <= CB_G, "one lane of the group writes each kept entry");
  constexpr int L = K + 1;                                      // K kept + the best dropped
  constexpr int RPW = 32 / CB_G;                                // rows of a warp pass
  __shared__ int s_drop[CB_THREADS / 32];
  __shared__ unsigned int s_flat[CB_THREADS / 32];
  const int h = blockIdx.y;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane & (CB_G - 1), grp = lane / CB_G;
  const float inv_cmk = 1.0f / (float)(C - K);
  const T* base = src + (size_t)h * ldh;
  int drop = 0;                                                 // bits of +0.0
  unsigned int flat = 0;
  uint32_t bad = 0;
  const long long r0 = (long long)blockIdx.x * CB_ROWS + (long long)warp * RPW * CB_PASSES;
  for (int pass = 0; pass < CB_PASSES; ++pass) {
    const long long nw = r0 + (long long)pass * RPW;
    if (nw >= N) break;                                         // warp-uniform; a group past N idles through the rounds
    const long long n = nw + grp;
    const bool valid = n < N;
    const T* row = base + (size_t)(valid ? n : nw) * C;
    float tv[L];
    int tc[L];
#pragma unroll
    for (int j = 0; j < L; ++j) { tv[j] = -INFINITY; tc[j] = INT_MAX; }
    for (int c0 = 0; valid && c0 < C; c0 += CB_G * CB_UNROLL) {
      float v[CB_UNROLL];
#pragma unroll
      for (int u = 0; u < CB_UNROLL; ++u) {                     // all loads of the batch in flight before any insert
        const int c = c0 + CB_G * u + g;
        v[u] = c < C ? slab_f(__ldcs(row + c)) : 0.f;
      }
#pragma unroll
      for (int u = 0; u < CB_UNROLL; ++u) {
        const int c = c0 + CB_G * u + g;
        if (c >= C) continue;
        if (!isfinite(v[u])) bad |= CODA_B200_FLAG_NONFINITE_INPUT;
        if (v[u] < 0.f || v[u] > 1.0001f) bad |= CODA_B200_FLAG_RANGE_INPUT;
        if (!cb_better(v[u], c, tv[L - 1], tc[L - 1])) continue;
        float nv = v[u];
        int nc = c;
#pragma unroll
        for (int j = 0; j < L; ++j) {                           // bubble the new pair into place (register-only)
          if (cb_better(nv, nc, tv[j], tc[j])) {
            const float sv = tv[j];
            const int sc = tc[j];
            tv[j] = nv; tc[j] = nc;
            nv = sv; nc = sc;
          }
        }
      }
    }
    float mine_v = 0.f, p0 = 0.f, s = 0.f;
    int mine_c = 0;
#pragma unroll
    for (int r = 0; r < L; ++r) {
      float bv = tv[0];
      int bc = tc[0];
#pragma unroll
      for (int o = CB_G >> 1; o > 0; o >>= 1) {                 // xor offsets < CB_G stay inside the group
        const float ov = __shfl_xor_sync(CODA_FULL, bv, o);
        const int oc = __shfl_xor_sync(CODA_FULL, bc, o);
        if (cb_better(ov, oc, bv, bc)) { bv = ov; bc = oc; }
      }
      if (tc[0] == bc) {                                        // the owner pops its head (classes are lane-unique)
#pragma unroll
        for (int j = 0; j + 1 < L; ++j) { tv[j] = tv[j + 1]; tc[j] = tc[j + 1]; }
        tv[L - 1] = -INFINITY;
        tc[L - 1] = INT_MAX;
      }
      if (r < K) {
        if (g == r) { mine_v = bv; mine_c = bc; }
        if (r == 0) { p0 = bv; s = bv; }
        else s += bv;                                           // compact_rest: left-to-right fp32 sum
      } else if (valid) {
        drop = max(drop, __float_as_int(bv));
      }
    }
    if (valid && g < K) {
      const size_t e = (size_t)h * out_ldh + (size_t)n * K + g;
      ids[e] = (uint16_t)mine_c;
      probs[e] = mine_v;
    }
    const float rest = (1.0f - s) * inv_cmk;
    if (valid && g == 0 && rest >= p0) ++flat;
  }
  bad = __reduce_or_sync(CODA_FULL, bad);
  drop = __reduce_max_sync(CODA_FULL, drop);
  flat = __reduce_add_sync(CODA_FULL, flat);
  if (lane == 0) {
    s_drop[warp] = drop;
    s_flat[warp] = flat;
    if (bad) atomicOr(flags, bad);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    int d = 0;
    unsigned int f = 0;
#pragma unroll
    for (int w = 0; w < CB_THREADS / 32; ++w) { d = max(d, s_drop[w]); f += s_flat[w]; }
    if (d > 0) atomicMax(dropped_bits + h, d);
    if (f) atomicAdd(flat_rows + h, (unsigned long long)f);
  }
}

template <typename T>
static int compact_build(const T* src, int64_t model_stride, int H, int64_t N, int C, int K, uint16_t* ids, float* probs,
                         int64_t out_stride, float* dropped_max, int64_t* flat_rows, uint32_t* flags,
                         coda_stream_t stream) {
  const long long grid = (N + CB_ROWS - 1) / CB_ROWS;
  CODA_CHECK_ARG(grid < (1LL << 31), "compact_build: N=%lld too large", (long long)N);
  const dim3 g((unsigned)grid, (unsigned)H);
  cudaStream_t st = as_stream(stream);
  int* db = reinterpret_cast<int*>(dropped_max);
  unsigned long long* fr = reinterpret_cast<unsigned long long*>(flat_rows);
#define CB_LAUNCH(KK) \
  k_compact_build<T, KK><<<g, CB_THREADS, 0, st>>>(src, (long long)model_stride, (long long)N, C, ids, probs, (long long)out_stride, db, fr, flags)
  switch (K) {
    case 1: CB_LAUNCH(1); break;
    case 2: CB_LAUNCH(2); break;
    case 3: CB_LAUNCH(3); break;
    case 4: CB_LAUNCH(4); break;
    case 8: CB_LAUNCH(8); break;
    default:
      coda_set_error("compact_build: K=%d not instantiated (1, 2, 3, 4, 8)", K);
      return CODA_B200_EINVAL;
  }
#undef CB_LAUNCH
  CODA_LAUNCH_OK("k_compact_build");
  return CODA_B200_OK;
}

extern "C" int coda_b200_compact_build(const void* src, int fmt, int64_t model_stride, int H, int64_t N, int C, int K,
                                       uint16_t* ids, float* probs, int64_t out_stride, float* dropped_max,
                                       int64_t* flat_rows, uint32_t* flags, coda_stream_t stream) {
  CODA_CHECK_ARG(src && ids && probs && dropped_max && flat_rows && flags, "compact_build: null pointer");
  CODA_CHECK_ARG(H >= 1 && H <= 65535 && N >= 1 && C >= 2 && C <= 4096 && K >= 1 && K < C,
                 "compact_build: bad dims H=%d N=%lld C=%d K=%d (1 <= K < C <= 4096)", H, (long long)N, C, K);
  CODA_CHECK_ARG(H == 1 || model_stride >= N * C, "compact_build: model_stride %lld < N*C", (long long)model_stride);
  CODA_CHECK_ARG(H == 1 || out_stride >= N * K, "compact_build: out_stride %lld < N*K", (long long)out_stride);
  return slab_dispatch(fmt, src, [&](auto p) {
    return compact_build(p, model_stride, H, N, C, K, ids, probs, out_stride, dropped_max, flat_rows, flags, stream);
  });
}

// ---- true losses of a compact slab: counts[h] = #{n : ids[h][n][0] == labels[n]} ------------------------------------
// ids[0] is the row's hard prediction (k_scan_compact), and for a slab compacted by k_compact_build torch.argmax's of the
// dense row, so these are the dense slab's accuracy counts.  One thread per item, one 64-bit atomic per CTA.
#define CTL_THREADS 256
#define CTL_ITEMS (CTL_THREADS * 4)

__global__ void __launch_bounds__(CTL_THREADS) k_true_loss_compact(const uint16_t* __restrict__ ids, long long ldh,
                                                                   long long N, int K,
                                                                   const long long* __restrict__ labels,
                                                                   unsigned long long* __restrict__ counts) {
  __shared__ unsigned int warp_cnt[CTL_THREADS / 32];
  const int h = blockIdx.y;
  const long long n0 = (long long)blockIdx.x * CTL_ITEMS;
  const uint16_t* base = ids + (size_t)h * ldh;
  unsigned int mine = 0;
  for (long long n = n0 + threadIdx.x; n < N && n < n0 + CTL_ITEMS; n += CTL_THREADS)
    mine += (long long)__ldg(base + (size_t)n * K) == __ldg(labels + n);
  mine = warp_sum(mine);
  if ((threadIdx.x & 31) == 0) warp_cnt[threadIdx.x >> 5] = mine;
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned int tot = 0;
#pragma unroll
    for (int w = 0; w < CTL_THREADS / 32; ++w) tot += warp_cnt[w];
    if (tot) atomicAdd(counts + h, (unsigned long long)tot);
  }
}

extern "C" int coda_b200_true_loss_counts_compact(const uint16_t* ids, int64_t model_stride, int H, int64_t N, int K,
                                                  const int64_t* labels, int64_t* counts, coda_stream_t stream) {
  CODA_CHECK_ARG(ids && labels && counts, "true_loss_counts_compact: null pointer");
  CODA_CHECK_ARG(H >= 1 && H <= 65535 && N >= 1 && K >= 1, "true_loss_counts_compact: bad dims H=%d N=%lld K=%d", H,
                 (long long)N, K);
  CODA_CHECK_ARG(H == 1 || model_stride >= N * K, "true_loss_counts_compact: model_stride %lld < N*K",
                 (long long)model_stride);
  const long long grid = (N + CTL_ITEMS - 1) / CTL_ITEMS;
  CODA_CHECK_ARG(grid < (1LL << 31), "true_loss_counts_compact: N=%lld too large", (long long)N);
  cudaStream_t st = as_stream(stream);
  CODA_CUDA_OK(cudaMemsetAsync(counts, 0, (size_t)H * sizeof(int64_t), st));
  k_true_loss_compact<<<dim3((unsigned)grid, (unsigned)H), CTL_THREADS, 0, st>>>(
      ids, (long long)model_stride, (long long)N, K, reinterpret_cast<const long long*>(labels),
      reinterpret_cast<unsigned long long*>(counts));
  CODA_LAUNCH_OK("k_true_loss_compact");
  return CODA_B200_OK;
}

CODA_MODULE_ANCHOR(compact_build, k_true_loss_compact)
