// Compact slab: top-K scores per (model, item) + a uniform remainder -- BASELINE.json configs[4] (M=1024, N=4e6,
// C=1000) is 16.4 TB as dense fp32 and cannot exist on 8 x 180 GB; the reference itself cannot run there
// (coda.py:227 materialises a second slab).  The compact form keeps, for every (h, n), the K highest-scoring
// classes (ids[h][n][K] u16, descending; probs[h][n][K] f32) and spreads the remaining mass evenly:
//
//     preds[h][n][c] = probs[h][n][j]                      if c == ids[h][n][j]
//                    = rest(h, n) = (1 - sum_j probs) / (C - K)   otherwise
//
// (24 bytes per (h, n) at K = 4: 98 GB for configs[4]).  Every slab-reading stage of the path has a twin here that
// works from this form and produces what the dense kernel would produce on the densified slab:
//   scan_compact        coda.py:193-194, 217-218 (+ util.py:13-14)   hard predictions, ensemble sums, pseudo labels
//   confusion_compact   coda.py:42       int64 fixed-point sums: bit-identical to the dense kernel on the densified slab
//   pi_full_compact     coda.py:227-229  U[n][c] = sum_h ( rest * rowsum(D[h][c]) + sum_j (p_j - rest) * D[h][c][id_j] )
//   pi_rank1_compact    coda.py:319      rank-1 refresh: preds[h][n][j_h] is a K-way match, no gather
// The class tables, rows, scoring pass and step kernels do not read the slab and are shared with the dense path.
#include "common.cuh"
#include "terms.cuh"

#define CK_MAX 8

template <int K>
__device__ __forceinline__ float compact_rest(const float (&p)[K], float inv_cmk) {
  float s = p[0];
#pragma unroll
  for (int j = 1; j < K; ++j) s += p[j];
  return (1.0f - s) * inv_cmk;
}

// one (model, item) entry: K ids + K scores; K = 4 with aligned arrays is one 8-byte and one 16-byte load
template <int K>
__device__ __forceinline__ void compact_load(const uint16_t* __restrict__ ids, const float* __restrict__ probs, size_t e,
                                             float (&p)[K], int (&id)[K]) {
  if (K == 4 && ((reinterpret_cast<uintptr_t>(ids + e) & 7) == 0) && ((reinterpret_cast<uintptr_t>(probs + e) & 15) == 0)) {
    const uint2 w = __ldg(reinterpret_cast<const uint2*>(ids + e));
    const float4 f = __ldg(reinterpret_cast<const float4*>(probs + e));
    id[0] = w.x & 0xFFFF; id[1] = w.x >> 16; id[2 % K] = w.y & 0xFFFF; id[3 % K] = w.y >> 16;
    p[0] = f.x; p[1 % K] = f.y; p[2 % K] = f.z; p[3 % K] = f.w;
  } else {
#pragma unroll
    for (int j = 0; j < K; ++j) {
      p[j] = __ldg(probs + e + j);
      id[j] = ids[e + j];
    }
  }
}

#define CK_DISPATCH(K, ...)                                    \
  do {                                                         \
    switch (K) {                                               \
      case 1: { constexpr int KK = 1; __VA_ARGS__; } break;           \
      case 2: { constexpr int KK = 2; __VA_ARGS__; } break;           \
      case 3: { constexpr int KK = 3; __VA_ARGS__; } break;           \
      case 4: { constexpr int KK = 4; __VA_ARGS__; } break;           \
      case 8: { constexpr int KK = 8; __VA_ARGS__; } break;           \
      default:                                                 \
        coda_set_error("compact slab: K=%d not instantiated (1, 2, 3, 4, 8)", K); \
        return CODA_B200_EINVAL;                               \
    }                                                          \
  } while (0)

// ---------------------------------------------------------------------------------------
// scan_compact: one thread per item (lanes <-> consecutive items: coalesced entry loads), models in order;
// the item's ensemble row lives in shared memory (row stride padded to an odd word count).
// ---------------------------------------------------------------------------------------
template <int K>
__global__ void __launch_bounds__(256) k_scan_compact(const uint16_t* __restrict__ ids, const float* __restrict__ probs,
                                                      int H, long long N, int C, long long model_stride_e,
                                                      uint16_t* __restrict__ hard, int32_t* __restrict__ pseudo,
                                                      uint8_t* __restrict__ disagree, float* __restrict__ ens_out,
                                                      uint32_t* __restrict__ flags) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int cpad = C | 1;
  float* E = reinterpret_cast<float*>(smem_raw);                 // [blockDim][cpad]
  const long long n = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const bool valid = n < N;
  float* row = E + (size_t)threadIdx.x * cpad;
  for (int c = 0; c < C; ++c) row[c] = 0.f;
  const float inv_cmk = 1.0f / (float)(C - K);
  float rsum = 0.f;
  uint32_t bad = 0;
  int first = -1, diff = 0;
  if (valid) {
    for (int h = 0; h < H; ++h) {
      const size_t e = (size_t)h * model_stride_e + (size_t)n * K;
      float p[K];
      int id[K];
      compact_load<K>(ids, probs, e, p, id);
#pragma unroll
      for (int j = 0; j < K; ++j) {
        if (!isfinite(p[j])) bad |= CODA_B200_FLAG_NONFINITE_INPUT;
        if (p[j] < 0.f || p[j] > 1.0001f || id[j] >= C) bad |= CODA_B200_FLAG_RANGE_INPUT;
      }
      const float r = compact_rest<K>(p, inv_cmk);
      if (r < -1e-6f) bad |= CODA_B200_FLAG_RANGE_INPUT;
      rsum += r;
#pragma unroll
      for (int j = 0; j < K; ++j)
        if (id[j] < C) row[id[j]] += p[j] - r;
      hard[(size_t)n * H + h] = (uint16_t)id[0];               // ids are sorted by score: the first is the argmax
      if (h == 0) first = id[0];
      else diff |= (id[0] != first);
    }
    float bv = -INFINITY;
    int bi = 0;
    const float fH = (float)H;
    for (int c = 0; c < C; ++c) {
      const float v = row[c] + rsum;
      if (ens_out) ens_out[(size_t)n * C + c] = v;
      const float mean = v / fH;                                 // util.py:14 mean(dim=0), then coda.py:194 argmax
      if (mean > bv) { bv = mean; bi = c; }
    }
    pseudo[n] = bi;
    disagree[n] = (uint8_t)(diff ? 1 : 0);
  }
  if (bad) atomicOr(flags, bad);
}

// ---------------------------------------------------------------------------------------
// scan_compact for large C: one warp per item, the item's [C] row in shared memory (one row per warp).  Lane l loads
// the entry of model h0 + l and stages its K (id, p - rest) pairs; the warp then applies models h0, h0 + 1, ... in
// ascending order, lane j < K making the model's j-th add (a model's K ids are distinct: the adds of one model never
// meet).  Every row[c] receives its adds in ascending h with k_scan_compact's arithmetic, and rsum is the same
// ascending fp32 sum, so hard / pseudo / disagree / ens have k_scan_compact's bits.
// ---------------------------------------------------------------------------------------
#define SCW_WARPS 8

template <int K>
__global__ void __launch_bounds__(SCW_WARPS * 32) k_scan_compact_warp(const uint16_t* __restrict__ ids,
                                                                     const float* __restrict__ probs, int H, long long N,
                                                                     int C, long long model_stride_e,
                                                                     uint16_t* __restrict__ hard, int32_t* __restrict__ pseudo,
                                                                     uint8_t* __restrict__ disagree,
                                                                     float* __restrict__ ens_out,
                                                                     uint32_t* __restrict__ flags) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float* row = reinterpret_cast<float*>(smem_raw) + (size_t)warp * C;                                   // [SCW_WARPS][C]
  int2* stg = reinterpret_cast<int2*>(smem_raw + (size_t)SCW_WARPS * C * 4) + (size_t)warp * 32 * K;   // [32][K] per warp
  const long long n = (long long)blockIdx.x * SCW_WARPS + warp;
  if (n >= N) return;                                           // whole warps only: no block-wide barrier below
  for (int c = lane; c < C; c += 32) row[c] = 0.f;
  const float inv_cmk = 1.0f / (float)(C - K);
  float rsum = 0.f;
  uint32_t bad = 0;
  int first = 0;
  bool diff = false;
  for (int h0 = 0; h0 < H; h0 += 32) {
    const int h = h0 + lane;
    float r = 0.f;
    int id0 = 0;
    bool dup = false;
    if (h < H) {
      float p[K];
      int id[K];
      compact_load<K>(ids, probs, (size_t)h * model_stride_e + (size_t)n * K, p, id);
#pragma unroll
      for (int j = 0; j < K; ++j) {
        if (!isfinite(p[j])) bad |= CODA_B200_FLAG_NONFINITE_INPUT;
        if (p[j] < 0.f || p[j] > 1.0001f || id[j] >= C) bad |= CODA_B200_FLAG_RANGE_INPUT;
      }
      r = compact_rest<K>(p, inv_cmk);
      if (r < -1e-6f) bad |= CODA_B200_FLAG_RANGE_INPUT;
#pragma unroll
      for (int j = 0; j < K; ++j) {
        stg[lane * K + j] = make_int2(id[j], __float_as_int(p[j] - r));
#pragma unroll
        for (int i = 0; i < j; ++i) dup |= id[i] == id[j];
      }
      hard[(size_t)n * H + h] = (uint16_t)id[0];               // ids are sorted by score: the first is the argmax
      id0 = id[0];
    }
    if (h0 == 0) first = __shfl_sync(CODA_FULL, id0, 0);
    diff |= __any_sync(CODA_FULL, h < H && id0 != first);
    // a hand-built entry that repeats an id: this chunk's adds go one after another from lane 0, in k_scan_compact's order
    const bool serial = __any_sync(CODA_FULL, dup);
    __syncwarp();                                              // the staged pairs (and, the first time, the zeroed row)
    const int hn = min(32, H - h0);
    for (int k = 0; k < hn; ++k) {
      rsum += __shfl_sync(CODA_FULL, r, k);
      if (!serial && lane < K) {
        const int2 a = stg[k * K + lane];
        if (a.x < C) row[a.x] += __int_as_float(a.y);
      } else if (serial && lane == 0) {
        for (int j = 0; j < K; ++j) {
          const int2 a = stg[k * K + j];
          if (a.x < C) row[a.x] += __int_as_float(a.y);
        }
      }
      __syncwarp();                                            // the next model may add to the same class
    }
  }
  float bv = -INFINITY;
  int bi = INT_MAX;
  const float fH = (float)H;
  for (int c = lane; c < C; c += 32) {
    const float v = row[c] + rsum;
    if (ens_out) ens_out[(size_t)n * C + c] = v;
    const float mean = v / fH;                                 // util.py:14 mean(dim=0), then coda.py:194 argmax
    if (mean > bv) { bv = mean; bi = c; }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {                           // the largest mean, the first class among equal ones
    const float ov = __shfl_xor_sync(CODA_FULL, bv, o);
    const int oi = __shfl_xor_sync(CODA_FULL, bi, o);
    if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
  }
  bad = __reduce_or_sync(CODA_FULL, bad);
  if (lane == 0) {
    pseudo[n] = bi == INT_MAX ? 0 : bi;
    disagree[n] = (uint8_t)(diff ? 1 : 0);
    if (bad) atomicOr(flags, bad);
  }
}

// one thread per item holds a [C] row per thread in shared memory: it runs up to C = 1599 (32-thread blocks), but its
// blocks shrink from C = 200.  On an H100 (H = 64, N = 1e5) the warp kernel is faster from C = 400 at K = 4 and 8 and
// slower at C = 200, K = 8 (BASELINE §9), so it takes over at C = 400.
#define SCAN_WARP_FROM_C 400

// kernel: 0 = chosen by C, 1 = one thread per item (C <= SCAN_THREAD_MAX_C), 2 = one warp per item
extern "C" int coda_b200_scan_compact_kernel(const uint16_t* ids, const float* probs, int64_t model_stride, int H,
                                             int64_t N, int C, int K, uint16_t* hard, int32_t* pseudo,
                                             uint8_t* disagree, float* ens_out, uint32_t* flags, int kernel,
                                             coda_stream_t stream) {
  CODA_CHECK_ARG(ids && probs && hard && pseudo && disagree && flags, "scan_compact: null pointer");
  CODA_CHECK_ARG(K >= 1 && K <= CK_MAX && K < C && H >= 1 && N >= 1, "scan_compact: bad dims (K=%d)", K);
  CODA_CHECK_ARG(C <= 4096, "scan_compact: C=%d too large for the compact path (C <= 4096)", C);
  CODA_CHECK_ARG(kernel >= 0 && kernel <= 2, "scan_compact: bad kernel %d", kernel);
  if (kernel == 0) kernel = C >= SCAN_WARP_FROM_C ? 2 : 1;
  if (kernel == 2) {
    const size_t smem = (size_t)SCW_WARPS * ((size_t)C * 4 + (size_t)32 * K * sizeof(int2));
    const long long grid = (N + SCW_WARPS - 1) / SCW_WARPS;
    CODA_CHECK_ARG(grid < (1LL << 31), "scan_compact: N=%lld too large", (long long)N);
    CK_DISPATCH(K, {
      CODA_CUDA_OK(cudaFuncSetAttribute(k_scan_compact_warp<KK>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
      k_scan_compact_warp<KK><<<(unsigned)grid, SCW_WARPS * 32, smem, as_stream(stream)>>>(
          ids, probs, H, N, C, (long long)model_stride, hard, pseudo, disagree, ens_out, flags);
    });
    CODA_LAUNCH_OK("k_scan_compact_warp");
    return CODA_B200_OK;
  }
  const int cpad = C | 1;
  int threads = 256;
  while (threads > 32 && (size_t)threads * cpad * 4 > 200 * 1024) threads >>= 1;
  const size_t smem = (size_t)threads * cpad * 4;
  CODA_CHECK_ARG(smem <= 200 * 1024, "scan_compact: C=%d too large for one thread per item", C);
  const long long grid = (N + threads - 1) / threads;
  CK_DISPATCH(K, {
    CODA_CUDA_OK(cudaFuncSetAttribute(k_scan_compact<KK>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k_scan_compact<KK><<<(unsigned)grid, threads, smem, as_stream(stream)>>>(ids, probs, H, N, C, (long long)model_stride,
                                                                             hard, pseudo, disagree, ens_out, flags);
  });
  CODA_LAUNCH_OK("k_scan_compact");
  return CODA_B200_OK;
}

extern "C" int coda_b200_scan_compact(const uint16_t* ids, const float* probs, int64_t model_stride, int H, int64_t N,
                                      int C, int K, uint16_t* hard, int32_t* pseudo, uint8_t* disagree, float* ens_out,
                                      uint32_t* flags, coda_stream_t stream) {
  return coda_b200_scan_compact_kernel(ids, probs, model_stride, H, N, C, K, hard, pseudo, disagree, ens_out, flags, 0,
                                       stream);
}

// ---------------------------------------------------------------------------------------
// confusion_compact: conf_fx[h][y][id_j] += fx(p_j) - fx(rest), conf_rest[h][y] += fx(rest)  (y = pseudo label of n).
// conf[h][y][j] of the densified slab == conf_fx[h][y][j] + conf_rest[h][y] exactly (integer sums).
// grid = (item chunks, H); lanes <-> consecutive items.
// ---------------------------------------------------------------------------------------
template <int K>
__global__ void __launch_bounds__(256) k_confusion_compact(const uint16_t* __restrict__ ids, const float* __restrict__ probs,
                                                           const int32_t* __restrict__ pseudo, long long N, int C,
                                                           long long model_stride_e, float fxs,
                                                           unsigned long long* __restrict__ conf_fx,
                                                           unsigned long long* __restrict__ conf_rest) {
  const int h = blockIdx.y;
  const long long n = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= N) return;
  const float inv_cmk = 1.0f / (float)(C - K);
  const size_t e = (size_t)h * model_stride_e + (size_t)n * K;
  float p[K];
  int id[K];
  compact_load<K>(ids, probs, e, p, id);
  const float r = compact_rest<K>(p, inv_cmk);
  const long long fr = to_fx(r, fxs);
  const int y = pseudo[n];
  unsigned long long* tab = conf_fx + ((size_t)h * C + y) * C;
  if (fr) atomicAdd(conf_rest + (size_t)h * C + y, (unsigned long long)fr);
#pragma unroll
  for (int j = 0; j < K; ++j) {
    const long long v = to_fx(p[j], fxs) - fr;
    if (v && id[j] < C) atomicAdd(tab + id[j], (unsigned long long)v);
  }
}

extern "C" int coda_b200_confusion_compact(const uint16_t* ids, const float* probs, int64_t model_stride,
                                           const int32_t* pseudo, int H, int64_t N, int C, int K, int fx_shift,
                                           int64_t* conf_fx, int64_t* conf_rest, coda_stream_t stream) {
  CODA_CHECK_ARG(ids && probs && pseudo && conf_fx && conf_rest, "confusion_compact: null pointer");
  CODA_CHECK_ARG(K >= 1 && K <= CK_MAX && K < C, "confusion_compact: bad K=%d", K);
  CODA_CHECK_ARG(fx_shift >= 8 && fx_shift <= 46, "confusion_compact: bad fx_shift %d", fx_shift);
  dim3 grid((unsigned)((N + 255) / 256), (unsigned)H);
  CK_DISPATCH(K, (k_confusion_compact<KK><<<grid, 256, 0, as_stream(stream)>>>(
                         ids, probs, pseudo, N, C, (long long)model_stride, exp2f((float)fx_shift),
                         reinterpret_cast<unsigned long long*>(conf_fx), reinterpret_cast<unsigned long long*>(conf_rest))));
  CODA_LAUNCH_OK("k_confusion_compact");
  return CODA_B200_OK;
}

// ---------------------------------------------------------------------------------------
// D helpers for pi_full_compact: DT[h][s][c] = D[h][c][s] (the column the top-K entry selects becomes a contiguous
// row) and RS[h][c] = sum_s D[h][c][s].
// ---------------------------------------------------------------------------------------
__global__ void k_transpose_D(const float* __restrict__ D, int C, float* __restrict__ DT) {
  __shared__ float tile[32][33];
  const int h = blockIdx.z;
  const int c0 = blockIdx.y * 32, s0 = blockIdx.x * 32;
  const float* src = D + (size_t)h * C * C;
  float* dst = DT + (size_t)h * C * C;
  for (int r = threadIdx.y; r < 32; r += 8) {
    const int c = c0 + r, s = s0 + threadIdx.x;
    tile[r][threadIdx.x] = (c < C && s < C) ? src[(size_t)c * C + s] : 0.f;
  }
  __syncthreads();
  for (int r = threadIdx.y; r < 32; r += 8) {
    const int s = s0 + r, c = c0 + threadIdx.x;
    if (s < C && c < C) dst[(size_t)s * C + c] = tile[threadIdx.x][r];
  }
}

__global__ void k_rowsum_D(const float* __restrict__ D, long long rows, int C, float* __restrict__ RS) {
  const int lane = threadIdx.x & 31;
  const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const float* src = D + (size_t)row * C;
  float s = 0.f;
  for (int j = lane; j < C; j += 32) s += src[j];
  s = warp_sum(s);
  if (lane == 0) RS[row] = s;
}

// one warp per item, the item's U row in registers (C <= 32 * KCU); models in order.
template <int KCU, int K>
__global__ void __launch_bounds__(256) k_pi_full_compact(const uint16_t* __restrict__ ids, const float* __restrict__ probs,
                                                         int H, long long N, int C, long long model_stride_e,
                                                         const float* __restrict__ DT, const float* __restrict__ RS,
                                                         float* __restrict__ U) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const float inv_cmk = 1.0f / (float)(C - K);
  for (long long n = (long long)blockIdx.x * 8 + warp; n < N; n += (long long)gridDim.x * 8) {
    float u[KCU];
#pragma unroll
    for (int k = 0; k < KCU; ++k) u[k] = 0.f;
    for (int h = 0; h < H; ++h) {
      const size_t e = (size_t)h * model_stride_e + (size_t)n * K;
      float p[K];
      int id[K];
      compact_load<K>(ids, probs, e, p, id);          // broadcast loads (every lane the same address)
      const float r = compact_rest<K>(p, inv_cmk);
      const float* rs = RS + (size_t)h * C;
#pragma unroll
      for (int k = 0; k < KCU; ++k) {
        const int c = lane + 32 * k;
        if (c < C) u[k] = fmaf(r, __ldg(rs + c), u[k]);
      }
#pragma unroll
      for (int j = 0; j < K; ++j) {
        if (id[j] >= C) continue;
        const float w = p[j] - r;
        const float* col = DT + ((size_t)h * C + id[j]) * C;
#pragma unroll
        for (int k = 0; k < KCU; ++k) {
          const int c = lane + 32 * k;
          if (c < C) u[k] = fmaf(w, __ldg(col + c), u[k]);
        }
      }
    }
#pragma unroll
    for (int k = 0; k < KCU; ++k) {
      const int c = lane + 32 * k;
      if (c < C) U[(size_t)n * C + c] = u[k];
    }
  }
}

// C > 1024: the same per-warp body on the class window [c0, c0 + 1024) of blockIdx.y (c0 = 1024 blockIdx.y): the loads
// of a DT row and of RS stay contiguous, and every element gets k_pi_full_compact's fmaf chain over (h, j).
#define PFC_WIN 1024
template <int K>
__global__ void __launch_bounds__(256, 1) k_pi_full_compact_win(const uint16_t* __restrict__ ids, const float* __restrict__ probs,
                                                             int H, long long N, int C, long long model_stride_e,
                                                             const float* __restrict__ DT, const float* __restrict__ RS,
                                                             float* __restrict__ U) {
  constexpr int KCU = PFC_WIN / 32;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int c0 = blockIdx.y * PFC_WIN;
  const float inv_cmk = 1.0f / (float)(C - K);
  for (long long n = (long long)blockIdx.x * 8 + warp; n < N; n += (long long)gridDim.x * 8) {
    float u[KCU];
#pragma unroll
    for (int k = 0; k < KCU; ++k) u[k] = 0.f;
    for (int h = 0; h < H; ++h) {
      const size_t e = (size_t)h * model_stride_e + (size_t)n * K;
      float p[K];
      int id[K];
      compact_load<K>(ids, probs, e, p, id);          // broadcast loads (every lane the same address)
      const float r = compact_rest<K>(p, inv_cmk);
      const float* rs = RS + (size_t)h * C + c0;
#pragma unroll
      for (int k = 0; k < KCU; ++k) {
        const int c = lane + 32 * k;
        if (c0 + c < C) u[k] = fmaf(r, __ldg(rs + c), u[k]);
      }
#pragma unroll
      for (int j = 0; j < K; ++j) {
        if (id[j] >= C) continue;
        const float w = p[j] - r;
        const float* col = DT + ((size_t)h * C + id[j]) * C + c0;
#pragma unroll
        for (int k = 0; k < KCU; ++k) {
          const int c = lane + 32 * k;
          if (c0 + c < C) u[k] = fmaf(w, __ldg(col + c), u[k]);
        }
      }
    }
#pragma unroll
    for (int k = 0; k < KCU; ++k) {
      const int c = lane + 32 * k;
      if (c0 + c < C) U[(size_t)n * C + c0 + c] = u[k];
    }
  }
}

extern "C" int coda_b200_pi_full_compact(const uint16_t* ids, const float* probs, int64_t model_stride, const float* D,
                                         int H, int64_t N, int C, int K, float* DT_scratch, float* RS_scratch, float* U,
                                         coda_stream_t stream) {
  CODA_CHECK_ARG(ids && probs && D && DT_scratch && RS_scratch && U, "pi_full_compact: null pointer");
  CODA_CHECK_ARG(K >= 1 && K <= CK_MAX && K < C && C <= 4096, "pi_full_compact: K=%d C=%d out of range", K, C);
  cudaStream_t st = as_stream(stream);
  dim3 tg((unsigned)((C + 31) / 32), (unsigned)((C + 31) / 32), (unsigned)H), tb(32, 8);
  k_transpose_D<<<tg, tb, 0, st>>>(D, C, DT_scratch);
  CODA_LAUNCH_OK("k_transpose_D");
  const long long rows = (long long)H * C;
  k_rowsum_D<<<(unsigned)((rows + 7) / 8), 256, 0, st>>>(D, rows, C, RS_scratch);
  CODA_LAUNCH_OK("k_rowsum_D");
  int grid = (int)min((long long)(N + 7) / 8, (long long)coda_sm_count() * 8);
  if (grid < 1) grid = 1;
  if (C > PFC_WIN) {
    const dim3 wg((unsigned)grid, (unsigned)((C + PFC_WIN - 1) / PFC_WIN));
    CK_DISPATCH(K, (k_pi_full_compact_win<KK><<<wg, 256, 0, st>>>(ids, probs, H, N, C, (long long)model_stride, DT_scratch,
                                                                  RS_scratch, U)));
    CODA_LAUNCH_OK("k_pi_full_compact_win");
    return CODA_B200_OK;
  }
#define LAUNCH_PFC(KCU) \
  CK_DISPATCH(K, (k_pi_full_compact<KCU, KK><<<grid, 256, 0, st>>>(ids, probs, H, N, C, (long long)model_stride, DT_scratch, RS_scratch, U)))
  if (C <= 32) LAUNCH_PFC(1);
  else if (C <= 64) LAUNCH_PFC(2);
  else if (C <= 128) LAUNCH_PFC(4);
  else if (C <= 256) LAUNCH_PFC(8);
  else if (C <= 512) LAUNCH_PFC(16);
  else LAUNCH_PFC(32);
#undef LAUNCH_PFC
  CODA_LAUNCH_OK("k_pi_full_compact");
  return CODA_B200_OK;
}

// ---------------------------------------------------------------------------------------
// pi_rank1_compact: U[n][t] += lr * sum_h preds[h][n][j_h] from the compact form.  Gather list (built by the step
// kernels with coda_step_t.compact_k > 0): term = {off = model h, sg = +-1, str = class j}: value = K-way match.
// lanes <-> consecutive items (coalesced 8/16-byte entry loads), then the warp walks its 32 rows of U.
// ---------------------------------------------------------------------------------------
// KCU: C <= 32 * KCU keeps the int64 column sums (and one U row) in registers; KCU = 0: any C, shared-memory sums
template <int K, int KCU>
__global__ void __launch_bounds__(256) k_pi_rank1_compact(const uint16_t* __restrict__ ids, const float* __restrict__ probs,
                                                          const float* __restrict__ E, long long N, int C,
                                                          long long model_stride_e, const long long* __restrict__ sel,
                                                          const int32_t* __restrict__ hdr, const R1Term* __restrict__ gterms,
                                                          float lr, float fxs, float* __restrict__ U,
                                                          unsigned long long* __restrict__ pisum_fx,
                                                          uint32_t* __restrict__ flags) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  constexpr int NACC = KCU > 0 ? 8 : 1;                                         // KCU > 0: one [C] per warp; KCU == 0: one
  long long* wacc_all = reinterpret_cast<long long*>(smem_raw);                 // [NACC][C]   for the block
  R1Term* terms = reinterpret_cast<R1Term*>(wacc_all + (size_t)NACC * C);       // [nt]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int t = (int)sel[1];
  const int nt = hdr[0], tp = hdr[1];
  long long* wacc = wacc_all + (size_t)(KCU > 0 ? warp : 0) * C;
  if (KCU > 0)
    for (int c = lane; c < C; c += 32) wacc[c] = 0;
  else
    for (int c = threadIdx.x; c < C; c += blockDim.x) wacc[c] = 0;
  for (int k = threadIdx.x; k < nt; k += blockDim.x) terms[k] = gterms[k];
  __syncthreads();
  const float inv_cmk = 1.0f / (float)(C - K);
  uint32_t bad = 0;
  long long racc[KCU > 0 ? KCU : 1];
#pragma unroll
  for (int k = 0; k < (KCU > 0 ? KCU : 1); ++k) racc[k] = 0;
  for (long long n0 = (long long)blockIdx.x * 256 + warp * 32; n0 < N; n0 += (long long)gridDim.x * 256) {
    const long long n = n0 + lane;
    float d = 0.f;
    if (n < N) {
      if (tp >= 0) d = __ldg(E + (size_t)n * C + tp);
      long long cur = -1;
      float p[K], r = 0.f;
      int id[K];
#pragma unroll
      for (int j = 0; j < K; ++j) { p[j] = 0.f; id[j] = -1; }
      for (int k = 0; k < nt; ++k) {
        const R1Term tm = terms[k];
        if (tm.off != cur) {                         // the two terms of one model share its entry
          cur = tm.off;
          compact_load<K>(ids, probs, (size_t)cur * model_stride_e + (size_t)n * K, p, id);
          r = compact_rest<K>(p, inv_cmk);
        }
        float v = r;
#pragma unroll
        for (int j = 0; j < K; ++j)
          if (id[j] == tm.str) v = p[j];
        d = fmaf(tm.sg, v, d);
      }
    }
    const float dl = lr * d;
    const int rows = (int)min(32LL, N - n0);
    for (int r2 = 0; r2 < rows; ++r2) {
      const float dr = __shfl_sync(CODA_FULL, dl, r2);
      float* urow = U + (size_t)(n0 + r2) * C;
      if (KCU > 0) {
        constexpr int KR = KCU > 0 ? KCU : 1;
        float u[KR];
        float s = 0.f;
        // every load of the row before the one store into it: a store between them orders the later loads behind it
        // (possible alias) and the row costs KR dependent memory round trips instead of one (ncu: 15 us per row)
#pragma unroll
        for (int k = 0; k < KR; ++k) {
          const int c = lane + 32 * k;
          u[k] = c < C ? urow[c] : 0.f;
        }
#pragma unroll
        for (int k = 0; k < KR; ++k) {
          if (lane + 32 * k == t) u[k] += dr;
          s += u[k];
        }
#pragma unroll
        for (int k = 0; k < KR; ++k)
          if (lane + 32 * k == t) urow[t] = u[k];
        s = warp_sum(s);
        if (!isfinite(s)) bad |= CODA_B200_FLAG_NONFINITE_PI;
        const float den = fmaxf(s, 1e-12f);                             // coda.py:230 clamp_(min=1e-12)
        const float rden = 1.0f / den;
#pragma unroll
        for (int k = 0; k < KR; ++k) racc[k] += to_fx(row_quot(u[k], den, rden), fxs);
        continue;
      }
      float s = 0.f, ut = 0.f;
      for (int c = lane; c < C; c += 32) {      // loads only (see above); column t is stored afterwards by its lane
        float u = urow[c];
        if (c == t) {
          u += dr;
          ut = u;
        }
        s += u;
      }
      if (lane == (t & 31)) urow[t] = ut;
      s = warp_sum(s);
      if (!isfinite(s)) bad |= CODA_B200_FLAG_NONFINITE_PI;
      const float den = fmaxf(s, 1e-12f);                               // coda.py:230 clamp_(min=1e-12)
      const float rden = 1.0f / den;
      for (int c = lane; c < C; c += 32)        // column t was rewritten by this lane; integer sums: any order, same bits
        atomicAdd(reinterpret_cast<unsigned long long*>(wacc) + c, (unsigned long long)to_fx(row_quot(urow[c], den, rden), fxs));
    }
  }
  if (KCU > 0) {
#pragma unroll
    for (int k = 0; k < (KCU > 0 ? KCU : 1); ++k) {
      const int c = lane + 32 * k;
      if (c < C) wacc[c] = racc[k];
    }
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    long long s2 = 0;
    for (int w = 0; w < NACC; ++w) s2 += wacc_all[(size_t)w * C + c];
    if (s2) atomicAdd(pisum_fx + c, (unsigned long long)s2);
  }
  if (bad) atomicOr(flags, bad);
}

extern "C" int coda_b200_pi_rank1_compact(const uint16_t* ids, const float* probs, int64_t model_stride, const float* ens,
                                          int H, int64_t N, int C, int K, const int64_t* sel, double lr, int fx_shift,
                                          const int32_t* terms, float* U, int64_t* pisum_fx, uint32_t* flags,
                                          coda_stream_t stream) {
  CODA_CHECK_ARG(ids && probs && sel && terms && U && pisum_fx && flags, "pi_rank1_compact: null pointer");
  CODA_CHECK_ARG(K >= 1 && K <= CK_MAX && K < C && 2 * H <= R1_MAXT, "pi_rank1_compact: bad dims");
  CODA_CHECK_ARG(C <= 4096, "pi_rank1_compact: C=%d too large", C);
  const size_t smem = (size_t)(C <= 1024 ? 8 : 1) * C * 8 + (size_t)2 * H * sizeof(R1Term);   // NACC of the KCU below
  int grid = (int)min((long long)(N + 255) / 256, (long long)coda_sm_count() * 4);
  if (grid < 1) grid = 1;
#define LAUNCH_R1C(KCU)                                                                                                  \
  CK_DISPATCH(K, {                                                                                                       \
    CODA_CUDA_OK(cudaFuncSetAttribute(k_pi_rank1_compact<KK, KCU>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
    k_pi_rank1_compact<KK, KCU><<<grid, 256, smem, as_stream(stream)>>>(                                                  \
        ids, probs, ens, N, C, (long long)model_stride, reinterpret_cast<const long long*>(sel), terms,                  \
        reinterpret_cast<const R1Term*>(terms + 2), (float)lr, exp2f((float)fx_shift), U,                                \
        reinterpret_cast<unsigned long long*>(pisum_fx), flags);                                                         \
  })
  if (C <= 128) LAUNCH_R1C(4);
  else if (C <= 512) LAUNCH_R1C(16);
  else if (C <= 1024) LAUNCH_R1C(32);
  else LAUNCH_R1C(0);
#undef LAUNCH_R1C
  CODA_LAUNCH_OK("k_pi_rank1_compact");
  return CODA_B200_OK;
}

// ---------------------------------------------------------------------------------------
// Inverted index of the compact slab: for every (model h, class c) the items whose top-K list holds c, as
// {item, probs - rest} pairs.  The rank-1 refresh needs sum_h preds[h][n][j_h] for ONE class j_h per model:
//
//     sum_h preds[h][n][j_h] = R[n] + sum_{h : j_h in topK(h, n)} (p_{h,n,j_h} - rest(h, n)),    R[n] = sum_h rest(h, n)
//
// so instead of scanning the whole slab every step (24 bytes per (h, n): 12 GB per shard at configs[4]) a step reads
// the H lists (h, j_h) -- N K / C entries each on average, 16 MB in all -- and scatters them into a per-item int64
// fixed-point accumulator (order-independent, so the result does not depend on how the lists were filled or on the
// shard count), then makes the one pass over U it has to make anyway.  Built once: count -> prefix sums (host
// plumbing) -> fill.  Same bytes as the slab itself (8 per entry).
// ---------------------------------------------------------------------------------------
#define CIDX_ITEMS 4096      // items per CTA and model in the count / fill passes

// counts[h][c] += #{(n, k) : ids[h][n][k] == c}, n in this CTA's chunk (shared-memory histogram first)
__global__ void __launch_bounds__(256) k_cidx_count(const uint16_t* __restrict__ ids, long long model_stride_e, long long N,
                                                    int C, int K, unsigned long long* __restrict__ counts) {
  extern __shared__ int s_hist[];
  const int h = blockIdx.y;
  for (int c = threadIdx.x; c < C; c += blockDim.x) s_hist[c] = 0;
  __syncthreads();
  const long long n0 = (long long)blockIdx.x * CIDX_ITEMS, n1 = min(N, n0 + CIDX_ITEMS);
  const uint16_t* base = ids + (size_t)h * model_stride_e;
  for (long long e = n0 * K + threadIdx.x; e < n1 * K; e += blockDim.x) {
    const int c = base[e];
    if (c < C) atomicAdd(&s_hist[c], 1);
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += blockDim.x)
    if (s_hist[c]) atomicAdd(counts + (size_t)h * C + c, (unsigned long long)s_hist[c]);
}

// second pass: every CTA reserves one contiguous range per class it meets (one global atomic each), then places its
// entries inside those ranges with shared-memory cursors.  ent[pos] = {item, float bits of (p - rest)}.
template <int K>
__global__ void __launch_bounds__(256) k_cidx_fill(const uint16_t* __restrict__ ids, const float* __restrict__ probs,
                                                   long long model_stride_e, long long N, int C,
                                                   unsigned long long* __restrict__ cursor, uint2* __restrict__ ent) {
  extern __shared__ int s_mem[];
  int* s_cnt = s_mem;                                                       // [C] entries of this chunk per class
  int* s_cur = s_mem + C;                                                   // [C] placed so far
  unsigned long long* s_base = reinterpret_cast<unsigned long long*>(s_mem + 2 * C + ((2 * C) & 1));   // [C] reserved range start
  const int h = blockIdx.y;
  for (int c = threadIdx.x; c < C; c += blockDim.x) { s_cnt[c] = 0; s_cur[c] = 0; }
  __syncthreads();
  const long long n0 = (long long)blockIdx.x * CIDX_ITEMS, n1 = min(N, n0 + CIDX_ITEMS);
  const uint16_t* ibase = ids + (size_t)h * model_stride_e;
  for (long long e = n0 * K + threadIdx.x; e < n1 * K; e += blockDim.x) {
    const int c = ibase[e];
    if (c < C) atomicAdd(&s_cnt[c], 1);
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += blockDim.x)
    if (s_cnt[c]) s_base[c] = atomicAdd(cursor + (size_t)h * C + c, (unsigned long long)s_cnt[c]);
  __syncthreads();
  const float inv_cmk = 1.0f / (float)(C - K);
  for (long long n = n0 + threadIdx.x; n < n1; n += blockDim.x) {
    float p[K];
    int id[K];
    compact_load<K>(ids, probs, (size_t)h * model_stride_e + (size_t)n * K, p, id);
    const float r = compact_rest<K>(p, inv_cmk);
#pragma unroll
    for (int j = 0; j < K; ++j) {
      if (id[j] < C) {
        const unsigned long long pos = s_base[id[j]] + (unsigned long long)atomicAdd(&s_cur[id[j]], 1);
        ent[pos] = make_uint2((unsigned)n, __float_as_uint(p[j] - r));
      }
    }
  }
}

// R[n] = sum_h rest(h, n), models in order (one thread per item)
template <int K>
__global__ void __launch_bounds__(256) k_cidx_rest(const uint16_t* __restrict__ ids, const float* __restrict__ probs,
                                                   long long model_stride_e, int H, long long N, int C,
                                                   float* __restrict__ R) {
  const long long n = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= N) return;
  const float inv_cmk = 1.0f / (float)(C - K);
  float s = 0.f;
  for (int h = 0; h < H; ++h) {
    float p[K];
    int id[K];
    compact_load<K>(ids, probs, (size_t)h * model_stride_e + (size_t)n * K, p, id);
    s += compact_rest<K>(p, inv_cmk);
  }
  R[n] = s;
}

extern "C" int coda_b200_compact_index_count(const uint16_t* ids, int64_t model_stride, int H, int64_t N, int C, int K,
                                             int64_t* counts, coda_stream_t stream) {
  CODA_CHECK_ARG(ids && counts, "compact_index_count: null pointer");
  CODA_CHECK_ARG(H >= 1 && N >= 1 && N < (1LL << 32) && K >= 1 && K <= CK_MAX && (size_t)C * 4 <= 160 * 1024,
                 "compact_index_count: bad dims");
  const dim3 grid((unsigned)((N + CIDX_ITEMS - 1) / CIDX_ITEMS), (unsigned)H);
  const size_t smem = (size_t)C * 4;
  CODA_CUDA_OK(cudaFuncSetAttribute(k_cidx_count, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  k_cidx_count<<<grid, 256, smem, as_stream(stream)>>>(ids, (long long)model_stride, N, C, K,
                                                       reinterpret_cast<unsigned long long*>(counts));
  CODA_LAUNCH_OK("k_cidx_count");
  return CODA_B200_OK;
}

extern "C" int coda_b200_compact_index_fill(const uint16_t* ids, const float* probs, int64_t model_stride, int H, int64_t N,
                                            int C, int K, int64_t* cursor, void* entries, float* rest_sum,
                                            coda_stream_t stream) {
  CODA_CHECK_ARG(ids && probs && cursor && entries && rest_sum, "compact_index_fill: null pointer");
  CODA_CHECK_ARG(H >= 1 && N >= 1 && N < (1LL << 32) && K >= 1 && K <= CK_MAX && K < C && (size_t)C * 16 + 8 <= 160 * 1024,
                 "compact_index_fill: bad dims");
  const dim3 grid((unsigned)((N + CIDX_ITEMS - 1) / CIDX_ITEMS), (unsigned)H);
  const size_t smem = (size_t)C * 16 + 8;
  CK_DISPATCH(K, {
    CODA_CUDA_OK(cudaFuncSetAttribute(k_cidx_fill<KK>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k_cidx_fill<KK><<<grid, 256, smem, as_stream(stream)>>>(ids, probs, (long long)model_stride, N, C,
                                                            reinterpret_cast<unsigned long long*>(cursor),
                                                            reinterpret_cast<uint2*>(entries));
    k_cidx_rest<KK><<<(unsigned)((N + 255) / 256), 256, 0, as_stream(stream)>>>(ids, probs, (long long)model_stride, H, N, C,
                                                                                 rest_sum);
  });
  CODA_LAUNCH_OK("k_cidx_fill");
  return CODA_B200_OK;
}

// ---- the rank-1 refresh from the index ------------------------------------------------------------------------
// scatter: CTA (x, h) walks its share of list (h, jvec[h]); delta_fx[n] += (p - rest) in int64 fixed point
__global__ void __launch_bounds__(256) k_r1i_scatter(const long long* __restrict__ off, const uint2* __restrict__ ent,
                                                     const int32_t* __restrict__ jvec, const int32_t* __restrict__ hdr,
                                                     int C, float fxs, unsigned long long* __restrict__ delta) {
  if (hdr[0] == 0 && hdr[1] < 0) return;                      // no label was applied in this step (see apply_label)
  const int h = blockIdx.y;
  const int j = jvec[h];
  const long long lo = off[(size_t)h * C + j], hi = off[(size_t)h * C + j + 1];
  for (long long i = lo + (long long)blockIdx.x * blockDim.x + threadIdx.x; i < hi; i += (long long)gridDim.x * blockDim.x) {
    const uint2 e = __ldg(ent + i);
    atomicAdd(delta + e.x, (unsigned long long)to_fx(__uint_as_float(e.y), fxs));
  }
}

// rows: d = R[n] + delta[n] (then cleared), U[n][t] += lr d, normalise, column sums -- the row walk of k_pi_rank1_compact
template <int KCU>
__global__ void __launch_bounds__(256) k_r1i_rows(const float* __restrict__ R, unsigned long long* __restrict__ delta,
                                                  long long N, int C, const long long* __restrict__ sel,
                                                  const int32_t* __restrict__ hdr, float lr, float inv_fxd, float fxs,
                                                  float* __restrict__ U, unsigned long long* __restrict__ pisum_fx,
                                                  uint32_t* __restrict__ flags) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  constexpr int NACC = KCU > 0 ? 8 : 1;                                         // as in k_pi_rank1_compact
  long long* wacc_all = reinterpret_cast<long long*>(smem_raw);                 // [NACC][C]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int t = (int)sel[1];
  const bool valid = !(hdr[0] == 0 && hdr[1] < 0);
  long long* wacc = wacc_all + (size_t)(KCU > 0 ? warp : 0) * C;
  if (KCU > 0)
    for (int c = lane; c < C; c += 32) wacc[c] = 0;
  else
    for (int c = threadIdx.x; c < C; c += blockDim.x) wacc[c] = 0;
  __syncthreads();
  uint32_t bad = 0;
  long long racc[KCU > 0 ? KCU : 1];
#pragma unroll
  for (int k = 0; k < (KCU > 0 ? KCU : 1); ++k) racc[k] = 0;
  for (long long n0 = (long long)blockIdx.x * 256 + warp * 32; n0 < N; n0 += (long long)gridDim.x * 256) {
    const long long n = n0 + lane;
    float d = 0.f;
    if (n < N && valid) {
      const long long dv = (long long)delta[n];
      if (dv) delta[n] = 0ull;
      d = R[n] + (float)dv * inv_fxd;
    }
    const float dl = lr * d;
    const int rows = (int)min(32LL, N - n0);
    for (int r2 = 0; r2 < rows; ++r2) {
      const float dr = __shfl_sync(CODA_FULL, dl, r2);
      float* urow = U + (size_t)(n0 + r2) * C;
      if (KCU > 0) {
        constexpr int KR = KCU > 0 ? KCU : 1;
        float u[KR];
        float s = 0.f;
        // every load of the row before the one store into it: a store between them orders the later loads behind it
        // (possible alias) and the row costs KR dependent memory round trips instead of one (ncu: 15 us per row)
#pragma unroll
        for (int k = 0; k < KR; ++k) {
          const int c = lane + 32 * k;
          u[k] = c < C ? urow[c] : 0.f;
        }
#pragma unroll
        for (int k = 0; k < KR; ++k) {
          if (lane + 32 * k == t) u[k] += dr;
          s += u[k];
        }
#pragma unroll
        for (int k = 0; k < KR; ++k)
          if (lane + 32 * k == t) urow[t] = u[k];
        s = warp_sum(s);
        if (!isfinite(s)) bad |= CODA_B200_FLAG_NONFINITE_PI;
        const float den = fmaxf(s, 1e-12f);                             // coda.py:230 clamp_(min=1e-12)
        const float rden = 1.0f / den;
#pragma unroll
        for (int k = 0; k < KR; ++k) racc[k] += to_fx(row_quot(u[k], den, rden), fxs);
        continue;
      }
      float s = 0.f, ut = 0.f;
      for (int c = lane; c < C; c += 32) {      // loads only (see above); column t is stored afterwards by its lane
        float u = urow[c];
        if (c == t) {
          u += dr;
          ut = u;
        }
        s += u;
      }
      if (lane == (t & 31)) urow[t] = ut;
      s = warp_sum(s);
      if (!isfinite(s)) bad |= CODA_B200_FLAG_NONFINITE_PI;
      const float den = fmaxf(s, 1e-12f);                               // coda.py:230 clamp_(min=1e-12)
      const float rden = 1.0f / den;
      for (int c = lane; c < C; c += 32)        // column t was rewritten by this lane; integer sums: any order, same bits
        atomicAdd(reinterpret_cast<unsigned long long*>(wacc) + c, (unsigned long long)to_fx(row_quot(urow[c], den, rden), fxs));
    }
  }
  if (KCU > 0) {
#pragma unroll
    for (int k = 0; k < (KCU > 0 ? KCU : 1); ++k) {
      const int c = lane + 32 * k;
      if (c < C) wacc[c] = racc[k];
    }
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    long long s2 = 0;
    for (int w = 0; w < NACC; ++w) s2 += wacc_all[(size_t)w * C + c];
    if (s2) atomicAdd(pisum_fx + c, (unsigned long long)s2);
  }
  if (bad) atomicOr(flags, bad);
}

#define CIDX_FX_SHIFT 40     // |sum_h (p - rest)| <= H <= 2^11: 2^51 at most

extern "C" int coda_b200_pi_rank1_index(const int64_t* offsets, const void* entries, const float* rest_sum,
                                        const int32_t* jvec, int H, int64_t N, int C, const int64_t* sel, double lr,
                                        int fx_shift, const int32_t* terms, int64_t* delta, float* U, int64_t* pisum_fx,
                                        uint32_t* flags, coda_stream_t stream) {
  CODA_CHECK_ARG(offsets && entries && rest_sum && jvec && sel && terms && delta && U && pisum_fx && flags,
                 "pi_rank1_index: null pointer");
  CODA_CHECK_ARG(H >= 1 && H <= 2048 && N >= 1 && C >= 2, "pi_rank1_index: bad dims");
  CODA_CHECK_ARG(C <= 4096, "pi_rank1_index: C=%d too large", C);
  const size_t smem = (size_t)(C <= 1024 ? 8 : 1) * C * 8;                     // NACC of the KCU below
  k_r1i_scatter<<<dim3(8, (unsigned)H), 256, 0, as_stream(stream)>>>(
      reinterpret_cast<const long long*>(offsets), reinterpret_cast<const uint2*>(entries), jvec, terms, C,
      exp2f((float)CIDX_FX_SHIFT), reinterpret_cast<unsigned long long*>(delta));
  CODA_LAUNCH_OK("k_r1i_scatter");
  int grid = (int)min((long long)(N + 255) / 256, (long long)coda_sm_count() * 8);
  if (grid < 1) grid = 1;
#define LAUNCH_R1I(KCU)                                                                                              \
  do {                                                                                                               \
    CODA_CUDA_OK(cudaFuncSetAttribute(k_r1i_rows<KCU>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));     \
    k_r1i_rows<KCU><<<grid, 256, smem, as_stream(stream)>>>(                                                         \
        rest_sum, reinterpret_cast<unsigned long long*>(delta), N, C, reinterpret_cast<const long long*>(sel), terms, \
        (float)lr, exp2f(-(float)CIDX_FX_SHIFT), exp2f((float)fx_shift), U,                                          \
        reinterpret_cast<unsigned long long*>(pisum_fx), flags);                                                     \
  } while (0)
  if (C <= 128) LAUNCH_R1I(4);
  else if (C <= 512) LAUNCH_R1I(16);
  else if (C <= 1024) LAUNCH_R1I(32);
  else LAUNCH_R1I(0);
#undef LAUNCH_R1I
  CODA_LAUNCH_OK("k_r1i_rows");
  return CODA_B200_OK;
}

CODA_MODULE_ANCHOR(compact, k_transpose_D)
