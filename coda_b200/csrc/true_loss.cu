// True losses of a prediction slab held as N-range pieces: per-model counts of items whose arg-max class equals the
// label (coda/oracle.py:9-21 with the accuracy loss of coda/options.py:5-8), one launch per piece.
//
// A CTA takes one model h and R consecutive items of it.  preds[h][n0 .. n0+R) is one contiguous run of R*C elements,
// staged into shared memory with 16-byte loads (scalar head and tail around the aligned body, so any model stride or
// N-range view works), then a group of G lanes reduces each row to its arg-max.  Each CTA adds its count with one
// 64-bit atomic: integer sums, the same for every piece count and launch order.
#include "common.cuh"

#include <limits.h>

#include <algorithm>

#define TL_THREADS 256
#define TL_TILE_BYTES 32768
#define TL_MAX_SMEM (200 * 1024)

// torch.argmax on the device: a NaN beats every number (the first NaN wins), equal values go to the lower index
__device__ __forceinline__ bool tl_better(float v, int i, float bv, int bi) {
  if (isnan(v)) return !isnan(bv) || i < bi;
  if (isnan(bv)) return false;
  return v > bv || (v == bv && i < bi);
}

template <typename T>
__global__ void __launch_bounds__(TL_THREADS) k_true_loss(const T* __restrict__ preds, long long ldh, long long N, int C,
                                                          int R, int G, const long long* __restrict__ labels,
                                                          unsigned long long* __restrict__ counts) {
  extern __shared__ __align__(16) unsigned char tl_smem[];
  __shared__ unsigned int warp_cnt[TL_THREADS / 32];
  const int h = blockIdx.y;
  const long long n0 = (long long)blockIdx.x * R;
  const int tn = (int)min((long long)R, N - n0);
  const T* src = preds + (size_t)h * ldh + (size_t)n0 * C;
  const long long E = (long long)tn * C;
  // element i of the run lives at byte mis + i*sizeof(T) of shared memory, so the aligned body maps onto aligned smem
  const int mis = (int)(reinterpret_cast<uintptr_t>(src) & 15);
  constexpr int V = 16 / sizeof(T);
  const long long head = min(E, (long long)(((16 - mis) & 15) / (int)sizeof(T)));
  const long long nvec = (E - head) / V;
  T* buf = reinterpret_cast<T*>(tl_smem + mis);
  for (long long i = threadIdx.x; i < head; i += TL_THREADS) buf[i] = src[i];
  const uint4* vsrc = reinterpret_cast<const uint4*>(src + head);
  uint4* vdst = reinterpret_cast<uint4*>(buf + head);
  long long k = threadIdx.x;
  for (; k + 3 * TL_THREADS < nvec; k += 4 * TL_THREADS) {   // four 16-byte loads in flight per thread
    const uint4 a = __ldcs(vsrc + k), b = __ldcs(vsrc + k + TL_THREADS);
    const uint4 c = __ldcs(vsrc + k + 2 * TL_THREADS), d = __ldcs(vsrc + k + 3 * TL_THREADS);
    vdst[k] = a; vdst[k + TL_THREADS] = b; vdst[k + 2 * TL_THREADS] = c; vdst[k + 3 * TL_THREADS] = d;
  }
  for (; k < nvec; k += TL_THREADS) vdst[k] = __ldcs(vsrc + k);
  for (long long i = head + nvec * V + threadIdx.x; i < E; i += TL_THREADS) buf[i] = src[i];
  __syncthreads();

  const int lg = threadIdx.x & (G - 1);
  const int grp = threadIdx.x / G, ngrp = TL_THREADS / G;
  unsigned int mine = 0;
  for (int r0 = 0; r0 < tn; r0 += ngrp) {              // block-uniform trip count: every warp shuffles converged
    const int r = r0 + grp;
    float bv = -INFINITY;
    int bi = INT_MAX;
    if (r < tn) {
      const T* row = buf + (size_t)r * C;
      for (int c = lg; c < C; c += G) {
        const float v = slab_f(row[c]);
        if (tl_better(v, c, bv, bi)) { bv = v; bi = c; }
      }
    }
    for (int o = G >> 1; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(CODA_FULL, bv, o);
      const int oi = __shfl_xor_sync(CODA_FULL, bi, o);
      if (tl_better(ov, oi, bv, bi)) { bv = ov; bi = oi; }
    }
    if (lg == 0 && r < tn && __ldg(labels + n0 + r) == (long long)bi) ++mine;
  }
  mine = warp_sum(mine);
  if ((threadIdx.x & 31) == 0) warp_cnt[threadIdx.x >> 5] = mine;
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned int tot = 0;
#pragma unroll
    for (int w = 0; w < TL_THREADS / 32; ++w) tot += warp_cnt[w];
    if (tot) atomicAdd(counts + h, (unsigned long long)tot);
  }
}

template <typename T>
static int true_loss_counts(const T* preds, int64_t model_stride, int H, int64_t N, int C, const int64_t* labels,
                            int64_t* counts, coda_stream_t stream) {
  const size_t row_bytes = (size_t)C * sizeof(T);
  CODA_CHECK_ARG(row_bytes + 16 <= TL_MAX_SMEM, "true_loss_counts: C=%d rows do not fit shared memory", C);
  const long long R = std::max<long long>(1, std::min<long long>(N, TL_TILE_BYTES / (long long)row_bytes));
  int G = 1;                                            // lanes per row: up to 8 elements each, at most a warp
  while (G < 32 && (long long)G * 8 < C) G <<= 1;
  const size_t smem = (size_t)R * row_bytes + 16;
  const long long grid = (N + R - 1) / R;
  CODA_CHECK_ARG(grid < (1LL << 31), "true_loss_counts: N=%lld too large", (long long)N);
  cudaStream_t st = as_stream(stream);
  CODA_CUDA_OK(cudaMemsetAsync(counts, 0, (size_t)H * sizeof(int64_t), st));
  CODA_CUDA_OK(cudaFuncSetAttribute(k_true_loss<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  k_true_loss<T><<<dim3((unsigned)grid, (unsigned)H), TL_THREADS, smem, st>>>(
      preds, (long long)model_stride, (long long)N, C, (int)R, G, reinterpret_cast<const long long*>(labels),
      reinterpret_cast<unsigned long long*>(counts));
  CODA_LAUNCH_OK("k_true_loss");
  return CODA_B200_OK;
}

extern "C" int coda_b200_true_loss_counts(const void* preds, int fmt, int64_t model_stride, int H, int64_t N, int C,
                                          const int64_t* labels, int64_t* counts, coda_stream_t stream) {
  CODA_CHECK_ARG(preds && labels && counts, "true_loss_counts: null pointer");
  CODA_CHECK_ARG(H >= 1 && H <= 65535 && N >= 1 && C >= 1, "true_loss_counts: bad dims H=%d N=%lld C=%d", H,
                 (long long)N, C);
  CODA_CHECK_ARG(H == 1 || model_stride >= N * C, "true_loss_counts: model_stride %lld < N*C",
                 (long long)model_stride);
  return slab_dispatch(fmt, preds, [&](auto p) {
    return true_loss_counts(p, model_stride, H, N, C, labels, counts, stream);
  });
}

CODA_MODULE_ANCHOR(true_loss, k_true_loss<float>)
