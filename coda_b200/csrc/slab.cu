// Slab-streaming kernels of the CODA hot path (HBM-bound passes over the (H, N, C) fp32
// prediction slab) and the Bayesian posterior update.
//
//   scan_slab          reference coda.py:193-194 (ensemble mean -> pseudo labels),
//                      coda.py:217-218, 263, 316 (per-model argmax), coda.py:215-219 (unanimity)
//   confusion_accum    coda.py:42   (einsum 'nc,hnj->hcj' with one-hot pseudo labels)
//   init_dirichlets    coda.py:43, 46-63, 196
//   pi_full            coda.py:227-229 (einsum 'hcs,hns->hnc' summed over h, never materialised)
//   pi_reduce          coda.py:230-233
//   label_row / label_apply / pi_rank1   coda.py:316-319 (posterior update + marginal refresh,
//                      restated as the rank-1 column update it algebraically is)
#include "common.cuh"
#include "terms.cuh"

#include <type_traits>

// ---------------------------------------------------------------------------------------
// scan_slab: one pass over the slab.  CTA = tile of TN points, all H models.
// ---------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(256) k_scan_slab(const T* __restrict__ preds, long long ldh, int H, long long N, int C,
                                                   int TN, uint16_t* __restrict__ hard,
                                                   int32_t* __restrict__ pseudo, uint8_t* __restrict__ disagree,
                                                   float* __restrict__ ens_out, uint32_t* __restrict__ flags) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  float* ens = reinterpret_cast<float*>(smem_raw);                       // [TN][C]
  uint16_t* hard_t = reinterpret_cast<uint16_t*>(ens + (size_t)TN * C);  // [TN][H]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarp = blockDim.x >> 5;
  const long long n0 = (long long)blockIdx.x * TN;
  const int tn = (int)min((long long)TN, N - n0);
  for (int i = threadIdx.x; i < TN * C; i += blockDim.x) ens[i] = 0.f;
  __syncthreads();
  uint32_t bad = 0;
  for (int h = 0; h < H; ++h) {
    const T* base = preds + (size_t)h * ldh + (size_t)n0 * C;
    for (int p = warp; p < tn; p += nwarp) {
      const T* row = base + (size_t)p * C;
      float* erow = ens + (size_t)p * C;
      float bv = -INFINITY;
      int bi = 0x7fffffff;
      for (int c = lane; c < C; c += 32) {
        float v = ldg_f(row + c);
        if (!isfinite(v)) bad |= CODA_B200_FLAG_NONFINITE_INPUT;
        if (v < 0.f || v > 1.0001f) bad |= CODA_B200_FLAG_RANGE_INPUT;
        erow[c] += v;
        if (v > bv) { bv = v; bi = c; }
      }
      warp_argmax(bv, bi);
      if (lane == 0) hard_t[(size_t)p * H + h] = (uint16_t)(bi == 0x7fffffff ? 0 : bi);
    }
  }
  __syncthreads();
  // hard predictions: contiguous [tn][H] block
  {
    uint16_t* dst = hard + (size_t)n0 * H;
    for (int i = threadIdx.x; i < tn * H; i += blockDim.x) dst[i] = hard_t[i];
  }
  if (ens_out) {   // E[n][c] = sum_h preds[h][n][c], reused by pi_rank1's ensemble shortcut
    float* dst = ens_out + (size_t)n0 * C;
    for (int i = threadIdx.x; i < tn * C; i += blockDim.x) dst[i] = ens[i];
  }
  const float fH = (float)H;
  for (int p = warp; p < tn; p += nwarp) {
    const float* erow = ens + (size_t)p * C;
    float bv = -INFINITY;
    int bi = 0x7fffffff;
    for (int c = lane; c < C; c += 32) {
      float v = erow[c] / fH;   // util.py:14 mean(dim=0), then coda.py:194 argmax
      if (v > bv) { bv = v; bi = c; }
    }
    warp_argmax(bv, bi);
    const uint16_t* hr = hard_t + (size_t)p * H;
    const uint16_t h0 = hr[0];
    int diff = 0;
    for (int h = lane; h < H; h += 32) diff |= (hr[h] != h0);
    diff = __any_sync(CODA_FULL, diff);
    if (lane == 0) {
      pseudo[n0 + p] = (bi == 0x7fffffff ? 0 : bi);
      disagree[n0 + p] = (uint8_t)(diff ? 1 : 0);
    }
  }
  if (bad) atomicOr(flags, bad);
}

// Fast path (C <= 128, N*C % 4 == 0): the [TN x C] tile of every model is one contiguous blob, staged into
// shared memory by 1-D bulk TMA (cp.async.bulk + mbarrier) through a SS_ST-deep ring, so HBM reads run ahead
// of the arg-max / ensemble arithmetic.  Each warp owns 4 rows of the tile (ILP over the four shuffle chains);
// the ensemble sums live in registers.
#define SS_TN 32
#define SS_ST 4
template <int KC, typename T>
__global__ void __launch_bounds__(256) k_scan_slab_tma(const T* __restrict__ preds, long long ldh, int H, long long N, int C,
                                                       uint16_t* __restrict__ hard, int32_t* __restrict__ pseudo,
                                                       uint8_t* __restrict__ disagree, float* __restrict__ ens_out,
                                                       uint32_t* __restrict__ flags) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int tile_floats = SS_TN * C;
  const size_t buf_bytes = ((size_t)tile_floats * sizeof(T) + 127) / 128 * 128;
  T* bufs = reinterpret_cast<T*>(smem_raw);                                            // [SS_ST][tile]
  uint16_t* hard_t = reinterpret_cast<uint16_t*>(smem_raw + SS_ST * buf_bytes);         // [SS_TN][H]
  uint64_t* full = reinterpret_cast<uint64_t*>(smem_raw + SS_ST * buf_bytes + (((size_t)SS_TN * H * 2 + 15) / 16) * 16);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long n0 = (long long)blockIdx.x * SS_TN;
  const int tn = (int)min((long long)SS_TN, N - n0);
  const uint32_t bytes = (uint32_t)tn * C * sizeof(T);  // multiple of 16: callers guarantee (tn * C * sizeof(T)) % 16 == 0
  if (threadIdx.x == 0) {
    for (int s = 0; s < SS_ST; ++s) mbar_init(&full[s], 1);
    mbar_fence_init();
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int s = 0; s < SS_ST && s < H; ++s) {
      mbar_expect_tx(&full[s], bytes);
      tma_load_1d(reinterpret_cast<unsigned char*>(bufs) + s * buf_bytes, preds + (size_t)s * ldh + (size_t)n0 * C, bytes, &full[s]);
    }
  }
  float ens[4][KC];
#pragma unroll
  for (int r = 0; r < 4; ++r)
#pragma unroll
    for (int k = 0; k < KC; ++k) ens[r][k] = 0.f;
  uint32_t bad = 0;
  for (int h = 0; h < H; ++h) {
    const int s = h % SS_ST;
    mbar_wait(&full[s], (h / SS_ST) & 1);
    const T* buf = reinterpret_cast<const T*>(reinterpret_cast<const unsigned char*>(bufs) + s * buf_bytes);
    float bv[4];
    int bi[4];
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const int p = warp + 8 * r;
      bv[r] = -INFINITY;
      bi[r] = 0x7fffffff;
      if (p < tn) {
#pragma unroll
        for (int k = 0; k < KC; ++k) {
          const int c = lane + 32 * k;
          if (c < C) {
            const float v = slab_f(buf[p * C + c]);
            if (!isfinite(v)) bad |= CODA_B200_FLAG_NONFINITE_INPUT;
            if (v < 0.f || v > 1.0001f) bad |= CODA_B200_FLAG_RANGE_INPUT;
            ens[r][k] += v;
            if (v > bv[r]) { bv[r] = v; bi[r] = c; }
          }
        }
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        const float ov = __shfl_xor_sync(CODA_FULL, bv[r], o);
        const int oi = __shfl_xor_sync(CODA_FULL, bi[r], o);
        if (ov > bv[r] || (ov == bv[r] && oi < bi[r])) { bv[r] = ov; bi[r] = oi; }
      }
    }
    if (lane == 0) {
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        const int p = warp + 8 * r;
        if (p < tn) hard_t[(size_t)p * H + h] = (uint16_t)(bi[r] == 0x7fffffff ? 0 : bi[r]);
      }
    }
    __syncthreads();                                   // everyone is done with buf[s]
    if (threadIdx.x == 0 && h + SS_ST < H) {
      mbar_expect_tx(&full[s], bytes);
      tma_load_1d(reinterpret_cast<unsigned char*>(bufs) + s * buf_bytes, preds + (size_t)(h + SS_ST) * ldh + (size_t)n0 * C, bytes,
                  &full[s]);
    }
  }
  {
    uint16_t* dst = hard + (size_t)n0 * H;
    for (int i = threadIdx.x; i < tn * H; i += blockDim.x) dst[i] = hard_t[i];
  }
  const float fH = (float)H;
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    const int p = warp + 8 * r;
    if (p >= tn) continue;
    float bv = -INFINITY;
    int bi = 0x7fffffff;
#pragma unroll
    for (int k = 0; k < KC; ++k) {
      const int c = lane + 32 * k;
      if (c < C) {
        if (ens_out) ens_out[(size_t)(n0 + p) * C + c] = ens[r][k];
        const float v = ens[r][k] / fH;              // util.py:14 mean(dim=0), then coda.py:194 argmax
        if (v > bv) { bv = v; bi = c; }
      }
    }
    warp_argmax(bv, bi);
    const uint16_t* hr = hard_t + (size_t)p * H;
    const uint16_t h0 = hr[0];
    int diff = 0;
    for (int h = lane; h < H; h += 32) diff |= (hr[h] != h0);
    diff = __any_sync(CODA_FULL, diff);
    if (lane == 0) {
      pseudo[n0 + p] = (bi == 0x7fffffff ? 0 : bi);
      disagree[n0 + p] = (uint8_t)(diff ? 1 : 0);
    }
  }
  if (bad) atomicOr(flags, bad);
}

template <typename T>
static int scan_slab(const T* preds, int64_t model_stride, int H, int64_t N, int C, uint16_t* hard, int32_t* pseudo,
                     uint8_t* disagree, float* ens_out, uint32_t* flags, coda_stream_t stream) {
  CODA_CHECK_ARG(preds && hard && pseudo && disagree && flags, "scan_slab: null pointer");
  CODA_CHECK_ARG(model_stride >= (int64_t)N * C, "scan_slab: model_stride %lld < N*C", (long long)model_stride);
  const long long ldh = model_stride;
  CODA_CHECK_ARG(H >= 1 && C >= 2 && C <= 65535 && N >= 1, "scan_slab: bad dims H=%d N=%lld C=%d", H, (long long)N, C);
  constexpr int E16 = 16 / sizeof(T);                       // elements per 16 bytes: every bulk copy is whole 16-byte units
  if (C <= 128 && ldh % E16 == 0 && ((long long)SS_TN * C) % E16 == 0 && ((N % SS_TN) * C) % E16 == 0 &&
      (reinterpret_cast<uintptr_t>(preds) & 15) == 0) {
    const size_t buf_bytes = ((size_t)SS_TN * C * sizeof(T) + 127) / 128 * 128;
    const size_t smem = SS_ST * buf_bytes + (((size_t)SS_TN * H * 2 + 15) / 16) * 16 + SS_ST * 8;
    if (smem <= 200 * 1024) {
      const long long grid = (N + SS_TN - 1) / SS_TN;
      cudaStream_t st = as_stream(stream);
#define LAUNCH_SS(KC)                                                                                             \
  do {                                                                                                            \
    CODA_CUDA_OK(cudaFuncSetAttribute(k_scan_slab_tma<KC, T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
    k_scan_slab_tma<KC, T><<<(unsigned)grid, 256, smem, st>>>(preds, ldh, H, N, C, hard, pseudo, disagree, ens_out, flags); \
  } while (0)
      if (C <= 32) LAUNCH_SS(1);
      else if (C <= 64) LAUNCH_SS(2);
      else if (C <= 96) LAUNCH_SS(3);
      else LAUNCH_SS(4);
#undef LAUNCH_SS
      CODA_LAUNCH_OK("k_scan_slab_tma");
      return CODA_B200_OK;
    }
  }
  int TN = 32;
  size_t need;
  while (true) {
    need = (size_t)TN * C * 4 + (size_t)TN * H * 2;
    if (need <= 200 * 1024 || TN == 1) break;
    TN >>= 1;
  }
  CODA_CHECK_ARG(need <= 200 * 1024, "scan_slab: H=%d C=%d does not fit shared memory", H, C);
  CODA_CUDA_OK(cudaFuncSetAttribute(k_scan_slab<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)need));
  long long grid = (N + TN - 1) / TN;
  k_scan_slab<T><<<(unsigned)grid, 256, need, as_stream(stream)>>>(preds, ldh, H, N, C, TN, hard, pseudo, disagree, ens_out, flags);
  CODA_LAUNCH_OK("k_scan_slab");
  return CODA_B200_OK;
}

extern "C" int coda_b200_scan_slab(const float* preds, int64_t model_stride, int H, int64_t N, int C, uint16_t* hard,
                                   int32_t* pseudo, uint8_t* disagree, float* ens_out, uint32_t* flags,
                                   coda_stream_t stream) {
  return scan_slab(preds, model_stride, H, N, C, hard, pseudo, disagree, ens_out, flags, stream);
}

extern "C" int coda_b200_scan_slab_x(const void* preds, int fmt, int64_t model_stride, int H, int64_t N, int C,
                                     uint16_t* hard, int32_t* pseudo, uint8_t* disagree, float* ens_out, uint32_t* flags,
                                     coda_stream_t stream) {
  return slab_dispatch(fmt, preds, [&](auto* p) {
    return scan_slab(p, model_stride, H, N, C, hard, pseudo, disagree, ens_out, flags, stream);
  });
}

// ---------------------------------------------------------------------------------------
// confusion_accum: conf_fx[h][pseudo_n][j] += fx(preds[h][n][j]); int64 fixed point so the
// result does not depend on summation order or on how N is sharded across GPUs.
// grid = (chunks, H).  Shared-memory table when C*C*8 fits, global atomics otherwise.
// ---------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(256) k_confusion_accum(const T* __restrict__ preds, long long ldh,
                                                         const int32_t* __restrict__ pseudo, int H, long long N,
                                                         int C, float fxs, long long chunk, int use_smem,
                                                         unsigned long long* __restrict__ conf_fx) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  unsigned long long* tab = reinterpret_cast<unsigned long long*>(smem_raw);  // [C][C]
  const int h = blockIdx.y;
  const long long n_lo = (long long)blockIdx.x * chunk;
  const long long n_hi = min(N, n_lo + chunk);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarp = blockDim.x >> 5;
  unsigned long long* gtab = conf_fx + (size_t)h * C * C;
  if (use_smem) {
    for (int i = threadIdx.x; i < C * C; i += blockDim.x) tab[i] = 0ull;
    __syncthreads();
  }
  unsigned long long* dst_tab = use_smem ? tab : gtab;
  for (long long n = n_lo + warp; n < n_hi; n += nwarp) {
    const int y = pseudo[n];
    const T* row = preds + (size_t)h * ldh + (size_t)n * C;
    unsigned long long* dst = dst_tab + (size_t)y * C;
    for (int j = lane; j < C; j += 32) {
      long long v = to_fx(ldg_f(row + j), fxs);
      if (v != 0) atomicAdd(dst + j, (unsigned long long)v);
    }
  }
  if (use_smem) {
    __syncthreads();
    for (int i = threadIdx.x; i < C * C; i += blockDim.x) {
      unsigned long long v = tab[i];
      if (v) atomicAdd(gtab + i, v);
    }
  }
}

// Class-sorted variant: `order` lists the items grouped by pseudo label, so one warp walks a run of items,
// keeps the int64 column sums of the current class in registers (lane <-> column j) and flushes them with a
// handful of global atomics when the class changes -- no shared-memory atomics on the slab-sized stream.
#define CS_RUN 256
template <int KC, typename T>
__global__ void __launch_bounds__(256) k_confusion_sorted(const T* __restrict__ preds, long long ldh,
                                                          const int32_t* __restrict__ pseudo,
                                                          const int32_t* __restrict__ order, int H, long long N, int C,
                                                          float fxs, unsigned long long* __restrict__ conf_fx) {
  const int h = blockIdx.y;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long i0 = ((long long)blockIdx.x * 8 + warp) * CS_RUN;
  const long long i1 = min(N, i0 + CS_RUN);
  if (i0 >= N) return;
  const T* slab = preds + (size_t)h * ldh;
  unsigned long long* tab = conf_fx + (size_t)h * C * C;
  long long acc[KC];
#pragma unroll
  for (int k = 0; k < KC; ++k) acc[k] = 0;
  int cur = -1;
  auto flush = [&]() {
    if (cur < 0) return;
#pragma unroll
    for (int k = 0; k < KC; ++k) {
      const int j = lane + 32 * k;
      if (j < C && acc[k]) atomicAdd(tab + (size_t)cur * C + j, (unsigned long long)acc[k]);
      acc[k] = 0;
    }
  };
  for (long long i = i0; i < i1; i += 4) {
    int n[4], y[4];
    float v[4][KC];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const long long ii = min(i + q, i1 - 1);
      n[q] = order[ii];
      y[q] = pseudo[n[q]];
    }
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const T* row = slab + (size_t)n[q] * C;
#pragma unroll
      for (int k = 0; k < KC; ++k) {
        const int j = lane + 32 * k;
        v[q][k] = j < C ? ldg_f(row + j) : 0.f;
      }
    }
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      if (i + q >= i1) break;
      if (y[q] != cur) {
        flush();
        cur = y[q];
      }
#pragma unroll
      for (int k = 0; k < KC; ++k) acc[k] += to_fx(v[q][k], fxs);
    }
  }
  flush();
}

template <typename T>
static int confusion_sorted(const T* preds, int64_t model_stride, const int32_t* pseudo, const int32_t* order, int H,
                            int64_t N, int C, int fx_shift, int64_t* conf_fx, coda_stream_t stream) {
  const long long ldh = model_stride;
  CODA_CHECK_ARG(preds && pseudo && order && conf_fx, "confusion_sorted: null pointer");
  CODA_CHECK_ARG(fx_shift >= 8 && fx_shift <= 46, "confusion_sorted: bad fx_shift %d", fx_shift);
  CODA_CHECK_ARG(C <= 128, "confusion_sorted: C=%d > 128 (use confusion_accum)", C);
  const long long runs = (N + CS_RUN - 1) / CS_RUN;
  dim3 grid((unsigned)((runs + 7) / 8), (unsigned)H);
  const float fxs = exp2f((float)fx_shift);
  unsigned long long* out = reinterpret_cast<unsigned long long*>(conf_fx);
  cudaStream_t st = as_stream(stream);
  if (C <= 32) k_confusion_sorted<1, T><<<grid, 256, 0, st>>>(preds, ldh, pseudo, order, H, N, C, fxs, out);
  else if (C <= 64) k_confusion_sorted<2, T><<<grid, 256, 0, st>>>(preds, ldh, pseudo, order, H, N, C, fxs, out);
  else if (C <= 96) k_confusion_sorted<3, T><<<grid, 256, 0, st>>>(preds, ldh, pseudo, order, H, N, C, fxs, out);
  else k_confusion_sorted<4, T><<<grid, 256, 0, st>>>(preds, ldh, pseudo, order, H, N, C, fxs, out);
  CODA_LAUNCH_OK("k_confusion_sorted");
  return CODA_B200_OK;
}

extern "C" int coda_b200_confusion_sorted(const float* preds, int64_t model_stride, const int32_t* pseudo,
                                          const int32_t* order, int H, int64_t N, int C, int fx_shift,
                                          int64_t* conf_fx, coda_stream_t stream) {
  return confusion_sorted(preds, model_stride, pseudo, order, H, N, C, fx_shift, conf_fx, stream);
}

extern "C" int coda_b200_confusion_sorted_x(const void* preds, int fmt, int64_t model_stride, const int32_t* pseudo,
                                            const int32_t* order, int H, int64_t N, int C, int fx_shift,
                                            int64_t* conf_fx, coda_stream_t stream) {
  return slab_dispatch(fmt, preds, [&](auto* p) {
    return confusion_sorted(p, model_stride, pseudo, order, H, N, C, fx_shift, conf_fx, stream);
  });
}

template <typename T>
static int confusion_accum(const T* preds, int64_t model_stride, const int32_t* pseudo, int H, int64_t N, int C,
                           int fx_shift, int64_t* conf_fx, coda_stream_t stream) {
  CODA_CHECK_ARG(preds && pseudo && conf_fx, "confusion_accum: null pointer");
  CODA_CHECK_ARG(fx_shift >= 8 && fx_shift <= 46, "confusion_accum: bad fx_shift %d", fx_shift);
  size_t tab = (size_t)C * C * 8;
  int use_smem = tab <= 160 * 1024;
  size_t smem = use_smem ? tab : 0;
  if (use_smem) CODA_CUDA_OK(cudaFuncSetAttribute(k_confusion_accum<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  long long chunk = 8192;
  long long chunks = (N + chunk - 1) / chunk;
  dim3 grid((unsigned)chunks, (unsigned)H);
  k_confusion_accum<T><<<grid, 256, smem, as_stream(stream)>>>(preds, (long long)model_stride, pseudo, H, N, C, exp2f((float)fx_shift), chunk, use_smem,
                                                              reinterpret_cast<unsigned long long*>(conf_fx));
  CODA_LAUNCH_OK("k_confusion_accum");
  return CODA_B200_OK;
}

extern "C" int coda_b200_confusion_accum(const float* preds, int64_t model_stride, const int32_t* pseudo, int H,
                                         int64_t N, int C, int fx_shift, int64_t* conf_fx, coda_stream_t stream) {
  return confusion_accum(preds, model_stride, pseudo, H, N, C, fx_shift, conf_fx, stream);
}

extern "C" int coda_b200_confusion_accum_x(const void* preds, int fmt, int64_t model_stride, const int32_t* pseudo, int H,
                                           int64_t N, int C, int fx_shift, int64_t* conf_fx, coda_stream_t stream) {
  return slab_dispatch(fmt, preds, [&](auto* p) {
    return confusion_accum(p, model_stride, pseudo, H, N, C, fx_shift, conf_fx, stream);
  });
}

// ---------------------------------------------------------------------------------------
// init_dirichlets: D = multiplier * (base + prior_strength * conf / max(rowsum, 1e-6))
// one warp per (h, c) row.
// ---------------------------------------------------------------------------------------
__global__ void k_init_dirichlets(const long long* __restrict__ conf_fx, const long long* __restrict__ conf_rest,
                                  int H, int C, int shift,
                                  float prior_strength, float multiplier, int uniform_prior,
                                  float* __restrict__ D) {
  const int lane = threadIdx.x & 31;
  const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= (long long)H * C) return;
  const int c = (int)(row % C);
  const long long* src = conf_fx + row * C;
  const long long rest = conf_rest ? conf_rest[row] : 0;          // compact slab: carried by every column of the row
  float rs = 0.f;
  for (int j = lane; j < C; j += 32) rs += (float)from_fx(src[j] + rest, shift);
  rs = warp_sum(rs);
  rs = fmaxf(rs, 1e-6f);                                        // coda.py:43 clamp_min(1e-6)
  const float off = uniform_prior ? (float)(2.0 / C) : (float)(1.0 / (C - 1));   // coda.py:53, 57
  for (int j = lane; j < C; j += 32) {
    float conf = (float)from_fx(src[j] + rest, shift) / rs;
    float base = (!uniform_prior && j == c) ? 1.0f : off;       // coda.py:60 fill_diagonal_(1.0)
    D[row * C + j] = multiplier * (base + prior_strength * conf);  // coda.py:63, 196
  }
}

extern "C" int coda_b200_init_dirichlets(const int64_t* conf_fx, const int64_t* conf_rest, int H, int C, int fx_shift,
                                         double prior_strength, double multiplier, int uniform_prior, float* D,
                                         coda_stream_t stream) {
  CODA_CHECK_ARG(conf_fx && D, "init_dirichlets: null pointer");
  long long rows = (long long)H * C;
  int wpb = 8;
  k_init_dirichlets<<<(unsigned)((rows + wpb - 1) / wpb), wpb * 32, 0, as_stream(stream)>>>(
      reinterpret_cast<const long long*>(conf_fx), reinterpret_cast<const long long*>(conf_rest), H, C, fx_shift,
      (float)prior_strength, (float)multiplier,
      uniform_prior, D);
  CODA_LAUNCH_OK("k_init_dirichlets");
  return CODA_B200_OK;
}

// ---------------------------------------------------------------------------------------
// pi_full: U[n][c] = sum_h sum_s D[h][c][s] * preds[h][n][s]   (fp32 SIMT GEMM, K = H*C)
// CTA: 64 points x 128 classes (grid.y walks the class blocks); thread (pg, cg) owns 4 points x 8 classes.
// COMP (C > 128, where no tensor-core pass exists): compensated (Kahan) accumulation.  There the diagonal term puts the
// accumulator near 1 and the H*C off-diagonal terms are each about one ulp of it; a plain chain rounds every one of them
// the same way and drifts by 1e-4 relative at C = 3200 (1e-3 at H = 128), the compensated chain stays at a few ulps.
// ---------------------------------------------------------------------------------------
#define PF_TN 64
#define PF_TC 128
#define PF_SK 32
template <typename T, bool COMP>
__global__ void __launch_bounds__(256) k_pi_full(const T* __restrict__ preds, long long ldh,
                                                 const float* __restrict__ D, int H, long long N, int C,
                                                 float* __restrict__ U) {
  __shared__ float As[PF_TN][PF_SK + 1];
  __shared__ float Bs[PF_TC][PF_SK + 1];
  const int tid = threadIdx.x;
  const int pg = tid >> 4, cg = tid & 15;
  const long long n0 = (long long)blockIdx.x * PF_TN;
  const int c0 = blockIdx.y * PF_TC;
  float acc[4][8], cmp[4][8];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int k = 0; k < 8; ++k) acc[i][k] = cmp[i][k] = 0.f;
  for (int h = 0; h < H; ++h) {
    const T* Ah = preds + (size_t)h * ldh;
    const float* Dh = D + ((size_t)h * C) * C;
    for (int s0 = 0; s0 < C; s0 += PF_SK) {
      __syncthreads();
      for (int e = tid; e < PF_TN * PF_SK; e += 256) {
        int r = e >> 5, col = e & 31;
        long long n = n0 + r;
        int s = s0 + col;
        As[r][col] = (n < N && s < C) ? ldg_f(Ah + (size_t)n * C + s) : 0.f;
      }
      for (int e = tid; e < PF_TC * PF_SK; e += 256) {
        int r = e >> 5, col = e & 31;
        int c = c0 + r, s = s0 + col;
        Bs[r][col] = (c < C && s < C) ? __ldg(Dh + (size_t)c * C + s) : 0.f;
      }
      __syncthreads();
#pragma unroll 8
      for (int s = 0; s < PF_SK; ++s) {
        float a[4], b[8];
#pragma unroll
        for (int i = 0; i < 4; ++i) a[i] = As[pg * 4 + i][s];
#pragma unroll
        for (int k = 0; k < 8; ++k) b[k] = Bs[cg + 16 * k][s];
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int k = 0; k < 8; ++k) {
            if (COMP) {
              const float y = fmaf(a[i], b[k], -cmp[i][k]);
              const float t = acc[i][k] + y;
              cmp[i][k] = (t - acc[i][k]) - y;
              acc[i][k] = t;
            } else {
              acc[i][k] = fmaf(a[i], b[k], acc[i][k]);
            }
          }
      }
    }
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    long long n = n0 + pg * 4 + i;
    if (n >= N) continue;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      int c = c0 + cg + 16 * k;
      if (c < C) U[(size_t)n * C + c] = acc[i][k];
    }
  }
}

template <typename T>
static int pi_full(const T* preds, int64_t model_stride, const float* D, int H, int64_t N, int C, float* U,
                   coda_stream_t stream) {
  CODA_CHECK_ARG(preds && D && U, "pi_full: null pointer");
  dim3 grid((unsigned)((N + PF_TN - 1) / PF_TN), (unsigned)((C + PF_TC - 1) / PF_TC));
  if (C > PF_TC)
    k_pi_full<T, true><<<grid, 256, 0, as_stream(stream)>>>(preds, (long long)model_stride, D, H, N, C, U);
  else
    k_pi_full<T, false><<<grid, 256, 0, as_stream(stream)>>>(preds, (long long)model_stride, D, H, N, C, U);
  CODA_LAUNCH_OK("k_pi_full");
  return CODA_B200_OK;
}

extern "C" int coda_b200_pi_full(const float* preds, int64_t model_stride, const float* D, int H, int64_t N, int C,
                                 float* U, coda_stream_t stream) {
  return pi_full(preds, model_stride, D, H, N, C, U, stream);
}

extern "C" int coda_b200_pi_full_x(const void* preds, int fmt, int64_t model_stride, const float* D, int H, int64_t N,
                                   int C, float* U, coda_stream_t stream) {
  return slab_dispatch(fmt, preds, [&](auto* p) { return pi_full(p, model_stride, D, H, N, C, U, stream); });
}

// ---------------------------------------------------------------------------------------
// shared tail of pi_reduce / pi_rank1: one warp normalises one row of U and adds the per-class
// column sums of pi_hat_xi (fixed point) into the block's shared-memory vector wacc[C] with 64-bit
// shared atomics.  One [C] vector per block (not one per warp) keeps C = 4096 at 32 KB; the sums
// are integers, so the order of the atomics does not change their bits.
// ---------------------------------------------------------------------------------------
__device__ __forceinline__ void row_accumulate(float* __restrict__ urow, int C, int lane, float fxs, int t,
                                               float delta_t, float* __restrict__ xi_out,
                                               long long* __restrict__ wacc, uint32_t& bad) {
  float s = 0.f, ut = 0.f;
  for (int c = lane; c < C; c += 32) {      // loads only: a store inside this loop would order every later load behind it
    float u = urow[c];                       // (possible alias) and turn the row into C / 32 dependent round trips
    if (c == t) {
      u += delta_t;
      ut = u;
    }
    s += u;
  }
  if (t >= 0 && lane == (t & 31)) urow[t] = ut;
  s = warp_sum(s);
  if (!isfinite(s)) bad |= CODA_B200_FLAG_NONFINITE_PI;
  const float den = fmaxf(s, 1e-12f);                               // coda.py:230 clamp_(min=1e-12)
  const float rden = 1.0f / den;
  for (int c = lane; c < C; c += 32) {
    float xi = row_quot(urow[c], den, rden);   // column t was rewritten above by this same lane

    if (xi_out) xi_out[c] = xi;
    atomicAdd(reinterpret_cast<unsigned long long*>(wacc) + c, (unsigned long long)to_fx(xi, fxs));
  }
}

__global__ void __launch_bounds__(256) k_pi_reduce(float* __restrict__ U, long long N, int C, float fxs,
                                                   float* __restrict__ xi_out,
                                                   unsigned long long* __restrict__ pisum_fx,
                                                   uint32_t* __restrict__ flags) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  long long* wacc = reinterpret_cast<long long*>(smem_raw);           // [C] the block's column sums
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarp = blockDim.x >> 5;
  for (int c = threadIdx.x; c < C; c += blockDim.x) wacc[c] = 0;
  __syncthreads();
  uint32_t bad = 0;
  for (long long n = (long long)blockIdx.x * nwarp + warp; n < N; n += (long long)gridDim.x * nwarp)
    row_accumulate(U + (size_t)n * C, C, lane, fxs, -1, 0.f, xi_out ? xi_out + (size_t)n * C : nullptr, wacc, bad);
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    const long long s = wacc[c];
    if (s) atomicAdd(pisum_fx + c, (unsigned long long)s);
  }
  if (bad) atomicOr(flags, bad);
}

extern "C" int coda_b200_pi_reduce(float* U, int64_t N, int C, int fx_shift, float* xi_out, int64_t* pisum_fx,
                                   uint32_t* flags, coda_stream_t stream) {
  CODA_CHECK_ARG(U && pisum_fx && flags, "pi_reduce: null pointer");
  size_t smem = (size_t)C * 8;
  CODA_CHECK_ARG(smem <= 200 * 1024, "pi_reduce: C=%d too large", C);
  CODA_CUDA_OK(cudaFuncSetAttribute(k_pi_reduce, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  long long want = (N + 7) / 8;
  int grid = (int)min(want, (long long)coda_sm_count() * 8);
  k_pi_reduce<<<grid, 256, smem, as_stream(stream)>>>(U, N, C, exp2f((float)fx_shift), xi_out,
                                                      reinterpret_cast<unsigned long long*>(pisum_fx), flags);
  CODA_LAUNCH_OK("k_pi_reduce");
  return CODA_B200_OK;
}

// ---------------------------------------------------------------------------------------
// posterior update (coda.py:316-317) and the marginal refresh it triggers (coda.py:319),
// restated:  D[h, t, j_h] += lr   with j_h = p_h(idx)   changes only row t of every D[h], so
//   U[n, t] += lr * sum_h preds[h, n, j_h]      and every other column of U is untouched.
// (the label itself -- owner's p_h(idx), labeled mark, D update, gather list -- is in step.cu)
// pi_rank1    : gathers one float per (h, n) (one 32 B sector each), updates column t of U,
//               renormalises rows on the fly and re-accumulates sum_n pi_hat_xi[n, :]
// ---------------------------------------------------------------------------------------
// ---------------------------------------------------------------------------------------
// class-major shadow copy  T[s][c][n] = preds[h_s][n][c]  for a subset of models (as many as spare HBM
// allows, least accurate first).  The rank-1 refresh needs ONE float per (model, item): from the reference
// layout that costs a 64-byte DRAM fetch each, from the shadow it is a coalesced 4-byte read.
// grid = (ceil(N/32), ceil(C/32), S), block = (32, 8)
// ---------------------------------------------------------------------------------------
template <typename E>
__global__ void k_shadow_transpose(const E* __restrict__ preds, long long ldh, long long N, int C,
                                   const int32_t* __restrict__ model_of_slot, long long cs, E* __restrict__ T) {
  __shared__ E tile[32][33];
  const int s = blockIdx.z, h = model_of_slot[s];
  const long long n0 = (long long)blockIdx.x * 32;
  const int c0 = blockIdx.y * 32;
  const E* src = preds + (size_t)h * ldh;
  for (int r = threadIdx.y; r < 32; r += 8) {
    const long long n = n0 + r;
    const int c = c0 + threadIdx.x;
    tile[r][threadIdx.x] = (n < N && c < C) ? __ldg(src + (size_t)n * C + c) : E();
  }
  __syncthreads();
  E* dst = T + (size_t)s * C * cs;
  for (int r = threadIdx.y; r < 32; r += 8) {
    const int c = c0 + r;
    const long long n = n0 + threadIdx.x;
    if (c < C && n < N) dst[(size_t)c * cs + n] = tile[threadIdx.x][r];
  }
}

template <typename E>
static int shadow_build(const E* preds, int64_t model_stride, int H, int64_t N, int C, const int32_t* model_of_slot,
                        int S, int64_t col_stride, E* T, coda_stream_t stream) {
  CODA_CHECK_ARG(preds && model_of_slot && T && S >= 1 && S <= H && col_stride >= N, "shadow_build: bad arguments");
  long long gx = (N + 31) / 32;
  CODA_CHECK_ARG(gx <= 0x7fffffffLL && S <= 65535, "shadow_build: grid too large");
  dim3 grid((unsigned)gx, (unsigned)((C + 31) / 32), (unsigned)S), block(32, 8);
  k_shadow_transpose<E><<<grid, block, 0, as_stream(stream)>>>(preds, (long long)model_stride, N, C, model_of_slot,
                                                               (long long)col_stride, T);
  CODA_LAUNCH_OK("k_shadow_transpose");
  return CODA_B200_OK;
}

extern "C" int coda_b200_shadow_build(const float* preds, int64_t model_stride, int H, int64_t N, int C,
                                      const int32_t* model_of_slot, int S, int64_t col_stride, float* T,
                                      coda_stream_t stream) {
  return shadow_build(preds, model_stride, H, N, C, model_of_slot, S, col_stride, T, stream);
}

extern "C" int coda_b200_shadow_build_x(const void* preds, int fmt, int64_t model_stride, int H, int64_t N, int C,
                                        const int32_t* model_of_slot, int S, int64_t col_stride, void* T,
                                        coda_stream_t stream) {
  return slab_dispatch(fmt, preds, [&](auto* p) {
    using E = std::remove_const_t<std::remove_pointer_t<decltype(p)>>;
    return shadow_build(p, model_stride, H, N, C, model_of_slot, S, col_stride, static_cast<E*>(T), stream);
  });
}

// register variant of row_accumulate for C <= 32 * KC: NR rows per call (all loads issued before the first
// reduction), the int64 column sums stay in registers
template <int KC, int NR>
__device__ __forceinline__ void rows_accumulate_reg(float* __restrict__ U, long long row0, int nrows, int rstride,
                                                    int C, int lane, float fxs, int t, const float (&dv)[NR],
                                                    long long (&racc)[KC], uint32_t& bad) {
  float u[NR][KC];
#pragma unroll
  for (int r = 0; r < NR; ++r) {
    const bool ok = r * rstride < nrows;
    const float* urow = U + (size_t)(row0 + (ok ? r * rstride : 0)) * C;
#pragma unroll
    for (int k = 0; k < KC; ++k) {
      const int c = lane + 32 * k;
      u[r][k] = (ok && c < C) ? urow[c] : 0.f;
    }
  }
#pragma unroll
  for (int r = 0; r < NR; ++r) {
    if (r * rstride >= nrows) break;
    float* urow = U + (size_t)(row0 + r * rstride) * C;
    float s = 0.f;
#pragma unroll
    for (int k = 0; k < KC; ++k) {
      const int c = lane + 32 * k;
      if (c == t) {
        u[r][k] += dv[r];
        urow[c] = u[r][k];
      }
      s += u[r][k];
    }
    s = warp_sum(s);
    if (!isfinite(s)) bad |= CODA_B200_FLAG_NONFINITE_PI;
    const float den = fmaxf(s, 1e-12f);                             // coda.py:230 clamp_(min=1e-12)
    const float rden = 1.0f / den;
#pragma unroll
    for (int k = 0; k < KC; ++k) racc[k] += to_fx(row_quot(u[r][k], den, rden), fxs);
  }
}

// The gather list is read by every lane at the same index: the constant cache serves that as a uniform load, shared
// memory as a broadcast LDS through the MIO pipe (measured: 0.37 ms vs 0.55 ms for the kernel below at cfg3).  The
// constant bank is per device and shared by every stream of the process, so it is cut into slots: a caller that owns
// a slot (coda_b200_pi_rank1's const_slot >= 0; coda_b200.engine hands them out per device) gets the constant path,
// anyone else the shared-memory copy.
#define R1_CONST_TERMS 3584                        // 56 KB of the 64 KB constant bank
__constant__ R1Term c_terms_bank[R1_CONST_TERMS];

#define R1_TN 256
#define R1_GU 16                                   // gathers in flight per lane
#define R1_NR 4                                    // U rows in flight per warp
// T: slab element type.  A 16-bit slab keeps the ensemble sums in fp32 behind their own base pointer `ensb`: the first
// term of a list with a majority class (hdr[1] >= 0) is read from there, every other term from the slab.  For fp32 both
// live behind `preds` (ensb is not read).  Term order and the fmaf chain are the same either way.
template <typename T, int KC, bool CONST_TERMS = false>
__global__ void __launch_bounds__(256, 4) k_pi_rank1(const T* __restrict__ preds, const float* __restrict__ ensb,
                                                  long long N, int C, const long long* __restrict__ sel,
                                                  const int32_t* __restrict__ hdr, const R1Term* __restrict__ gterms,
                                                  int const_base, float lr, float fxs,
                                                  float* __restrict__ U, unsigned long long* __restrict__ pisum_fx,
                                                  uint32_t* __restrict__ flags) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  constexpr int NACC = KC > 0 ? 8 : 1;                                           // KC > 0: one [C] per warp; KC == 0: one
  long long* wacc_all = reinterpret_cast<long long*>(smem_raw);                 // [NACC][C]   for the block (row_accumulate)
  R1Term* s_terms = reinterpret_cast<R1Term*>(wacc_all + (size_t)NACC * C);     // [nt] gather list (broadcast reads)
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int t = (int)sel[1];
  const int nt = hdr[0];
  const bool ens_f32 = !std::is_same<T, float>::value && hdr[1] >= 0;
  if (!CONST_TERMS)
    for (int k = threadIdx.x; k < nt; k += blockDim.x) s_terms[k] = gterms[k];
  const R1Term* c_terms = CONST_TERMS ? (c_terms_bank + const_base) : s_terms;
  long long* wacc = wacc_all + (size_t)(KC > 0 ? warp : 0) * C;
  if (KC > 0)
    for (int c = lane; c < C; c += 32) wacc[c] = 0;
  else
    for (int c = threadIdx.x; c < C; c += blockDim.x) wacc[c] = 0;
  long long racc[KC > 0 ? KC : 1];
#pragma unroll
  for (int k = 0; k < (KC > 0 ? KC : 1); ++k) racc[k] = 0;
  __syncthreads();
  uint32_t bad = 0;
  // one warp = 32 consecutive items: lane i gathers item i's increment, then the warp walks the 32 rows of U
  // (increment handed over by shuffle).  No block-level barrier inside the loop, warps run independently.
  const long long wstride = (long long)gridDim.x * R1_TN;
  for (long long n0 = (long long)blockIdx.x * R1_TN + warp * 32; n0 < N; n0 += wstride) {
    const long long n = n0 + lane;
    float d = 0.f;
    if (n < N) {
      int k = 0;
      if (ens_f32) {
        d = fmaf(c_terms[0].sg, __ldg(ensb + c_terms[0].off + n * c_terms[0].str), d);
        k = 1;
      }
      for (; k + R1_GU <= nt; k += R1_GU) {
        float v[R1_GU];
#pragma unroll
        for (int q = 0; q < R1_GU; ++q) v[q] = ldg_f(preds + c_terms[k + q].off + n * c_terms[k + q].str);
#pragma unroll
        for (int q = 0; q < R1_GU; ++q) d = fmaf(c_terms[k + q].sg, v[q], d);
      }
      for (; k < nt; ++k) d = fmaf(c_terms[k].sg, ldg_f(preds + c_terms[k].off + n * c_terms[k].str), d);
    }
    const float dl = lr * d;
    const int rows = (int)min(32LL, N - n0);
    if (KC > 0) {
      for (int r = 0; r < rows; r += R1_NR) {
        float dv[R1_NR];
#pragma unroll
        for (int i = 0; i < R1_NR; ++i) dv[i] = __shfl_sync(CODA_FULL, dl, (r + i) & 31);
        rows_accumulate_reg<(KC > 0 ? KC : 1), R1_NR>(U, n0 + r, rows - r, 1, C, lane, fxs, t, dv, racc, bad);
      }
    } else {
      for (int r = 0; r < rows; ++r) {
        const float dr = __shfl_sync(CODA_FULL, dl, r);
        row_accumulate(U + (size_t)(n0 + r) * C, C, lane, fxs, t, dr, nullptr, wacc, bad);
      }
    }
  }
  if (KC > 0) {
#pragma unroll
    for (int k = 0; k < (KC > 0 ? KC : 1); ++k) {
      const int c = lane + 32 * k;
      if (c < C) wacc[c] = racc[k];
    }
  }
  __syncthreads();          // every warp's column sums are in shared memory
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    long long s2 = 0;
    for (int w = 0; w < NACC; ++w) s2 += wacc_all[(size_t)w * C + c];
    if (s2) atomicAdd(pisum_fx + c, (unsigned long long)s2);
  }
  if (bad) atomicOr(flags, bad);
}

template <typename T>
static int pi_rank1(const T* preds, const float* ensb, int H, int64_t N, int C, const int64_t* sel, double lr,
                    int fx_shift, const int32_t* terms /*[2 + 8H]*/, float* U, int64_t* pisum_fx, uint32_t* flags,
                    int ctas_per_sm, int const_slot, coda_stream_t stream) {
  CODA_CHECK_ARG(preds && sel && terms && U && pisum_fx && flags, "pi_rank1: null pointer");
  CODA_CHECK_ARG(2 * H <= R1_MAXT, "pi_rank1: H=%d too large", H);
  CODA_CHECK_ARG((reinterpret_cast<uintptr_t>(terms) & 7) == 0, "pi_rank1: terms must be 8-byte aligned");
  const int32_t* hdr = terms;                                                  // 2 ints
  const R1Term* tlist = reinterpret_cast<const R1Term*>(terms + 2);            // <= 2H x 16 bytes
  cudaStream_t st = as_stream(stream);
  size_t smem = (size_t)(C <= 128 ? 8 : 1) * C * 8 + (size_t)2 * H * sizeof(R1Term);   // NACC of the KC chosen below
  CODA_CHECK_ARG(smem <= 200 * 1024, "pi_rank1: C=%d too large", C);
  long long want = (N + R1_TN - 1) / R1_TN;
  if (ctas_per_sm < 1 || ctas_per_sm > 8) ctas_per_sm = 8;
  int grid = (int)min(want, (long long)coda_sm_count() * ctas_per_sm);
  // constant-bank slot of this caller (see c_terms_bank): the list is copied device-to-device on the launching stream
  const int slot_terms = (2 * H + 63) / 64 * 64;
  const bool use_const = const_slot >= 0 && (long long)(const_slot + 1) * slot_terms <= R1_CONST_TERMS && C <= 128;
  const int const_base = use_const ? const_slot * slot_terms : 0;
  if (use_const)
    CODA_CUDA_OK(cudaMemcpyToSymbolAsync(c_terms_bank, tlist, (size_t)2 * H * sizeof(R1Term),
                                         (size_t)const_base * sizeof(R1Term), cudaMemcpyDeviceToDevice, st));
#define LAUNCH_R1(KC)                                                                                          \
  do {                                                                                                         \
    if (use_const) {                                                                                           \
      CODA_CUDA_OK(cudaFuncSetAttribute(k_pi_rank1<T, KC, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
      k_pi_rank1<T, KC, true><<<grid, 256, smem, st>>>(preds, ensb, N, C, reinterpret_cast<const long long*>(sel), hdr, \
                                            tlist, const_base, (float)lr, exp2f((float)fx_shift), U,           \
                                            reinterpret_cast<unsigned long long*>(pisum_fx), flags);           \
      break;                                                                                                   \
    }                                                                                                          \
    CODA_CUDA_OK(cudaFuncSetAttribute(k_pi_rank1<T, KC>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
    k_pi_rank1<T, KC><<<grid, 256, smem, st>>>(preds, ensb, N, C, reinterpret_cast<const long long*>(sel), hdr,    \
                                            tlist, 0, (float)lr, exp2f((float)fx_shift), U,                    \
                                            reinterpret_cast<unsigned long long*>(pisum_fx), flags);           \
  } while (0)
  if (C <= 32) LAUNCH_R1(1);
  else if (C <= 64) LAUNCH_R1(2);
  else if (C <= 128) LAUNCH_R1(4);
  else LAUNCH_R1(0);
#undef LAUNCH_R1
  CODA_LAUNCH_OK("k_pi_rank1");
  return CODA_B200_OK;
}

extern "C" int coda_b200_pi_rank1(const float* preds, const float* ens, int H, int64_t N, int C, const int64_t* sel,
                                  double lr, int fx_shift, const int32_t* terms /*[2 + 8H]*/, float* U,
                                  int64_t* pisum_fx, uint32_t* flags, int ctas_per_sm, int const_slot,
                                  coda_stream_t stream) {
  return pi_rank1(preds, preds, H, N, C, sel, lr, fx_shift, terms, U, pisum_fx, flags, ctas_per_sm, const_slot, stream);
}

extern "C" int coda_b200_pi_rank1_x(const void* preds, int fmt, const float* ens_base, int H, int64_t N, int C,
                                    const int64_t* sel, double lr, int fx_shift, const int32_t* terms, float* U,
                                    int64_t* pisum_fx, uint32_t* flags, int ctas_per_sm, int const_slot,
                                    coda_stream_t stream) {
  CODA_CHECK_ARG(fmt == CODA_B200_SLAB_F32 || ens_base, "pi_rank1: a 16-bit slab needs the fp32 ensemble base pointer");
  return slab_dispatch(fmt, preds, [&](auto* p) {
    return pi_rank1(p, fmt == CODA_B200_SLAB_F32 ? static_cast<const float*>(preds) : ens_base, H, N, C, sel, lr,
                    fx_shift, terms, U, pisum_fx, flags, ctas_per_sm, const_slot, stream);
  });
}

CODA_MODULE_ANCHOR(slab, k_init_dirichlets)
