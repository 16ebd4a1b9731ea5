// Scoring only a sample of items (--prefilter-n, coda.py:221-223, 239): the reference integrates rows for its
// candidate ids only, so a step with prefilter_n = m needs the EIG of m items, not of all N.
//
//   sample_plan   one CTA: the sample's heavy rows (|Z| >= 2) as a class-major work list -- per class a base, tiles of
//                 <= width same-class positions, {0, tile count} in tile_off form, the heavy-row count -- and the
//                 output slot of every sampled item's heavy rows (slot = hoff[j] + its k-th heavy row).
//   sample_fill   one warp per sample position: the H-bit mask of each heavy row from `hard`, bit for bit what
//                 pair_fill wrote for that row, its class and its slot, at a position of its class's range.
//   pair_rows_tc / pair_rows (unchanged) run over that list in their device-`sel` form (sel[1] = 0, tile_off =
//                 {0, tile count}: a fixed grid, graph-capturable), writing the rows through row_of into a scratch.
//   sample_gains  gain of every template row and every scratch row: k_row_gains' arithmetic, row count on the device.
//   sample_eig    eig of every sampled item: the per-item arithmetic of the full pass's assembly (eig_item.cuh).
//
// A row's bits depend only on its own mask, its class's tables and the fixed K chunking, not on the rows that share
// its tile, so a scratch row equals the cached row of the same (item, class), and a sampled item's eig equals what the
// full pass computes for it (tests/test_prefilter_sample.py checks both).
#include "common.cuh"
#include "eig_item.cuh"

#define SP_THREADS 1024

// exclusive block scan of one value per thread; returns the block total to every thread
__device__ __forceinline__ long long sp_block_scan(long long v, long long* sh, long long& total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  long long x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const long long y = __shfl_up_sync(CODA_FULL, x, o);
    if (lane >= o) x += y;
  }
  if (lane == 31) sh[warp] = x;
  __syncthreads();
  if (warp == 0) {
    long long w = lane < SP_THREADS / 32 ? sh[lane] : 0;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const long long y = __shfl_up_sync(CODA_FULL, w, o);
      if (lane >= o) w += y;
    }
    sh[lane] = w;                            // inclusive warp totals
  }
  __syncthreads();
  const long long excl = x - v + (warp > 0 ? sh[warp - 1] : 0);
  total = sh[SP_THREADS / 32 - 1];
  __syncthreads();
  return excl;
}

__global__ void __launch_bounds__(SP_THREADS) k_sample_plan(const int32_t* __restrict__ items, int m,
                                                           const int32_t* __restrict__ ent_off,
                                                           const int32_t* __restrict__ ent_row,
                                                           const uint16_t* __restrict__ ent_cls,
                                                           const int32_t* __restrict__ heavy_off, long long T, int C,
                                                           int width, int32_t* __restrict__ hoff,
                                                           int32_t* __restrict__ cursor, int4* __restrict__ tiles,
                                                           long long* __restrict__ tile_off, long long* __restrict__ nheavy) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  int* cnt = reinterpret_cast<int*>(smem_raw);               // [C] heavy rows of the sample per class
  __shared__ long long sh[SP_THREADS / 32];
  for (int c = threadIdx.x; c < C; c += SP_THREADS) cnt[c] = 0;
  __syncthreads();
  // slots: exclusive prefix of the sampled items' heavy-row counts, in sample order
  long long carry = 0;
  for (int j0 = 0; j0 < m; j0 += SP_THREADS) {
    const int j = j0 + threadIdx.x;
    long long v = 0;
    if (j < m) {
      const int n = items[j];
      if (n >= 0) {
        v = heavy_off[n + 1] - heavy_off[n];
        for (int e = ent_off[n]; e < ent_off[n + 1]; ++e)
          if (ent_row[e] >= T) atomicAdd(&cnt[ent_cls[e]], 1);
      }
    }
    long long tot;
    const long long ex = sp_block_scan(v, sh, tot);
    if (j < m) hoff[j] = (int32_t)(carry + ex);
    carry += tot;
  }
  __syncthreads();
  // class bases and tiles: one class per tile, <= width positions each
  long long pos_carry = 0, tile_carry = 0;
  for (int c0 = 0; c0 < C; c0 += SP_THREADS) {
    const int c = c0 + threadIdx.x;
    const long long k = c < C ? cnt[c] : 0;
    const long long nt = (k + width - 1) / width;
    long long ptot, ttot;
    const long long pb = pos_carry + sp_block_scan(k, sh, ptot);
    const long long tb = tile_carry + sp_block_scan(nt, sh, ttot);
    if (c < C) {
      cursor[c] = (int32_t)pb;
      for (long long t = 0; t < nt; ++t)
        tiles[tb + t] = make_int4(c, (int)(pb + width * t), (int)min((long long)width, k - width * t), 0);
    }
    pos_carry += ptot;
    tile_carry += ttot;
  }
  if (threadIdx.x == 0) {
    hoff[m] = (int32_t)carry;
    tile_off[0] = 0;
    tile_off[1] = tile_carry;
    *nheavy = carry;
  }
}

__global__ void __launch_bounds__(256) k_sample_fill(const int32_t* __restrict__ items, int m,
                                                    const uint16_t* __restrict__ hard, int H, int W,
                                                    const int32_t* __restrict__ ent_off,
                                                    const int32_t* __restrict__ ent_row,
                                                    const uint16_t* __restrict__ ent_cls,
                                                    const int32_t* __restrict__ heavy_off, long long T,
                                                    const int32_t* __restrict__ hoff, int32_t* __restrict__ cursor,
                                                    uint32_t* __restrict__ zmask, int32_t* __restrict__ row_of,
                                                    uint16_t* __restrict__ row_cls) {
  const int lane = threadIdx.x & 31;
  const long long j = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (j >= m) return;
  const int n = items[j];
  if (n < 0) return;
  const uint16_t* hrow = hard + (size_t)n * H;
  for (int e = ent_off[n]; e < ent_off[n + 1]; ++e) {
    const int r = ent_row[e];
    if (r < T) continue;                                      // a template row: no mask of its own
    const int c = ent_cls[e];
    const int slot = hoff[j] + (int)(r - T - heavy_off[n]);   // the item's heavy rows are consecutive row ids
    uint32_t myword = 0;                                      // mask words as pair_fill builds them: lane w <- word w
    for (int w = 0; w < W; ++w) {
      const int h = w * 32 + lane;
      const uint32_t bits = __ballot_sync(CODA_FULL, h < H && hrow[h] == c);
      if (lane == w) myword = bits;
    }
    int q = 0;
    if (lane == 0) q = atomicAdd(&cursor[c], 1);
    q = __shfl_sync(CODA_FULL, q, 0);
    if (lane < W) zmask[(size_t)q * W + lane] = myword;
    if (lane == 0) {
      row_of[q] = slot;
      row_cls[slot] = (uint16_t)c;
    }
  }
}

// gain of rows [0, T + *nheavy): templates from `tmpl`, the rest from `scratch`.  Per row, lane l sums
// gain4 over the columns 4 l + 128 i in ascending i, then the warp sum: the order of k_row_gains / k_row_gains_any.
__device__ __forceinline__ float4 sp_ld_stream4(const float4* p) {
  float4 v;
  asm volatile("ld.global.cs.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p));
  return v;
}

__device__ __forceinline__ float sp_gain4(const float4 ph, const float4 pb, const float4 m, const float4 fm, float pic) {
  float g = fm.x - ent_term(m.x + pic * (ph.x - pb.x));
  g += fm.y - ent_term(m.y + pic * (ph.y - pb.y));
  g += fm.z - ent_term(m.z + pic * (ph.z - pb.z));
  g += fm.w - ent_term(m.w + pic * (ph.w - pb.w));
  return g;
}

__global__ void __launch_bounds__(256) k_sample_gains(const float* __restrict__ tmpl, const float* __restrict__ scratch,
                                                     const uint16_t* __restrict__ row_cls,
                                                     const long long* __restrict__ nheavy, long long T, int H, int Hp,
                                                     const float* __restrict__ PB, const float* __restrict__ m0,
                                                     const float* __restrict__ pi_hat, float* __restrict__ gain) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  float* m0s = reinterpret_cast<float*>(smem_raw);
  float* fm0 = m0s + Hp;
  for (int h = threadIdx.x; h < Hp; h += blockDim.x) {
    const float m = h < H ? m0[h] : 0.f;
    m0s[h] = m;
    fm0[h] = ent_term(m);
  }
  __syncthreads();
  const long long nrows = T + *nheavy;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (long long r = (long long)blockIdx.x * 8 + warp; r < nrows; r += (long long)gridDim.x * 8) {
    const int c = r < T ? (int)(r / (1 + H)) : (int)row_cls[r - T];
    const float pic = pi_hat[c];
    const float* row = r < T ? tmpl + (size_t)r * Hp : scratch + (size_t)(r - T) * Hp;
    const float* pb = PB + (size_t)c * Hp;
    float g = 0.f;
    for (int hq = lane * 4; hq < Hp; hq += 128) {
      const float4 ph = sp_ld_stream4(reinterpret_cast<const float4*>(row + hq));
      const float4 p4 = __ldg(reinterpret_cast<const float4*>(pb + hq));
      const float4 m4 = *reinterpret_cast<const float4*>(m0s + hq);
      const float4 f4 = *reinterpret_cast<const float4*>(fm0 + hq);
      g += sp_gain4(ph, p4, m4, f4, pic);
    }
    g = warp_sum(g);
    if (lane == 0) gain[r] = g;
  }
}

struct SampleEigArgs {
  const int32_t* items;
  int m;
  const int32_t* hoff;
  const float* U;
  int C;
  long long T;
  const int32_t* ent_off;
  const int32_t* ent_row;
  const uint16_t* ent_cls;
  const int32_t* heavy_off;
  const float* gain;        // [T + heavy rows of the sample]
  float* eig;
  uint32_t* flags;
};

// the gain of row r of item n at sample position j: a template row in place, a heavy row at its slot
__device__ __forceinline__ float sp_gain_at(const SampleEigArgs& a, int n, int j, int r) {
  return r < a.T ? __ldg(a.gain + r) : __ldg(a.gain + a.T + a.hoff[j] + (r - a.T - a.heavy_off[n]));
}

// the full pass's 8-lane assembly (C <= 128, <= 32 entries per item): one 8-lane group per sample position
template <int KC8>
__global__ void __launch_bounds__(256) k_sample_eig_g8(const SampleEigArgs a) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  float* g0 = reinterpret_cast<float*>(smem_raw);
  const int C = a.C;
  const int H1 = (int)(a.T / C);
  for (int c = threadIdx.x; c < C; c += blockDim.x) g0[c] = a.gain[(size_t)c * H1];
  __syncthreads();
  const int g = threadIdx.x & 7;
  const long long j = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 3;
  const int n = j < a.m ? a.items[j] : -1;
  if (__all_sync(CODA_FULL, n < 0)) return;
  const int nn = n < 0 ? 0 : n;                              // a group without an item computes on item 0 and writes nothing
  const float* urow = a.U + (size_t)nn * C;
  float u[KC8];
#pragma unroll
  for (int k = 0; k < KC8; ++k) {
    const int c = g + 8 * k;
    u[k] = c < C ? __ldg(urow + c) : 0.f;
  }
  const int e0 = a.ent_off[nn], ne = n < 0 ? 0 : a.ent_off[nn + 1] - e0;
  int er[4], ec[4];
  float eg[4], eu[4];
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const int e = g + 8 * q;
    er[q] = -1; ec[q] = 0; eg[q] = 0.f; eu[q] = 0.f;
    if (e < ne) {
      er[q] = __ldg(a.ent_row + e0 + e);
      ec[q] = __ldg(a.ent_cls + e0 + e);
      eg[q] = sp_gain_at(a, nn, n < 0 ? 0 : (int)j, er[q]);
      eu[q] = __ldg(urow + ec[q]);
    }
  }
  float s, e;
  g8_item_sums<KC8>(u, er, ec, eu, eg, g0, C, g, s, e);
  if (g == 0 && n >= 0) {
    const float v = eig_value(e, s);
    a.eig[n] = v;
    if (!isfinite(v)) atomicOr(a.flags, CODA_B200_FLAG_NONFINITE_EIG);
  }
}

// the full pass's one-warp assembly (any C, any number of entries): one warp per sample position
template <int KC>
__global__ void __launch_bounds__(256) k_sample_eig_warp(const SampleEigArgs a) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  float* g0 = reinterpret_cast<float*>(smem_raw);
  const int C = a.C;
  const int H1 = (int)(a.T / C);
  for (int c = threadIdx.x; c < C; c += blockDim.x) g0[c] = a.gain[(size_t)c * H1];
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const long long j = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (j >= a.m) return;
  const int n = a.items[j];
  if (n < 0) return;
  constexpr int KR = KC > 0 ? KC : 1;
  const float* urow = a.U + (size_t)n * C;
  float u[KR];
  if (KC > 0) {
#pragma unroll
    for (int k = 0; k < KR; ++k) {
      const int c = lane + 32 * k;
      u[k] = c < C ? __ldg(urow + c) : 0.f;
    }
  }
  float s, e;
  warp_item_sums<KC>(urow, u, C, a.ent_off[n], a.ent_off[n + 1], a.ent_row, a.ent_cls, g0,
                     [&](int r) { return sp_gain_at(a, n, (int)j, r); }, lane, s, e);
  if (lane == 0) {
    const float v = eig_value(e, s);
    a.eig[n] = v;
    if (!isfinite(v)) atomicOr(a.flags, CODA_B200_FLAG_NONFINITE_EIG);
  }
}

extern "C" int coda_b200_sample_plan(const int32_t* items, int m, const int32_t* ent_off, const int32_t* ent_row,
                                     const uint16_t* ent_cls, const int32_t* heavy_off, int H, int C, int width,
                                     int32_t* hoff, int32_t* cursor, int32_t* tiles, int64_t* tile_off,
                                     int64_t* nheavy, coda_stream_t stream) {
  CODA_CHECK_ARG(items && ent_off && ent_row && ent_cls && heavy_off && hoff && cursor && tiles && tile_off && nheavy,
                 "sample_plan: null pointer");
  CODA_CHECK_ARG(m >= 1 && H >= 1 && C >= 2 && (width == 32 || width == 128), "sample_plan: bad m=%d C=%d width=%d",
                 m, C, width);
  const size_t smem = (size_t)C * 4;
  CODA_CHECK_ARG(smem <= 200 * 1024, "sample_plan: C=%d too large", C);
  CODA_CUDA_OK(cudaFuncSetAttribute(k_sample_plan, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  k_sample_plan<<<1, SP_THREADS, smem, as_stream(stream)>>>(items, m, ent_off, ent_row, ent_cls, heavy_off,
                                                            (long long)C * (1 + H), C, width, hoff, cursor,
                                                            reinterpret_cast<int4*>(tiles),
                                                            reinterpret_cast<long long*>(tile_off),
                                                            reinterpret_cast<long long*>(nheavy));
  CODA_LAUNCH_OK("k_sample_plan");
  return CODA_B200_OK;
}

extern "C" int coda_b200_sample_fill(const int32_t* items, int m, const uint16_t* hard, int H, int C,
                                     const int32_t* ent_off, const int32_t* ent_row, const uint16_t* ent_cls,
                                     const int32_t* heavy_off, const int32_t* hoff, int32_t* cursor, uint32_t* zmask,
                                     int32_t* row_of, uint16_t* row_cls, coda_stream_t stream) {
  CODA_CHECK_ARG(items && hard && ent_off && ent_row && ent_cls && heavy_off && hoff && cursor && zmask && row_of &&
                 row_cls, "sample_fill: null pointer");
  CODA_CHECK_ARG(m >= 1 && H >= 1 && H <= 1024, "sample_fill: bad m=%d H=%d", m, H);
  const int W = (H + 31) / 32;
  k_sample_fill<<<(unsigned)((m + 7) / 8), 256, 0, as_stream(stream)>>>(items, m, hard, H, W, ent_off, ent_row,
                                                                       ent_cls, heavy_off, (long long)C * (1 + H),
                                                                       hoff, cursor, zmask, row_of, row_cls);
  CODA_LAUNCH_OK("k_sample_fill");
  return CODA_B200_OK;
}

extern "C" int coda_b200_sample_gains(const float* tmpl, const float* scratch, const uint16_t* row_cls, int64_t cap,
                                      const int64_t* nheavy, int H, int C, const float* PB, const float* m0,
                                      const float* pi_hat, float* gain, coda_stream_t stream) {
  CODA_CHECK_ARG(tmpl && scratch && row_cls && nheavy && PB && m0 && pi_hat && gain && cap >= 0,
                 "sample_gains: null pointer");
  const int Hp = (H + 31) / 32 * 32;
  const long long T = (long long)C * (1 + H);
  int grid = (int)min((T + cap + 7) / 8, (long long)coda_sm_count() * 8);
  if (grid < 1) grid = 1;
  k_sample_gains<<<grid, 256, (size_t)2 * Hp * 4, as_stream(stream)>>>(tmpl, scratch, row_cls,
                                                                       reinterpret_cast<const long long*>(nheavy), T,
                                                                       H, Hp, PB, m0, pi_hat, gain);
  CODA_LAUNCH_OK("k_sample_gains");
  return CODA_B200_OK;
}

extern "C" int coda_b200_sample_eig(const int32_t* items, int m, const int32_t* hoff, const float* U, int C, int H,
                                    const int32_t* ent_off, const int32_t* ent_row, const uint16_t* ent_cls,
                                    const int32_t* heavy_off, const float* gain, int max_entries, float* eig,
                                    uint32_t* flags, coda_stream_t stream) {
  CODA_CHECK_ARG(items && hoff && U && ent_off && ent_row && ent_cls && heavy_off && gain && eig && flags,
                 "sample_eig: null pointer");
  CODA_CHECK_ARG(m >= 1 && C >= 2 && H >= 1, "sample_eig: bad dims");
  SampleEigArgs a;
  a.items = items; a.m = m; a.hoff = hoff; a.U = U; a.C = C; a.T = (long long)C * (1 + H);
  a.ent_off = ent_off; a.ent_row = ent_row; a.ent_cls = ent_cls; a.heavy_off = heavy_off; a.gain = gain;
  a.eig = eig; a.flags = flags;
  const size_t smem = (size_t)C * 4;
  CODA_CHECK_ARG(smem <= 220 * 1024, "sample_eig: C=%d does not fit shared memory", C);
  cudaStream_t st = as_stream(stream);
  // the kernel the full pass (coda_b200_gain_eig) takes for this C and max_entries, so the same arithmetic
  if (C <= 128 && max_entries >= 0 && max_entries <= 32) {
    const unsigned grid = (unsigned)((m + 31) / 32);
#define LAUNCH_SG8(K8) k_sample_eig_g8<K8><<<grid, 256, smem, st>>>(a)
    if (C <= 32) LAUNCH_SG8(4);
    else if (C <= 64) LAUNCH_SG8(8);
    else if (C <= 104) LAUNCH_SG8(13);
    else LAUNCH_SG8(16);
#undef LAUNCH_SG8
    CODA_LAUNCH_OK("k_sample_eig_g8");
    return CODA_B200_OK;
  }
  const unsigned grid = (unsigned)((m + 7) / 8);
#define LAUNCH_SW(KC)                                                                                              \
  do {                                                                                                             \
    CODA_CUDA_OK(cudaFuncSetAttribute(k_sample_eig_warp<KC>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
    k_sample_eig_warp<KC><<<grid, 256, smem, st>>>(a);                                                             \
  } while (0)
  if (C <= 32) LAUNCH_SW(1);
  else if (C <= 64) LAUNCH_SW(2);
  else if (C <= 128) LAUNCH_SW(4);
  else LAUNCH_SW(0);
#undef LAUNCH_SW
  CODA_LAUNCH_OK("k_sample_eig_warp");
  return CODA_B200_OK;
}

CODA_MODULE_ANCHOR(sample, k_sample_plan)
