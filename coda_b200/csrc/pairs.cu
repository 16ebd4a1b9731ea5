// Hypothetical-update "pairs" and the fused EIG quadrature kernel.
//
// A pair is (item b, class c) with the set Z = {h : p_h(b) = c} of models that would be "hit"
// if b were labeled c (coda.py:150-168).  Three exact reductions of the reference's dense
// (B, C, H, P) iteration space (coda.py:261-279):
//   * Z empty      -> the result depends on c only: one "template" pair per class;
//   * Z = {h'}     -> depends on (c, h') only: H template pairs per class;
//   * |Z| >= 2     -> a "heavy" pair, stored with its H-bit mask.
// Two orderings of the same rows:
//   * ROW ids (what is stored: cached P(best | hypothetical) rows, gains): the T = C*(1+H) template rows first,
//     class-major (c*(1+H) + 0 = Z empty, + 1 + h' = Z = {h'}), then the heavy rows ITEM-major -- the heavy rows of
//     item n are contiguous, ascending class -- so the per-step scoring pass (gain.cu) streams them in item order;
//   * the class-major WORK LIST the row kernels tile over: positions [cls_base[c], cls_base[c+1]) =
//     [z0 template | H singleton templates | heavy rows of c], with zmask[q] (the H-bit set Z) and row_of[q].
// Every item keeps a CSR entry list (row id, class), one entry per distinct predicted class, ascending class.
//
//   pair_count / pair_templates / pair_fill     build the structure from the hard predictions
//   pair_rows     coda.py:267-276 for a tile of 32 same-class rows: D = exp(Z . dL),
//                 prob = D . G_{z}, normalise (coda.py:114), information gain per row
#include "common.cuh"

#include <stdlib.h>

// ---------------------------------------------------------------------------------------
// structure build: one warp per item
// ---------------------------------------------------------------------------------------
__device__ __forceinline__ void warp_histogram(const uint16_t* __restrict__ hrow, int H, int lane, int* cnt) {
  for (int h = lane; h < H; h += 32) atomicAdd(&cnt[hrow[h]], 1);
  __syncwarp();
}
__device__ __forceinline__ void warp_histogram_clear(const uint16_t* __restrict__ hrow, int H, int lane, int* cnt) {
  __syncwarp();
  for (int h = lane; h < H; h += 32) cnt[hrow[h]] = 0;
  __syncwarp();
}

__global__ void __launch_bounds__(256) k_pair_count(const uint16_t* __restrict__ hard, int H, long long N, int C,
                                                    int32_t* __restrict__ ent_cnt, int32_t* __restrict__ heavy_cnt,
                                                    int32_t* __restrict__ cls_heavy) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  int* cnt_all = reinterpret_cast<int*>(smem_raw);   // [8][C]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  int* cnt = cnt_all + (size_t)warp * C;
  for (int c = lane; c < C; c += 32) cnt[c] = 0;
  __syncwarp();
  for (long long n = (long long)blockIdx.x * 8 + warp; n < N; n += (long long)gridDim.x * 8) {
    const uint16_t* hrow = hard + (size_t)n * H;
    warp_histogram(hrow, H, lane, cnt);
    int distinct = 0, heavy = 0;
    for (int c0 = 0; c0 < C; c0 += 32) {
      int c = c0 + lane;
      int k = c < C ? cnt[c] : 0;
      distinct += __popc(__ballot_sync(CODA_FULL, k >= 1));
      heavy += __popc(__ballot_sync(CODA_FULL, k >= 2));
      if (k >= 2) atomicAdd(&cls_heavy[c], 1);
    }
    if (lane == 0) {
      ent_cnt[n] = distinct;
      heavy_cnt[n] = heavy;
    }
    warp_histogram_clear(hrow, H, lane, cnt);
  }
}

// templates: pid = cls_base[c] + 0 (Z empty), cls_base[c] + 1 + h' (Z = {h'})
__global__ void k_pair_templates(int H, int C, int W, const long long* __restrict__ cls_base,
                                 uint32_t* __restrict__ zmask, int32_t* __restrict__ row_of) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)C * (H + 1)) return;
  const int c = (int)(i / (H + 1)), k = (int)(i % (H + 1));
  const long long pid = cls_base[c] + k;
  row_of[pid] = (int32_t)i;                       // template row id = c * (1 + H) + k
  for (int w = 0; w < W; ++w) zmask[(size_t)pid * W + w] = (k >= 1 && ((k - 1) >> 5) == w) ? (1u << ((k - 1) & 31)) : 0u;
}

__global__ void __launch_bounds__(256) k_pair_fill(const uint16_t* __restrict__ hard, int H, long long N, int C, int W,
                                                   const int32_t* __restrict__ ent_off,
                                                   const int32_t* __restrict__ heavy_off,
                                                   const long long* __restrict__ cls_base,
                                                   int32_t* __restrict__ cls_cursor, int32_t* __restrict__ ent_row,
                                                   uint16_t* __restrict__ ent_cls, uint32_t* __restrict__ zmask,
                                                   int32_t* __restrict__ row_of, uint16_t* __restrict__ row_cls) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  int* cnt_all = reinterpret_cast<int*>(smem_raw);   // [8][C]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  int* cnt = cnt_all + (size_t)warp * C;
  for (int c = lane; c < C; c += 32) cnt[c] = 0;
  __syncwarp();
  for (long long n = (long long)blockIdx.x * 8 + warp; n < N; n += (long long)gridDim.x * 8) {
    const uint16_t* hrow = hard + (size_t)n * H;
    warp_histogram(hrow, H, lane, cnt);
    int pos = ent_off[n];
    int next_row = C * (H + 1) + heavy_off[n];      // next heavy row id of this item
    for (int c0 = 0; c0 < C; c0 += 32) {
      const int cl = c0 + lane;
      const int k = cl < C ? cnt[cl] : 0;
      uint32_t present = __ballot_sync(CODA_FULL, k >= 1);
      while (present) {
        const int src = __ffs(present) - 1;
        present &= present - 1;
        const int c = c0 + src;
        const int kc = __shfl_sync(CODA_FULL, k, src);
        // mask words: lane w ends up holding word w  (H <= 1024)
        uint32_t myword = 0;
        for (int w = 0; w < W; ++w) {
          const int h = w * 32 + lane;
          const uint32_t bits = __ballot_sync(CODA_FULL, h < H && hrow[h] == c);
          if (lane == w) myword = bits;
        }
        int row;
        if (kc == 1) {
          const uint32_t has = __ballot_sync(CODA_FULL, myword != 0);
          const int wl = __ffs(has) - 1;
          const uint32_t word = __shfl_sync(CODA_FULL, myword, wl);
          const int hp = wl * 32 + (__ffs(word) - 1);
          row = c * (H + 1) + 1 + hp;                       // singleton template row
        } else {
          int slot = 0;
          if (lane == 0) slot = atomicAdd(&cls_cursor[c], 1);
          slot = __shfl_sync(CODA_FULL, slot, 0);
          const long long q = cls_base[c] + 1 + H + slot;     // position in the class-major work list
          row = next_row++;
          if (lane < W) zmask[(size_t)q * W + lane] = myword;
          if (lane == 0) {
            row_of[q] = row;
            row_cls[row - C * (H + 1)] = (uint16_t)c;
          }
        }
        if (lane == 0) {
          ent_row[pos] = row;
          ent_cls[pos] = (uint16_t)c;
        }
        ++pos;
      }
    }
    warp_histogram_clear(hrow, H, lane, cnt);
  }
}

extern "C" int coda_b200_pair_count(const uint16_t* hard, int H, int64_t N, int C, int32_t* ent_cnt,
                                    int32_t* heavy_cnt, int32_t* cls_heavy, coda_stream_t stream) {
  CODA_CHECK_ARG(hard && ent_cnt && heavy_cnt && cls_heavy, "pair_count: null pointer");
  CODA_CHECK_ARG(H <= 1024, "pair_count: H=%d > 1024 not supported", H);
  size_t smem = (size_t)8 * C * 4;
  CODA_CHECK_ARG(smem <= 200 * 1024, "pair_count: C=%d too large", C);
  CODA_CUDA_OK(cudaFuncSetAttribute(k_pair_count, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  int grid = (int)min((long long)(N + 7) / 8, (long long)coda_sm_count() * 8);
  k_pair_count<<<grid, 256, smem, as_stream(stream)>>>(hard, H, N, C, ent_cnt, heavy_cnt, cls_heavy);
  CODA_LAUNCH_OK("k_pair_count");
  return CODA_B200_OK;
}

extern "C" int coda_b200_pair_fill(const uint16_t* hard, int H, int64_t N, int C, const int32_t* ent_off,
                                   const int32_t* heavy_off, const int64_t* cls_base, int32_t* cls_cursor,
                                   int32_t* ent_row, uint16_t* ent_cls, uint32_t* zmask, int32_t* row_of,
                                   uint16_t* row_cls, coda_stream_t stream) {
  CODA_CHECK_ARG(hard && ent_off && heavy_off && cls_base && cls_cursor && ent_row && ent_cls && zmask && row_of && row_cls,
                 "pair_fill: null pointer");
  CODA_CHECK_ARG(H <= 1024, "pair_fill: H=%d > 1024 not supported", H);
  const int W = (H + 31) / 32;
  long long nt = (long long)C * (H + 1);
  k_pair_templates<<<(unsigned)((nt + 255) / 256), 256, 0, as_stream(stream)>>>(
      H, C, W, reinterpret_cast<const long long*>(cls_base), zmask, row_of);
  CODA_LAUNCH_OK("k_pair_templates");
  size_t smem = (size_t)8 * C * 4;
  CODA_CUDA_OK(cudaFuncSetAttribute(k_pair_fill, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  int grid = (int)min((long long)(N + 7) / 8, (long long)coda_sm_count() * 8);
  k_pair_fill<<<grid, 256, smem, as_stream(stream)>>>(hard, H, N, C, W, ent_off, heavy_off,
                                                      reinterpret_cast<const long long*>(cls_base), cls_cursor,
                                                      ent_row, ent_cls, zmask, row_of, row_cls);
  CODA_LAUNCH_OK("k_pair_fill");
  return CODA_B200_OK;
}

// ---------------------------------------------------------------------------------------
// pair_rows: the fused quadrature for a tile of TPAIR same-class pairs (SIMT fp32).
//   phase A  logD[p][x] = sum_h z[p][h] * dL[c][h][x]      threads <-> quadrature node x
//   phase B  a_k[p][h]  = sum_x G_k[c][x][h] * D[p][x]      threads <-> model h  (k = miss, hit)
//   final    prob = z ? a_1 : a_0 ; normalise over h ; gain = sum_h f(m0) - f(m0 + pi_c (ph - PB_c))
// ---------------------------------------------------------------------------------------
#define TPAIR 32
#define TPAD (TPAIR + 4)   // padded row (floats): 16-byte aligned, conflict-free 128-bit rows
#define NODES 256

struct PairRowsArgs {
  const int4* tiles;          // (class, first pid, count, unused)
  const uint32_t* zmask;      // [npairs][W]   (work-list order)
  const int32_t* row_of;      // [npairs]      work-list position -> row id
  const float* dL;            // [C][H][P]
  const float* G0T;           // [C][P][Hp]
  const float* G1T;           // [C][P][Hp]
  const float* PB;            // [C][Hp]
  const float* m0;            // [Hp]
  const float* pi_hat;        // [C]
  float* ph_cache;            // [npairs][Hp] or null
  float* gain;                // [npairs]
  uint32_t* flags;
  const long long* sel;       // optional: device-resident {idx, class}; then only that class's tiles run
  const long long* tile_off;  // [C+1] first tile of every class (needed with sel)
  int H, Hp, W;
};

template <int HB>   // models per pass: 32, 64, 128 or 256
__global__ void __launch_bounds__(256) k_pair_rows(PairRowsArgs a, int tile0) {
  constexpr int NG = 256 / HB;        // pair groups working side by side in phase B
  constexpr int PPG = TPAIR / NG;     // pairs per group
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int H = a.H, Hp = a.Hp, W = a.W;
  float* Ds = reinterpret_cast<float*>(smem_raw);                 // [NODES][TPAD]
  float* zf = Ds + NODES * TPAD;                                  // [Hp][TPAD]   (phase A)
  float* Ps = zf;                                                 // [TPAIR][Hp]  (phase B, aliases zf)
  const size_t zf_floats = (size_t)Hp * TPAD > (size_t)TPAIR * Hp ? (size_t)Hp * TPAD : (size_t)TPAIR * Hp;
  uint32_t* zs = reinterpret_cast<uint32_t*>(zf + zf_floats);     // [TPAIR][W]
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (a.sel) {   // host-free loop: the class to refresh is only known on the device
    const long long t = a.sel[1];
    tile0 = (int)a.tile_off[t];
    if ((long long)blockIdx.x >= a.tile_off[t + 1] - a.tile_off[t]) return;
  }
  const int4 tile = a.tiles[tile0 + blockIdx.x];
  const int c = tile.x, pid0 = tile.y, cnt = tile.z;

  for (int i = tid; i < TPAIR * W; i += 256) {
    int p = i / W, w = i % W;
    zs[i] = p < cnt ? a.zmask[(size_t)(pid0 + p) * W + w] : 0u;
  }
  __syncthreads();
  for (int i = tid; i < Hp * TPAIR; i += 256) {
    int h = i / TPAIR, p = i % TPAIR;
    zf[h * TPAD + p] = (float)((zs[p * W + (h >> 5)] >> (h & 31)) & 1u);
  }
  __syncthreads();

  // ---- phase A -------------------------------------------------------------------------
  {
    float acc[TPAIR];
#pragma unroll
    for (int p = 0; p < TPAIR; ++p) acc[p] = 0.f;
    const float* dl = a.dL + (size_t)c * H * NODES + tid;
    int h = 0;
    for (; h + 4 <= H; h += 4) {
      float d[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) d[k] = __ldg(dl + (size_t)(h + k) * NODES);
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float4* zr = reinterpret_cast<const float4*>(zf + (h + k) * TPAD);
#pragma unroll
        for (int q = 0; q < TPAIR / 4; ++q) {
          float4 z4 = zr[q];
          acc[4 * q + 0] = fmaf(z4.x, d[k], acc[4 * q + 0]);
          acc[4 * q + 1] = fmaf(z4.y, d[k], acc[4 * q + 1]);
          acc[4 * q + 2] = fmaf(z4.z, d[k], acc[4 * q + 2]);
          acc[4 * q + 3] = fmaf(z4.w, d[k], acc[4 * q + 3]);
        }
      }
    }
    for (; h < H; ++h) {
      float d = __ldg(dl + (size_t)h * NODES);
      const float4* zr = reinterpret_cast<const float4*>(zf + h * TPAD);
#pragma unroll
      for (int q = 0; q < TPAIR / 4; ++q) {
        float4 z4 = zr[q];
        acc[4 * q + 0] = fmaf(z4.x, d, acc[4 * q + 0]);
        acc[4 * q + 1] = fmaf(z4.y, d, acc[4 * q + 1]);
        acc[4 * q + 2] = fmaf(z4.z, d, acc[4 * q + 2]);
        acc[4 * q + 3] = fmaf(z4.w, d, acc[4 * q + 3]);
      }
    }
    float4* drow = reinterpret_cast<float4*>(Ds + tid * TPAD);
#pragma unroll
    for (int q = 0; q < TPAIR / 4; ++q)
      drow[q] = make_float4(expf(acc[4 * q + 0]), expf(acc[4 * q + 1]), expf(acc[4 * q + 2]), expf(acc[4 * q + 3]));
  }
  __syncthreads();   // Ds complete; zf no longer needed (Ps aliases it)

  // ---- phase B -------------------------------------------------------------------------
  {
    const int hl = tid % HB, grp = tid / HB;
    const int pbase = grp * PPG;
    for (int h0 = 0; h0 < Hp; h0 += HB) {
      const int h = h0 + hl;
      float a0[PPG], a1[PPG];
#pragma unroll
      for (int p = 0; p < PPG; ++p) { a0[p] = 0.f; a1[p] = 0.f; }
      if (h < Hp) {
        const float* g0p = a.G0T + (size_t)c * NODES * Hp + h;
        const float* g1p = a.G1T + (size_t)c * NODES * Hp + h;
        for (int x = 0; x < NODES; x += 4) {
          float g0[4], g1[4];
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            g0[k] = __ldg(g0p + (size_t)(x + k) * Hp);
            g1[k] = __ldg(g1p + (size_t)(x + k) * Hp);
          }
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            const float4* dr = reinterpret_cast<const float4*>(Ds + (x + k) * TPAD + pbase);
#pragma unroll
            for (int q = 0; q < PPG / 4; ++q) {
              float4 d4 = dr[q];
              a0[4 * q + 0] = fmaf(g0[k], d4.x, a0[4 * q + 0]);
              a0[4 * q + 1] = fmaf(g0[k], d4.y, a0[4 * q + 1]);
              a0[4 * q + 2] = fmaf(g0[k], d4.z, a0[4 * q + 2]);
              a0[4 * q + 3] = fmaf(g0[k], d4.w, a0[4 * q + 3]);
              a1[4 * q + 0] = fmaf(g1[k], d4.x, a1[4 * q + 0]);
              a1[4 * q + 1] = fmaf(g1[k], d4.y, a1[4 * q + 1]);
              a1[4 * q + 2] = fmaf(g1[k], d4.z, a1[4 * q + 2]);
              a1[4 * q + 3] = fmaf(g1[k], d4.w, a1[4 * q + 3]);
            }
          }
        }
        const int wsel = h >> 5, bsel = h & 31;
#pragma unroll
        for (int p = 0; p < PPG; ++p) {
          const uint32_t bit = (zs[(pbase + p) * W + wsel] >> bsel) & 1u;
          Ps[(size_t)(pbase + p) * Hp + h] = bit ? a1[p] : a0[p];
        }
      }
    }
  }
  __syncthreads();

  // ---- normalise + information gain: one warp per pair ---------------------------------
  const bool want_gain = a.gain != nullptr;       // cache-only refresh: m0 / pi_hat may not be final yet
  const float pic = want_gain ? a.pi_hat[c] : 0.f;
  const float* pbrow = a.PB + (size_t)c * Hp;
  uint32_t bad = 0;
  for (int p = warp; p < cnt; p += 8) {
    const float* pr = Ps + (size_t)p * Hp;
    const int row = a.row_of[pid0 + p];
    float s = 0.f;
    for (int h = lane; h < H; h += 32) s += pr[h];
    s = warp_sum(s);
    if (!isfinite(s)) bad |= CODA_B200_FLAG_NONFINITE_EIG;
    const float den = fmaxf(s, 1e-30f);                         // coda.py:114
    if (s < 0.9999e-30f) bad |= CODA_B200_FLAG_ROWSUM_WARN;     // util.py:37-39: the normalised row does not sum to 1
    float g = 0.f;
    float* cache = a.ph_cache ? a.ph_cache + (size_t)row * Hp : nullptr;
    for (int h = lane; h < Hp; h += 32) {
      float ph = 0.f;
      if (h < H) {
        ph = pr[h] / den;
        if (ph < -1e-12f) bad |= CODA_B200_FLAG_NEGATIVE_PROB;  // util.py:33-35
        if (want_gain) {
          const float m = a.m0[h];
          const float mix = m + pic * (ph - pbrow[h]);          // coda.py:274-275
          g += ent_term(m) - ent_term(mix);                     // coda.py:254, 276
        }
      }
      if (cache) cache[h] = ph;
    }
    if (want_gain) {
      g = warp_sum(g);
      if (lane == 0) a.gain[row] = g;
    }
  }
  if (bad) atomicOr(a.flags, bad);
}

static size_t pair_rows_smem(int Hp, int W) {
  size_t zf_floats = (size_t)Hp * TPAD > (size_t)TPAIR * Hp ? (size_t)Hp * TPAD : (size_t)TPAIR * Hp;
  return ((size_t)NODES * TPAD + zf_floats) * 4 + (size_t)TPAIR * W * 4;
}

extern "C" int coda_b200_pair_rows(const int32_t* tiles, int tile_lo, int tile_hi, const uint32_t* zmask,
                                   const int32_t* row_of, const float* dL, const float* G0T, const float* G1T, const float* PB,
                                   const float* m0, const float* pi_hat, int H, float* ph_cache, float* gain,
                                   const int64_t* sel, const int64_t* tile_off, uint32_t* flags,
                                   coda_stream_t stream) {
  CODA_CHECK_ARG(tiles && zmask && row_of && dL && G0T && G1T && PB && flags, "pair_rows: null pointer");
  CODA_CHECK_ARG((gain && m0 && pi_hat) || (!gain && ph_cache), "pair_rows: need gain (+m0, pi_hat) or ph_cache");
  CODA_CHECK_ARG(H >= 1 && H <= 1024, "pair_rows: H=%d out of range", H);
  if (tile_hi <= tile_lo) return CODA_B200_OK;
  PairRowsArgs a;
  a.tiles = reinterpret_cast<const int4*>(tiles);
  a.zmask = zmask; a.row_of = row_of; a.dL = dL; a.G0T = G0T; a.G1T = G1T; a.PB = PB; a.m0 = m0; a.pi_hat = pi_hat;
  a.ph_cache = ph_cache; a.gain = gain; a.flags = flags;
  a.sel = reinterpret_cast<const long long*>(sel);
  a.tile_off = reinterpret_cast<const long long*>(tile_off);
  CODA_CHECK_ARG(!sel || tile_off, "pair_rows: sel needs tile_off");
  a.H = H; a.Hp = (H + 31) / 32 * 32; a.W = a.Hp / 32;
  const size_t smem = pair_rows_smem(a.Hp, a.W);
  CODA_CHECK_ARG(smem <= 227 * 1024, "pair_rows: H=%d needs %zu B shared memory", H, smem);
  const int ntiles = tile_hi - tile_lo;
  cudaStream_t st = as_stream(stream);
#define LAUNCH_PR(HB)                                                                                        \
  do {                                                                                                       \
    CODA_CUDA_OK(cudaFuncSetAttribute(k_pair_rows<HB>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
    k_pair_rows<HB><<<ntiles, 256, smem, st>>>(a, tile_lo);                                                  \
  } while (0)
  if (a.Hp <= 32) LAUNCH_PR(32);
  else if (a.Hp <= 64) LAUNCH_PR(64);
  else if (a.Hp <= 128) LAUNCH_PR(128);
  else LAUNCH_PR(256);
#undef LAUNCH_PR
  CODA_LAUNCH_OK("k_pair_rows");
  return CODA_B200_OK;
}


CODA_MODULE_ANCHOR(pairs, k_pair_count)
