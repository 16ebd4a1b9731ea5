// pair_rows on the Hopper tensor cores (wgmma, fp32 accumulators in registers), for Hp = 32..256 models.
//
// Same arithmetic as k_pair_rows (pairs.cu) for a tile of 128 same-class pairs, cast as two GEMMs:
//
//   phase A   logD[128 x 256] = Z[128 x Hp] . dL_c[Hp x 256]             K = Hp (models)
//             Z in {0,1} is exact in bf16; dL is split into 3 bf16 limbs (24 mantissa bits) -> 3 MMAs
//   epilogue  D = exp(logD)  (registers -> exp -> two bf16 limbs -> shared memory, A-operand layout)
//   phase B   prob_k[128 x Hp] = D[128 x 256] . G_k[256 x Hp],  k = miss, hit    K = 256 (quadrature nodes)
//             D = Dhi + Dlo, G = Ghi + Glo (bf16 limbs); Dhi.Ghi + Dhi.Glo + Dlo.Ghi -> 3 MMAs per table
//   epilogue  select hit/miss column by the pair's mask bit, normalise over models (coda.py:114), information gain
//             (coda.py:274-276), cached row write.
//
// Two consumer warpgroups, one per 64 pairs of the tile; every MMA is a wgmma m64n32k16 (one 32-model / 32-node column
// block; 32 models are also one word of the pair's mask).  Operands are staged by 1-D bulk TMA (cp.async.bulk, no tensor
// map): the class tables are stored in HBM already in the no-swizzle K-major core-matrix order (8 rows x 16 bytes per
// core, see tables.cu), so one K-chunk of all limbs is a single contiguous blob.  The accumulators of phase B for both
// tables over all Hp columns would not fit the register file at Hp > 128, so phase B then runs in two passes over
// column halves (the G stream is read twice; it is per class and stays in L2 across the class's tiles).
#include "common.cuh"

#include <cuda_bf16.h>

namespace {

constexpr int TC_M = 128;        // pairs per tile
constexpr int TC_NODES = 256;    // quadrature nodes
constexpr int KA = 32;           // models per phase-A chunk
constexpr int KB = 16;           // nodes per phase-B chunk
constexpr int STAGES_A = 3;
constexpr int STAGES_B = 3;
constexpr int TC_THREADS = 256;  // 2 warpgroups x 64 pairs
constexpr int NBMAX = 4;         // 32-column blocks per phase-B pass

struct TcArgs {
  const int4* tiles;             // (class, first pid, count <= 128, unused)
  const uint32_t* zmask;         // [npairs][W]   (work-list order)
  const int32_t* row_of;         // [npairs]      work-list position -> row id
  const __nv_bfloat16* dLb;      // [C][Hp/KA][3][TC_NODES x KA]      core-matrix order, rows = nodes
  const __nv_bfloat16* Gb;       // [C][TC_NODES/KB][4][Hp x KB]      core-matrix order, rows = models
  const float* PB;               // [C][Hp]
  const float* m0;               // [Hp]
  const float* pi_hat;           // [C]
  float* ph_cache;               // [npairs][Hp] or null
  float* gain;                   // [npairs] or null
  uint32_t* flags;
  const long long* sel;
  const long long* tile_off;
  int H, Hp, W;
};

// D[64 x 32] (+)= A[64 x 16] . B[16 x 32]^T, both operands bf16 in shared memory (K-major), fp32 accumulators
__device__ __forceinline__ void mma_n32(float (&d)[16], uint64_t adesc, uint64_t bdesc, uint32_t accum) {
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "setp.ne.b32 p, %18, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, 0, 0;\n\t"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
        "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(adesc), "l"(bdesc), "r"(accum));
}

__device__ __forceinline__ uint32_t pack_bf16(float a, float b) {
  __nv_bfloat162 t = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&t);
}

// byte offset of element (row r, column k) of an operand tile stored as [k_core][r_core][8 rows][8 bf16]
__device__ __forceinline__ uint32_t core_off(int r, int k, int rows) {
  return (uint32_t)(((k >> 3) * (rows >> 3) + (r >> 3)) * 128 + (r & 7) * 16 + (k & 7) * 2);
}

// accumulator fragment of wgmma m64nN (fp32): register 4 j + 2 i + e holds row (16 warp + lane / 4 + 8 i),
// column (8 j + 2 (lane % 4) + e)
__device__ __forceinline__ int frag_col(int j, int e, int lane) { return 8 * j + 2 * (lane & 3) + e; }

__global__ void __launch_bounds__(TC_THREADS, 1) k_pair_rows_tc(TcArgs a, int tile0) {
  extern __shared__ __align__(1024) unsigned char smem[];
  const int H = a.H, Hp = a.Hp, W = a.W;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int wg = warp >> 2;                                   // warpgroup: pairs [64 wg, 64 wg + 64)
  const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);    // this thread's two pairs: r0 and r0 + 8
  if (a.sel) {
    const long long t = a.sel[1];
    tile0 = (int)a.tile_off[t];
    if ((long long)blockIdx.x >= a.tile_off[t + 1] - a.tile_off[t]) return;
  }
  const int4 tile = a.tiles[tile0 + blockIdx.x];
  const int c = tile.x, pid0 = tile.y, cnt = tile.z;

  // ---- shared memory carve-up ----------------------------------------------------------------
  // [0, 64K)           phase A: Z operand                       | phase B: D hi
  // [64K, 208K)        phase A: 3 stages x 48K (3 limbs x 256 x KA bf16)
  // [64K, 128K)                                                 | phase B: D lo
  // [128K, 224K)                                                | phase B: 3 stages x 32K (4 tables x Hp x KB)
  // tail               barriers, m0 / PB rows
  unsigned char* opA = smem;
  unsigned char* stg = smem + 128 * 1024;
  unsigned char* stgA = smem + 64 * 1024;
  unsigned char* tail = stg + 96 * 1024;
  uint64_t* fullA = reinterpret_cast<uint64_t*>(tail);        // [STAGES_A]
  uint64_t* emptyA = fullA + STAGES_A;                        // [STAGES_A]
  uint64_t* fullB = emptyA + STAGES_A;                        // [STAGES_B]
  uint64_t* emptyB = fullB + STAGES_B;                        // [STAGES_B]
  float* m0s = reinterpret_cast<float*>(emptyB + STAGES_B + 2);   // [Hp]
  float* pbs = m0s + Hp;                                      // [Hp]

  const int nka = Hp / KA;                       // phase-A chunks
  constexpr int nkb = TC_NODES / KB;             // phase-B chunks per pass
  const int nblk = Hp / 32;                      // 32-model column blocks
  const int npass = nblk > NBMAX ? 2 : 1;
  const int nb0 = (nblk + npass - 1) / npass;    // blocks of pass 0 (pass 1 takes the rest)
  const int nqb = npass * nkb;                   // phase-B chunks over all passes
  const uint32_t bytesA = 3u * TC_NODES * KA * 2u;          // per stage
  const uint32_t tabB = (uint32_t)Hp * KB * 2u;             // one table, one chunk
  const uint32_t bytesB = 4u * tabB;
  const unsigned char* srcA = reinterpret_cast<const unsigned char*>(a.dLb) + (size_t)c * nka * bytesA;
  const unsigned char* srcB = reinterpret_cast<const unsigned char*>(a.Gb) + (size_t)c * nkb * bytesB;

  if (tid == 0) {
    for (int i = 0; i < STAGES_A; ++i) { mbar_init(&fullA[i], 1); mbar_init(&emptyA[i], TC_THREADS / 32); }
    for (int i = 0; i < STAGES_B; ++i) { mbar_init(&fullB[i], 1); mbar_init(&emptyB[i], TC_THREADS / 32); }
    mbar_fence_init();
  }
  const bool want_gain = a.gain != nullptr;
  for (int h = tid; h < Hp; h += TC_THREADS) {
    m0s[h] = (want_gain && h < H) ? a.m0[h] : 0.f;
    pbs[h] = a.PB[(size_t)c * Hp + h];
  }
  // ---- Z operand: row = pair, K = models, bf16 {0, 1} ------------------------------------------
#pragma unroll 1
  for (int i = tid; i < TC_M * W; i += TC_THREADS) {
    const int row = i % TC_M, w = i / TC_M;
    const uint32_t z = row < cnt ? a.zmask[(size_t)(pid0 + row) * W + w] : 0u;
#pragma unroll
    for (int q = 0; q < 4; ++q) {   // 8 models -> one 16-byte core row
      const uint32_t b = z >> (8 * q);
      uint4 v;
      v.x = ((b & 1u) ? 0x3F80u : 0u) | ((b & 2u) ? 0x3F800000u : 0u);
      v.y = ((b & 4u) ? 0x3F80u : 0u) | ((b & 8u) ? 0x3F800000u : 0u);
      v.z = ((b & 16u) ? 0x3F80u : 0u) | ((b & 32u) ? 0x3F800000u : 0u);
      v.w = ((b & 64u) ? 0x3F80u : 0u) | ((b & 128u) ? 0x3F800000u : 0u);
      *reinterpret_cast<uint4*>(opA + core_off(row, w * 32 + q * 8, TC_M)) = v;
    }
  }
  fence_proxy_async_smem();
  __syncthreads();
  if (tid == 0) {
    for (int kc = 0; kc < STAGES_A && kc < nka; ++kc) {
      mbar_expect_tx(&fullA[kc], bytesA);
      tma_load_1d(stgA + (size_t)kc * 48 * 1024, srcA + (size_t)kc * bytesA, bytesA, &fullA[kc]);
    }
  }
  const uint32_t opA_s = smem_u32(opA), stg_s = smem_u32(stg), stgA_s = smem_u32(stgA);
  const uint32_t a_rows = (uint32_t)(wg * 8) * 128;          // this warpgroup's 8 row cores
  constexpr uint32_t LBO_A = (TC_M / 8) * 128;

  // ---- phase A: logD = Z . dL (3 limbs) --------------------------------------------------------
  // Thread 0 refills the stage of chunk kc - 1 once both warpgroups have released it, STAGES_A - 1 chunks ahead.
  float acc[2][NBMAX][16];        // phase A: acc[b / 4][b % 4] = node block b; phase B: acc[table][block]
  for (int kc = 0; kc < nka; ++kc) {
    const int s = kc % STAGES_A;
    if (tid == 0 && kc >= 1 && kc - 1 + STAGES_A < nka) {
      const int q = kc - 1 + STAGES_A, sq = q % STAGES_A;
      mbar_wait(&emptyA[sq], ((kc - 1) / STAGES_A) & 1);
      mbar_expect_tx(&fullA[sq], bytesA);
      tma_load_1d(stgA + (size_t)sq * 48 * 1024, srcA + (size_t)q * bytesA, bytesA, &fullA[sq]);
    }
    __syncwarp();
    mbar_wait(&fullA[s], (kc / STAGES_A) & 1);
    wg_fence();
#pragma unroll
    for (int limb = 0; limb < 3; ++limb) {
#pragma unroll
      for (int ks = 0; ks < KA / 16; ++ks) {
        // A: Z tile [k_core][16 r_core], this warpgroup's rows; advance 2 k-cores per K = 16 step
        const uint64_t ad = wg_desc(opA_s + (uint32_t)(kc * (KA / 8) + ks * 2) * LBO_A + a_rows, LBO_A, 128);
        const uint32_t bb = stgA_s + (uint32_t)s * 48 * 1024 + (uint32_t)limb * (TC_NODES * KA * 2) +
                            (uint32_t)(ks * 2) * (TC_NODES / 8) * 128;
        const uint32_t first = (kc | limb | ks) ? 1u : 0u;
#pragma unroll
        for (int b = 0; b < TC_NODES / 32; ++b)   // B: limb tile [4 k_core][32 r_core], 32-node block b
          mma_n32(acc[b >> 2][b & 3], ad, wg_desc(bb + (uint32_t)b * 4 * 128, (TC_NODES / 8) * 128, 128), first);
      }
    }
    wg_commit();
    wg_wait0();
    __syncwarp();
    if (lane == 0) mbar_arrive(&emptyA[s]);
  }
  __syncthreads();                               // every phase-A read is done: D lo and the phase-B stages may land

  if (tid == 0) {
    for (int q = 0; q < STAGES_B && q < nqb; ++q) {
      mbar_expect_tx(&fullB[q], bytesB);
      tma_load_1d(stg + (size_t)q * 32 * 1024, srcB + (size_t)(q % nkb) * bytesB, bytesB, &fullB[q]);
    }
  }

  // ---- epilogue A: D = exp(logD) -> bf16 hi / lo limbs in the A-operand layout ---------------------
  {
    unsigned char* dhi = opA;
    unsigned char* dlo = opA + 64 * 1024;
#pragma unroll
    for (int b = 0; b < TC_NODES / 32; ++b) {
#pragma unroll
      for (int j = 0; j < 4; ++j) {
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          const float* v = &acc[b >> 2][b & 3][4 * j + 2 * i];
          const float d0 = __expf(v[0]), d1 = __expf(v[1]);   // ex2.approx: 2 ulp, far inside the 16-bit limb pair D is cut into
          const __nv_bfloat16 h0 = __float2bfloat16_rn(d0), h1 = __float2bfloat16_rn(d1);
          const uint32_t hi = (uint32_t)__bfloat16_as_ushort(h0) | ((uint32_t)__bfloat16_as_ushort(h1) << 16);
          const uint32_t lo = pack_bf16(d0 - __bfloat162float(h0), d1 - __bfloat162float(h1));
          const uint32_t off = core_off(r0 + 8 * i, b * 32 + frag_col(j, 0, lane), TC_M);
          *reinterpret_cast<uint32_t*>(dhi + off) = hi;
          *reinterpret_cast<uint32_t*>(dlo + off) = lo;
        }
      }
    }
  }
  fence_proxy_async_smem();
  __syncthreads();

  // ---- phase B: prob_k = D . G_k, one pass per column half --------------------------------------------
  float keep[NBMAX][16];          // selected probabilities of pass 0 when there are two passes
  float sum[2] = {0.f, 0.f};      // row sums of rows r0, r0 + 8 (this thread's columns)
  const uint32_t lboB = (uint32_t)(Hp / 8) * 128;
  for (int pass = 0; pass < npass; ++pass) {
    const int blo = pass * nb0, nbp = min(nblk - blo, nb0);
    for (int kc = 0; kc < nkb; ++kc) {
      const int q = pass * nkb + kc, s = q % STAGES_B;
      if (tid == 0 && q >= 1 && q - 1 + STAGES_B < nqb) {
        const int qn = q - 1 + STAGES_B, sn = qn % STAGES_B;
        mbar_wait(&emptyB[sn], ((q - 1) / STAGES_B) & 1);
        mbar_expect_tx(&fullB[sn], bytesB);
        tma_load_1d(stg + (size_t)sn * 32 * 1024, srcB + (size_t)(qn % nkb) * bytesB, bytesB, &fullB[sn]);
      }
      __syncwarp();
      mbar_wait(&fullB[s], (q / STAGES_B) & 1);
      wg_fence();
      const uint64_t ahi = wg_desc(opA_s + (uint32_t)(kc * 2) * LBO_A + a_rows, LBO_A, 128);
      const uint64_t alo = wg_desc(opA_s + 64 * 1024 + (uint32_t)(kc * 2) * LBO_A + a_rows, LBO_A, 128);
      const uint32_t sb = stg_s + (uint32_t)s * 32 * 1024 + (uint32_t)blo * 4 * 128;
      const uint32_t first = kc ? 1u : 0u;
#pragma unroll
      for (int k = 0; k < 2; ++k) {              // k = 0 miss table (G0), 1 hit table (G1)
#pragma unroll
        for (int b = 0; b < NBMAX; ++b) {
          if (b < nbp) {                         // warp-uniform
            const uint64_t ghi = wg_desc(sb + (uint32_t)(2 * k) * tabB + (uint32_t)b * 4 * 128, lboB, 128);
            const uint64_t glo = wg_desc(sb + (uint32_t)(2 * k + 1) * tabB + (uint32_t)b * 4 * 128, lboB, 128);
            mma_n32(acc[k][b], ahi, ghi, first);
            mma_n32(acc[k][b], ahi, glo, 1u);
            mma_n32(acc[k][b], alo, ghi, 1u);
          }
        }
      }
      wg_commit();
      wg_wait0();
      __syncwarp();
      if (lane == 0) mbar_arrive(&emptyB[s]);
    }
    // select hit / miss by the pair's mask bit; the selection lands in keep (pass 0 of two) or acc[0] (last pass)
#pragma unroll
    for (int b = 0; b < NBMAX; ++b) {
      if (b < nbp) {
        uint32_t z[2];                           // mask words (32 models) of both rows for this block
#pragma unroll
        for (int i = 0; i < 2; ++i) z[i] = r0 + 8 * i < cnt ? a.zmask[(size_t)(pid0 + r0 + 8 * i) * W + blo + b] : 0u;
#pragma unroll
        for (int r = 0; r < 16; ++r) {
          const int i = (r >> 1) & 1, col = frag_col(r >> 2, r & 1, lane);
          const float v = ((z[i] >> col) & 1u) ? acc[1][b][r] : acc[0][b][r];
          sum[i] += v;
          if (pass + 1 < npass) keep[b][r] = v;
          else acc[0][b][r] = v;
        }
      }
    }
  }

  // ---- epilogue B: normalise, gain, cached rows --------------------------------------------------
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    sum[i] += __shfl_xor_sync(CODA_FULL, sum[i], 1);
    sum[i] += __shfl_xor_sync(CODA_FULL, sum[i], 2);
  }
  const float pic = want_gain ? a.pi_hat[c] : 0.f;
  uint32_t bad = 0;
  float g[2] = {0.f, 0.f};
  int orow[2];
  float* cache[2];
  float rden[2];
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int row = r0 + 8 * i;
    orow[i] = row < cnt ? a.row_of[pid0 + row] : 0;
    cache[i] = (a.ph_cache && row < cnt) ? a.ph_cache + (size_t)orow[i] * Hp : nullptr;
    rden[i] = 1.0f / fmaxf(sum[i], 1e-30f);                       // coda.py:114
    if (row < cnt && (lane & 3) == 0) {
      if (!isfinite(sum[i])) bad |= CODA_B200_FLAG_NONFINITE_EIG;
      if (sum[i] < 0.9999e-30f) bad |= CODA_B200_FLAG_ROWSUM_WARN;   // util.py:37-39
    }
  }
#pragma unroll
  for (int pass = 0; pass < 2; ++pass) {
    if (pass < npass) {
      const int blo = pass * nb0, nbp = min(nblk - blo, nb0);
#pragma unroll
      for (int b = 0; b < NBMAX; ++b) {
        if (b < nbp) {
#pragma unroll
          for (int r = 0; r < 16; r += 2) {
            const int i = (r >> 1) & 1;
            const int h0 = (blo + b) * 32 + frag_col(r >> 2, 0, lane);
            float ph[2];
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int h = h0 + e;
              const float v = (pass + 1 < npass) ? keep[b][r + e] : acc[0][b][r + e];
              ph[e] = h < H ? v * rden[i] : 0.f;
              if (ph[e] < -1e-12f) bad |= CODA_B200_FLAG_NEGATIVE_PROB;          // util.py:33-35
              if (want_gain && h < H) {
                const float m = m0s[h];
                g[i] += ent_term(m) - ent_term(m + pic * (ph[e] - pbs[h]));      // coda.py:254, 274-276
              }
            }
            if (cache[i]) *reinterpret_cast<float2*>(cache[i] + h0) = make_float2(ph[0], ph[1]);
          }
        }
      }
    }
  }
  if (want_gain) {
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      g[i] += __shfl_xor_sync(CODA_FULL, g[i], 1);
      g[i] += __shfl_xor_sync(CODA_FULL, g[i], 2);
      if ((lane & 3) == 0 && r0 + 8 * i < cnt) a.gain[orow[i]] = g[i];
    }
  }
  if (bad) atomicOr(a.flags, bad);
}

}  // namespace

extern "C" int coda_b200_pair_rows_tc(const int32_t* tiles128, int tile_lo, int tile_hi, const uint32_t* zmask,
                                      const int32_t* row_of, const void* dLb, const void* Gb, const float* PB, const float* m0,
                                      const float* pi_hat, int H, float* ph_cache, float* gain, const int64_t* sel,
                                      const int64_t* tile_off, uint32_t* flags, coda_stream_t stream) {
  CODA_CHECK_ARG(tiles128 && zmask && row_of && dLb && Gb && PB && flags, "pair_rows_tc: null pointer");
  CODA_CHECK_ARG((gain && m0 && pi_hat) || (!gain && ph_cache), "pair_rows_tc: need gain (+m0, pi_hat) or ph_cache");
  CODA_CHECK_ARG(!sel || tile_off, "pair_rows_tc: sel needs tile_off");
  const int Hp = (H + 31) / 32 * 32;
  CODA_CHECK_ARG(H >= 1 && Hp <= 256, "pair_rows_tc: H=%d needs the SIMT kernel", H);
  if (tile_hi <= tile_lo) return CODA_B200_OK;
  TcArgs a;
  a.tiles = reinterpret_cast<const int4*>(tiles128);
  a.zmask = zmask;
  a.row_of = row_of;
  a.dLb = reinterpret_cast<const __nv_bfloat16*>(dLb);
  a.Gb = reinterpret_cast<const __nv_bfloat16*>(Gb);
  a.PB = PB; a.m0 = m0; a.pi_hat = pi_hat; a.ph_cache = ph_cache; a.gain = gain; a.flags = flags;
  a.sel = reinterpret_cast<const long long*>(sel);
  a.tile_off = reinterpret_cast<const long long*>(tile_off);
  a.H = H; a.Hp = Hp; a.W = Hp / 32;
  const size_t smem = (size_t)(128 + 96) * 1024 + 256 + (size_t)2 * Hp * 4;
  CODA_CUDA_OK(cudaFuncSetAttribute(k_pair_rows_tc, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  k_pair_rows_tc<<<tile_hi - tile_lo, TC_THREADS, smem, as_stream(stream)>>>(a, tile_lo);
  CODA_LAUNCH_OK("k_pair_rows_tc");
  return CODA_B200_OK;
}

CODA_MODULE_ANCHOR(pairs_tc, k_pair_rows_tc)
