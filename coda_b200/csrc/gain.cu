// The per-step scoring pass, item-major: per-item expected information gain from the gain of every row.
//
//   gain(b, c) = H_before - H_after(b, c) = sum_h f(m0_h) - f(m0_h + pi_hat[c] * (PH[b,c,h] - PB[c,h]))   coda.py:254, 274-276
//   eig[b]     = sum_c pi_hat_xi[b,c] * gain(b, c)                                                          coda.py:278
//              = (sum_c U[b,c] * g0[c] + sum_{entries} U[b,c_e] * (gain_e - g0[c_e])) / max(sum_c U[b,c], 1e-12)
//
// with g0[c] the gain of the "no model predicts c" template row and one entry per distinct predicted class of
// the item.  The gains of all rows come from row_gains (cached rows) or pair_rows (no cache); the assembly looks
// them up.  An item's entries and its U row are contiguous in HBM: a warp that walks items in order streams them.
// Candidate filter (coda.py:215-219, 239) and the arg-max with runner-up (coda.py:306-309) ride along.
// The per-item arithmetic of k_gain_eig / k_eig_assemble_g8 and the per-row arithmetic of k_row_gains are restated
// for the sampled scoring pass (eig_item.cuh, sample.cu); a change to one order of operations must be made to both.
#include "common.cuh"

#define GE_THREADS 384
#define GE_WARPS (GE_THREADS / 32)

struct GainEigArgs {
  const float* U;
  long long N;
  int C, H;
  const int32_t* ent_off;
  const int32_t* ent_row;
  const uint16_t* ent_cls;
  const float* gain;
  const uint8_t* labeled;
  const uint8_t* disagree;
  long long n_offset;
  float* eig;
  long long* partials;
  uint32_t* flags;
  const int32_t* ell_row;     // optional ELL copy of the entry lists: [N][ell_k] row ids (-1 = empty) ...
  const uint16_t* ell_cls;    // ... and classes
  int ell_k;
};

__device__ __forceinline__ float gain4(const float4 ph, const float4 pb, const float4 m, const float4 fm, float pic) {
  float g = fm.x - ent_term(m.x + pic * (ph.x - pb.x));
  g += fm.y - ent_term(m.y + pic * (ph.y - pb.y));
  g += fm.z - ent_term(m.z + pic * (ph.z - pb.z));
  g += fm.w - ent_term(m.w + pic * (ph.w - pb.w));
  return g;
}

// one warp per item, any C and any number of entries per item (the 8-lane assembly below takes C <= 128 and
// <= 32 entries).  KC: C <= 32 * KC keeps the item's U row in registers (KC = 0: any C, the row is re-read).
template <int KC>
__global__ void __launch_bounds__(GE_THREADS, 2) k_gain_eig(GainEigArgs a) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int C = a.C, H = a.H;
  float* g0 = reinterpret_cast<float*>(smem_raw);                        // [C]   gain of the empty-set template row
  __shared__ float s_v[2][GE_WARPS], s_v2[2][GE_WARPS];
  __shared__ long long s_i[2][GE_WARPS], s_c[GE_WARPS];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  for (int c = tid; c < C; c += GE_THREADS) g0[c] = a.gain[(size_t)c * (1 + H)];
  __syncthreads();

  Best2 bA = best2_empty(), bB = best2_empty();
  long long cntA = 0;
  uint32_t bad = 0;
  constexpr int KR = KC > 0 ? KC : 1;
  const long long nw = (long long)gridDim.x * GE_WARPS;
  long long n = (long long)blockIdx.x * GE_WARPS + warp;
  int e0 = 0, e1 = 0;
  if (n < a.N) {
    e0 = __ldg(a.ent_off + n); e1 = __ldg(a.ent_off + n + 1);
  }
  while (n < a.N) {
    // offsets of the next item this warp will visit: one memory latency ahead
    const long long nn = n + nw;
    int ne0 = 0, ne1 = 0;
    if (nn < a.N) {
      ne0 = __ldg(a.ent_off + nn); ne1 = __ldg(a.ent_off + nn + 1);
    }
    const float* urow = a.U + (size_t)n * C;
    float u[KR];
    float s = 0.f, e = 0.f;
    if (KC > 0) {
#pragma unroll
      for (int k = 0; k < KR; ++k) {
        const int c = lane + 32 * k;
        u[k] = c < C ? __ldg(urow + c) : 0.f;
      }
    }
    for (int eb = e0; eb < e1; eb += 32) {       // one trip unless an item has > 32 distinct predicted classes
      int r = -1, c = 0;
      if (eb + lane < e1) {
        r = __ldg(a.ent_row + eb + lane);
        c = __ldg(a.ent_cls + eb + lane);
      }
      const float myg = r >= 0 ? __ldg(a.gain + r) : 0.f;
      // correction of this chunk's entries: xi_c * (gain - gain of the empty-set template)
      float ucls = 0.f;
      if (KC > 0) {
#pragma unroll
        for (int k = 0; k < KR; ++k) {
          const float t = __shfl_sync(CODA_FULL, u[k], c & 31);
          if ((c >> 5) == k) ucls = t;
        }
      } else if (r >= 0) {
        ucls = __ldg(urow + c);
      }
      if (r >= 0) e = fmaf(ucls, myg - g0[c], e);
    }
    if (KC > 0) {
#pragma unroll
      for (int k = 0; k < KR; ++k) {
        const int c = lane + 32 * k;
        s += u[k];
        if (c < C) e = fmaf(u[k], g0[c], e);
      }
    } else {
      for (int c = lane; c < C; c += 32) {
        const float v = __ldg(urow + c);
        s += v;
        e = fmaf(v, g0[c], e);
      }
    }
    s = warp_sum(s);
    e = warp_sum(e);
    if (lane == 0) {
      const float v = e / fmaxf(s, 1e-12f);                 // coda.py:230 clamp, coda.py:278
      a.eig[n] = v;
      if (!isfinite(v)) bad |= CODA_B200_FLAG_NONFINITE_EIG;
      if (!a.labeled[n]) {
        best2_add(bB, v, a.n_offset + n);
        if (a.disagree[n]) {
          best2_add(bA, v, a.n_offset + n);
          ++cntA;
        }
      }
    }
    n = nn; e0 = ne0; e1 = ne1;
  }
  if (lane == 0) {
    s_v[0][warp] = bA.v; s_i[0][warp] = bA.i; s_v2[0][warp] = bA.v2;
    s_v[1][warp] = bB.v; s_i[1][warp] = bB.i; s_v2[1][warp] = bB.v2;
    s_c[warp] = cntA;
  }
  __syncthreads();
  if (tid == 0) {
    Best2 fa = best2_empty(), fb = best2_empty();
    long long cn = 0;
    for (int w = 0; w < GE_WARPS; ++w) {
      best2_merge(fa, Best2{s_v[0][w], s_i[0][w], s_v2[0][w]});
      best2_merge(fb, Best2{s_v[1][w], s_i[1][w], s_v2[1][w]});
      cn += s_c[w];
    }
    rec_store(a.partials + (size_t)blockIdx.x * REC_W, fa, cn, fb);
  }
  if (bad) atomicOr(a.flags, bad);
}

// ---------------------------------------------------------------------------------------
// row_gains: information gain of every heavy row from its cached P(best | hypothetical) row.  HBM-bound stream
// over the item-major row cache: one warp per chunk of 32 consecutive rows, four rows (4 KB) in flight per warp,
// rows read with the streaming hint so that the class rows PB[c] (100 KB at cfg3, a different class for every
// row) stay resident in L1.  Hp = 128 * NQ.
// ---------------------------------------------------------------------------------------
__device__ __forceinline__ float4 ld_stream4(const float4* p) {
  float4 v;
  asm volatile("ld.global.cs.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p));
  return v;
}

template <int NQ>
__global__ void __launch_bounds__(256) k_row_gains(const float* __restrict__ rows, const uint16_t* __restrict__ row_cls,
                                                   long long nrows, long long T, int H, const float* __restrict__ PB,
                                                   const float* __restrict__ m0, const float* __restrict__ pi_hat,
                                                   float* __restrict__ gain) {
  constexpr int Hp = 128 * NQ;
  constexpr int CH = 32;   // rows per warp chunk
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float4 m[NQ], fm[NQ];
#pragma unroll
  for (int q = 0; q < NQ; ++q) {
    const int h = (q * 32 + lane) * 4;
    float4 v = __ldg(reinterpret_cast<const float4*>(m0) + q * 32 + lane);
    if (h + 0 >= H) v.x = 0.f;
    if (h + 1 >= H) v.y = 0.f;
    if (h + 2 >= H) v.z = 0.f;
    if (h + 3 >= H) v.w = 0.f;
    m[q] = v;
    fm[q] = make_float4(ent_term(v.x), ent_term(v.y), ent_term(v.z), ent_term(v.w));
  }
  const long long nchunks = (nrows + CH - 1) / CH;
  for (long long ch = (long long)blockIdx.x * 8 + warp; ch < nchunks; ch += (long long)gridDim.x * 8) {
    const long long p0 = ch * CH;
    const long long p1 = min(nrows, p0 + CH);
    // classes of the whole chunk, one per lane: template rows (r < T) are class-major, heavy rows carry row_cls
    int mycls = 0;
    if (p0 + lane < p1) mycls = (p0 + lane < T) ? (int)((p0 + lane) / (1 + H)) : (int)row_cls[p0 + lane - T];
    for (long long i = p0; i < p1; i += 4) {
      float4 a[4][NQ];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const long long r = min(i + j, nrows - 1);
        const float4* rp = reinterpret_cast<const float4*>(rows + (size_t)r * Hp);
#pragma unroll
        for (int q = 0; q < NQ; ++q) a[j][q] = ld_stream4(rp + q * 32 + lane);
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const long long r = i + j;
        if (r < p1) {
          const int c = __shfl_sync(CODA_FULL, mycls, (int)(r - p0));
          const float pic = __ldg(pi_hat + c);
          const float4* pb = reinterpret_cast<const float4*>(PB + (size_t)c * Hp);
          float g = 0.f;
#pragma unroll
          for (int q = 0; q < NQ; ++q) g += gain4(a[j][q], __ldg(pb + q * 32 + lane), m[q], fm[q], pic);
          g = warp_sum(g);
          if (lane == 0) gain[r] = g;
        }
      }
    }
  }
}

// any Hp (multiple of 32): m0 / f(m0) in shared memory, one row at a time
__global__ void __launch_bounds__(256) k_row_gains_any(const float* __restrict__ rows, const uint16_t* __restrict__ row_cls,
                                                       long long nrows, long long T, int H, int Hp, const float* __restrict__ PB,
                                                       const float* __restrict__ m0, const float* __restrict__ pi_hat,
                                                       float* __restrict__ gain) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  float* m0s = reinterpret_cast<float*>(smem_raw);
  float* fm0 = m0s + Hp;
  for (int h = threadIdx.x; h < Hp; h += blockDim.x) {
    const float m = h < H ? m0[h] : 0.f;
    m0s[h] = m;
    fm0[h] = ent_term(m);
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (long long r = (long long)blockIdx.x * 8 + warp; r < nrows; r += (long long)gridDim.x * 8) {
    const int c = r < T ? (int)(r / (1 + H)) : (int)row_cls[r - T];
    const float pic = pi_hat[c];
    const float* row = rows + (size_t)r * Hp;
    const float* pb = PB + (size_t)c * Hp;
    float g = 0.f;
    for (int hq = lane * 4; hq < Hp; hq += 128) {
      const float4 ph = ld_stream4(reinterpret_cast<const float4*>(row + hq));
      const float4 p4 = __ldg(reinterpret_cast<const float4*>(pb + hq));
      const float4 m4 = *reinterpret_cast<const float4*>(m0s + hq);
      const float4 f4 = *reinterpret_cast<const float4*>(fm0 + hq);
      g += gain4(ph, p4, m4, f4, pic);
    }
    g = warp_sum(g);
    if (lane == 0) gain[r] = g;
  }
}

extern "C" int coda_b200_row_gains(const float* ph_cache, const uint16_t* row_cls, int64_t n_heavy, int H, int C,
                                   const float* PB, const float* m0, const float* pi_hat, float* gain,
                                   coda_stream_t stream) {
  CODA_CHECK_ARG(ph_cache && PB && m0 && pi_hat && gain && (row_cls || n_heavy == 0), "row_gains: null pointer");
  const int Hp = (H + 31) / 32 * 32;
  const long long T = (long long)C * (1 + H);
  const long long nrows = T + (n_heavy > 0 ? n_heavy : 0);      // template rows first, then the heavy rows: one stream
  const float* rows = ph_cache;
  float* g = gain;
  cudaStream_t st = as_stream(stream);
  if (Hp % 128 == 0 && Hp <= 512) {
    int grid = (int)min((long long)(nrows + 255) / 256, (long long)coda_sm_count() * 6);
    if (grid < 1) grid = 1;
#define LAUNCH_RG(NQ) k_row_gains<NQ><<<grid, 256, 0, st>>>(rows, row_cls, nrows, T, H, PB, m0, pi_hat, g)
    if (Hp == 128) LAUNCH_RG(1);
    else if (Hp == 256) LAUNCH_RG(2);
    else if (Hp == 384) LAUNCH_RG(3);
    else LAUNCH_RG(4);
#undef LAUNCH_RG
    CODA_LAUNCH_OK("k_row_gains");
    return CODA_B200_OK;
  }
  int grid = (int)min((long long)(nrows + 7) / 8, (long long)coda_sm_count() * 8);
  if (grid < 1) grid = 1;
  k_row_gains_any<<<grid, 256, (size_t)2 * Hp * 4, st>>>(rows, row_cls, nrows, T, H, Hp, PB, m0, pi_hat, g);
  CODA_LAUNCH_OK("k_row_gains_any");
  return CODA_B200_OK;
}

// ---------------------------------------------------------------------------------------
// eig assembly from per-row gains, 8 lanes per item (C <= 128, <= 32 entries per item): four items per warp
// instruction, IT8 batches in flight; three dependent load levels (offsets -> entries + U row -> gains), each
// issued for all items of the batch before the first use.
// ---------------------------------------------------------------------------------------
// The arguments are read in place from the parameter bank (__grid_constant__): left free to copy them, ptxas schedules
// the C <= 64 and C <= 104 instantiations differently, about 1 us per step slower at cfg3 on an H100 (700 W).
constexpr int IT8 = 2;     // items per 8-lane group and iteration
template <int KC8>
__global__ void __launch_bounds__(256, 2) k_eig_assemble_g8(const __grid_constant__ GainEigArgs a, int nblocks_rec) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  float* g0 = reinterpret_cast<float*>(smem_raw);   // [C]
  __shared__ float s_v[2][8], s_v2[2][8];
  __shared__ long long s_i[2][8], s_c[8];
  const int C = a.C;
  for (int c = threadIdx.x; c < C; c += blockDim.x) g0[c] = a.gain[(size_t)c * (1 + a.H)];
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane & 7, grp = lane >> 3;
  Best2 bA = best2_empty(), bB = best2_empty();
  long long cntA = 0;
  uint32_t bad = 0;
  const long long per_iter = (long long)gridDim.x * 8 * 4 * IT8;
  // the loop bound is warp-uniform (full-mask shuffles inside); a group past the end clamps its loads and skips its writes
  for (long long wb = ((long long)blockIdx.x * 8 + warp) * 4 * IT8; wb < a.N; wb += per_iter) {
    const long long nb = wb + grp * IT8;
    int e0[IT8], ne[IT8];
    if (!a.ell_row) {
#pragma unroll
      for (int i = 0; i < IT8; ++i) {
        const long long n = min(nb + i, a.N - 1);
        e0[i] = __ldg(a.ent_off + n);
        ne[i] = __ldg(a.ent_off + n + 1) - e0[i];
      }
    }
    float u[IT8][KC8];
    int er[IT8][4], ec[IT8][4];
#pragma unroll
    for (int i = 0; i < IT8; ++i) {
      const long long n = min(nb + i, a.N - 1);
      const float* urow = a.U + (size_t)n * C;
#pragma unroll
      for (int k = 0; k < KC8; ++k) {
        const int c = g + 8 * k;
        u[i][k] = c < C ? __ldg(urow + c) : 0.f;
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int e = g + 8 * j;
        er[i][j] = -1; ec[i][j] = 0;
        if (a.ell_row) {     // the entry address follows from the item index: one dependent load level less
          if (e < a.ell_k) {
            er[i][j] = __ldg(a.ell_row + (size_t)n * a.ell_k + e);
            ec[i][j] = __ldg(a.ell_cls + (size_t)n * a.ell_k + e);
          }
        } else if (e < ne[i]) {
          er[i][j] = __ldg(a.ent_row + e0[i] + e);
          ec[i][j] = __ldg(a.ent_cls + e0[i] + e);
        }
      }
    }
    float eg[IT8][4], eu[IT8][4];
#pragma unroll
    for (int i = 0; i < IT8; ++i) {
      const long long n = min(nb + i, a.N - 1);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        eg[i][j] = 0.f; eu[i][j] = 0.f;
        if (er[i][j] >= 0) {
          eg[i][j] = __ldg(a.gain + er[i][j]);
          eu[i][j] = __ldg(a.U + (size_t)n * C + ec[i][j]);
        }
      }
    }
#pragma unroll
    for (int i = 0; i < IT8; ++i) {
      const long long n = nb + i;
      float s = 0.f, e = 0.f;
#pragma unroll
      for (int k = 0; k < KC8; ++k) {
        const int c = g + 8 * k;
        s += u[i][k];
        if (c < C) e = fmaf(u[i][k], g0[c], e);
      }
#pragma unroll
      for (int j = 0; j < 4; ++j)
        if (er[i][j] >= 0) e = fmaf(eu[i][j], eg[i][j] - g0[ec[i][j]], e);
#pragma unroll
      for (int o = 4; o > 0; o >>= 1) {
        s += __shfl_xor_sync(CODA_FULL, s, o);
        e += __shfl_xor_sync(CODA_FULL, e, o);
      }
      if (g == 0 && n < a.N) {
        const float v = e / fmaxf(s, 1e-12f);                // coda.py:230, 278
        a.eig[n] = v;
        if (!isfinite(v)) bad |= CODA_B200_FLAG_NONFINITE_EIG;
        if (!a.labeled[n]) {
          best2_add(bB, v, a.n_offset + n);
          if (a.disagree[n]) {
            best2_add(bA, v, a.n_offset + n);
            ++cntA;
          }
        }
      }
    }
  }
  best2_warp(bA);
  best2_warp(bB);
  cntA = warp_sum(cntA);
  if (lane == 0) {
    s_v[0][warp] = bA.v; s_i[0][warp] = bA.i; s_v2[0][warp] = bA.v2;
    s_v[1][warp] = bB.v; s_i[1][warp] = bB.i; s_v2[1][warp] = bB.v2;
    s_c[warp] = cntA;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    Best2 fa = best2_empty(), fb = best2_empty();
    long long cn = 0;
    for (int w = 0; w < 8; ++w) {
      best2_merge(fa, Best2{s_v[0][w], s_i[0][w], s_v2[0][w]});
      best2_merge(fb, Best2{s_v[1][w], s_i[1][w], s_v2[1][w]});
      cn += s_c[w];
    }
    rec_store(a.partials + (size_t)blockIdx.x * REC_W, fa, cn, fb);
    // the caller merges a fixed number of records: blocks beyond this grid leave empty ones
    if (blockIdx.x == 0)
      for (int b = gridDim.x; b < nblocks_rec; ++b) rec_store(a.partials + (size_t)b * REC_W, best2_empty(), 0, best2_empty());
  }
  if (bad) atomicOr(a.flags, bad);
}

extern "C" int coda_b200_eig_blocks(int64_t N, int H, int C) {
  (void)H; (void)C;
  long long want = (N + GE_WARPS - 1) / GE_WARPS;
  long long cap = (long long)coda_sm_count() * 4;
  return (int)(want < cap ? (want < 1 ? 1 : want) : cap);
}

extern "C" int coda_b200_gain_eig(const float* U, int64_t N, int C, int H, const int32_t* ent_off,
                                  const int32_t* ent_row, const uint16_t* ent_cls, const float* gain,
                                  const uint8_t* labeled, const uint8_t* disagree, int64_t n_offset, int max_entries,
                                  const int32_t* ell_row, const uint16_t* ell_cls, int ell_k, float* eig,
                                  int64_t* partials, uint32_t* flags, coda_stream_t stream) {
  CODA_CHECK_ARG(U && ent_off && ent_row && ent_cls && gain && labeled && disagree && eig && partials && flags,
                 "gain_eig: null pointer");
  CODA_CHECK_ARG(N >= 1 && C >= 2 && H >= 1, "gain_eig: bad dims");
  GainEigArgs a;
  a.U = U; a.N = N; a.C = C; a.H = H;
  a.ent_off = ent_off; a.ent_row = ent_row; a.ent_cls = ent_cls; a.gain = gain;
  a.labeled = labeled; a.disagree = disagree; a.n_offset = n_offset; a.eig = eig;
  a.partials = reinterpret_cast<long long*>(partials); a.flags = flags;
  a.ell_row = (ell_row && ell_cls && ell_k >= 1 && ell_k <= 32) ? ell_row : nullptr;
  a.ell_cls = ell_cls; a.ell_k = ell_k;
  const size_t smem = (size_t)C * 4;                     // g0
  CODA_CHECK_ARG(smem <= 220 * 1024, "gain_eig: C=%d does not fit shared memory", C);
  const int grid = coda_b200_eig_blocks(N, H, C);
  cudaStream_t st = as_stream(stream);
  if (C <= 128 && max_entries >= 0 && max_entries <= 32) {
    // 8-lane groups: the grid may be smaller than the record count the caller merges (block 0 writes empty records)
    int g8 = (int)min((long long)(N + 31) / 32, (long long)min(grid, coda_sm_count() * 2));
    if (g8 < 1) g8 = 1;
#define LAUNCH_G8(K8) k_eig_assemble_g8<K8><<<g8, 256, smem, st>>>(a, grid)
    if (C <= 32) LAUNCH_G8(4);
    else if (C <= 64) LAUNCH_G8(8);
    else if (C <= 104) LAUNCH_G8(13);
    else LAUNCH_G8(16);
#undef LAUNCH_G8
    CODA_LAUNCH_OK("k_eig_assemble_g8");
    return CODA_B200_OK;
  }
#define LAUNCH_GE(KC)                                                                                        \
  do {                                                                                                       \
    CODA_CUDA_OK(cudaFuncSetAttribute(k_gain_eig<KC>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
    k_gain_eig<KC><<<grid, GE_THREADS, smem, st>>>(a);                                                        \
  } while (0)
  if (C <= 32) LAUNCH_GE(1);
  else if (C <= 64) LAUNCH_GE(2);
  else if (C <= 128) LAUNCH_GE(4);
  else LAUNCH_GE(0);
#undef LAUNCH_GE
  CODA_LAUNCH_OK("k_gain_eig");
  return CODA_B200_OK;
}

// ELL copy of the per-item entry lists for the 8-lane assembly: ell_row[n][k] = row id or -1, ell_cls[n][k] = class.
__global__ void k_ell_build(const int32_t* __restrict__ ent_off, const int32_t* __restrict__ ent_row,
                            const uint16_t* __restrict__ ent_cls, long long N, int K, int32_t* __restrict__ ell_row,
                            uint16_t* __restrict__ ell_cls) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N * K) return;
  const long long n = i / K;
  const int k = (int)(i % K);
  const int o = ent_off[n] + k;
  const bool has = o < ent_off[n + 1];
  ell_row[i] = has ? ent_row[o] : -1;
  ell_cls[i] = has ? ent_cls[o] : (uint16_t)0;
}

extern "C" int coda_b200_ell_build(const int32_t* ent_off, const int32_t* ent_row, const uint16_t* ent_cls, int64_t N,
                                   int K, int32_t* ell_row, uint16_t* ell_cls, coda_stream_t stream) {
  CODA_CHECK_ARG(ent_off && ent_row && ent_cls && ell_row && ell_cls && K >= 1 && K <= 32, "ell_build: bad arguments");
  const long long tot = (long long)N * K;
  k_ell_build<<<(unsigned)((tot + 255) / 256), 256, 0, as_stream(stream)>>>(ent_off, ent_row, ent_cls, N, K, ell_row, ell_cls);
  CODA_LAUNCH_OK("k_ell_build");
  return CODA_B200_OK;
}

CODA_MODULE_ANCHOR(gain, k_ell_build)
