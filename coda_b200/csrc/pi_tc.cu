// pi_full on the Hopper tensor cores (wgmma):  U[n][c] = sum_h sum_s preds[h][n][s] * D[h][c][s]   (coda.py:227-229)
//
// A skinny GEMM: M = N items, N = C classes, K = H*C.  One CTA owns a tile of 128 items (64 when C is too large for two
// such stages in shared memory) and walks the H models; per model the tile's block of the slab is ONE contiguous blob
// (51 KB at C = 100), fetched by one 1-D bulk TMA copy together with the model's D limbs.  fp32 does not go through the
// tensor cores, so both operands are cut into two fp16 limbs, x = hi + 2^-12 lo  (11 + 11 significant bits: 2^-22
// relative at worst, a quarter of an fp32 ulp on average; lo is stored scaled so that it stays a normal fp16 number),
// and three products are formed per K = 16 chunk:
//
//     main  += A_hi . B_hi                    (22-bit products: exact in the fp32 accumulator)
//     corr  += A_hi . B_lo + A_lo . B_hi      (carries the 2^12 scale; A_lo . B_lo ~ 2^-22 is dropped)
//
// preds lie in [0, 1]; D (Dirichlet parameters) is multiplied by a power of two chosen from max |D| so that it stays
// inside the fp16 range, and U is scaled back at the end (exact).  The tensor core accumulates in fp32 with truncation,
// which biases a long chain of positive terms; so the two accumulators are folded every G (= 4) models into fp32
// registers (round-to-nearest adds) and restarted.  Against an fp64 contraction the result is closer than the
// 25 600-term fp32 FMA chain of the SIMT kernel (slab.cu: k_pi_full), see
// tests/test_gpu_parity.py::test_tensor_core_marginals_match_fp64.
//
// Each warpgroup owns 64 items.  The A limbs never touch shared memory: every thread converts the fp32 slab values of
// its own wgmma A fragment (2 items x 4 classes of the chunk) to fp16 limbs in registers.  B (the D limbs, pre-packed by
// k_pi_w_limbs in the K-major core-matrix order) is read by wgmma straight from the staged blob, in 16-class blocks.
// Thread 0 refills the stage of model h - 1 with model h - 1 + S once both warpgroups have released it.
// Every wait is bounded: a pipeline that stops sets CODA_B200_FLAG_PIPELINE_TIMEOUT and the kernel drains out.
//
// A 16-bit slab (fp16 / bf16) is widened to fp32 as the A fragment is loaded, then split into the same two limbs, so it
// gives the bits of its fp32 widening.  Its tile of 128 items is 25 600 bytes at C = 100, but a tile (or a model) need not
// start on a 16-byte boundary: the bulk copy takes the tile's 16-byte aligned interior and thread 0 copies the few
// elements before and after it, so every shape the fp32 slab takes here is taken by the 16-bit slab too.
#include "common.cuh"

#include <stdlib.h>
#include <type_traits>

namespace {

constexpr int PT_WG = 64;                 // items per warpgroup
constexpr int PT_MAXB = 8;                // 16-class blocks (Np <= 128)
constexpr int PT_MAX_STAGES = 6;
constexpr float PT_LO_SCALE = 4096.f;     // lo limbs are stored times 2^12
constexpr long long PT_TIMEOUT_CYCLES = 4000000000LL;   // ~2 s
constexpr size_t PT_SMEM_BUDGET = 227 * 1024;
constexpr size_t PT_TAIL = 256;           // barriers + abort flag

struct PiTcArgs {
  const void* preds;          // float, __half or __nv_bfloat16 (the kernel's T)
  long long ldh;              // elements between models
  const unsigned char* wb;    // [H][KC][2 k_cores][2 Np/8 (hi | lo)][8][8] fp16, then the 16-byte header (max |D| bits)
  const uint32_t* dmax;       // header: bits of max |D|
  float* U;
  uint32_t* flags;
  long long N;
  int H, C, Np, KC;
  int rows;                   // items per CTA: 64 x warpgroups
  int S;                      // stages (one model each)
  uint32_t xbytes;            // stage offset of the D limbs (the items block, + 16 bytes of alignment slack for 16-bit
                              // slabs, rounded up to 128 bytes)
  uint32_t sbytes;            // bytes per stage
  int G;                      // models per accumulator fold
};

// power of two that brings max |D| below 2^15 (fp16 overflows at 65504); 0 when no scaling is needed
__device__ __forceinline__ int pt_down_shift(uint32_t maxbits) {
  const int e = (int)((maxbits >> 23) & 0xffu) - 127;
  return max(0, e - 14);
}

// try_wait with a suspend-time hint: the warp is parked by the hardware until the phase completes (or ~the hint elapses)
__device__ __forceinline__ bool pt_try(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t"
      "}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity), "r"(20000u)
      : "memory");
  return ok != 0;
}

// false = the pipeline was aborted (here or by another thread)
__device__ __forceinline__ bool pt_wait(uint64_t* bar, uint32_t parity, volatile int* abort_s) {
  if (pt_try(bar, parity)) return true;
  const long long t0 = clock64();
  for (;;) {
    if (pt_try(bar, parity)) return true;
    if (*abort_s) return false;
    if (clock64() - t0 > PT_TIMEOUT_CYCLES) {
      *abort_s = 1;
      return false;
    }
  }
}

// AND of `ok` over the 128 threads of warpgroup `wg` (named barrier 1 + wg; 0 is __syncthreads): the wgmma instructions
// are warpgroup-wide, so a pipeline abort has to be agreed by the whole warpgroup before any of its warps leaves the loop
__device__ __forceinline__ bool wg_all(bool ok, int wg) {
  uint32_t r;
  asm volatile(
      "{\n\t"
      ".reg .pred p, q;\n\t"
      "setp.ne.u32 p, %1, 0;\n\t"
      "bar.red.and.pred q, %2, 128, p;\n\t"
      "selp.u32 %0, 1, 0, q;\n\t"
      "}"
      : "=r"(r)
      : "r"((uint32_t)ok), "r"(1 + wg)
      : "memory");
  return r != 0;
}

// D[64 x 16] (+)= A[64 x 16] . B[16 x 16]^T: A fp16 from registers (wgmma A fragment), B fp16 in shared memory (K-major)
__device__ __forceinline__ void mma_n16(float (&d)[8], const uint32_t (&a)[4], uint64_t bdesc, uint32_t accum) {
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "setp.ne.b32 p, %13, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7}, {%8, %9, %10, %11}, %12, p, 1, 1, 0;\n\t"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(accum));
}

// two floats -> packed fp16 hi limbs and packed fp16 lo limbs:  x = hi + lo / 4096 (+ 2^-22 x at worst)
__device__ __forceinline__ void pt_split2(float a, float b, uint32_t& hi, uint32_t& lo) {
  const __half2 h = __floats2half2_rn(a, b);
  const float2 hf = __half22float2(h);
  const __half2 l = __floats2half2_rn((a - hf.x) * PT_LO_SCALE, (b - hf.y) * PT_LO_SCALE);   // a - hi is exact
  hi = *reinterpret_cast<const uint32_t*>(&h);
  lo = *reinterpret_cast<const uint32_t*>(&l);
}

// ---- max |D| (bit pattern; D is finite and positive in every valid run, NaN / Inf end up as NaN in U) ---------------
__global__ void __launch_bounds__(256) k_pi_w_max(const float* __restrict__ D, long long n, uint32_t* __restrict__ out) {
  uint32_t m = 0;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    m = max(m, __float_as_uint(fabsf(D[i])));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = max(m, __shfl_xor_sync(CODA_FULL, m, o));
  if ((threadIdx.x & 31) == 0 && m) atomicMax(out, m);
}

// ---- D -> fp16 limbs in the B-operand order: one blob per (model, K chunk) -----------------------------------------
// blob = [k_core 2][n_core 2 Np/8: hi limbs, then lo limbs][8 classes][8 s] fp16;  class = n_core*8 + r,  s = chunk*16 + k_core*8 + e
__global__ void __launch_bounds__(256) k_pi_w_limbs(const float* __restrict__ D, int H, int C, int Np, int KC,
                                                    const uint32_t* __restrict__ dmax, __half* __restrict__ wb) {
  const long long per_limb = (long long)2 * Np * 8;           // elements of one limb of one chunk (= Np x 16)
  const long long total = (long long)H * KC * per_limb;
  const float down = __uint_as_float((uint32_t)(127 - pt_down_shift(*dmax)) << 23);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int e = (int)(i & 7), r = (int)((i >> 3) & 7);
    long long q = i >> 6;
    const int ncore = (int)(q % (Np / 8));
    q /= (Np / 8);
    const int kcore = (int)(q & 1);
    q >>= 1;
    const int kc = (int)(q % KC);
    const int h = (int)(q / KC);
    const int c = ncore * 8 + r, s = kc * 16 + kcore * 8 + e;
    const float v = (c < C && s < C) ? D[((size_t)h * C + c) * C + s] * down : 0.f;
    const __half hi = __float2half_rn(v);
    const __half lo = __float2half_rn((v - __half2float(hi)) * PT_LO_SCALE);
    const long long blob = ((long long)h * KC + kc) * 2 * per_limb;
    const long long within = ((long long)kcore * (2 * Np / 8) + ncore) * 64 + r * 8 + e;
    wb[blob + within] = hi;
    wb[blob + (long long)(Np / 8) * 64 + within] = lo;
  }
}

// two consecutive classes of one item -> fp32 (the fp32 slab keeps its 8-byte load)
__device__ __forceinline__ float2 pt_ld2(const float* p) { return *reinterpret_cast<const float2*>(p); }
template <typename T>
__device__ __forceinline__ float2 pt_ld2(const T* p) { return make_float2(slab_f(p[0]), slab_f(p[1])); }

template <typename T>
__global__ void __launch_bounds__(2 * 128, 1) k_pi_full_tc(PiTcArgs a) {
  constexpr bool WIDE = std::is_same<T, float>::value;
  const T* preds = static_cast<const T*>(a.preds);
  extern __shared__ __align__(1024) unsigned char smem[];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int H = a.H, C = a.C, Np = a.Np, KC = a.KC, S = a.S, G = a.G;
  const int nb = Np / 16;                                     // 16-class blocks
  const long long n0 = (long long)blockIdx.x * a.rows;
  const int cnt = (int)min((long long)a.rows, a.N - n0);
  const int r0 = (warp >> 2) * PT_WG + (warp & 3) * 16 + (lane >> 2);   // this thread's items: r0 and r0 + 8
  const int nwarps = blockDim.x >> 5;

  uint64_t* full = reinterpret_cast<uint64_t*>(smem + (size_t)S * a.sbytes);
  uint64_t* empty = full + PT_MAX_STAGES;
  volatile int* abort_s = reinterpret_cast<volatile int*>(empty + PT_MAX_STAGES);
  if (tid == 0) {
    for (int i = 0; i < S; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], nwarps);
    }
    *abort_s = (*a.flags & CODA_B200_FLAG_PIPELINE_TIMEOUT) ? 1 : 0;          // an earlier CTA already gave up
    mbar_fence_init();
  }
  __syncthreads();
  const uint32_t xbytes = (uint32_t)cnt * C * (uint32_t)sizeof(T), dbytes = (uint32_t)KC * Np * 64u;
  // byte offset of this CTA's tile of model h inside its stage: 0 for fp32; for a 16-bit slab the stage holds the
  // tile's bytes from the 16-byte boundary at or below its first element
  auto tile_pad = [&](int h) -> uint32_t {
    return WIDE ? 0u : (uint32_t)(reinterpret_cast<uintptr_t>(preds + (size_t)h * a.ldh + (size_t)n0 * C) & 15);
  };
  auto load = [&](int h) {
    unsigned char* st = smem + (size_t)(h % S) * a.sbytes;
    uint64_t* bar = &full[h % S];
    const T* src = preds + (size_t)h * a.ldh + (size_t)n0 * C;
    if (WIDE) {
      mbar_expect_tx(bar, xbytes + dbytes);
      tma_load_1d(st, src, xbytes, bar);
    } else {
      // [lo, hi): whole 16-byte units of the tile by bulk copy; the elements before lo and from hi on by this thread
      const uintptr_t b = reinterpret_cast<uintptr_t>(src), e = b + xbytes, b0 = b & ~(uintptr_t)15;
      uintptr_t lo = (b + 15) & ~(uintptr_t)15, hi = e & ~(uintptr_t)15;
      if (hi <= lo) lo = hi = e;
      for (uintptr_t x = b; x < lo; x += sizeof(T))
        *reinterpret_cast<T*>(st + (x - b0)) = __ldg(reinterpret_cast<const T*>(x));
      for (uintptr_t x = hi; x < e; x += sizeof(T))
        *reinterpret_cast<T*>(st + (x - b0)) = __ldg(reinterpret_cast<const T*>(x));
      mbar_expect_tx(bar, (uint32_t)(hi - lo) + dbytes);        // arrive (release): the stores above are visible
      if (hi > lo) tma_load_1d(st + (lo - b0), reinterpret_cast<const void*>(lo), (uint32_t)(hi - lo), bar);
    }
    tma_load_1d(st + a.xbytes, a.wb + (size_t)h * dbytes, dbytes, bar);
  };
  if (tid == 0)
    for (int h = 0; h < S && h < H; ++h) load(h);

  float mainv[PT_MAXB][8], corr[PT_MAXB][8], tot[PT_MAXB][8];
#pragma unroll
  for (int b = 0; b < PT_MAXB; ++b)
#pragma unroll
    for (int i = 0; i < 8; ++i) tot[b][i] = 0.f;
  const uint32_t lbo = (uint32_t)(2 * Np / 8) * 128, lo_off = (uint32_t)(Np / 8) * 128, chunk_bytes = (uint32_t)Np * 64u;
  const bool in0 = r0 < cnt, in1 = r0 + 8 < cnt;
  bool ok = true;
  for (int h = 0; h < H && ok; ++h) {
    const int s = h % S;
    if (tid == 0 && h >= 1 && h - 1 + S < H) {
      if (pt_wait(&empty[(h - 1) % S], ((h - 1) / S) & 1, abort_s)) load(h - 1 + S);
    }
    __syncwarp();
    ok = wg_all(pt_wait(&full[s], (h / S) & 1, abort_s), warp >> 2);
    if (!ok) break;
    const unsigned char* st = smem + (size_t)s * a.sbytes;
    const T* x0 = reinterpret_cast<const T*>(st + tile_pad(h)) + (size_t)r0 * C;
    const T* x1 = x0 + (size_t)8 * C;
    const uint32_t dst = smem_u32(st + a.xbytes);
    const bool restart = h % G == 0;
    for (int kc = 0; kc < KC; ++kc) {
      // this thread's A fragment: items r0, r0 + 8 x classes c0, c0 + 1, c0 + 8, c0 + 9 of the chunk (C % 4 == 0)
      const int c0 = kc * 16 + 2 * (lane & 3);
      const float2 z = make_float2(0.f, 0.f);
      const float2 v00 = (in0 && c0 < C) ? pt_ld2(x0 + c0) : z;
      const float2 v10 = (in1 && c0 < C) ? pt_ld2(x1 + c0) : z;
      const float2 v01 = (in0 && c0 + 8 < C) ? pt_ld2(x0 + c0 + 8) : z;
      const float2 v11 = (in1 && c0 + 8 < C) ? pt_ld2(x1 + c0 + 8) : z;
      uint32_t ahi[4], alo[4];
      pt_split2(v00.x, v00.y, ahi[0], alo[0]);
      pt_split2(v10.x, v10.y, ahi[1], alo[1]);
      pt_split2(v01.x, v01.y, ahi[2], alo[2]);
      pt_split2(v11.x, v11.y, ahi[3], alo[3]);
      const uint32_t bc = dst + (uint32_t)kc * chunk_bytes;
      const uint32_t acc = (restart && kc == 0) ? 0u : 1u;
      wg_fence();
#pragma unroll
      for (int b = 0; b < PT_MAXB; ++b) {
        if (b < nb) {                                         // warp-uniform
          const uint64_t bhi = wg_desc(bc + (uint32_t)b * 256u, lbo, 128);
          const uint64_t blo = wg_desc(bc + lo_off + (uint32_t)b * 256u, lbo, 128);
          mma_n16(mainv[b], ahi, bhi, acc);                   // main (+)= A_hi . D_hi
          mma_n16(corr[b], ahi, blo, acc);                    // corr (+)= A_hi . D_lo
          mma_n16(corr[b], alo, bhi, 1u);                     // corr  += A_lo . D_hi
        }
      }
      wg_commit();
      wg_wait0();
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty[s]);
    if ((h + 1) % G == 0 || h + 1 == H) {
#pragma unroll
      for (int b = 0; b < PT_MAXB; ++b)
#pragma unroll
        for (int i = 0; i < 8; ++i) tot[b][i] = fmaf(corr[b][i], 1.0f / PT_LO_SCALE, tot[b][i] + mainv[b][i]);
    }
  }
  __syncthreads();
  if (tid == 0 && *abort_s) atomicOr(a.flags, CODA_B200_FLAG_PIPELINE_TIMEOUT);
  if (*abort_s) return;
  // accumulator fragment: register 4 j + 2 i + e of block b = item r0 + 8 i, class 16 b + 8 j + 2 (lane % 4) + e
  const float up = __uint_as_float((uint32_t)(127 + pt_down_shift(*a.dmax)) << 23);      // undo the D range scaling
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    if (r0 + 8 * i >= cnt) continue;
    float* urow = a.U + (size_t)(n0 + r0 + 8 * i) * C;
#pragma unroll
    for (int b = 0; b < PT_MAXB; ++b) {
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        const int col = 16 * b + 8 * j + 2 * (lane & 3);
        if (b < nb && col < C)                                // C % 4 == 0: both classes in range
          *reinterpret_cast<float2*>(urow + col) = make_float2(tot[b][4 * j + 2 * i] * up, tot[b][4 * j + 2 * i + 1] * up);
      }
    }
  }
}

struct PiTcPlan {
  int rows, stages;
  uint32_t xbytes, sbytes;
  size_t smem;
};

// two warpgroups (128 items per CTA) when two stages fit shared memory, else one; then as many stages as fit
PiTcPlan pi_tc_plan(int C, int Np, int KC, size_t esz) {
  PiTcPlan p;
  const size_t dbytes = (size_t)KC * Np * 64;
  const size_t slack = esz == 4 ? 0 : 16;                       // 16-bit tiles may start mid 16-byte unit
  for (p.rows = 2 * PT_WG; ; p.rows -= PT_WG) {
    p.xbytes = (uint32_t)(((size_t)p.rows * C * esz + slack + 127) & ~(size_t)127);
    p.sbytes = (uint32_t)(p.xbytes + dbytes);
    if (2 * (size_t)p.sbytes + PT_TAIL <= PT_SMEM_BUDGET || p.rows == PT_WG) break;
  }
  p.stages = (int)min((size_t)PT_MAX_STAGES, (PT_SMEM_BUDGET - PT_TAIL) / p.sbytes);
  p.smem = (size_t)p.stages * p.sbytes + PT_TAIL;
  return p;
}

}  // namespace

extern "C" int coda_b200_pi_full_tc_ok(int H, int64_t N, int C, int64_t model_stride) {
  return H >= 1 && N >= 1 && C >= 16 && C <= 128 && C % 4 == 0 && model_stride % 4 == 0;
}

// a 16-bit slab is staged at any element alignment (see the file comment): the model stride does not matter
extern "C" int coda_b200_pi_full_tc_ok_x(int fmt, int H, int64_t N, int C, int64_t model_stride) {
  if (fmt == CODA_B200_SLAB_F32) return coda_b200_pi_full_tc_ok(H, N, C, model_stride);
  return (fmt == CODA_B200_SLAB_F16 || fmt == CODA_B200_SLAB_BF16) && H >= 1 && N >= 1 && C >= 16 && C <= 128 &&
         C % 4 == 0;
}

extern "C" size_t coda_b200_pi_full_tc_scratch_bytes(int H, int C) {
  const int Np = (C + 15) / 16 * 16, KC = (C + 15) / 16;
  return (size_t)H * KC * 2 * Np * 16 * 2 + 16;
}

template <typename T>
static int pi_full_tc(const T* preds, int fmt, int64_t model_stride, const float* D, int H, int64_t N, int C, float* U,
                      void* scratch, uint32_t* flags, coda_stream_t stream) {
  CODA_CHECK_ARG(preds && D && U && scratch && flags, "pi_full_tc: null pointer");
  CODA_CHECK_ARG(coda_b200_pi_full_tc_ok_x(fmt, H, N, C, model_stride),
                 "pi_full_tc: needs 16 <= C <= 128, C %% 4 == 0 and (fp32) a 16-byte aligned model stride (C=%d)", C);
  CODA_CHECK_ARG((sizeof(T) != 4 || ((uintptr_t)preds & 15) == 0) && ((uintptr_t)U & 15) == 0 &&
                     ((uintptr_t)scratch & 15) == 0,
                 "pi_full_tc: preds (fp32), U and scratch must be 16-byte aligned");
  const int Np = (C + 15) / 16 * 16, KC = (C + 15) / 16;
  unsigned char* wb = reinterpret_cast<unsigned char*>(scratch);
  uint32_t* dmax = reinterpret_cast<uint32_t*>(wb + coda_b200_pi_full_tc_scratch_bytes(H, C) - 16);
  CODA_CUDA_OK(cudaMemsetAsync(dmax, 0, 16, as_stream(stream)));
  k_pi_w_max<<<coda_sm_count(), 256, 0, as_stream(stream)>>>(D, (long long)H * C * C, dmax);
  CODA_LAUNCH_OK("k_pi_w_max");
  k_pi_w_limbs<<<coda_sm_count() * 4, 256, 0, as_stream(stream)>>>(D, H, C, Np, KC, dmax, reinterpret_cast<__half*>(wb));
  CODA_LAUNCH_OK("k_pi_w_limbs");
  const PiTcPlan plan = pi_tc_plan(C, Np, KC, sizeof(T));
  CODA_CHECK_ARG(plan.stages >= 2, "pi_full_tc: C=%d does not fit shared memory", C);
  PiTcArgs a;
  a.preds = preds; a.ldh = model_stride; a.wb = wb; a.dmax = dmax; a.U = U; a.flags = flags;
  a.N = N; a.H = H; a.C = C; a.Np = Np; a.KC = KC;
  a.rows = plan.rows; a.S = plan.stages; a.xbytes = plan.xbytes; a.sbytes = plan.sbytes;
  // models per fold: the truncating fp32 accumulate of the tensor core loses up to 2^-24 per K = 8 sub-step of the chain
  const char* genv = getenv("CODA_B200_PI_DRAIN");
  a.G = genv ? max(1, min(16, atoi(genv))) : 4;
  CODA_CUDA_OK(cudaFuncSetAttribute(k_pi_full_tc<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)plan.smem));
  const long long grid = (N + plan.rows - 1) / plan.rows;
  k_pi_full_tc<T><<<(unsigned)grid, 2 * plan.rows, plan.smem, as_stream(stream)>>>(a);
  CODA_LAUNCH_OK("k_pi_full_tc");
  return CODA_B200_OK;
}

extern "C" int coda_b200_pi_full_tc(const float* preds, int64_t model_stride, const float* D, int H, int64_t N, int C,
                                    float* U, void* scratch, uint32_t* flags, coda_stream_t stream) {
  return pi_full_tc(preds, CODA_B200_SLAB_F32, model_stride, D, H, N, C, U, scratch, flags, stream);
}

extern "C" int coda_b200_pi_full_tc_x(const void* preds, int fmt, int64_t model_stride, const float* D, int H, int64_t N,
                                      int C, float* U, void* scratch, uint32_t* flags, coda_stream_t stream) {
  return slab_dispatch(fmt, preds, [&](auto* p) {
    return pi_full_tc(p, fmt, model_stride, D, H, N, C, U, scratch, flags, stream);
  });
}

CODA_MODULE_ANCHOR(pi_tc, k_pi_w_max)
