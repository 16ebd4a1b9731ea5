// Beta quadrature tables (the P(best) mixture over classes is in step.cu).
//
// The reference (coda.py:77-119) evaluates, for every hypothetical (item b, class c), the
// pdf / cumulative-trapezoid cdf of H Beta distributions on a 256-node grid.  Only three
// distinct Betas exist per (model h, class c):  before=(a, b), miss=(a, b+w), hit=(a+w, b)
// (coda.py:150-168), so they are tabulated once per class and the per-item work reduces to
//
//   prob_h(b, c) = sum_x G_{z_h}[c][x][h] * D_{b,c}(x),      D_{b,c}(x) = exp(sum_{h in Z} dL[c][h][x])
//
// with Z = {h : p_h(b) = c}, z_h = [h in Z] and
//   dL[c][h][x]  = L_hit - L_miss                       (L = log(max(cdf, 1e-30)), coda.py:104)
//   G0[c][x][h]  = wq[x] * pdf_miss[h][x] * exp(clamp(S0_c[x] - L_miss[h][x], -80, 80))
//   G1[c][x][h]  = wq[x] * pdf_hit [h][x] * exp(clamp(S0_c[x] - L_hit [h][x], -80, 80))
//   S0_c[x]      = sum_h L_miss[h][x]                   (coda.py:107 leave-one-out product)
//   wq           = trapezoid weights of the fp32 grid   (coda.py:111 torch.trapz)
// The +-80 clamp of coda.py:107 is applied to the class-level factor; it differs from the
// reference's per-item clamp only where the integrand is below e^-80 (see DESIGN.md).
// PB[c][h] is the "before" row P(h best | class c) (coda.py:245-251, 325-332), normalised.
//
// Tables are built in fp64 from fp32 inputs and rounded to fp32 once.
#include "common.cuh"

#include <cuda_bf16.h>

#define TP_ 256   // quadrature nodes == threads per block in the table kernels

__device__ __forceinline__ double block_scan_incl(double v, double* wsum /*[8]*/) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    double t = __shfl_up_sync(CODA_FULL, v, o);
    if (lane >= o) v += t;
  }
  if (lane == 31) wsum[warp] = v;
  __syncthreads();
  double off = 0.0;
  for (int w = 0; w < warp; ++w) off += wsum[w];
  __syncthreads();
  return v + off;
}

// grid = (H, ncls); block = 256 threads, one per node.
__global__ void __launch_bounds__(TP_) k_beta_nodes(const float* __restrict__ D, const float* __restrict__ grid_x,
                                                    int H, int C, int cls_lo, float w,
                                                    const long long* __restrict__ sel,
                                                    double* __restrict__ pdf_s, double* __restrict__ L_s,
                                                    uint32_t* __restrict__ flags) {
  if (sel) cls_lo = (int)sel[1];   // device-resident class (host-free loop)
  __shared__ double red[8];
  __shared__ double wsum[8];
  __shared__ double pdf_sh[TP_];
  __shared__ double lgn[3];     // lgamma(a+b) - lgamma(a) - lgamma(b) per variant: node-independent
  const int h = blockIdx.x, ci = blockIdx.y, c = cls_lo + ci, x = threadIdx.x;
  const int ncls = gridDim.y;
  const float* drow = D + ((size_t)h * C + c) * C;
  // rowsum (coda.py:24): accumulate in double, round once to fp32
  double part = 0.0;
  for (int j = x; j < C; j += TP_) part += (double)drow[j];
  part = warp_sum(part);
  if ((x & 31) == 0) red[x >> 5] = part;
  __syncthreads();
  double rs = 0.0;
  for (int k = 0; k < 8; ++k) rs += red[k];
  const float alpha = drow[c];
  const float beta = (float)rs - alpha;                          // coda.py:24
  const float xf = grid_x[x];
  const double lx = log((double)xf);
  const double l1x = log((double)(1.0f - xf));                    // fp32 (1 - x) as the reference forms it
  const float dxf = x > 0 ? (xf - grid_x[x - 1]) : 0.f;           // coda.py:100 (fp32 difference)
  uint32_t bad = 0;
  if (x < 3) {
    const float a = alpha + (x == 2 ? w : 0.f), b = beta + (x == 1 ? w : 0.f);
    lgn[x] = lgamma((double)(a + b)) - (lgamma((double)a) + lgamma((double)b));
  }
  __syncthreads();
  for (int v = 0; v < 3; ++v) {
    const float a = alpha + (v == 2 ? w : 0.f);                   // coda.py:165
    const float b = beta + (v == 1 ? w : 0.f);                    // coda.py:166
    // torch.distributions.Dirichlet.log_prob (dirichlet.py:90-97) on [x, 1-x] with conc [a, b]
    const double am1 = (double)(a - 1.0f), bm1 = (double)(b - 1.0f);
    const double t1 = (am1 == 0.0) ? 0.0 : am1 * lx;              // xlogy(0, .) = 0
    const double t2 = (bm1 == 0.0) ? 0.0 : bm1 * l1x;
    const double lp = (t1 + t2) + lgn[v];
    const double pdf = exp(lp);
    if (!isfinite(pdf) || !(a > 0.f) || !(b > 0.f)) bad |= CODA_B200_FLAG_NONFINITE_TABLE;
    __syncthreads();
    pdf_sh[x] = pdf;
    __syncthreads();
    const double inc = x > 0 ? 0.5 * (pdf + pdf_sh[x - 1]) * (double)dxf : 0.0;   // coda.py:101
    const double cdf = block_scan_incl(inc, wsum);
    const double L = log(fmax(cdf, (double)1e-30f));              // coda.py:104
    const size_t o = (((size_t)v * ncls + ci) * H + h) * TP_ + x;
    pdf_s[o] = pdf;
    L_s[o] = L;
  }
  if (bad) atomicOr(flags, bad);
}

// grid = (ncls, nsplit); block = (256 nodes, NP parts).  Every CTA forms S0 / SB for its class: part p sums the
// models h = p, p + NP, ... and the partial sums are combined in a fixed order, so every CTA (and every replica on
// every GPU) computes the same bits.  Then part p of CTA (ci, sl) writes dL, G0T, G1T and the raw "before"
// integrals for the models h = sl + nsplit * (p + NP * i).
#define HSPLIT 8
template <int NP>
__global__ void __launch_bounds__(TP_ * NP) k_beta_combine(const double* __restrict__ pdf_s, const double* __restrict__ L_s,
                                                          const float* __restrict__ grid_x, int H, int Hp, int cls_lo,
                                                          const long long* __restrict__ sel, float* __restrict__ dL,
                                                          float* __restrict__ G0T, float* __restrict__ G1T,
                                                          __nv_bfloat16* __restrict__ dLb, __nv_bfloat16* __restrict__ Gb,
                                                          double* __restrict__ pb_raw, uint32_t* __restrict__ flags) {
  if (sel) cls_lo = (int)sel[1];
  __shared__ double part[NP][8];
  __shared__ double s0p[NP][TP_], sbp[NP][TP_];
  const int ci = blockIdx.x, c = cls_lo + ci, x = threadIdx.x, p = threadIdx.y, ncls = gridDim.x;
  const int lane = x & 31, warp = x >> 5;
  const size_t plane = (size_t)ncls * H * TP_;
  const double* Lb = L_s + 0 * plane + (size_t)ci * H * TP_;
  const double* Lm = L_s + 1 * plane + (size_t)ci * H * TP_;
  const double* Lh = L_s + 2 * plane + (size_t)ci * H * TP_;
  const double* pb = pdf_s + 0 * plane + (size_t)ci * H * TP_;
  const double* pm = pdf_s + 1 * plane + (size_t)ci * H * TP_;
  const double* ph = pdf_s + 2 * plane + (size_t)ci * H * TP_;
  // trapezoid weight of node x from the fp32 grid differences (coda.py:111)
  const float xf = grid_x[x];
  const float dl_ = x > 0 ? xf - grid_x[x - 1] : 0.f;
  const float dr_ = x < TP_ - 1 ? grid_x[x + 1] - xf : 0.f;
  const double wq = 0.5 * ((double)dl_ + (double)dr_);
  {
    double a0 = 0.0, ab = 0.0;
    for (int h = p; h < H; h += NP) {
      a0 += Lm[(size_t)h * TP_ + x];
      ab += Lb[(size_t)h * TP_ + x];
    }
    s0p[p][x] = a0;
    sbp[p][x] = ab;
  }
  __syncthreads();
  double S0 = 0.0, SB = 0.0;
#pragma unroll
  for (int q = 0; q < NP; ++q) {      // fixed order
    S0 += s0p[q][x];
    SB += sbp[q][x];
  }
  uint32_t bad = 0;
  const int niter = (H + gridDim.y * NP - 1) / (gridDim.y * NP);
  for (int it = 0; it < niter; ++it) {
    const int h = blockIdx.y + gridDim.y * (p + NP * it);
    double ib = 0.0;
    if (h < H) {
      const size_t o = (size_t)h * TP_ + x;
      const double lm = Lm[o], lh = Lh[o], lb = Lb[o];
      const double g0 = wq * pm[o] * exp(fmin(fmax(S0 - lm, -80.0), 80.0));
      const double g1 = wq * ph[o] * exp(fmin(fmax(S0 - lh, -80.0), 80.0));
      ib = wq * pb[o] * exp(fmin(fmax(SB - lb, -80.0), 80.0));
      const float g0f = (float)g0, g1f = (float)g1;
      if (!isfinite(g0f) || !isfinite(g1f) || !isfinite(ib)) bad |= CODA_B200_FLAG_NONFINITE_TABLE;
      const float dlf = (float)(lh - lm);
      dL[((size_t)c * H + h) * TP_ + x] = dlf;
      G0T[((size_t)c * TP_ + x) * Hp + h] = g0f;
      G1T[((size_t)c * TP_ + x) * Hp + h] = g1f;
      if (dLb) {
        // tensor-core operand tables (pairs_tc.cu): bf16 limbs in the wgmma no-swizzle K-major core-matrix order
        // [k_core][r_core][8 rows][8 elements].  dLb tile: rows = nodes, K = 32 models; Gb tile: rows = models, K = 16 nodes.
        const __nv_bfloat16 d0 = __float2bfloat16_rn(dlf);
        const float r1 = dlf - __bfloat162float(d0);
        const __nv_bfloat16 d1 = __float2bfloat16_rn(r1);
        const __nv_bfloat16 d2 = __float2bfloat16_rn(r1 - __bfloat162float(d1));
        const size_t nka = (size_t)Hp / 32;
        const size_t ta = ((size_t)c * nka + (h >> 5)) * 3 * (TP_ * 32);
        const size_t ea = (size_t)((((h & 31) >> 3) * (TP_ / 8) + (x >> 3)) * 64 + (x & 7) * 8 + (h & 7));
        dLb[ta + 0 * (TP_ * 32) + ea] = d0;
        dLb[ta + 1 * (TP_ * 32) + ea] = d1;
        dLb[ta + 2 * (TP_ * 32) + ea] = d2;
        const __nv_bfloat16 a0 = __float2bfloat16_rn(g0f), b0 = __float2bfloat16_rn(g1f);
        const __nv_bfloat16 a1 = __float2bfloat16_rn(g0f - __bfloat162float(a0));
        const __nv_bfloat16 b1 = __float2bfloat16_rn(g1f - __bfloat162float(b0));
        const size_t tsz = (size_t)Hp * 16;
        const size_t tb = ((size_t)c * (TP_ / 16) + (x >> 4)) * 4 * tsz;
        const size_t eb = (size_t)((((x & 15) >> 3) * (Hp / 8) + (h >> 3)) * 64 + (h & 7) * 8 + (x & 7));
        Gb[tb + 0 * tsz + eb] = a0;
        Gb[tb + 1 * tsz + eb] = a1;
        Gb[tb + 2 * tsz + eb] = b0;
        Gb[tb + 3 * tsz + eb] = b1;
      }
    }
    ib = warp_sum(ib);
    __syncthreads();
    if (lane == 0) part[p][warp] = ib;
    __syncthreads();
    if (x == 0 && h < H) {
      double sum = 0.0;
      for (int w8 = 0; w8 < 8; ++w8) sum += part[p][w8];   // fixed order
      pb_raw[(size_t)ci * Hp + h] = sum;
    }
  }
  if (bad) atomicOr(flags, bad);
}

// PB row: normalise the raw integrals over h (coda.py:114).  grid = (ncls), block = 256.
__global__ void __launch_bounds__(TP_) k_pb_normalize(const double* __restrict__ pb_raw, int H, int Hp, int cls_lo,
                                                      const long long* __restrict__ sel, float* __restrict__ PB,
                                                      uint32_t* __restrict__ flags) {
  if (sel) cls_lo = (int)sel[1];
  __shared__ double red[8];
  const int ci = blockIdx.x, c = cls_lo + ci, x = threadIdx.x;
  const double* row = pb_raw + (size_t)ci * Hp;
  double tot = 0.0;
  for (int h = x; h < H; h += TP_) tot += row[h];
  tot = warp_sum(tot);
  if ((x & 31) == 0) red[x >> 5] = tot;
  __syncthreads();
  double total = 0.0;
  for (int k = 0; k < 8; ++k) total += red[k];
  if (!isfinite(total) && x == 0) atomicOr(flags, CODA_B200_FLAG_NONFINITE_TABLE);
  total = fmax(total, (double)1e-30f);
  for (int h = x; h < Hp; h += TP_) PB[(size_t)c * Hp + h] = h < H ? (float)(row[h] / total) : 0.f;
}

extern "C" size_t coda_b200_tables_scratch_bytes(int H, int ncls) {
  const int Hp = (H + 31) / 32 * 32;
  return (size_t)2 * 3 * ncls * H * TP_ * sizeof(double) + (size_t)ncls * Hp * sizeof(double);
}

extern "C" int coda_b200_beta_tables(const float* D, const float* grid_x, int H, int C, int P, double hyp_w,
                                     int cls_lo, int cls_hi, const int64_t* sel, void* scratch, float* dL,
                                     float* G0T, float* G1T, float* PB, void* dLb, void* Gb, uint32_t* flags,
                                     coda_stream_t stream) {
  CODA_CHECK_ARG(D && grid_x && scratch && dL && G0T && G1T && PB && flags, "beta_tables: null pointer");
  CODA_CHECK_ARG(P == TP_, "beta_tables: P must be %d", TP_);
  CODA_CHECK_ARG((dLb == nullptr) == (Gb == nullptr), "beta_tables: dLb and Gb go together");
  if (sel) { cls_lo = 0; cls_hi = 1; }   // one class, index read from sel[1] on the device
  CODA_CHECK_ARG(0 <= cls_lo && cls_lo < cls_hi && cls_hi <= C, "beta_tables: bad class range [%d,%d)", cls_lo, cls_hi);
  const int ncls = cls_hi - cls_lo;
  const long long* seld = reinterpret_cast<const long long*>(sel);
  const int Hp = (H + 31) / 32 * 32;
  double* pdf_s = reinterpret_cast<double*>(scratch);
  double* L_s = pdf_s + (size_t)3 * ncls * H * TP_;
  double* pb_raw = L_s + (size_t)3 * ncls * H * TP_;
  dim3 g1((unsigned)H, (unsigned)ncls);
  k_beta_nodes<<<g1, TP_, 0, as_stream(stream)>>>(D, grid_x, H, C, cls_lo, (float)hyp_w, seld, pdf_s, L_s, flags);
  CODA_LAUNCH_OK("k_beta_nodes");
  {
    // the S0 / SB sums are split over four parts per node in BOTH launch shapes: a class table must carry the same bits
    // whether it was built alone (per-step refresh, on the critical path of a sharded step) or in a batch (construction,
    // checkpoint resume).  Few classes: spread the models over more CTAs.
    const int split = ncls >= 16 ? (H / 4 < HSPLIT ? (H / 4 > 0 ? H / 4 : 1) : HSPLIT) : (H <= 4 ? 1 : (H / 4 < 64 ? H / 4 : 64));
    dim3 g2((unsigned)ncls, (unsigned)split), b2(TP_, 4);
    k_beta_combine<4><<<g2, b2, 0, as_stream(stream)>>>(pdf_s, L_s, grid_x, H, Hp, cls_lo, seld, dL, G0T, G1T,
                                                        reinterpret_cast<__nv_bfloat16*>(dLb), reinterpret_cast<__nv_bfloat16*>(Gb), pb_raw, flags);
  }
  CODA_LAUNCH_OK("k_beta_combine");
  k_pb_normalize<<<ncls, TP_, 0, as_stream(stream)>>>(pb_raw, H, Hp, cls_lo, seld, PB, flags);
  CODA_LAUNCH_OK("k_pb_normalize");
  return CODA_B200_OK;
}


CODA_MODULE_ANCHOR(tables, k_beta_nodes)
