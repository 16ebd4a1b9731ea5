// ModelPicker's epsilon grid search on the device (coda_b200/eps_search.py, DESIGN.md §5b): many whole ModelPicker
// runs per launch.  A run is one (epsilon, realisation) pair: a pool of P items of the task, labelled for B steps.
// Each CTA carries the runs of one realisation for a block of epsilons and executes every step of them with no host
// involvement; a step of a run is what one step of ModelPicker.run_steps does on the same pool (k_mp_entropy<true>,
// the arg-min with its exact ties, k_bl_draw, k_select_kth_dev, k_bl_step), with the same arithmetic and the same
// Philox draws, so a run is bit for bit the device loop's.
#include "modelpicker.cuh"

#define MR_THREADS 256
#define MR_WARPS (MR_THREADS / 32)
#define MR_MAX_RUNS 32              // runs per CTA: the item loop keeps the active runs of an item in one 32-bit mask
#define MR_STEP_THREADS 256         // BL_THREADS of k_bl_step, whose fp64 posterior sum order the step restates
#define MR_ERR_NO_PICK 1u           // flags bit: a step found no tied item (a non-finite entropy)

struct MrArgs {
  const uint16_t* hard;             // [N][H]
  const int64_t* labels;            // [N]
  const uint8_t* disagree;          // [N]
  const int64_t* pool;              // [R][P] item of each pool position
  const float* gammas;              // [E] fp32 gamma of each epsilon
  const int64_t* keys;              // [E][R] Philox key of each run
  int H, C, P, B, E, ecta;
  long long R, r0;                  // all realisations; the first one of this launch
  float* ent;                       // scratch [CTAs of the launch][ecta][P]
  uint8_t* lab;                     // scratch [CTAs of the launch][ecta][P]
  int32_t* picks;                   // [E][R][B] pool position labelled at each step
  int32_t* best;                    // [E][R][B] best model after each step
  uint8_t* pick_tie;                // [E][R][B] the pick was drawn among > 1 exact ties
  uint8_t* best_tie;                // [E][R][B] the best model was drawn among > 1 exact ties
  uint32_t* flags;
};

static size_t mr_smem(int H, int ec) {
  const size_t Hp = (size_t)((H + 31) & ~31);
  return (size_t)ec * (2 * H * sizeof(double) + 5 * sizeof(double) + MR_WARPS * sizeof(double) + 2 * sizeof(long long) +
                       H * sizeof(float) + sizeof(float) + H * sizeof(int)) +
         MR_WARPS * Hp * sizeof(uint16_t);
}

// p_h, p_h log2 p_h, S, B and the no-group entropy of run e's posterior (one warp, as every warp of k_mp_entropy does)
__device__ __forceinline__ void mr_prologue(const float* post, double* sp, double* spl, double* sS, double* sB,
                                            double* sHn, int H, int lane) {
  for (int h = lane; h < H; h += 32) mp_post_terms(post[h], sp[h], spl[h]);
  __syncwarp();
  double S, B;
  mp_sums(sp, spl, H, lane, S, B);
  if (lane == 0) {
    *sS = S;
    *sB = B;
    *sHn = mp_h_none(S, B);
  }
}

__device__ __forceinline__ int mr_warp_max(int v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = max(v, __shfl_xor_sync(CODA_FULL, v, o));
  return v;
}

// the j-th (ascending) index i < n with pred(i), -1 if there is none; every lane gets the answer
template <typename Pred>
__device__ __forceinline__ int mr_kth(int n, long long j, int lane, Pred pred) {
  for (int i0 = 0; i0 < n; i0 += 32) {
    const int i = i0 + lane;
    const unsigned b = __ballot_sync(CODA_FULL, i < n && pred(i));
    const int c = __popc(b);
    if (j < c) {
      unsigned w = b;
      for (; j > 0; --j) w &= w - 1;
      return i0 + __ffs(w) - 1;
    }
    j -= c;
  }
  return -1;
}

__global__ void __launch_bounds__(MR_THREADS) k_mp_runs(const MrArgs a) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int H = a.H, P = a.P, EC = a.ecta, Hp = (H + 31) & ~31;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int e0 = blockIdx.x * EC, ne = min(EC, a.E - e0);
  const long long r = a.r0 + blockIdx.y;
  double* sp = reinterpret_cast<double*>(smem_raw);     // [EC][H]
  double* spl = sp + (size_t)EC * H;                    // [EC][H]
  double* sS = spl + (size_t)EC * H;
  double* sB = sS + EC;
  double* sHn = sB + EC;
  double* sGm1 = sHn + EC;
  double* sGlg = sGm1 + EC;
  double* wacc = sGlg + EC;                             // [MR_WARPS][EC] the item's acc per run (lane 0 of the warp)
  long long* nd = reinterpret_cast<long long*>(wacc + MR_WARPS * EC);   // unlabeled items some model disagrees on
  long long* key = nd + EC;
  float* post = reinterpret_cast<float*>(key + EC);     // [EC][H]
  float* gam = post + (size_t)EC * H;
  int* counts = reinterpret_cast<int*>(gam + EC);       // [EC][H] correct labels
  uint16_t* row = reinterpret_cast<uint16_t*>(counts + (size_t)EC * H) + (size_t)warp * Hp;
  const size_t cta = (size_t)blockIdx.y * gridDim.x + blockIdx.x;
  float* ent = a.ent + cta * EC * P;
  uint8_t* lab = a.lab + cta * EC * P;
  const int64_t* pool = a.pool + (size_t)r * P;

  // ModelPicker's initial state: posterior 1 / H (torch.ones(H) / H), no labels
  const float p0 = __fdiv_rn(1.0f, (float)H);
  for (int i = threadIdx.x; i < ne * P; i += MR_THREADS) lab[i] = 0;
  for (int i = threadIdx.x; i < ne * H; i += MR_THREADS) {
    post[i] = p0;
    counts[i] = 0;
  }
  if (warp == 0) {
    int nd0 = 0;
    for (int n = lane; n < P; n += 32) nd0 += a.disagree[pool[n]] != 0;
    nd0 = warp_sum(nd0);
    if (lane < ne) {
      const int e = lane;
      const double g = (double)a.gammas[e0 + e];
      gam[e] = a.gammas[e0 + e];
      sGm1[e] = g - 1.0;
      sGlg[e] = g * log2(g);
      nd[e] = nd0;
      key[e] = (long long)a.keys[(size_t)(e0 + e) * a.R + r];
    }
  }
  __syncthreads();
  for (int e = warp; e < ne; e += MR_WARPS)
    mr_prologue(post + (size_t)e * H, sp + (size_t)e * H, spl + (size_t)e * H, sS + e, sB + e, sHn + e, H, lane);
  __syncthreads();

  for (int s = 0; s < a.B; ++s) {
    // every unlabeled pool item under every run this CTA carries; its hard row is read once for all of them
    for (int n = warp; n < P; n += MR_WARPS) {
      const long long g = pool[n];
      const bool dis = a.disagree[g] != 0;
      unsigned act = 0;
      for (int e = 0; e < ne; ++e) {
        if (lab[(size_t)e * P + n]) continue;
        if (nd[e] > 0 && !dis) {                         // agreeing items are masked while disagreeing ones are left
          if (lane == 0) ent[(size_t)e * P + n] = INFINITY;
          continue;
        }
        act |= 1u << e;
      }
      if (!act) continue;                                // warp-uniform
      const uint16_t* src = a.hard + (size_t)g * H;
      for (int h = lane; h < H; h += 32) row[h] = src[h];
      __syncwarp();
      double* acc = wacc + warp * EC;
      if (lane == 0)
        for (unsigned m = act; m; m &= m - 1) acc[__ffs(m) - 1] = 0.0;
      int K = 0;
      for_each_group(row, H, lane, [&](uint16_t, unsigned mine) {
        for (unsigned m = act; m; m &= m - 1) {
          const int e = __ffs(m) - 1;
          const double t = mp_group_term(sp + (size_t)e * H, spl + (size_t)e * H, mine, lane, sS[e], sB[e], sGm1[e],
                                         sGlg[e]);
          if (lane == 0) acc[e] += t;
        }
        ++K;
      });
      if (lane == 0)
        for (unsigned m = act; m; m &= m - 1) {
          const int e = __ffs(m) - 1;
          ent[(size_t)e * P + n] = mp_item_entropy(acc[e], K, a.C, sHn[e]);
        }
      __syncwarp();
    }
    __syncthreads();

    // one warp per run: the pick, its label, the counts, the posterior, the best model, the next step's prologue
    for (int e = warp; e < ne; e += MR_WARPS) {
      const float* ev = ent + (size_t)e * P;
      uint8_t* lv = lab + (size_t)e * P;
      float mn = 0.f;
      int cnt = 0;                                       // {value, count} merges as vc_merge does
      for (int n = lane; n < P; n += 32) {
        if (lv[n]) continue;
        const float v = ev[n];
        if (cnt == 0 || v < mn) { mn = v; cnt = 1; }
        else if (v == mn) ++cnt;
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        const float v = __shfl_xor_sync(CODA_FULL, mn, o);
        const int c = __shfl_xor_sync(CODA_FULL, cnt, o);
        if (c == 0) continue;
        if (cnt == 0 || v < mn) { mn = v; cnt = c; }
        else if (v == mn) cnt += c;
      }
      const long long k = cnt > 1 ? bl_tie_pick(bl_philox(key[e], s, 0u), cnt) : 0;
      const int pick = mr_kth(P, k, lane, [&](int n) { return !lv[n] && ev[n] == mn; });
      const size_t o = ((size_t)(e0 + e) * a.R + r) * a.B + s;
      if (pick < 0) {                                    // warp-uniform
        if (lane == 0) {
          atomicOr(a.flags, MR_ERR_NO_PICK);
          a.picks[o] = -1;
          a.best[o] = -1;
        }
        continue;
      }
      const long long g = pool[pick];
      const long long lab_g = a.labels[g];
      const uint16_t* src = a.hard + (size_t)g * H;
      float* pe = post + (size_t)e * H;
      int* ce = counts + (size_t)e * H;
      const float gf = gam[e];
      for (int h = lane; h < H; h += 32) {
        const bool agree = (long long)src[h] == lab_g;
        ce[h] += agree ? 1 : 0;
        if (agree) pe[h] = __fmul_rn(pe[h], gf);
      }
      __syncwarp();
      double tot = 0.0;
      for (int w = 0; w < MR_STEP_THREADS / 32; ++w) {
        double part = 0.0;
        for (int h = w * 32 + lane; h < H; h += MR_STEP_THREADS) part += (double)pe[h];
        tot += warp_sum(part);
      }
      const float sf = (float)tot;
      int mx = INT_MIN;
      for (int h = lane; h < H; h += 32) {
        pe[h] = __fdiv_rn(pe[h], sf);
        mx = max(mx, ce[h]);
      }
      mx = mr_warp_max(mx);
      int cntb = 0;
      for (int h0 = 0; h0 < H; h0 += 32) cntb += __popc(__ballot_sync(CODA_FULL, h0 + lane < H && ce[h0 + lane] == mx));
      const long long j = cntb > 1 ? bl_tie_pick(bl_philox(key[e], s + 1, 1u), cntb) : 0;
      const int bm = mr_kth(H, j, lane, [&](int h) { return ce[h] == mx; });
      if (lane == 0) {
        lv[pick] = 1;
        if (a.disagree[g]) nd[e] -= 1;
        a.picks[o] = pick;
        a.best[o] = bm;
        a.pick_tie[o] = cnt > 1;
        a.best_tie[o] = cntb > 1;
      }
      __syncwarp();
      mr_prologue(pe, sp + (size_t)e * H, spl + (size_t)e * H, sS + e, sB + e, sHn + e, H, lane);
    }
    __syncthreads();
  }
}

struct MrPlan {
  int ecta, eblocks;
  long long rchunk;
  size_t smem, scratch;
};

// runs per CTA: as many epsilons as the shared memory holds (at most MR_MAX_RUNS), spread evenly over the blocks;
// realisations per launch: one wave of resident CTAs, so that a launch lasts about as long as one CTA's runs
static int mr_plan(int H, int E, int P, long long R, MrPlan* pl) {
  int dev = 0, optin = 0;
  CODA_CUDA_OK(cudaGetDevice(&dev));
  CODA_CUDA_OK(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
  int ec = min(E, MR_MAX_RUNS);
  while (ec > 1 && mr_smem(H, ec) > (size_t)optin) --ec;
  CODA_CHECK_ARG(mr_smem(H, ec) <= (size_t)optin, "mp_runs: H=%d needs more shared memory than the device has", H);
  pl->eblocks = (E + ec - 1) / ec;
  pl->ecta = (E + pl->eblocks - 1) / pl->eblocks;
  pl->smem = mr_smem(H, pl->ecta);
  CODA_CUDA_OK(cudaFuncSetAttribute(k_mp_runs, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)pl->smem));
  int per_sm = 0;
  CODA_CUDA_OK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_mp_runs, MR_THREADS, pl->smem));
  const long long wave = (long long)max(per_sm, 1) * coda_sm_count();
  pl->rchunk = max(1LL, min(R, wave / pl->eblocks));
  pl->scratch = (size_t)pl->rchunk * pl->eblocks * pl->ecta * P * (sizeof(float) + sizeof(uint8_t));
  return CODA_B200_OK;
}

static int mr_shape_ok(int H, int E, int P, long long R, int B) {
  CODA_CHECK_ARG(H >= 1 && H <= 1024 && E >= 1 && P >= 1 && R >= 1 && B >= 1 && B <= P && R <= 65535LL * 65535LL,
                 "mp_runs: bad shape H=%d E=%d P=%d R=%lld B=%d", H, E, P, R, B);
  return CODA_B200_OK;
}

extern "C" int coda_b200_mp_runs_plan(int H, int E, int P, int64_t R, int B, int64_t* plan) {
  CODA_CHECK_ARG(plan, "mp_runs_plan: null pointer");
  if (int rc = mr_shape_ok(H, E, P, R, B)) return rc;
  MrPlan pl;
  if (int rc = mr_plan(H, E, P, R, &pl)) return rc;
  plan[0] = pl.ecta;
  plan[1] = pl.eblocks;
  plan[2] = pl.rchunk;
  plan[3] = (int64_t)pl.smem;
  plan[4] = (int64_t)pl.scratch;
  return CODA_B200_OK;
}

extern "C" int coda_b200_mp_runs(const uint16_t* hard, const int64_t* labels, const uint8_t* disagree, int H, int C,
                                 const int64_t* pool, int64_t R, int P, int B, const float* gammas,
                                 const int64_t* keys, int E, void* scratch, size_t scratch_bytes, int32_t* picks,
                                 int32_t* best, uint8_t* pick_tie, uint8_t* best_tie, uint32_t* flags,
                                 coda_stream_t stream) {
  CODA_CHECK_ARG(hard && labels && disagree && pool && gammas && keys && scratch && picks && best && pick_tie &&
                 best_tie && flags, "mp_runs: null pointer");
  CODA_CHECK_ARG(C >= 1, "mp_runs: bad C=%d", C);
  if (int rc = mr_shape_ok(H, E, P, R, B)) return rc;
  MrPlan pl;
  if (int rc = mr_plan(H, E, P, R, &pl)) return rc;
  CODA_CHECK_ARG(scratch_bytes >= pl.scratch, "mp_runs: scratch of %zu bytes, %zu needed", scratch_bytes, pl.scratch);
  MrArgs a;
  a.hard = hard; a.labels = labels; a.disagree = disagree; a.pool = pool; a.gammas = gammas; a.keys = keys;
  a.H = H; a.C = C; a.P = P; a.B = B; a.E = E; a.ecta = pl.ecta; a.R = R;
  a.ent = static_cast<float*>(scratch);
  a.lab = static_cast<uint8_t*>(scratch) + (size_t)pl.rchunk * pl.eblocks * pl.ecta * P * sizeof(float);
  a.picks = picks; a.best = best; a.pick_tie = pick_tie; a.best_tie = best_tie; a.flags = flags;
  for (long long r0 = 0; r0 < R; r0 += pl.rchunk) {
    a.r0 = r0;
    const dim3 grid((unsigned)pl.eblocks, (unsigned)min(pl.rchunk, R - r0));
    k_mp_runs<<<grid, MR_THREADS, pl.smem, as_stream(stream)>>>(a);
    CODA_LAUNCH_OK("k_mp_runs");
  }
  return CODA_B200_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// The search's oracle and yardstick: majority labels and per-realisation pool accuracies
// ---------------------------------------------------------------------------------------------------------------
// one warp per item: the class most models predict, the smallest class id among equal counts (np.unique + argmax)
__global__ void __launch_bounds__(MR_THREADS) k_majority(const uint16_t* __restrict__ hard, int H, long long N,
                                                        int64_t* __restrict__ labels) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int Hp = (H + 31) & ~31;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  uint16_t* row = reinterpret_cast<uint16_t*>(smem_raw) + (size_t)warp * Hp;
  const long long nw = (long long)gridDim.x * MR_WARPS;
  for (long long n = (long long)blockIdx.x * MR_WARPS + warp; n < N; n += nw) {
    const uint16_t* src = hard + (size_t)n * H;
    for (int h = lane; h < H; h += 32) row[h] = src[h];
    __syncwarp();
    int bc = 0, bm = 0;                                  // groups come in lowest-model order, not class order
    for_each_group(row, H, lane, [&](uint16_t c, unsigned mine) {
      const int m = warp_sum((int)__popc(mine));
      if (m > bm || (m == bm && (int)c < bc)) { bm = m; bc = c; }
    });
    if (lane == 0) labels[n] = bc;
    __syncwarp();
  }
}

extern "C" int coda_b200_majority(const uint16_t* hard, int H, int64_t N, int64_t* labels, coda_stream_t stream) {
  CODA_CHECK_ARG(hard && labels, "majority: null pointer");
  CODA_CHECK_ARG(H >= 1 && H <= 1024 && N >= 1, "majority: bad shape H=%d N=%lld", H, (long long)N);
  const size_t smem = (size_t)MR_WARPS * ((H + 31) & ~31) * sizeof(uint16_t);
  long long grid = (N + MR_WARPS - 1) / MR_WARPS;
  grid = min(grid, (long long)coda_sm_count() * 8);
  k_majority<<<(unsigned)grid, MR_THREADS, smem, as_stream(stream)>>>(hard, H, N, labels);
  CODA_LAUNCH_OK("k_majority");
  return CODA_B200_OK;
}

// acc[r][h] = the pool items of realisation r that model h predicts as labels[] has them
__global__ void __launch_bounds__(MR_THREADS) k_pool_accuracy(const uint16_t* __restrict__ hard,
                                                             const int64_t* __restrict__ labels, int H,
                                                             const int64_t* __restrict__ pool, int P,
                                                             int32_t* __restrict__ acc) {
  const long long r = blockIdx.x;
  const int64_t* pr = pool + (size_t)r * P;
  for (int h = threadIdx.x; h < H; h += MR_THREADS) {
    int c = 0;
    for (int p = 0; p < P; ++p) {
      const long long g = pr[p];
      c += (long long)hard[(size_t)g * H + h] == labels[g];
    }
    acc[(size_t)r * H + h] = c;
  }
}

extern "C" int coda_b200_pool_accuracy(const uint16_t* hard, const int64_t* labels, int H, const int64_t* pool,
                                       int64_t R, int P, int32_t* acc, coda_stream_t stream) {
  CODA_CHECK_ARG(hard && labels && pool && acc, "pool_accuracy: null pointer");
  CODA_CHECK_ARG(H >= 1 && H <= 1024 && R >= 1 && R < (1LL << 31) && P >= 1, "pool_accuracy: bad shape H=%d R=%lld P=%d",
                 H, (long long)R, P);
  k_pool_accuracy<<<(unsigned)R, MR_THREADS, 0, as_stream(stream)>>>(hard, labels, H, pool, P, acc);
  CODA_LAUNCH_OK("k_pool_accuracy");
  return CODA_B200_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// A search's pool table: the rows of one piece's items that a block of realisations draws, copied to table slots
// ---------------------------------------------------------------------------------------------------------------
// one warp per pair: out_hard[slot] = hard[item] (H u16 as V words), out_disagree[slot], out_labels[slot].  A row is
// 2H bytes, so with H a multiple of 8 (4, 2) every row starts 16 (8, 4) bytes into an aligned buffer.
template <typename V>
__global__ void __launch_bounds__(MR_THREADS) k_pool_gather(const uint16_t* __restrict__ hard,
                                                           const uint8_t* __restrict__ disagree,
                                                           const int64_t* __restrict__ labels, int H,
                                                           const int64_t* __restrict__ slots,
                                                           const int64_t* __restrict__ items, long long K,
                                                           uint16_t* __restrict__ out_hard,
                                                           uint8_t* __restrict__ out_disagree,
                                                           int64_t* __restrict__ out_labels) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int W = H * (int)sizeof(uint16_t) / (int)sizeof(V);
  const long long nw = (long long)gridDim.x * MR_WARPS;
  for (long long k = (long long)blockIdx.x * MR_WARPS + warp; k < K; k += nw) {
    const long long n = items[k], s = slots[k];
    const V* src = reinterpret_cast<const V*>(hard + (size_t)n * H);
    V* dst = reinterpret_cast<V*>(out_hard + (size_t)s * H);
    for (int w = lane; w < W; w += 32) dst[w] = src[w];
    if (lane == 0) {
      out_disagree[s] = disagree[n];
      out_labels[s] = labels[n];
    }
  }
}

extern "C" int coda_b200_pool_gather(const uint16_t* hard, const uint8_t* disagree, const int64_t* labels, int H,
                                     const int64_t* slots, const int64_t* items, int64_t K, uint16_t* out_hard,
                                     uint8_t* out_disagree, int64_t* out_labels, coda_stream_t stream) {
  CODA_CHECK_ARG(H >= 1 && H <= 1024 && K >= 0, "pool_gather: bad shape H=%d K=%lld", H, (long long)K);
  if (K == 0) return CODA_B200_OK;
  CODA_CHECK_ARG(hard && disagree && labels && slots && items && out_hard && out_disagree && out_labels,
                 "pool_gather: null pointer");
  CODA_CHECK_ARG(((uintptr_t)hard | (uintptr_t)out_hard) % 16 == 0, "pool_gather: hard tables must be 16-byte aligned");
  long long grid = (K + MR_WARPS - 1) / MR_WARPS;
  grid = min(grid, (long long)coda_sm_count() * 16);
  const cudaStream_t s = as_stream(stream);
  if (H % 8 == 0)
    k_pool_gather<uint4><<<(unsigned)grid, MR_THREADS, 0, s>>>(hard, disagree, labels, H, slots, items, K, out_hard,
                                                               out_disagree, out_labels);
  else if (H % 4 == 0)
    k_pool_gather<uint2><<<(unsigned)grid, MR_THREADS, 0, s>>>(hard, disagree, labels, H, slots, items, K, out_hard,
                                                               out_disagree, out_labels);
  else if (H % 2 == 0)
    k_pool_gather<uint32_t><<<(unsigned)grid, MR_THREADS, 0, s>>>(hard, disagree, labels, H, slots, items, K,
                                                                  out_hard, out_disagree, out_labels);
  else
    k_pool_gather<uint16_t><<<(unsigned)grid, MR_THREADS, 0, s>>>(hard, disagree, labels, H, slots, items, K,
                                                                  out_hard, out_disagree, out_labels);
  CODA_LAUNCH_OK("k_pool_gather");
  return CODA_B200_OK;
}

CODA_MODULE_ANCHOR(eps_search, k_mp_runs)
