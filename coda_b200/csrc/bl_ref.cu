// tie_rule="reference" of the competing selectors' host-free loop (include/coda_b200.h, "torch's generators on the
// device"): the draws the reference makes from torch's generators, made from device replicas of them.
//   CPU generator (at::mt19937): the MT19937 core of pyrandom.cuh.  torch keeps {left, next} where Python keeps pos;
//     the host converts (pos = 625 - left).  random() is one tempered word; randperm(n) is Fisher-Yates with
//     z = random() % (n - i), i = 0 .. n - 2, so randperm(n)[0] = random() % n followed by n - 2 more words;
//     randint(n) is random() % n below 2^28 and random64() % n (two words, the first the high half) from it.
//   CUDA generator (Philox4x32-10, {seed, offset}): randint(n, (1,)) is curand4 of curand_init(seed, 0, offset), x % n
//     below 2^28, and advances the offset by 4 (one element: one curand4 per thread, 4 counter words).
// Each kernel is one warp; the words of the CPU replica live in shared memory between a load and a store, as
// pyrandom.cuh's do.  Every shard runs the same kernels on the same global counts, so the replicas need no exchange.
#include "modelpicker.cuh"
#include "pyrandom.cuh"
#include <curand_kernel.h>

#define BR_STOP_NO_ITEM 3                    // ls[2]: no item was picked (include/coda_b200.h, loop words)
#define BR_RANDINT64 (1LL << 28)             // torch's randint switches to 64-bit draws here

// n words drawn and dropped: a twist per 624
__device__ __forceinline__ void tc_skip(PyRand& g, long long n) {
  while (n > 0) {
    if (g.pos >= PR_N) {
      pr_twist(g.mt);
      g.pos = 0;
    }
    const int a = (int)min(n, (long long)(PR_N - g.pos));
    g.pos += a;
    n -= a;
  }
}

// torch.randperm(n)[0] (2 <= n < 2^32 / 20, the 32-bit branch of randperm_cpu): n - 1 words
__device__ __forceinline__ long long tc_randperm0(PyRand& g, long long n) {
  const long long r = (long long)pr_next(g) % n;
  tc_skip(g, n - 2);
  return r;
}

// torch.randint(n, (1,)) on the CPU generator (n >= 1)
__device__ __forceinline__ long long tc_randint(PyRand& g, long long n) {
  if (n >= BR_RANDINT64) {
    const unsigned long long hi = pr_next(g), lo = pr_next(g);
    return (long long)(((hi << 32) | lo) % (unsigned long long)n);
  }
  return (long long)pr_next(g) % n;
}

// torch.randint(n, (1,), device="cuda") (1 <= n < 2^28) from {seed, offset}; the offset advances by 4
__device__ __forceinline__ long long tg_randint(long long* __restrict__ gs, long long n) {
  curandStatePhilox4_32_10_t s;
  curand_init((unsigned long long)gs[0], 0ull, (unsigned long long)gs[1], &s);
  const uint4 r = curand4(&s);
  __syncwarp();
  if ((threadIdx.x & 31) == 0) gs[1] += 4;
  return (long long)(r.x % (unsigned)n);
}

// Uncertainty / ModelPicker, in place of bl_draw: the k of this step's k-th item tie.  Uncertainty draws
// randperm(cnt)[0] when cnt > 1 items tie (uncertainty.py), ModelPicker randint(cnt) every step (modelpicker.py:70).
__global__ void __launch_bounds__(32) k_bl_draw_ref(const coda_bl_loop_t a, uint32_t* __restrict__ trng) {
  __shared__ uint32_t mt[PR_N];
  long long* ls = reinterpret_cast<long long*>(a.ls);
  if (ls[2]) return;
  const long long cnt = a.best[1];
  if (cnt < 1) {
    if (threadIdx.x == 0) ls[2] = BR_STOP_NO_ITEM;
    return;
  }
  const bool mp = a.method == CODA_B200_BL_MODELPICKER;
  if (!mp && cnt == 1) {
    if (threadIdx.x == 0) ls[3] = ls[4] = 0;
    return;
  }
  PyRand g{mt, pr_load(trng, mt)};
  const long long k = mp ? tc_randint(g, cnt) : tc_randperm0(g, cnt);
  pr_store(g, trng);
  if (threadIdx.x == 0) {
    ls[3] = k;
    ls[4] = cnt > 1;
  }
}

// After bl_step of a step that committed (ls[2] == 0): the best model again, from the sums bl_step left and with bl_step's
// arithmetic, its tie now drawn as the reference draws it -> hist_best of the step.  IID, Uncertainty, ActiveTesting
// and VMA: randperm(cnt)[0] on the CPU generator when cnt > 1 models tie (iid.py:52-55, activetesting.py:113-117);
// ModelPicker: randint(cnt) on the CUDA generator every step (modelpicker.py:109).  The r-th tie in ascending order.
__global__ void __launch_bounds__(32) k_bl_best_ref(const coda_bl_loop_t a, uint32_t* __restrict__ trng,
                                                    long long* __restrict__ grng) {
  __shared__ uint32_t mt[PR_N];
  __shared__ unsigned tie_w[32];
  const long long* ls = reinterpret_cast<const long long*>(a.ls);
  if (ls[2]) return;
  const int H = a.H, nwords = (H + 31) >> 5, lane = threadIdx.x;
  const long long M = ls[0], slot = (ls[5] - 1) % a.hist_cap;
  const bool lure = a.method == CODA_B200_BL_ACTIVETESTING || a.method == CODA_B200_BL_VMA;
  const bool mp = a.method == CODA_B200_BL_MODELPICKER;
  const double Ng = (double)a.n_global, m = (double)M;
  auto rv = [&](int h) -> double {                          // the value bl_step's best model minimises
    if (lure) return bl_lure_risk(a.s1[h], a.s2[h], Ng, m);
    return mp ? -(double)a.counts[h] : (double)a.counts[h];
  };
  double mn = INFINITY;
  for (int h = lane; h < H; h += 32) mn = fmin(mn, rv(h));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mn = fmin(mn, __shfl_xor_sync(CODA_FULL, mn, o));
  int cnt = 0;
  for (int w = 0; w < nwords; ++w) {
    const int h = w * 32 + lane;
    const unsigned b = __ballot_sync(CODA_FULL, h < H && rv(h) == mn);
    if (lane == 0) tie_w[w] = b;
    cnt += __popc(b);
  }
  __syncwarp();
  long long j = 0;
  if (mp) {
    j = tg_randint(grng, cnt);
  } else if (cnt > 1) {
    PyRand g{mt, pr_load(trng, mt)};
    j = tc_randperm0(g, cnt);
    pr_store(g, trng);
  }
  if (lane == 0) {
    int best = -1;
    for (int w = 0; w < nwords && best < 0; ++w) {
      unsigned b = tie_w[w];
      const int c = __popc(b);
      if (j < c) {
        for (; j > 0; --j) b &= b - 1;
        best = w * 32 + __ffs(b) - 1;
      } else {
        j -= c;
      }
    }
    a.hist_best[slot] = best;
  }
}

// the kernel-level check of the replicas: ops [nops][2] = {0, n}: randperm(n)[0] (CPU), {1, n}: randint(n) (CPU),
// {2, n}: randint(n) (CUDA); one output each
__global__ void __launch_bounds__(32) k_torch_rng_run(uint32_t* __restrict__ trng, long long* __restrict__ grng,
                                                      const long long* __restrict__ ops, int nops,
                                                      long long* __restrict__ out) {
  __shared__ uint32_t mt[PR_N];
  PyRand g{mt, pr_load(trng, mt)};
  for (int k = 0; k < nops; ++k) {
    const long long kind = ops[2 * k], n = ops[2 * k + 1];
    const long long r = kind == 0 ? (n > 1 ? tc_randperm0(g, n) : 0) : kind == 1 ? tc_randint(g, n) : tg_randint(grng, n);
    if (threadIdx.x == 0) out[k] = r;
    __syncwarp();
  }
  pr_store(g, trng);
}

static int br_loop_ok(const coda_bl_loop_t* a, const char* what) {
  CODA_CHECK_ARG(a && a->ls && a->flags && a->best, "%s: null pointer", what);
  CODA_CHECK_ARG(a->method >= CODA_B200_BL_IID && a->method <= CODA_B200_BL_MODELPICKER, "%s: bad method %d", what,
                 a->method);
  CODA_CHECK_ARG(a->H >= 1 && a->H <= 1024 && a->N >= 1 && a->n_global >= a->N && a->n_offset >= 0,
                 "%s: bad shape H=%d N=%lld", what, a->H, (long long)a->N);
  return CODA_B200_OK;
}

extern "C" int coda_b200_bl_draw_ref(const coda_bl_loop_t* a, uint32_t* cpu_rng, coda_stream_t stream) {
  if (int rc = br_loop_ok(a, "bl_draw_ref")) return rc;
  CODA_CHECK_ARG(a->method == CODA_B200_BL_UNCERTAINTY || a->method == CODA_B200_BL_MODELPICKER,
                 "bl_draw_ref: method %d draws no item tie from torch (use bl_draw)", a->method);
  CODA_CHECK_ARG(cpu_rng, "bl_draw_ref: null cpu_rng");
  CODA_CHECK_ARG(a->method == CODA_B200_BL_MODELPICKER || a->n_global < CODA_B200_RANDPERM32_MAX,
                 "bl_draw_ref: randperm over %lld items takes torch's 64-bit branch", (long long)a->n_global);
  k_bl_draw_ref<<<1, 32, 0, as_stream(stream)>>>(*a, cpu_rng);
  CODA_LAUNCH_OK("k_bl_draw_ref");
  return CODA_B200_OK;
}

extern "C" int coda_b200_bl_best_ref(const coda_bl_loop_t* a, uint32_t* cpu_rng, int64_t* cuda_rng,
                                     coda_stream_t stream) {
  if (int rc = br_loop_ok(a, "bl_best_ref")) return rc;
  const bool lure = a->method == CODA_B200_BL_ACTIVETESTING || a->method == CODA_B200_BL_VMA;
  const bool mp = a->method == CODA_B200_BL_MODELPICKER;
  CODA_CHECK_ARG(a->hist_best && a->hist_cap >= 1 && (lure ? (a->s1 && a->s2) : a->counts != nullptr) &&
                 (mp ? cuda_rng != nullptr : cpu_rng != nullptr), "bl_best_ref: null pointer");
  k_bl_best_ref<<<1, 32, 0, as_stream(stream)>>>(*a, cpu_rng, (long long*)cuda_rng);
  CODA_LAUNCH_OK("k_bl_best_ref");
  return CODA_B200_OK;
}

extern "C" int coda_b200_torch_rng_run(uint32_t* cpu_rng, int64_t* cuda_rng, const int64_t* ops, int nops, int64_t* out,
                                       coda_stream_t stream) {
  CODA_CHECK_ARG(cpu_rng && cuda_rng && ops && out && nops >= 0, "torch_rng_run: bad arguments");
  k_torch_rng_run<<<1, 32, 0, as_stream(stream)>>>(cpu_rng, (long long*)cuda_rng, (const long long*)ops, nops,
                                                   (long long*)out);
  CODA_LAUNCH_OK("k_torch_rng_run");
  return CODA_B200_OK;
}

CODA_MODULE_ANCHOR(bl_ref, k_bl_draw_ref)
