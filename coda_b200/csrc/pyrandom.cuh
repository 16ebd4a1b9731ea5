// Python's `random` module generator on the device, for loops whose number of draws depends on device data (the
// isclose tie breaks and the prefilter samples of CODA's host-free loop, DESIGN.md §4).
//
// State as CPython keeps it (random.getstate()[1]): the 624 MT19937 words, then the position 0..624 of the next word.
// genrand_uint32 is CPython's (twist every 624 words, then the tempering); on top of it:
//   pr_randbelow(n)   Random._randbelow_with_getrandbits: k = n.bit_length(), getrandbits(k) = word >> (32 - k),
//                     redrawn while >= n (1 <= n < 2^32); random.choice(seq) is seq[_randbelow(len(seq))]
//   pr_sample         random.sample(range(n), m), both branches (the pool when n <= setsize, else a set of positions)
// A generator belongs to ONE warp: every lane makes every call with the same arguments and gets the same result; the
// words live in shared memory.  Every shard holds a replica and advances it by globally known counts, so the replicas
// need no exchange.
#pragma once
#include "common.cuh"

#define PR_N 624
#define PR_M 397
#define PR_WORDS (PR_N + 1)

struct PyRand {
  uint32_t* mt;   // [624] shared
  int pos;        // warp-uniform
};

// The twist in three phases with a barrier between them.  Word kk reads the old kk and kk + 1 and word kk + 397
// (mod 624): old in [0, 227), written by the first phase in [227, 454), by the second in [454, 624) -- 623 reads the
// new words 0 and 396.  Inside a phase every lane reads all its inputs before any lane writes.
__device__ __forceinline__ void pr_twist(uint32_t* mt) {
  const int lane = threadIdx.x & 31;
#pragma unroll
  for (int ph = 0; ph < 3; ++ph) {
    const int lo = ph * 227, hi = ph == 2 ? PR_N : lo + 227;
    uint32_t nv[8];
#pragma unroll
    for (int r = 0; r < 8; ++r) {
      const int kk = lo + r * 32 + lane;
      if (kk < hi) {
        const uint32_t y = (mt[kk] & 0x80000000u) | (mt[kk + 1 == PR_N ? 0 : kk + 1] & 0x7fffffffu);
        nv[r] = mt[kk + PR_M < PR_N ? kk + PR_M : kk + PR_M - PR_N] ^ (y >> 1) ^ ((y & 1u) ? 0x9908b0dfu : 0u);
      }
    }
    __syncwarp();
#pragma unroll
    for (int r = 0; r < 8; ++r) {
      const int kk = lo + r * 32 + lane;
      if (kk < hi) mt[kk] = nv[r];
    }
    __syncwarp();
  }
}

__device__ __forceinline__ uint32_t pr_next(PyRand& g) {
  if (g.pos >= PR_N) {
    pr_twist(g.mt);
    g.pos = 0;
  }
  uint32_t y = g.mt[g.pos++];
  y ^= y >> 11;
  y ^= (y << 7) & 0x9d2c5680u;
  y ^= (y << 15) & 0xefc60000u;
  y ^= y >> 18;
  return y;
}

__device__ __forceinline__ long long pr_randbelow(PyRand& g, long long n) {
  const int k = 64 - __clzll(n);
  long long r;
  do {
    r = (long long)(pr_next(g) >> (32 - k));
  } while (r >= n);
  return r;
}

// random.sample(range(n), m) -> out[0 .. m).  pool: >= n ints (used when n <= setsize); seen: ceil(n / 32) words,
// zero on entry and on return (used otherwise).  setsize is Lib/random.py's, computed on the host (it depends on m only).
static __device__ void pr_sample(PyRand& g, long long n, int m, long long setsize, long long* out, int* pool, uint32_t* seen) {
  const int lane = threadIdx.x & 31;
  if (n <= setsize) {
    for (long long i = lane; i < n; i += 32) pool[i] = (int)i;
    __syncwarp();
    for (int i = 0; i < m; ++i) {
      const long long j = pr_randbelow(g, n - i);
      if (lane == 0) {
        out[i] = pool[j];
        pool[j] = pool[n - i - 1];
      }
    }
    __syncwarp();
    return;
  }
  for (int i = 0; i < m; ++i) {
    long long j;
    int dup;
    do {
      j = pr_randbelow(g, n);
      int d = 0;
      if (lane == 0) {
        const uint32_t bit = 1u << (j & 31), w = seen[j >> 5];
        d = (w & bit) != 0;
        if (!d) seen[j >> 5] = w | bit;
      }
      dup = __shfl_sync(CODA_FULL, d, 0);
    } while (dup);
    if (lane == 0) out[i] = j;
  }
  __syncwarp();
  for (int i = lane; i < m; i += 32) seen[out[i] >> 5] = 0u;   // the set bits are exactly the picked positions
  __syncwarp();
}

// CTA-wide: state [625] (global) -> mt (shared); returns the position
__device__ __forceinline__ int pr_load(const uint32_t* __restrict__ state, uint32_t* mt) {
  for (int i = threadIdx.x; i < PR_N; i += blockDim.x) mt[i] = state[i];
  __syncthreads();
  return (int)state[PR_N];
}
// the generator's warp, after its last draw
__device__ __forceinline__ void pr_store(const PyRand& g, uint32_t* __restrict__ state) {
  __syncwarp();
  for (int i = threadIdx.x & 31; i < PR_N; i += 32) state[i] = g.mt[i];
  if ((threadIdx.x & 31) == 0) state[PR_N] = (uint32_t)g.pos;
}
