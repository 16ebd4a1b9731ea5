// The select kernel of the fused step (step.cu) and what it shares with step_label, for the two translation units that
// launch it: step.cu the default variant, step_defer.cu the deferring one (tie_rule="reference").  Instantiated in one
// unit, the deferring variant would change how nvcc compiles the shared device functions into the default kernel.
#pragma once
#include "xchg.cuh"
#include "terms.cuh"

#define ST_THREADS 256

// step.cu keeps the helpers below external as they always were; a second unit makes its copies static
#ifndef STEP_LINKAGE
#define STEP_LINKAGE
#endif

// ---- shared tail: posterior update + gather list -------------------------------------------------------
// jv (shared memory) holds p_h(idx) for every model; t is the revealed class.
STEP_LINKAGE __device__ void apply_label(const coda_step_t& a, int t, const int* jv, int* cnt /*[C] shared*/, bool valid) {
  const int H = a.H, C = a.C, tid = threadIdx.x;
  unsigned long long* pz = reinterpret_cast<unsigned long long*>(a.pisum_fx);
  for (int c = tid; c < C; c += ST_THREADS) pz[c] = 0ull;            // pi_rank1 / pi_reduce accumulate into it next
  int32_t* hdr = a.terms;
  R1Term* terms = reinterpret_cast<R1Term*>(a.terms + 2);
  if (!valid) {
    if (tid == 0) { hdr[0] = 0; hdr[1] = -1; }
    return;
  }
  for (int h = tid; h < H; h += ST_THREADS) {
    a.jvec[h] = jv[h];
    a.D[((size_t)h * C + t) * C + jv[h]] += a.lr;                     // coda.py:317
  }
  __shared__ int s_tp, s_m, s_total;
  __shared__ int wtot[ST_THREADS / 32];
  for (int c = tid; c < C; c += ST_THREADS) cnt[c] = 0;
  __syncthreads();
  for (int h = tid; h < H; h += ST_THREADS) atomicAdd(&cnt[jv[h]], 1);
  __syncthreads();
  if (tid == 0) {
    int best = -1, bc = 0;
    for (int c = 0; c < C; ++c)
      if (cnt[c] > best) { best = cnt[c]; bc = c; }
    s_tp = bc;
    s_m = H - best;
  }
  __syncthreads();
  const int tp = s_tp, M = s_m;
  const bool ens = a.have_ens && 2 * M < H;
  // dense slab: the shortcut's base E[n][t'] is the first term of the list, read like any other term (coalesced from
  // the class-major ensemble slot when there is one); the compact kernels load it themselves from hdr[1]
  const bool ens_term = ens && a.compact_k == 0;
  if (ens_term && tid == 0) {
    const bool cm = a.ens_col_stride > 0;
    terms[0] = R1Term{a.ens_off + (long long)tp * (cm ? a.ens_col_stride : 1), 1.f, cm ? 1 : C};
  }
  // every model contributes 1 (direct), or 0 / 2 (ensemble shortcut) terms: exclusive scan over models, in order
  int carry = ens_term ? 1 : 0;
  const int lane = tid & 31, warp = tid >> 5;
  for (int h0 = 0; h0 < H; h0 += ST_THREADS) {
    const int h = h0 + tid;
    const int j = h < H ? jv[h] : 0;
    const int n = h < H ? (ens ? (j != tp ? 2 : 0) : 1) : 0;
    int incl = n;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int v = __shfl_up_sync(CODA_FULL, incl, o);
      if (lane >= o) incl += v;
    }
    if (lane == 31) wtot[warp] = incl;
    __syncthreads();
    int off = carry;
    for (int w = 0; w < warp; ++w) off += wtot[w];
    const int k = off + incl - n;
    if (n && a.compact_k > 0) {
      // compact slab: a term names (model, class); pi_rank1_compact resolves it by a K-way match
      terms[k] = R1Term{(long long)h, 1.f, j};
      if (n == 2) terms[k + 1] = R1Term{(long long)h, -1.f, tp};
    } else if (n && a.n_host > 0 && a.slot_of_model[h] >= H - a.n_host) {
      // host slot: column (slot - S, class) of the pinned host slots, item stride 0 until coda_b200_host_stage
      // copies it to a staging column and points the term there
      const long long hb = (long long)(a.slot_of_model[h] - (H - a.n_host)) * C * a.shadow_col_stride;
      terms[k] = R1Term{hb + (long long)j * a.shadow_col_stride, 1.f, 0};
      if (n == 2) terms[k + 1] = R1Term{hb + (long long)tp * a.shadow_col_stride, -1.f, 0};
    } else if (n) {
      const int slot = a.slot_of_model ? a.slot_of_model[h] : -1;
      // shadow: [slot][class][col_stride] (item stride 1); reference layout: [model][item][class] (item stride C)
      const long long base = slot >= 0 ? a.shadow_off + (long long)slot * C * a.shadow_col_stride : (long long)h * a.model_stride;
      const long long mul = slot >= 0 ? a.shadow_col_stride : 1;
      const int str = slot >= 0 ? 1 : C;
      terms[k] = R1Term{base + (long long)j * mul, 1.f, str};
      if (n == 2) terms[k + 1] = R1Term{base + (long long)tp * mul, -1.f, str};
    }
    if (tid == ST_THREADS - 1) s_total = off + incl;
    __syncthreads();
    carry = s_total;
  }
  if (tid == 0) {
    hdr[0] = carry;
    hdr[1] = ens ? tp : -1;
  }
}

// merge this shard's block records -> one record in `out` (shared memory, 8 words); every thread returns after a barrier
STEP_LINKAGE __device__ void merge_partials(const long long* __restrict__ partials, int nblocks, long long* out) {
  __shared__ float sv[2][ST_THREADS / 32], sv2[2][ST_THREADS / 32];
  __shared__ long long si[2][ST_THREADS / 32], sc[ST_THREADS / 32];
  Best2 A = best2_empty(), B = best2_empty();
  long long cn = 0;
  for (int r = threadIdx.x; r < nblocks; r += ST_THREADS) {
    Best2 ra, rb;
    long long c;
    rec_load(partials + (size_t)r * REC_W, ra, c, rb);
    best2_merge(A, ra);
    best2_merge(B, rb);
    cn += c;
  }
  best2_warp(A);
  best2_warp(B);
  cn = warp_sum(cn);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) {
    sv[0][warp] = A.v; si[0][warp] = A.i; sv2[0][warp] = A.v2;
    sv[1][warp] = B.v; si[1][warp] = B.i; sv2[1][warp] = B.v2;
    sc[warp] = cn;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    Best2 fa = best2_empty(), fb = best2_empty();
    long long c = 0;
    for (int w = 0; w < ST_THREADS / 32; ++w) {
      best2_merge(fa, Best2{sv[0][w], si[0][w], sv2[0][w]});
      best2_merge(fb, Best2{sv[1][w], si[1][w], sv2[1][w]});
      c += sc[w];
    }
    rec_store(out, fa, c, fb);
  }
  __syncthreads();
}

// pick = 1: host-free loop (select + label + update); pick = 0: merge + exchange only.
// DEFER (the loop's tie_rule="reference"): a step whose winner has an isclose runner-up commits nothing and sets
// *pending = 1 -- tie_band / tie_draw / step_label_if finish it; any other step commits as without DEFER, *pending = 0.
template <bool DEFER>
__global__ void __launch_bounds__(ST_THREADS) k_step_select(coda_step_t a, XchgView x, int pick, long long* pending) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int H = a.H, C = a.C, tid = threadIdx.x;
  const uint32_t hrow = xch_align16((uint32_t)H * 2);
  long long* rec = reinterpret_cast<long long*>(smem_raw);                  // [8]     stage: record
  uint16_t* rowA = reinterpret_cast<uint16_t*>(smem_raw + 64);              // [H]     stage: p_h(candidate A)
  uint16_t* rowB = reinterpret_cast<uint16_t*>(smem_raw + 64 + hrow);       // [H]     stage: p_h(candidate B)
  int* jv = reinterpret_cast<int*>(smem_raw + 64 + 2 * hrow);               // [H]
  int* cnt = jv + H;                                                        // [C]
  __shared__ long long s_g;
  __shared__ int s_src, s_useA, s_tie, s_t;
  __shared__ float s_v;
  merge_partials(reinterpret_cast<const long long*>(a.partials), a.nblocks, rec);
  if (pick) {
    const long long iA = rec[1], iB = rec[4];
    for (int h = tid; h < H; h += ST_THREADS) {
      rowA[h] = iA != IDX_NONE ? a.hard[(size_t)(iA - a.n_offset) * H + h] : (uint16_t)0;
      rowB[h] = iB != IDX_NONE ? a.hard[(size_t)(iB - a.n_offset) * H + h] : (uint16_t)0;
    }
    for (int h = H + tid; h < (int)(hrow / 2); h += ST_THREADS) { rowA[h] = 0; rowB[h] = 0; }
  }
  __syncthreads();
  unsigned long long ep = 0;
  bool ok = true;
  if (x.world > 1) {
    ep = xch_epoch(x, XCH_REC);
    xch_push(x, XCH_REC, ep, smem_raw, pick ? x.slot_bytes[XCH_REC] : 64u);
    ok = xch_wait(x, XCH_REC, ep);
  }
  if (tid == 0) {
    Best2 A = best2_empty(), B = best2_empty();
    long long cn = 0;
    int srcA = 0, srcB = 0;
    if (x.world > 1) {
      for (int s = 0; s < x.world; ++s) {
        Best2 ra, rb;
        long long c;
        rec_load(reinterpret_cast<const long long*>(xch_data(x, XCH_REC, ep, s)), ra, c, rb);
        const long long pa = A.i, pb = B.i;
        best2_merge(A, ra);
        best2_merge(B, rb);
        if (A.i != pa) srcA = s;
        if (B.i != pb) srcB = s;
        cn += c;
      }
    } else {
      rec_load(rec, A, cn, B);
    }
    rec_store(reinterpret_cast<long long*>(a.bestrec), A, cn, B);
    const bool useA = cn > 0;                                          // coda.py:239 `or` fallback
    const Best2& w = useA ? A : B;
    s_g = w.i;
    s_v = w.v;
    s_src = useA ? srcA : srcB;
    s_useA = useA ? 1 : 0;
    s_tie = (w.i != IDX_NONE && isclose_best(w.v2, w.v)) ? 1 : 0;      // coda.py:307: a second candidate isclose to the best
    if constexpr (DEFER) *pending = s_tie;
    if (!ok) atomicOr(a.flags, CODA_B200_FLAG_XCHG_TIMEOUT);
  }
  __syncthreads();
  bool stop = !pick;
  if constexpr (DEFER) stop = stop || s_tie;
  if (stop) {
    if (x.world > 1) xch_done(x, XCH_REC, ep);
    return;
  }
  const long long g = s_g;
  const bool valid = g != IDX_NONE;
  if (tid == 0) {
    const long long k = *a.step_ctr;
    int t = 0;
    long long loc = -1;
    if (valid) {
      t = (int)a.labels_global[g];                                     // oracle(idx), coda/oracle.py:23-24
      loc = g - a.n_offset;
      if (loc < 0 || loc >= a.N) loc = -1;
      if (loc >= 0) a.labeled[loc] = 1;                                // coda.py:323
      if (t < 0 || t >= C) t = 0;
    } else {
      atomicOr(a.flags, CODA_B200_FLAG_NO_CANDIDATE);
    }
    a.sel[0] = loc;
    a.sel[1] = t;
    s_t = t;
    if (a.hist_idx && a.hist_cap > 0) {
      const long long slot = k % a.hist_cap;
      a.hist_idx[slot] = valid ? g : -1;
      if (a.hist_q) a.hist_q[slot] = s_v;
      if (a.hist_tie) a.hist_tie[slot] = s_tie;
    }
    *a.step_ctr = k + 1;
  }
  // p_h(idx) of the winner: from the winning shard's record payload
  {
    const uint16_t* row;
    if (x.world > 1) {
      const unsigned char* d = xch_data(x, XCH_REC, ep, s_src);
      row = reinterpret_cast<const uint16_t*>(d + 64 + (s_useA ? 0 : hrow));
    } else {
      row = s_useA ? rowA : rowB;
    }
    for (int h = tid; h < H; h += ST_THREADS) jv[h] = row[h];
  }
  __syncthreads();
  apply_label(a, s_t, jv, cnt, valid);
  if (x.world > 1) {
    __syncthreads();
    xch_done(x, XCH_REC, ep);
  }
}

// ---- host side ----------------------------------------------------------------------------------------
static int check_step(const coda_step_t* st, const char* who) {
  CODA_CHECK_ARG(st, "%s: null state", who);
  CODA_CHECK_ARG(st->H >= 1 && st->H <= 1024 && st->C >= 2 && st->C <= 4096 && st->N >= 1, "%s: bad dims", who);
  CODA_CHECK_ARG(st->flags, "%s: flags missing", who);
  return CODA_B200_OK;
}

static size_t select_smem(int H, int C) { return 64 + 2 * (size_t)xch_align16((uint32_t)H * 2) + (size_t)H * 4 + (size_t)C * 4; }

// a translation unit instantiates only the variant it launches
template <bool DEFER>
static int launch_select(const coda_step_t* st, const coda_xchg_t* x, int pick, coda_stream_t stream,
                         int64_t* pending = nullptr) {
  if (int rc = check_step(st, "step_select")) return rc;
  CODA_CHECK_ARG(st->partials && st->nblocks >= 1 && st->bestrec, "step_select: selection buffers missing");
  if (pick) {
    CODA_CHECK_ARG(st->hard && st->labeled && st->D && st->jvec && st->sel && st->terms && st->pisum_fx && st->labels_global &&
                       st->step_ctr,
                   "step_select: null pointer");
    CODA_CHECK_ARG(2 * st->H <= R1_MAXT && (reinterpret_cast<uintptr_t>(st->terms) & 7) == 0, "step_select: bad terms buffer");
  }
  XchgView v;
  if (int rc = xchg_view_from(x, &v)) return rc;
  k_step_select<DEFER><<<1, ST_THREADS, select_smem(st->H, st->C), as_stream(stream)>>>(*st, v, pick, (long long*)pending);
  CODA_LAUNCH_OK("k_step_select");
  return CODA_B200_OK;
}

