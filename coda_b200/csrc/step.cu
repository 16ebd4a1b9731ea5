// Fused single-CTA step kernels: everything between two slab-sized passes of one acquisition step.
//
//   step_select   coda.py:306/309 (global arg-max over shards, first index), oracle(idx) from a device-resident label
//                 vector (coda/oracle.py:23-24), coda.py:316-317 (D[h][t][p_h(idx)] += lr), coda.py:323 (mark labeled),
//                 the gather list of the rank-1 marginal refresh -- the host-free loop
//   step_merge    the arg-max part only (API get_next_item_to_label; ties and random.choice stay with the host)
//   step_label    API add_label (coda.py:315-317) for a host-chosen (idx, class): the owner shard shares p_h(idx)
//   step_mixture  coda.py:232-233 pi_hat from the shards' column sums, coda.py:253/325-332 P(best), 254 H_before, 346 argmax
//   ties          coda.py:307 isclose scan against the global record;  report_gather: every shard's tie list to all
//
// Shards exchange their contributions through peer memory inside these kernels (xchg.cuh): no NCCL call and no
// extra launch sits between the scoring pass and the posterior update.
#include "xchg.cuh"
#include "terms.cuh"

#define ST_THREADS 256

// ---- shared tail: posterior update + gather list -------------------------------------------------------
// jv (shared memory) holds p_h(idx) for every model; t is the revealed class.
__device__ void apply_label(const coda_step_t& a, int t, const int* jv, int* cnt /*[C] shared*/, bool valid) {
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
__device__ void merge_partials(const long long* __restrict__ partials, int nblocks, long long* out) {
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

// pick = 1: host-free loop (select + label + update); pick = 0: merge + exchange only
__global__ void __launch_bounds__(ST_THREADS) k_step_select(coda_step_t a, XchgView x, int pick) {
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
    if (!ok) atomicOr(a.flags, CODA_B200_FLAG_XCHG_TIMEOUT);
  }
  __syncthreads();
  if (!pick) {
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

__global__ void __launch_bounds__(ST_THREADS) k_step_label(coda_step_t a, XchgView x) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int H = a.H, C = a.C, tid = threadIdx.x;
  const uint32_t hrow = xch_align16((uint32_t)H * 2);
  int* hdr = reinterpret_cast<int*>(smem_raw);                              // [4]  stage: {owner?, 0, 0, 0}
  uint16_t* row = reinterpret_cast<uint16_t*>(smem_raw + 16);               // [H]  stage: p_h(idx) on the owner
  int* jv = reinterpret_cast<int*>(smem_raw + 16 + hrow);                   // [H]
  int* cnt = jv + H;                                                        // [C]
  __shared__ int s_src;
  const long long loc = a.sel[0];
  const int t = (int)a.sel[1];
  const bool own = loc >= 0 && loc < a.N;
  if (tid < 4) hdr[tid] = (tid == 0 && own) ? 1 : 0;
  for (int h = tid; h < (int)(hrow / 2); h += ST_THREADS) row[h] = (own && h < H) ? a.hard[(size_t)loc * H + h] : (uint16_t)0;
  if (tid == 0) s_src = own ? x.rank : -1;
  __syncthreads();
  unsigned long long ep = 0;
  if (x.world > 1) {
    ep = xch_epoch(x, XCH_JROW);
    xch_push(x, XCH_JROW, ep, smem_raw, x.slot_bytes[XCH_JROW]);
    const bool ok = xch_wait(x, XCH_JROW, ep);
    if (tid == 0) {
      int src = -1;
      for (int s = 0; s < x.world; ++s)
        if (reinterpret_cast<const int*>(xch_data(x, XCH_JROW, ep, s))[0] == 1) src = s;
      s_src = src;
      if (!ok) atomicOr(a.flags, CODA_B200_FLAG_XCHG_TIMEOUT);
    }
    __syncthreads();
  }
  const int src = s_src;
  const bool valid = src >= 0 && t >= 0 && t < C;
  if (valid) {
    const uint16_t* r = x.world > 1 ? reinterpret_cast<const uint16_t*>(xch_data(x, XCH_JROW, ep, src) + 16) : row;
    for (int h = tid; h < H; h += ST_THREADS) jv[h] = r[h];
    if (tid == 0 && own) a.labeled[loc] = 1;                               // coda.py:323
  }
  __syncthreads();
  apply_label(a, valid ? t : 0, jv, cnt, valid);
  if (x.world > 1) {
    __syncthreads();
    xch_done(x, XCH_JROW, ep);
  }
}

__global__ void __launch_bounds__(ST_THREADS) k_step_mixture(coda_step_t a, XchgView x) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int H = a.H, C = a.C, Hp = (H + 31) / 32 * 32, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  long long* tot = reinterpret_cast<long long*>(smem_raw);                          // [C] (16-byte aligned stage)
  float* pis = reinterpret_cast<float*>(smem_raw + xch_align16((uint32_t)C * 8));   // [C]
  __shared__ long long red[ST_THREADS / 32];
  __shared__ float redv[ST_THREADS / 32];
  __shared__ int redi[ST_THREADS / 32];
  for (int c = tid; c < C; c += ST_THREADS) tot[c] = a.pisum_fx[c];
  for (int c = C + tid; c < (int)(xch_align16((uint32_t)C * 8) / 8); c += ST_THREADS) tot[c] = 0;
  __syncthreads();
  unsigned long long ep = 0;
  if (x.world > 1) {
    ep = xch_epoch(x, XCH_PISUM);
    xch_push(x, XCH_PISUM, ep, smem_raw, x.slot_bytes[XCH_PISUM]);
    const bool ok = xch_wait(x, XCH_PISUM, ep);
    if (!ok && tid == 0) atomicOr(a.flags, CODA_B200_FLAG_XCHG_TIMEOUT);
    for (int c = tid; c < C; c += ST_THREADS) {          // integer sums: exact, so the shard count leaves no trace
      long long s = 0;
      for (int r = 0; r < x.world; ++r) s += reinterpret_cast<const long long*>(xch_data(x, XCH_PISUM, ep, r))[c];
      tot[c] = s;
    }
    __syncthreads();
  }
  long long part = 0;
  for (int c = tid; c < C; c += ST_THREADS) part += tot[c];
  part = warp_sum(part);
  if (lane == 0) red[warp] = part;
  __syncthreads();
  long long total = 0;
  for (int w = 0; w < ST_THREADS / 32; ++w) total += red[w];
  const double dt = (double)total;
  for (int c = tid; c < C; c += ST_THREADS) {
    const float p = (float)((double)tot[c] / dt);                    // coda.py:232-233
    pis[c] = p;
    a.pi_hat[c] = p;
  }
  __syncthreads();
  float ent = 0.f, bv = -INFINITY;
  int bi = 0x7fffffff;
  uint32_t bad = 0;
  for (int h = tid; h < Hp; h += ST_THREADS) {
    float m = 0.f;
    if (h < H) {
      // m0[h] = sum_c pi_hat[c] PB[c][h] (coda.py:253 == coda.py:145): four interleaved partial sums keep the
      // L2 loads of PB in flight; the order is fixed, so every shard computes the same bits
      float m4[4] = {0.f, 0.f, 0.f, 0.f};
      int c = 0;
      for (; c + 4 <= C; c += 4) {
#pragma unroll
        for (int k = 0; k < 4; ++k) m4[k] = fmaf(pis[c + k], __ldg(a.PB + (size_t)(c + k) * Hp + h), m4[k]);
      }
      for (; c < C; ++c) m4[0] = fmaf(pis[c], __ldg(a.PB + (size_t)c * Hp + h), m4[0]);
      m = (m4[0] + m4[1]) + (m4[2] + m4[3]);
      if (!isfinite(m)) bad |= CODA_B200_FLAG_NONFINITE_PBEST;
      ent += ent_term(m);
      if (m > bv) { bv = m; bi = h; }
    }
    a.m0[h] = m;
  }
  ent = warp_sum(ent);
  warp_argmax(bv, bi);
  if (lane == 0) redv[warp] = ent;
  __syncthreads();
  float e = 0.f;
  for (int k = 0; k < ST_THREADS / 32; ++k) e += redv[k];
  __syncthreads();
  if (lane == 0) { redv[warp] = bv; redi[warp] = bi; }
  __syncthreads();
  if (tid == 0) {
    float b = redv[0];
    int i = redi[0];
    for (int k = 1; k < ST_THREADS / 32; ++k)
      if (redv[k] > b || (redv[k] == b && redi[k] < i)) { b = redv[k]; i = redi[k]; }
    *a.h_before = e;
    *a.best_model = (i == 0x7fffffff) ? 0 : i;
  }
  if (bad) atomicOr(a.flags, bad);
  if (x.world > 1) xch_done(x, XCH_PISUM, ep);
}

// ---- host side ----------------------------------------------------------------------------------------
static int check_step(const coda_step_t* st, const char* who) {
  CODA_CHECK_ARG(st, "%s: null state", who);
  CODA_CHECK_ARG(st->H >= 1 && st->H <= 1024 && st->C >= 2 && st->C <= 4096 && st->N >= 1, "%s: bad dims", who);
  CODA_CHECK_ARG(st->flags, "%s: flags missing", who);
  return CODA_B200_OK;
}

static size_t select_smem(int H, int C) { return 64 + 2 * (size_t)xch_align16((uint32_t)H * 2) + (size_t)H * 4 + (size_t)C * 4; }

static int launch_select(const coda_step_t* st, const coda_xchg_t* x, int pick, coda_stream_t stream) {
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
  k_step_select<<<1, ST_THREADS, select_smem(st->H, st->C), as_stream(stream)>>>(*st, v, pick);
  CODA_LAUNCH_OK("k_step_select");
  return CODA_B200_OK;
}

extern "C" int coda_b200_step_select(const coda_step_t* st, const coda_xchg_t* x, coda_stream_t stream) {
  return launch_select(st, x, 1, stream);
}
extern "C" int coda_b200_step_merge(const coda_step_t* st, const coda_xchg_t* x, coda_stream_t stream) {
  return launch_select(st, x, 0, stream);
}

extern "C" int coda_b200_step_label(const coda_step_t* st, const coda_xchg_t* x, coda_stream_t stream) {
  if (int rc = check_step(st, "step_label")) return rc;
  CODA_CHECK_ARG(st->hard && st->labeled && st->D && st->jvec && st->sel && st->terms && st->pisum_fx, "step_label: null pointer");
  CODA_CHECK_ARG(2 * st->H <= R1_MAXT && (reinterpret_cast<uintptr_t>(st->terms) & 7) == 0, "step_label: bad terms buffer");
  XchgView v;
  if (int rc = xchg_view_from(x, &v)) return rc;
  const size_t smem = 16 + (size_t)xch_align16((uint32_t)st->H * 2) + (size_t)st->H * 4 + (size_t)st->C * 4;
  k_step_label<<<1, ST_THREADS, smem, as_stream(stream)>>>(*st, v);
  CODA_LAUNCH_OK("k_step_label");
  return CODA_B200_OK;
}

extern "C" int coda_b200_step_mixture(const coda_step_t* st, const coda_xchg_t* x, coda_stream_t stream) {
  if (int rc = check_step(st, "step_mixture")) return rc;
  CODA_CHECK_ARG(st->pisum_fx && st->PB && st->pi_hat && st->m0 && st->h_before && st->best_model, "step_mixture: null pointer");
  XchgView v;
  if (int rc = xchg_view_from(x, &v)) return rc;
  const size_t smem = (size_t)xch_align16((uint32_t)st->C * 8) + (size_t)st->C * 4;
  k_step_mixture<<<1, ST_THREADS, smem, as_stream(stream)>>>(*st, v);
  CODA_LAUNCH_OK("k_step_mixture");
  return CODA_B200_OK;
}

__global__ void k_record_best(const long long* __restrict__ best_model, const long long* __restrict__ step_ctr,
                              int* __restrict__ hist_best, long long hist_cap) {
  const long long k = *step_ctr - 1;
  if (k >= 0) hist_best[k % hist_cap] = (int)*best_model;
}

extern "C" int coda_b200_record_best(const int64_t* best_model, const int64_t* step_ctr, int32_t* hist_best,
                                     int64_t hist_cap, coda_stream_t stream) {
  CODA_CHECK_ARG(best_model && step_ctr && hist_best, "record_best: null pointer");
  CODA_CHECK_ARG(hist_cap >= 1, "record_best: bad hist_cap %lld", (long long)hist_cap);
  k_record_best<<<1, 1, 0, as_stream(stream)>>>((const long long*)best_model, (const long long*)step_ctr, hist_best,
                                                hist_cap);
  CODA_LAUNCH_OK("k_record_best");
  return CODA_B200_OK;
}

// ---- tie scan against the GLOBAL record ---------------------------------------------------------------
// tie_hdr: {count, min tied global index}; tie_idx/tie_val hold up to `cap` entries (unordered).
__global__ void __launch_bounds__(256) k_ties(const float* __restrict__ eig, long long N,
                                              const uint8_t* __restrict__ labeled,
                                              const uint8_t* __restrict__ disagree, long long n_offset,
                                              const long long* __restrict__ best, int cap,
                                              long long* __restrict__ tie_hdr, long long* __restrict__ tie_idx,
                                              float* __restrict__ tie_val) {
  const bool useA = best[2] > 0;                                      // coda.py:239 `or` fallback
  const float bv = __int_as_float((int)(useA ? best[0] : best[3]));
  for (long long n = (long long)blockIdx.x * blockDim.x + threadIdx.x; n < N;
       n += (long long)gridDim.x * blockDim.x) {
    if (labeled[n]) continue;
    if (useA && !disagree[n]) continue;
    const float e = eig[n];
    if (isclose_best(e, bv)) {
      const long long g = n_offset + n;
      unsigned long long k = atomicAdd(reinterpret_cast<unsigned long long*>(tie_hdr), 1ull);
      atomicMin(tie_hdr + 1, g);
      if (k < (unsigned long long)cap) {
        tie_idx[k] = g;
        tie_val[k] = e;
      }
    }
  }
}

__global__ void k_ties_reset(long long* tie_hdr) {
  tie_hdr[0] = 0;
  tie_hdr[1] = IDX_NONE;
}

extern "C" int coda_b200_ties(const float* eig, int64_t N, const uint8_t* labeled, const uint8_t* disagree,
                              int64_t n_offset, const int64_t* best, int cap, int64_t* tie_hdr, int64_t* tie_idx,
                              float* tie_val, coda_stream_t stream) {
  CODA_CHECK_ARG(eig && labeled && disagree && best && tie_hdr && tie_idx && tie_val, "ties: null pointer");
  int grid = (int)min((long long)(N + 255) / 256, (long long)coda_sm_count() * 4);
  if (grid < 1) grid = 1;
  k_ties_reset<<<1, 1, 0, as_stream(stream)>>>(reinterpret_cast<long long*>(tie_hdr));
  k_ties<<<grid, 256, 0, as_stream(stream)>>>(eig, N, labeled, disagree, n_offset,
                                              reinterpret_cast<const long long*>(best), cap,
                                              reinterpret_cast<long long*>(tie_hdr),
                                              reinterpret_cast<long long*>(tie_idx), tie_val);
  CODA_LAUNCH_OK("k_ties");
  return CODA_B200_OK;
}

__global__ void __launch_bounds__(ST_THREADS) k_report_gather(const long long* __restrict__ rep, int rep_words,
                                                              long long* __restrict__ rep_all, XchgView x,
                                                              uint32_t* __restrict__ flags) {
  if (x.world <= 1) {
    for (int i = threadIdx.x; i < rep_words; i += ST_THREADS) rep_all[i] = rep[i];
    return;
  }
  const unsigned long long ep = xch_epoch(x, XCH_REPORT);
  xch_push(x, XCH_REPORT, ep, rep, (uint32_t)rep_words * 8u);
  const bool ok = xch_wait(x, XCH_REPORT, ep);
  if (!ok && threadIdx.x == 0) atomicOr(flags, CODA_B200_FLAG_XCHG_TIMEOUT);
  for (int s = 0; s < x.world; ++s) {
    const long long* src = reinterpret_cast<const long long*>(xch_data(x, XCH_REPORT, ep, s));
    for (int i = threadIdx.x; i < rep_words; i += ST_THREADS) rep_all[(size_t)s * rep_words + i] = src[i];
  }
  __syncthreads();
  xch_done(x, XCH_REPORT, ep);
}

extern "C" int coda_b200_report_gather(const int64_t* rep, int rep_words, int64_t* rep_all, const coda_xchg_t* x,
                                       uint32_t* flags, coda_stream_t stream) {
  CODA_CHECK_ARG(rep && rep_all && flags && rep_words >= 8 && rep_words % 2 == 0, "report_gather: bad arguments");
  CODA_CHECK_ARG((reinterpret_cast<uintptr_t>(rep) & 15) == 0, "report_gather: rep must be 16-byte aligned");
  XchgView v;
  if (int rc = xchg_view_from(x, &v)) return rc;
  CODA_CHECK_ARG(v.world == 1 || (uint32_t)rep_words * 8u <= v.slot_bytes[XCH_REPORT], "report_gather: report larger than its slot");
  k_report_gather<<<1, ST_THREADS, 0, as_stream(stream)>>>(reinterpret_cast<const long long*>(rep), rep_words,
                                                          reinterpret_cast<long long*>(rep_all), v, flags);
  CODA_LAUNCH_OK("k_report_gather");
  return CODA_B200_OK;
}
