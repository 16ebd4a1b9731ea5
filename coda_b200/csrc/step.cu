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
#include "step_select.cuh"

// GATED: the same on a step the deferring select left pending, and nothing otherwise (the word is equal on every shard:
// all shards exchange or none)
template <bool GATED>
__global__ void __launch_bounds__(ST_THREADS) k_step_label(coda_step_t a, XchgView x, const long long* pending) {
  if constexpr (GATED) {
    if (!*pending) return;
  }
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
extern "C" int coda_b200_step_select(const coda_step_t* st, const coda_xchg_t* x, coda_stream_t stream) {
  return launch_select<false>(st, x, 1, stream);
}
extern "C" int coda_b200_step_merge(const coda_step_t* st, const coda_xchg_t* x, coda_stream_t stream) {
  return launch_select<false>(st, x, 0, stream);
}

static int launch_label(const coda_step_t* st, const coda_xchg_t* x, const int64_t* pending, coda_stream_t stream) {
  if (int rc = check_step(st, "step_label")) return rc;
  CODA_CHECK_ARG(st->hard && st->labeled && st->D && st->jvec && st->sel && st->terms && st->pisum_fx, "step_label: null pointer");
  CODA_CHECK_ARG(2 * st->H <= R1_MAXT && (reinterpret_cast<uintptr_t>(st->terms) & 7) == 0, "step_label: bad terms buffer");
  XchgView v;
  if (int rc = xchg_view_from(x, &v)) return rc;
  const size_t smem = 16 + (size_t)xch_align16((uint32_t)st->H * 2) + (size_t)st->H * 4 + (size_t)st->C * 4;
  if (pending) {
    k_step_label<true><<<1, ST_THREADS, smem, as_stream(stream)>>>(*st, v, (const long long*)pending);
    CODA_LAUNCH_OK("k_step_label_if");
  } else {
    k_step_label<false><<<1, ST_THREADS, smem, as_stream(stream)>>>(*st, v, nullptr);
    CODA_LAUNCH_OK("k_step_label");
  }
  return CODA_B200_OK;
}

extern "C" int coda_b200_step_label(const coda_step_t* st, const coda_xchg_t* x, coda_stream_t stream) {
  return launch_label(st, x, nullptr, stream);
}

extern "C" int coda_b200_step_label_if(const coda_step_t* st, const coda_xchg_t* x, const int64_t* pending,
                                       coda_stream_t stream) {
  CODA_CHECK_ARG(pending, "step_label_if: null pending word");
  return launch_label(st, x, pending, stream);
}

extern "C" int coda_b200_step_mixture(const coda_step_t* st, const coda_xchg_t* x, coda_stream_t stream) {
  if (int rc = check_step(st, "step_mixture")) return rc;
  CODA_CHECK_ARG(st->pisum_fx && st->PB && st->pi_hat && st->m0 && st->h_before && st->best_model, "step_mixture: null pointer");
  XchgView v;
  if (int rc = xchg_view_from(x, &v)) return rc;
  const size_t smem = (size_t)xch_align16((uint32_t)st->C * 8) + (size_t)st->C * 4;   // 48 KB at C = 4096: over the default
  CODA_CUDA_OK(cudaFuncSetAttribute(k_step_mixture, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
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

CODA_MODULE_ANCHOR(step, k_step_mixture)
