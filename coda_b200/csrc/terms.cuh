// Gather list of the rank-1 marginal refresh (coda.py:319 restated; built by the step kernels, consumed by pi_rank1).
//   direct     : sum_h preds[h][n][j_h]                                  -> H terms
//   ensemble   : with t' = the most common j_h and E[n][c] = sum_h preds[h][n][c],
//                sum_h preds[h][n][j_h] = E[n][t'] + sum_{h: j_h != t'} (preds[h][n][j_h] - preds[h][n][t'])
//                -> 1 + 2*M terms (M = models that disagree with the majority on the labeled item): on the dense slab
//                the first term is E[n][t'] itself (sign +1), so the kernels need no special load for it
//                (the compact-slab kernels take t' from hdr[1] and read E themselves: 2*M terms there).
// A model with a shadow slot is read from the class-major shadow copy (item stride 1) instead of preds (item stride C);
// E is read from the shadow's class-major ensemble slot when there is one, else from the item-major ens (stride C).
// Memory: int32 hdr[2] = {nterms, t' or -1} followed by nterms x R1Term (8-byte aligned).
#pragma once
#include <stdint.h>

#define R1_MAXT 2048
struct R1Term {
  long long off;   // element offset relative to preds for item 0
  float sg;        // +1 / -1
  int str;         // element stride per item: C (reference layout) or 1 (shadow)
};
