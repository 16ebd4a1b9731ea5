// coda_b200_step_select_defer: k_step_select<true> (step_select.cuh), in a translation unit of its own.
#define STEP_LINKAGE static
#include "step_select.cuh"

extern "C" int coda_b200_step_select_defer(const coda_step_t* st, const coda_xchg_t* x, int64_t* pending,
                                           coda_stream_t stream) {
  CODA_CHECK_ARG(pending, "step_select_defer: null pending word");
  return launch_select<true>(st, x, 1, stream, pending);
}

CODA_MODULE_ANCHOR(step_defer, k_step_select<true>)
