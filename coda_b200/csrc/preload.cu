// coda_b200_preload_kernels: load every kernel of this library into the current device's context now.
//
// With CUDA's lazy loading (the default, and what torch asks for) a kernel's code is loaded at its first launch, and
// that load can wait for the kernels already running on the device.  Shards that share one GPU spin on each other
// inside the step kernels, so a shard whose first launch of some kernel comes after a peer's exchange kernel has
// started would wait for that peer, which waits for it: the exchange times out.  Loading everything up front, before
// any exchange can spin, removes the first-launch load from the step path.
//
// Every translation unit is a module of its own; each names one of its kernels through CODA_MODULE_ANCHOR, which
// leads to the unit's CUlibrary, whose kernels are enumerated and loaded (driver entry points through the runtime,
// so the library does not link libcuda).
#include "common.cuh"

#include <cuda.h>

#include <vector>

extern "C" {
const void* coda_anchor_baselines(void);
const void* coda_anchor_bl_ref(void);
const void* coda_anchor_compact(void);
const void* coda_anchor_compact_build(void);
const void* coda_anchor_eps_search(void);
const void* coda_anchor_gain(void);
const void* coda_anchor_host_stage(void);
const void* coda_anchor_pairs(void);
const void* coda_anchor_pairs_tc(void);
const void* coda_anchor_pi_tc(void);
const void* coda_anchor_sample(void);
const void* coda_anchor_slab(void);
const void* coda_anchor_step(void);
const void* coda_anchor_step_defer(void);
const void* coda_anchor_tables(void);
const void* coda_anchor_true_loss(void);
}

namespace {
typedef CUresult (*KernelGetLibrary)(CUlibrary*, CUkernel);
typedef CUresult (*LibraryGetKernelCount)(unsigned int*, CUlibrary);
typedef CUresult (*LibraryEnumerateKernels)(CUkernel*, unsigned int, CUlibrary);
typedef CUresult (*KernelGetFunction)(CUfunction*, CUkernel);
typedef CUresult (*FuncLoad)(CUfunction);

template <typename F>
int driver_fn(const char* name, F* out) {
  void* p = nullptr;
  cudaDriverEntryPointQueryResult q;
  CODA_CUDA_OK(cudaGetDriverEntryPointByVersion(name, &p, 12050, cudaEnableDefault, &q));
  CODA_CHECK_ARG(q == cudaDriverEntryPointSuccess && p, "preload_kernels: driver entry point %s not found", name);
  *out = reinterpret_cast<F>(p);
  return CODA_B200_OK;
}
}  // namespace

extern "C" int coda_b200_preload_kernels(int64_t* loaded_host) {
  CODA_CHECK_ARG(loaded_host, "preload_kernels: null pointer");
  KernelGetLibrary get_lib;
  LibraryGetKernelCount get_count;
  LibraryEnumerateKernels enumerate;
  KernelGetFunction get_fn;
  FuncLoad load;
  int rc;
  if ((rc = driver_fn("cuKernelGetLibrary", &get_lib)) || (rc = driver_fn("cuLibraryGetKernelCount", &get_count)) ||
      (rc = driver_fn("cuLibraryEnumerateKernels", &enumerate)) || (rc = driver_fn("cuKernelGetFunction", &get_fn)) ||
      (rc = driver_fn("cuFuncLoad", &load)))
    return rc;
  CODA_CUDA_OK(cudaFree(nullptr));                      // the current device's primary context exists
  const void* anchors[] = {coda_anchor_baselines(), coda_anchor_bl_ref(), coda_anchor_compact(), coda_anchor_eps_search(),
                           coda_anchor_gain(),      coda_anchor_pairs(),  coda_anchor_pairs_tc(), coda_anchor_pi_tc(),
                           coda_anchor_sample(),    coda_anchor_slab(),   coda_anchor_step(),     coda_anchor_step_defer(),
                           coda_anchor_tables(),    coda_anchor_true_loss(),  coda_anchor_compact_build(),
                           coda_anchor_host_stage()};
  int64_t loaded = 0;
  for (const void* a : anchors) {
    cudaKernel_t k;
    CODA_CUDA_OK(cudaGetKernel(&k, a));
    CUlibrary lib;
    CODA_CHECK_ARG(get_lib(&lib, reinterpret_cast<CUkernel>(k)) == CUDA_SUCCESS, "preload_kernels: cuKernelGetLibrary failed");
    unsigned int n = 0;
    CODA_CHECK_ARG(get_count(&n, lib) == CUDA_SUCCESS, "preload_kernels: cuLibraryGetKernelCount failed");
    std::vector<CUkernel> ks(n);
    CODA_CHECK_ARG(n == 0 || enumerate(ks.data(), n, lib) == CUDA_SUCCESS, "preload_kernels: cuLibraryEnumerateKernels failed");
    for (CUkernel kk : ks) {
      CUfunction f;
      CODA_CHECK_ARG(get_fn(&f, kk) == CUDA_SUCCESS, "preload_kernels: cuKernelGetFunction failed");
      CODA_CHECK_ARG(load(f) == CUDA_SUCCESS, "preload_kernels: cuFuncLoad failed");
      ++loaded;
    }
  }
  *loaded_host = loaded;
  return CODA_B200_OK;
}
