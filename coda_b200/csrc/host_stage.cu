// Host-resident slab (HostSlab): the per-step staging of host-slot columns for the rank-1 marginal refresh.
//
// With the slab in host memory every model has a class-major shadow slot; the slots that did not fit in HBM live in
// pinned host memory, mapped into the device's address space.  The step kernels (step_select.cuh, apply_label) emit a
// host slot's term as {element offset into the host slots, sign, item stride 0}.  Before pi_rank1 runs, the two
// kernels here copy each such column (cs slab elements, one (model, class) column of every item) over PCIe into a
// device staging column and point the term at it (item stride 1, offset relative to the slab base pi_rank1 reads).
// k_pi_rank1 is not changed: it sees a list of device terms in the same order with the same signs, so every item's
// fmaf chain is the one of a run with the whole slab on the device.
//
// The copy is bound by PCIe, not HBM: 16-byte loads, HS_UNROLL of them in flight per thread, over a small fixed grid
// (HS_GRID blocks) that leaves the SMs to the class-t tables and rows running on the side stream.  The grid does not
// depend on the list, so the launch can be captured in a CUDA graph; the term count is read on the device.
#include "common.cuh"
#include "terms.cuh"

#define HS_THREADS 256
#define HS_GRID 32
#define HS_UNROLL 8

// rank of every host term of the list (the order of the terms) -> s_src[rank] = its term index; returns the count.
// Every thread of the block returns the same count after a barrier.
static __device__ int host_terms(const int32_t* __restrict__ hdr, const R1Term* __restrict__ terms, int* s_src) {
  __shared__ int s_wsum[HS_THREADS / 32];
  __shared__ int s_carry;
  const int nt = hdr[0], tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (tid == 0) s_carry = 0;
  __syncthreads();
  for (int b = 0; b < nt; b += HS_THREADS) {
    const int k = b + tid;
    const bool host = k < nt && terms[k].str == 0;
    const unsigned m = __ballot_sync(CODA_FULL, host);
    if (lane == 0) s_wsum[warp] = __popc(m);
    __syncthreads();
    int off = s_carry;
    for (int w = 0; w < warp; ++w) off += s_wsum[w];
    if (host) s_src[off + __popc(m & ((1u << lane) - 1u))] = k;
    __syncthreads();
    if (tid == 0)
      for (int w = 0; w < HS_THREADS / 32; ++w) s_carry += s_wsum[w];
    __syncthreads();
  }
  return s_carry;
}

// staging column r <- host column of the r-th host term; cs16 = 16-byte units per column
__global__ void __launch_bounds__(HS_THREADS) k_host_stage(const int32_t* __restrict__ hdr,
                                                           const R1Term* __restrict__ terms,
                                                           const uint4* __restrict__ host, uint4* __restrict__ stage,
                                                           long long cs16, int esz16) {
  __shared__ int s_src[R1_MAXT];
  const int nh = host_terms(hdr, terms, s_src);
  const long long total = (long long)nh * cs16;
  const long long stride = (long long)gridDim.x * HS_THREADS;
  for (long long i0 = (long long)blockIdx.x * HS_THREADS + threadIdx.x; i0 < total; i0 += stride * HS_UNROLL) {
    uint4 v[HS_UNROLL];
#pragma unroll
    for (int u = 0; u < HS_UNROLL; ++u) {
      const long long i = i0 + u * stride;
      if (i < total) {
        const long long r = i / cs16, q = i - r * cs16;
        v[u] = host[terms[s_src[r]].off / esz16 + q];
      }
    }
#pragma unroll
    for (int u = 0; u < HS_UNROLL; ++u) {
      const long long i = i0 + u * stride;
      if (i < total) stage[i] = v[u];
    }
  }
}

// after the copy: point the r-th host term at staging column r; census += the columns staged
__global__ void __launch_bounds__(HS_THREADS) k_host_stage_terms(const int32_t* __restrict__ hdr, R1Term* terms,
                                                                 long long stage_off, long long cs,
                                                                 long long* census) {
  __shared__ int s_src[R1_MAXT];
  const int nh = host_terms(hdr, terms, s_src);
  for (int r = threadIdx.x; r < nh; r += HS_THREADS) {
    R1Term& t = terms[s_src[r]];
    t.off = stage_off + (long long)r * cs;
    t.str = 1;
  }
  if (threadIdx.x == 0 && census && nh) atomicAdd(reinterpret_cast<unsigned long long*>(census), (unsigned long long)nh);
}

extern "C" int coda_b200_host_stage(const coda_step_t* st, int fmt, int64_t* census, coda_stream_t stream) {
  CODA_CHECK_ARG(st, "host_stage: null state");
  if (st->n_host == 0) return CODA_B200_OK;
  CODA_CHECK_ARG(fmt == CODA_B200_SLAB_F32 || fmt == CODA_B200_SLAB_F16 || fmt == CODA_B200_SLAB_BF16,
                 "host_stage: unknown slab format %d", fmt);
  CODA_CHECK_ARG(st->terms && st->host_shadow && st->stage && st->n_host > 0 && st->n_host <= st->H && 2 * st->H <= R1_MAXT,
                 "host_stage: bad arguments");
  const int esz = fmt == CODA_B200_SLAB_F32 ? 4 : 2;
  const long long cs = st->shadow_col_stride;
  CODA_CHECK_ARG(cs >= st->N && (cs * esz) % 16 == 0, "host_stage: column stride %lld is not whole 16-byte units", cs);
  CODA_CHECK_ARG((reinterpret_cast<uintptr_t>(st->host_shadow) & 15) == 0 && (reinterpret_cast<uintptr_t>(st->stage) & 15) == 0 &&
                     (reinterpret_cast<uintptr_t>(st->terms) & 7) == 0,
                 "host_stage: host slots and staging must be 16-byte aligned, terms 8-byte aligned");
  const int32_t* hdr = st->terms;
  R1Term* terms = reinterpret_cast<R1Term*>(st->terms + 2);
  cudaStream_t s = as_stream(stream);
  // offsets count slab elements; a column is cs * esz bytes, a whole number of 16-byte units
  k_host_stage<<<HS_GRID, HS_THREADS, 0, s>>>(hdr, terms, static_cast<const uint4*>(st->host_shadow),
                                              static_cast<uint4*>(st->stage), cs * esz / 16, 16 / esz);
  CODA_LAUNCH_OK("k_host_stage");
  k_host_stage_terms<<<1, HS_THREADS, 0, s>>>(hdr, terms, (long long)st->stage_off, cs,
                                              reinterpret_cast<long long*>(census));
  CODA_LAUNCH_OK("k_host_stage_terms");
  return CODA_B200_OK;
}

// Page-lock an existing host allocation and map it into every device's address space.  The kernels read and write the
// host slots through the same address (unified addressing); a device where the registered address differs is refused.
extern "C" int coda_b200_host_register(void* ptr, size_t bytes) {
  CODA_CHECK_ARG(ptr && bytes > 0, "host_register: bad arguments");
  CODA_CUDA_OK(cudaHostRegister(ptr, bytes, cudaHostRegisterPortable | cudaHostRegisterMapped));
  void* dptr = nullptr;
  const cudaError_t e = cudaHostGetDevicePointer(&dptr, ptr, 0);
  if (e != cudaSuccess || dptr != ptr) {
    cudaHostUnregister(ptr);
    CODA_CHECK_ARG(false, "host_register: the device address of %zu registered bytes differs from the host address", bytes);
  }
  return CODA_B200_OK;
}

extern "C" int coda_b200_host_unregister(void* ptr) {
  CODA_CHECK_ARG(ptr, "host_unregister: null pointer");
  CODA_CUDA_OK(cudaHostUnregister(ptr));
  return CODA_B200_OK;
}

CODA_MODULE_ANCHOR(host_stage, k_host_stage)
