// Shared device/host helpers for libsonarfe (sm_90a only).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <cstdarg>
#include <cstdio>
#include <cstring>

#include "../../include/sonarfe.h"

namespace sfe {

// ---------------------------------------------------------------- error plumbing
void set_error(const char *fmt, ...);  // thread-local message behind sfe_last_error()

#define SFE_CUDA(call)                                                                      \
  do {                                                                                      \
    cudaError_t e_ = (call);                                                                \
    if (e_ != cudaSuccess) {                                                                \
      sfe::set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #call, cudaGetErrorString(e_)); \
      (void)cudaGetLastError(); /* do not leave the error for an unrelated later call */   \
      return SFE_ERR_CUDA;                                                                  \
    }                                                                                       \
  } while (0)

#define SFE_REQUIRE(cond, ...)         \
  do {                                 \
    if (!(cond)) {                     \
      sfe::set_error(__VA_ARGS__);     \
      return SFE_ERR_ARG;              \
    }                                  \
  } while (0)

// ---------------------------------------------------------------- context
struct Buffer {  // grow-only device scratch
  void *ptr = nullptr;
  size_t cap = 0;
};
// the slots of sfe_ctx::scratch, one per subsystem
enum { SCR_CFAR_FLAGS = 0, SCR_FEATX = 1, SCR_CLOUD = 2, SCR_ICP = 3, SCR_MISC = 4, SCR_CFAR_LUT = 5, SCR_DS_GRID = 6,
       SCR_MAP = 7, SCR_RO_MAP = 8, SCR_ICP_FILTER = 9, SCR_COUNT = 10 };

struct JpegState;  // jpeg.cu
struct PngState;   // png.cu
void destroy(JpegState *s);
void destroy(PngState *s);

}  // namespace sfe

struct sfe_ctx {
  int device = 0;
  cudaStream_t stream = nullptr;
  bool owns_stream = false;
  int sm_count = 0;         // SMs the persistent launches are sized for (sfe_ctx_set_grid_sms; default the device's)
  int device_sm_count = 0;  // the device's SM count
  int max_smem_optin = 0;
  sfe::Buffer scratch[sfe::SCR_COUNT];  // per-subsystem scratch
  sfe::Buffer stage_in[2];  // device staging for the *_host entry points
  sfe::Buffer stage_out[4];
  void *pinned = nullptr;   // small pinned host block for async result reads
  size_t pinned_cap = 0;
  uint64_t launches = 0;    // kernels launched through this context (bench: gpu_launches)
  // per-context caches (they describe buffers / attributes owned by THIS context, so they live here and not in
  // thread-local statics: a new context may get a recycled device address, two contexts may share a thread)
  double cfar_lut_key[6] = {-1, 0, 0, 0, 0, 0};  // parameters of the table held in scratch[SCR_CFAR_LUT]
  const void *cfar_lut_buf = nullptr;            // ... and the buffer it was uploaded to (null = none)
  // CTAs per SM of the persistent one-CTA launches (sfe::ctas_per_sm), by (kernel, threads, dynamic bytes); room for
  // every configuration one front-end step launches
  struct OccEntry { const void *fn; size_t smem; int threads, per_sm; } occ[16] = {};
  int occ_next = 0;
  sfe::JpegState *jpeg = nullptr;       // JPEG decoder state, created on first use
  sfe::PngState *png = nullptr;         // PNG decoder state, created on first use
  cudaStream_t copy_stream = nullptr;   // host flavours that overlap copies with kernels (featx.cu), created on first use
  cudaEvent_t copy_ev[4] = {};
  int *work = nullptr;  // device [SFE_WORK_COUNTERS]: work counters of the persistent kernels (sfe::next_work_item)
  sfe_icp_filters icp_filters = {};  // sfe_icp_set_filters
  bool has_icp_filters = false;
  sfe_icp_robust icp_robust = {};  // sfe_icp_set_robust
  bool has_icp_robust = false;
};

struct sfe_maps {  // per-geometry polar->Cartesian sampling table (featx.cu)
  int rows, cols;  // Cartesian image
  int R, B;        // polar image
  double width, height;
  void *table;     // device MapEntry[rows*cols]
  int32_t *inv_off;  // device [R*B + 1]: for every polar cell, the Cartesian pixels it can light ...
  int32_t *inv_idx;  // ... as a CSR list of pixel indices
  float *metres;     // device [cols + rows]: lateral metres of every column, then forward metres of every row
                     // (feature_extraction.py:235-237 evaluated per column / per row in float64 on the host)
  int device;
};

namespace sfe {
// Work counters in ctx->work, one per launch site; launches that may run at the same time (on different streams) use
// different counters, launches on one stream reuse theirs (each zeroes it first, stream-ordered).
enum { WORK_CART = 0, WORK_DS = 1, WORK_ICP = 2, SFE_WORK_COUNTERS = 5 };  // WORK_ICP: three, one per launch class

// (re)allocate if too small, stream-ordered on `stream` (default: ctx->stream).  A buffer must only grow on a stream
// that is ordered after every earlier user of the block and before every later one: the stream that uses it.
int ensure(sfe_ctx *ctx, Buffer &b, size_t bytes);
int ensure(sfe_ctx *ctx, Buffer &b, size_t bytes, cudaStream_t stream);
int ensure_pinned(sfe_ctx *ctx, size_t bytes);

// Carves sub-buffers out of one grow-only scratch block, 256 B aligned each.  Two passes over the same take() calls:
// the first (base null) sizes the block in `off`, the second, after ensure() and with base set, hands out pointers.
struct Carver {
  char *base = nullptr;
  size_t off = 0;
  void *take(size_t bytes) {
    void *p = base ? base + off : nullptr;
    off += (bytes + 255) & ~size_t(255);
    return p;
  }
};

// ---------------------------------------------------------------- one-CTA launches (api.cu)
// The largest n <= cap whose layout bytes_of(n) fits `budget`; bytes_of must not decrease with n.
template <class BytesOf>
int largest_layout(int cap, size_t budget, BytesOf bytes_of) {
  int lo = 0, hi = cap;
  while (lo < hi) {
    const int mid = lo + (hi - lo + 1) / 2;
    if (bytes_of(mid) <= budget) lo = mid;
    else hi = mid - 1;
  }
  return lo;
}
// *budget = the dynamic shared memory one CTA of `fn` may take on ctx's device: the opt-in limit less fn's static
// shared memory.
int cta_smem_budget(const sfe_ctx *ctx, const void *fn, size_t *budget);
// Lets `fn` take `bytes` of dynamic shared memory.  The attribute belongs to (function, device), not to a context, so
// it is only ever raised, process-wide: a launch on another thread's context never finds it lowered under its layout.
int raise_smem_limit(const sfe_ctx *ctx, const void *fn, size_t bytes);
// raise_smem_limit, then *per_sm = CTAs of `fn` per SM with `threads` threads and `bytes` of dynamic shared memory (at
// least 1), cached in the context.
int ctas_per_sm(sfe_ctx *ctx, const void *fn, int threads, size_t bytes, int *per_sm);

// ---------------------------------------------------------------- compressed pings (jpeg.cu, png.cu)
// Orientation (tag 0x0112 of IFD0) of a TIFF structure, as carried by JPEG's APP1 "Exif" segment and PNG's eXIf
// chunk; 1 when absent or unreadable.
inline int tiff_orientation(const uint8_t *t, int64_t tl) {
  if (tl < 8) return 1;
  const bool le = t[0] == 'I' && t[1] == 'I', be = t[0] == 'M' && t[1] == 'M';
  if (!le && !be) return 1;
  auto u16 = [&](int64_t o) { return le ? (t[o] | t[o + 1] << 8) : (t[o] << 8 | t[o + 1]); };
  auto u32 = [&](int64_t o) { return ((uint32_t)u16(le ? o + 2 : o) << 16) | (uint32_t)u16(le ? o : o + 2); };
  const int64_t ifd = u32(4);
  if (ifd + 2 > tl) return 1;
  const int cnt = u16(ifd);
  for (int k = 0; k < cnt; ++k) {
    const int64_t e = ifd + 2 + 12 * (int64_t)k;
    if (e + 12 > tl) break;
    if (u16(e) == 0x0112) return u16(e + 8);
  }
  return 1;
}

#ifdef __CUDACC__
// OpenCV 4.x cvtColor BGR2GRAY, 8-bit: fixed point with 15 fractional bits (the weights sum to 2^15, so three equal
// channels give the value back)
__host__ __device__ __forceinline__ uint8_t bgr2gray(int b, int g, int r) {
  return (uint8_t)((3735 * b + 19235 * g + 9798 * r + (1 << 14)) >> 15);
}
#endif

// cuTensorMapEncodeTiled through the runtime's driver entry point (no -lcuda needed)
int encode_tensor_map_3d(CUtensorMap *map, CUtensorMapDataType dt, size_t elem_bytes, const void *base,
                         uint64_t d0, uint64_t d1, uint64_t d2, uint32_t b0, uint32_t b1, uint32_t b2);

// ---------------------------------------------------------------- device PTX wrappers
#ifdef __CUDACC__
__device__ __forceinline__ uint32_t smem_u32(const void *p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t *bar) {
  asm volatile("{\n .reg .b64 st;\n mbarrier.arrive.shared::cta.b64 st, [%0];\n}" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t *bar, uint32_t bytes) {
  asm volatile("{\n .reg .b64 st;\n mbarrier.arrive.expect_tx.shared::cta.b64 st, [%0], %1;\n}" ::"r"(smem_u32(bar)),
               "r"(bytes)
               : "memory");
}
// try_wait with a suspend-time hint: a waiting thread may sleep in hardware until the phase completes (or the
// hint expires) instead of spinning on the barrier.
__device__ __forceinline__ bool mbar_try_wait(uint64_t *bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n .reg .pred p;\n mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n selp.u32 %0, 1, 0, p;\n}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity), "r"(1000000u)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}
// TMA: global -> shared tile load of a 3-D tensor (SASS: UTMALDG)
__device__ __forceinline__ void tma_load_3d(void *smem_dst, const CUtensorMap *map, uint64_t *bar, int c0, int c1,
                                            int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], "
      "[%2];" ::"r"(smem_u32(smem_dst)),
      "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
// TMA: shared -> global tile store (SASS: UTMASTG)
__device__ __forceinline__ void tma_store_3d(const CUtensorMap *map, const void *smem_src, int c0, int c1, int c2) {
  asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.tile.bulk_group [%0, {%2, %3, %4}], [%1];" ::"l"(map),
               "r"(smem_u32(smem_src)), "r"(c0), "r"(c1), "r"(c2)
               : "memory");
}
__device__ __forceinline__ void tma_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void tma_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
template <int N>
__device__ __forceinline__ void tma_wait_all() {
  asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory");
}
__device__ __forceinline__ void prefetch_tmap(const CUtensorMap *map) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(map) : "memory");
}
// Persistent CTAs: CTA c starts with work item c; every later item is the next one no CTA has taken yet (`counter`
// zero at launch), so CTAs that drew short items take more and a launch ends in a short tail instead of waiting for
// the CTAs whose static share (c, c + gridDim.x, ...) happened to be the longest.  All threads of the CTA call it;
// `bcast` is a CTA-shared int.
__device__ __forceinline__ int next_work_item(int *counter, int *bcast) {
  __syncthreads();  // every thread has read the previous item
  if (threadIdx.x == 0) *bcast = (int)gridDim.x + atomicAdd(counter, 1);
  __syncthreads();
  return *bcast;
}
__device__ __forceinline__ void named_bar_sync(int id, int nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}
#endif  // __CUDACC__

}  // namespace sfe
