// libsonarfe C ABI: context, error reporting, host-buffer conveniences.
// Declarations and reference citations: include/sonarfe.h.
#include <cudaTypedefs.h>

#include <algorithm>
#include <iterator>
#include <map>
#include <mutex>
#include <vector>

#include "grid.cuh"
#include "stages.cuh"

namespace sfe {

static thread_local char g_err[512] = "";

void set_error(const char *fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int ensure(sfe_ctx *ctx, Buffer &b, size_t bytes) { return ensure(ctx, b, bytes, ctx->stream); }

int ensure(sfe_ctx *ctx, Buffer &b, size_t bytes, cudaStream_t stream) {
  if (bytes <= b.cap) return SFE_OK;
  // grow-only; the old block may still be in use by enqueued work -> stream-ordered free
  if (b.ptr) SFE_CUDA(cudaFreeAsync(b.ptr, stream));
  if (b.ptr == ctx->cfar_lut_buf) ctx->cfar_lut_buf = nullptr;  // the cached table went with the block
  b.ptr = nullptr, b.cap = 0;
  size_t want = bytes + bytes / 4 + 256;
  SFE_CUDA(cudaMallocAsync(&b.ptr, want, stream));
  b.cap = want;
  return SFE_OK;
}

int ensure_pinned(sfe_ctx *ctx, size_t bytes) {
  if (bytes <= ctx->pinned_cap) return SFE_OK;
  if (ctx->pinned) {
    SFE_CUDA(cudaStreamSynchronize(ctx->stream));
    SFE_CUDA(cudaFreeHost(ctx->pinned));
  }
  ctx->pinned = nullptr, ctx->pinned_cap = 0;
  SFE_CUDA(cudaMallocHost(&ctx->pinned, bytes * 2));
  ctx->pinned_cap = bytes * 2;
  return SFE_OK;
}

static std::mutex g_fn_mu;                                    // guards the two tables below
static std::map<const void *, size_t> g_static_smem;          // kernel -> its static shared memory
static std::map<std::pair<int, const void *>, size_t> g_dyn;  // (device, kernel) -> dynamic shared memory allowed

int cta_smem_budget(const sfe_ctx *ctx, const void *fn, size_t *budget) {
  std::lock_guard<std::mutex> lock(g_fn_mu);
  auto it = g_static_smem.find(fn);
  if (it == g_static_smem.end()) {  // a property of the kernel, the same on every device: read once
    cudaFuncAttributes attr;
    SFE_CUDA(cudaFuncGetAttributes(&attr, fn));
    it = g_static_smem.emplace(fn, attr.sharedSizeBytes).first;
  }
  *budget = (size_t)ctx->max_smem_optin - it->second;
  return SFE_OK;
}

int raise_smem_limit(const sfe_ctx *ctx, const void *fn, size_t bytes) {
  std::lock_guard<std::mutex> lock(g_fn_mu);
  size_t &cur = g_dyn[{ctx->device, fn}];
  if (bytes > cur) {
    SFE_CUDA(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
    cur = bytes;
  }
  return SFE_OK;
}

int ctas_per_sm(sfe_ctx *ctx, const void *fn, int threads, size_t bytes, int *per_sm) {
  int rc = raise_smem_limit(ctx, fn, bytes);
  if (rc != SFE_OK) return rc;
  for (const auto &e : ctx->occ)
    if (e.fn == fn && e.smem == bytes && e.threads == threads) {
      *per_sm = e.per_sm;
      return SFE_OK;
    }
  int q = 1;
  SFE_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&q, fn, threads, bytes));
  *per_sm = q < 1 ? 1 : q;
  ctx->occ[ctx->occ_next] = {fn, bytes, threads, *per_sm};
  ctx->occ_next = (ctx->occ_next + 1) % (int)std::size(ctx->occ);
  return SFE_OK;
}

int encode_tensor_map_3d(CUtensorMap *map, CUtensorMapDataType dt, size_t es, const void *base, uint64_t d0,
                         uint64_t d1, uint64_t d2, uint32_t b0, uint32_t b1, uint32_t b2) {
  static PFN_cuTensorMapEncodeTiled_v12000 encode = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void *fn = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      encode = reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(fn);
  });
  if (!encode) {
    set_error("cuTensorMapEncodeTiled is not available from the driver");
    return SFE_ERR_CUDA;
  }
  cuuint64_t dims[3] = {d0, d1, d2};
  cuuint64_t strides[2] = {d0 * es, d0 * d1 * es};  // bytes, dims 1..2
  cuuint32_t box[3] = {b0, b1, b2};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = encode(map, dt, 3, const_cast<void *>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                      CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                      CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed (CUresult %d) for dims (%llu,%llu,%llu) box (%u,%u,%u)", (int)r,
              (unsigned long long)d0, (unsigned long long)d1, (unsigned long long)d2, b0, b1, b2);
    return SFE_ERR_CUDA;
  }
  return SFE_OK;
}

}  // namespace sfe

using namespace sfe;

extern "C" {

int sfe_version(void) { return SFE_VERSION; }
const char *sfe_last_error(void) { return g_err; }

int sfe_ctx_create(int device, void *cuda_stream, int own_stream, sfe_ctx **out) {
  SFE_REQUIRE(out != nullptr, "sfe_ctx_create: null out pointer");
  *out = nullptr;
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess || n == 0) {
    set_error("sfe_ctx_create: no CUDA device available (%s); libsonarfe has no CPU fallback",
              e == cudaSuccess ? "device count 0" : cudaGetErrorString(e));
    return SFE_ERR_CUDA;
  }
  SFE_REQUIRE(device >= 0 && device < n, "sfe_ctx_create: device %d out of range [0, %d)", device, n);
  SFE_CUDA(cudaSetDevice(device));
  cudaDeviceProp prop;
  SFE_CUDA(cudaGetDeviceProperties(&prop, device));
  if (prop.major != 9 || prop.minor != 0) {
    set_error("sfe_ctx_create: device %d is sm_%d%d; this library is built for sm_90a (H100) only", device,
              prop.major, prop.minor);
    return SFE_ERR_UNSUPPORTED;
  }
  sfe_ctx *ctx = new sfe_ctx();
  ctx->device = device;
  ctx->sm_count = ctx->device_sm_count = prop.multiProcessorCount;
  ctx->max_smem_optin = (int)prop.sharedMemPerBlockOptin;
  if (!own_stream) {
    ctx->stream = (cudaStream_t)cuda_stream;
  } else {
    cudaError_t e2 = cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking);
    if (e2 != cudaSuccess) {
      set_error("cudaStreamCreate: %s", cudaGetErrorString(e2));
      delete ctx;
      return SFE_ERR_CUDA;
    }
    ctx->owns_stream = true;
  }
  if (cudaMalloc((void **)&ctx->work, SFE_WORK_COUNTERS * sizeof(int)) != cudaSuccess) {
    set_error("sfe_ctx_create: cudaMalloc of the work counters failed");
    (void)cudaGetLastError();
    if (ctx->owns_stream) cudaStreamDestroy(ctx->stream);
    delete ctx;
    return SFE_ERR_CUDA;
  }
  *out = ctx;
  return SFE_OK;
}

void sfe_ctx_destroy(sfe_ctx *ctx) {
  if (!ctx) return;
  cudaSetDevice(ctx->device);
  cudaStreamSynchronize(ctx->stream);
  sfe::destroy(ctx->jpeg);
  sfe::destroy(ctx->png);
  for (auto &b : ctx->scratch)
    if (b.ptr) cudaFree(b.ptr);
  for (auto &b : ctx->stage_in)
    if (b.ptr) cudaFree(b.ptr);
  for (auto &b : ctx->stage_out)
    if (b.ptr) cudaFree(b.ptr);
  if (ctx->pinned) cudaFreeHost(ctx->pinned);
  if (ctx->work) cudaFree(ctx->work);
  if (ctx->copy_stream) {
    cudaStreamSynchronize(ctx->copy_stream);
    cudaStreamDestroy(ctx->copy_stream);
  }
  for (auto ev : ctx->copy_ev)
    if (ev) cudaEventDestroy(ev);
  if (ctx->owns_stream) cudaStreamDestroy(ctx->stream);
  delete ctx;
}

int sfe_sync(sfe_ctx *ctx) {
  SFE_REQUIRE(ctx != nullptr, "sfe_sync: null context");
  SFE_CUDA(cudaStreamSynchronize(ctx->stream));
  return SFE_OK;
}

uint64_t sfe_launch_count(const sfe_ctx *ctx) { return ctx ? ctx->launches : 0; }

int sfe_ctx_set_grid_sms(sfe_ctx *ctx, int sms, int32_t *effective) {
  SFE_REQUIRE(ctx != nullptr, "sfe_ctx_set_grid_sms: null context");
  ctx->sm_count = sms >= 1 ? std::min(sms, ctx->device_sm_count) : ctx->device_sm_count;
  if (effective) *effective = ctx->sm_count;
  return SFE_OK;
}

int sfe_ctx_occupancy(const sfe_ctx *ctx, int32_t *threads, int32_t *smem, int32_t *per_sm, int capacity,
                      int32_t *n) {
  SFE_REQUIRE(ctx && n && capacity >= 0 && (capacity == 0 || (threads && smem && per_sm)),
              "sfe_ctx_occupancy: null argument");
  const int size = (int)std::size(ctx->occ);
  const bool wrapped = ctx->occ[ctx->occ_next].fn != nullptr;  // (the ring is full: its oldest entry is next)
  int k = 0;
  for (int i = 0; i < size; ++i) {
    const auto &e = ctx->occ[((wrapped ? ctx->occ_next : 0) + i) % size];
    if (!e.fn) continue;
    if (k < capacity) threads[k] = e.threads, smem[k] = (int32_t)e.smem, per_sm[k] = e.per_sm;
    ++k;
  }
  *n = k;
  return SFE_OK;
}

int sfe_copy_to_host(sfe_ctx *ctx, void *dst_host, const void *src_dev, uint64_t bytes) {
  SFE_REQUIRE(ctx && (bytes == 0 || (dst_host && src_dev)), "sfe_copy_to_host: null argument");
  if (bytes == 0) return SFE_OK;
  SFE_CUDA(cudaSetDevice(ctx->device));
  SFE_CUDA(cudaMemcpyAsync(dst_host, src_dev, (size_t)bytes, cudaMemcpyDeviceToHost, ctx->stream));
  SFE_CUDA(cudaStreamSynchronize(ctx->stream));
  return SFE_OK;
}

int sfe_cfar_dev(sfe_ctx *ctx, const void *img_dev, int dtype, int n_frames, int R, int B, int alg, int train_hs,
                 int guard_hs, int k, double tau, int gate_enable, double gate_threshold, uint8_t *mask_dev,
                 float *thr_dev, uint32_t *bits_dev) {
  SFE_REQUIRE(ctx != nullptr, "sfe_cfar_dev: null context");
  SFE_CUDA(cudaSetDevice(ctx->device));
  return cfar_run(ctx, ctx->stream, img_dev, dtype, n_frames, R, B, alg, train_hs, guard_hs, k, tau, gate_enable,
                  gate_threshold, mask_dev, thr_dev, bits_dev);
}

int sfe_cfar_host(sfe_ctx *ctx, const void *img_host, int dtype, int n_frames, int R, int B, int alg, int train_hs,
                  int guard_hs, int k, double tau, int gate_enable, double gate_threshold, uint8_t *mask_host,
                  float *thr_host) {
  SFE_REQUIRE(ctx != nullptr, "sfe_cfar_host: null context");
  SFE_REQUIRE(dtype == SFE_U8 || dtype == SFE_F32, "sfe_cfar_host: dtype must be SFE_U8 or SFE_F32");
  SFE_REQUIRE(n_frames >= 0 && R >= 0 && B >= 0, "sfe_cfar_host: negative shape");
  SFE_CUDA(cudaSetDevice(ctx->device));
  const size_t cells = (size_t)n_frames * R * B;
  if (cells == 0) return SFE_OK;
  SFE_REQUIRE(img_host != nullptr && mask_host != nullptr, "sfe_cfar_host: null image or mask pointer");
  const size_t es = dtype == SFE_U8 ? 1 : 4;
  int rc;
  if ((rc = ensure(ctx, ctx->stage_in[0], cells * es)) != SFE_OK) return rc;
  if ((rc = ensure(ctx, ctx->stage_out[0], cells)) != SFE_OK) return rc;
  if (thr_host && (rc = ensure(ctx, ctx->stage_out[1], cells * sizeof(float))) != SFE_OK) return rc;
  SFE_CUDA(cudaMemcpyAsync(ctx->stage_in[0].ptr, img_host, cells * es, cudaMemcpyHostToDevice, ctx->stream));
  rc = cfar_run(ctx, ctx->stream, ctx->stage_in[0].ptr, dtype, n_frames, R, B, alg, train_hs, guard_hs, k, tau, gate_enable,
                gate_threshold, (uint8_t *)ctx->stage_out[0].ptr, thr_host ? (float *)ctx->stage_out[1].ptr : nullptr,
                nullptr);
  if (rc != SFE_OK) return rc;
  SFE_CUDA(cudaMemcpyAsync(mask_host, ctx->stage_out[0].ptr, cells, cudaMemcpyDeviceToHost, ctx->stream));
  if (thr_host)
    SFE_CUDA(cudaMemcpyAsync(thr_host, ctx->stage_out[1].ptr, cells * sizeof(float), cudaMemcpyDeviceToHost,
                             ctx->stream));
  SFE_CUDA(cudaStreamSynchronize(ctx->stream));
  return SFE_OK;
}

}  // extern "C"

// ============================================================================ clouds / match / ICP
extern "C" {

int sfe_downsample_dev(sfe_ctx *ctx, const float *pts_dev, const int32_t *off_dev, int n_clouds, int dim, int n_max,
                       float resolution, float *out_pts_dev, int32_t *out_idx_dev, int32_t *out_count_dev) {
  SFE_REQUIRE(ctx != nullptr, "sfe_downsample_dev: null context");
  SFE_CUDA(cudaSetDevice(ctx->device));
  return downsample_run(ctx, ctx->stream, {pts_dev, off_dev, nullptr, n_max}, n_clouds, dim, resolution, out_pts_dev,
                        out_idx_dev, out_count_dev, DS_ANY_SIZE, SCR_CLOUD, WORK_DS);
}

int sfe_downsample_frames_dev(sfe_ctx *ctx, const float *pts_dev, const int32_t *off_dev, const int32_t *cnt_dev,
                              int n_clouds, int n_max, int frame_points, float resolution, float *out_pts_dev,
                              int32_t *out_idx_dev, int32_t *out_count_dev) {
  SFE_REQUIRE(ctx != nullptr, "sfe_downsample_frames_dev: null context");
  SFE_REQUIRE(frame_points > 0, "sfe_downsample_frames_dev: frame_points must be positive (got %d)", frame_points);
  SFE_CUDA(cudaSetDevice(ctx->device));
  return downsample_run(ctx, ctx->stream, {pts_dev, off_dev, cnt_dev, n_max}, n_clouds, 2, resolution, out_pts_dev,
                        out_idx_dev, out_count_dev, frame_points, SCR_CLOUD, WORK_DS);
}

int sfe_downsample_cta_limit(sfe_ctx *ctx, int dim, int32_t *limit) {
  SFE_REQUIRE(ctx && limit, "sfe_downsample_cta_limit: null pointer");
  SFE_REQUIRE(dim == 2 || dim == 3, "sfe_downsample_cta_limit: points must have 2 or 3 columns (got %d)", dim);
  SFE_CUDA(cudaSetDevice(ctx->device));
  int n;
  const int rc = downsample_cta_limit(ctx, &n, dim);
  if (rc == SFE_OK) *limit = n;
  return rc;
}

int sfe_remove_outlier_dev(sfe_ctx *ctx, const float *pts_dev, const int32_t *off_dev, int n_clouds, int dim,
                           int n_max, double radius, int min_points, float *out_pts_dev, int32_t *out_idx_dev,
                           int32_t *out_count_dev) {
  SFE_REQUIRE(ctx != nullptr, "sfe_remove_outlier_dev: null context");
  SFE_CUDA(cudaSetDevice(ctx->device));
  return remove_outlier_run(ctx, ctx->stream, {pts_dev, off_dev, nullptr, n_max}, n_clouds, dim, radius, min_points,
                            out_pts_dev, out_idx_dev, out_count_dev, 0);
}

static int cloud_filter_host(sfe_ctx *ctx, int which, const float *pts_host, int n, int dim, float resolution,
                             double radius, int min_points, float *out_pts_host, int32_t *out_idx_host,
                             int32_t *n_out) {
  SFE_REQUIRE(ctx && n_out, "cloud filter: null context or n_out");
  SFE_REQUIRE(n >= 0, "cloud filter: negative point count");
  SFE_REQUIRE(dim == 2 || dim == 3, "cloud filter: points must have 2 or 3 columns (got %d)", dim);
  *n_out = 0;
  if (n == 0) return SFE_OK;
  SFE_REQUIRE(pts_host && out_pts_host && out_idx_host, "cloud filter: null pointer");
  SFE_CUDA(cudaSetDevice(ctx->device));
  Carver cv;
  for (int pass = 0; pass < 2; ++pass) {
    cv.off = 0;
    float *d_pts = (float *)cv.take(sizeof(float) * (size_t)n * dim);
    int32_t *d_off = (int32_t *)cv.take(2 * sizeof(int32_t));
    float *d_out = (float *)cv.take(sizeof(float) * (size_t)n * dim);
    int32_t *d_idx = (int32_t *)cv.take(sizeof(int32_t) * (size_t)n);
    int32_t *d_cnt = (int32_t *)cv.take(sizeof(int32_t));
    if (pass == 0) {
      int rc = ensure(ctx, ctx->stage_in[1], cv.off);
      if (rc != SFE_OK) return rc;
      cv.base = (char *)ctx->stage_in[1].ptr;
      continue;
    }
    const int32_t off[2] = {0, n};
    SFE_CUDA(cudaMemcpyAsync(d_pts, pts_host, sizeof(float) * (size_t)n * dim, cudaMemcpyHostToDevice, ctx->stream));
    SFE_CUDA(cudaMemcpyAsync(d_off, off, sizeof(off), cudaMemcpyHostToDevice, ctx->stream));
    const PackedClouds in{d_pts, d_off, nullptr, n};
    int rc = which == 0 ? downsample_run(ctx, ctx->stream, in, 1, dim, resolution, d_out, d_idx, d_cnt, DS_ANY_SIZE,
                                         SCR_CLOUD, WORK_DS)
                        : remove_outlier_run(ctx, ctx->stream, in, 1, dim, radius, min_points, d_out, d_idx, d_cnt, 0);
    if (rc != SFE_OK) return rc;
    SFE_CUDA(cudaMemcpyAsync(n_out, d_cnt, sizeof(int32_t), cudaMemcpyDeviceToHost, ctx->stream));
    SFE_CUDA(cudaMemcpyAsync(out_pts_host, d_out, sizeof(float) * (size_t)n * dim, cudaMemcpyDeviceToHost,
                             ctx->stream));
    SFE_CUDA(cudaMemcpyAsync(out_idx_host, d_idx, sizeof(int32_t) * (size_t)n, cudaMemcpyDeviceToHost, ctx->stream));
    SFE_CUDA(cudaStreamSynchronize(ctx->stream));
  }
  return SFE_OK;
}

int sfe_downsample_host(sfe_ctx *ctx, const float *pts_host, int n, int dim, float resolution, float *out_pts_host,
                        int32_t *out_idx_host, int32_t *n_out) {
  return cloud_filter_host(ctx, 0, pts_host, n, dim, resolution, 0.0, 0, out_pts_host, out_idx_host, n_out);
}

int sfe_remove_outlier_host(sfe_ctx *ctx, const float *pts_host, int n, int dim, double radius, int min_points,
                            float *out_pts_host, int32_t *out_idx_host, int32_t *n_out) {
  return cloud_filter_host(ctx, 1, pts_host, n, dim, 0.f, radius, min_points, out_pts_host, out_idx_host, n_out);
}

int sfe_match_dev(sfe_ctx *ctx, const float *ref_pts_dev, const int32_t *ref_off_dev, const float *in_pts_dev,
                  const int32_t *in_off_dev, int n_pairs, int n_ref_max, float max_dist, int32_t *ids_dev,
                  float *dists_dev) {
  SFE_REQUIRE(ctx != nullptr, "sfe_match_dev: null context");
  SFE_CUDA(cudaSetDevice(ctx->device));
  return match_run(ctx, ctx->stream, {ref_pts_dev, ref_off_dev, nullptr, n_ref_max},
                   {in_pts_dev, in_off_dev, nullptr, 0}, n_pairs, max_dist, ids_dev, dists_dev);
}

int sfe_match_knn_dev(sfe_ctx *ctx, const float *ref_pts_dev, const int32_t *ref_off_dev, const float *in_pts_dev,
                      const int32_t *in_off_dev, int n_pairs, int n_ref_max, int knn, float max_dist, int32_t *ids_dev,
                      float *dists_dev) {
  SFE_REQUIRE(ctx != nullptr, "sfe_match_knn_dev: null context");
  SFE_CUDA(cudaSetDevice(ctx->device));
  return match_knn_run(ctx, ctx->stream, {ref_pts_dev, ref_off_dev, nullptr, n_ref_max},
                       {in_pts_dev, in_off_dev, nullptr, 0}, n_pairs, knn, max_dist, ids_dev, dists_dev);
}

int sfe_match_dim_dev(sfe_ctx *ctx, const float *ref_pts_dev, const int32_t *ref_off_dev, const float *in_pts_dev,
                      const int32_t *in_off_dev, int n_pairs, int dim, int n_ref_max, float max_dist, int32_t *ids_dev,
                      float *dists_dev) {
  SFE_REQUIRE(ctx != nullptr, "sfe_match_dim_dev: null context");
  SFE_CUDA(cudaSetDevice(ctx->device));
  return match_knn_run(ctx, ctx->stream, {ref_pts_dev, ref_off_dev, nullptr, n_ref_max},
                       {in_pts_dev, in_off_dev, nullptr, 0}, n_pairs, 1, max_dist, ids_dev, dists_dev, dim);
}

int sfe_match_knn_dim_dev(sfe_ctx *ctx, const float *ref_pts_dev, const int32_t *ref_off_dev, const float *in_pts_dev,
                          const int32_t *in_off_dev, int n_pairs, int dim, int n_ref_max, int knn, float max_dist,
                          int32_t *ids_dev, float *dists_dev) {
  SFE_REQUIRE(ctx != nullptr, "sfe_match_knn_dim_dev: null context");
  SFE_CUDA(cudaSetDevice(ctx->device));
  return match_knn_run(ctx, ctx->stream, {ref_pts_dev, ref_off_dev, nullptr, n_ref_max},
                       {in_pts_dev, in_off_dev, nullptr, 0}, n_pairs, knn, max_dist, ids_dev, dists_dev, dim);
}

// sfe_match[_knn][_dim]_host (`name` in messages): one pair of dim-column clouds, results [knn][n_in]
static int match_host(sfe_ctx *ctx, const char *name, const float *ref_host, int n_ref, const float *in_host, int n_in,
                      int knn, float max_dist, int32_t *ids_host, float *dists_host, int dim = 2) {
  SFE_REQUIRE(ctx != nullptr, "%s: null context", name);
  SFE_REQUIRE(n_ref >= 0 && n_in >= 0, "%s: negative point count", name);
  SFE_REQUIRE(knn >= 1 && knn <= GRID_KNN_MAX, "%s: knn %d is not supported (1..%d)", name, knn, GRID_KNN_MAX);
  SFE_REQUIRE(dim == 2 || dim == 3, "%s: points must have 2 or 3 columns (got %d)", name, dim);
  if (n_in == 0) return SFE_OK;
  SFE_REQUIRE(in_host && ids_host && dists_host && (ref_host || n_ref == 0), "%s: null pointer", name);
  SFE_CUDA(cudaSetDevice(ctx->device));
  const size_t out = (size_t)knn * n_in;
  Carver cv;
  for (int pass = 0; pass < 2; ++pass) {
    cv.off = 0;
    float *d_ref = (float *)cv.take(sizeof(float) * dim * (size_t)(n_ref > 0 ? n_ref : 1));
    float *d_in = (float *)cv.take(sizeof(float) * dim * (size_t)n_in);
    int32_t *d_off = (int32_t *)cv.take(4 * sizeof(int32_t));
    int32_t *d_ids = (int32_t *)cv.take(sizeof(int32_t) * out);
    float *d_d = (float *)cv.take(sizeof(float) * out);
    if (pass == 0) {
      int rc = ensure(ctx, ctx->stage_in[1], cv.off);
      if (rc != SFE_OK) return rc;
      cv.base = (char *)ctx->stage_in[1].ptr;
      continue;
    }
    const int32_t off[4] = {0, n_ref, 0, n_in};
    if (n_ref > 0)
      SFE_CUDA(cudaMemcpyAsync(d_ref, ref_host, sizeof(float) * dim * (size_t)n_ref, cudaMemcpyHostToDevice, ctx->stream));
    SFE_CUDA(cudaMemcpyAsync(d_in, in_host, sizeof(float) * dim * (size_t)n_in, cudaMemcpyHostToDevice, ctx->stream));
    SFE_CUDA(cudaMemcpyAsync(d_off, off, sizeof(off), cudaMemcpyHostToDevice, ctx->stream));
    int rc = match_knn_run(ctx, ctx->stream, {d_ref, d_off, nullptr, n_ref}, {d_in, d_off + 2, nullptr, n_in}, 1, knn,
                           max_dist, d_ids, d_d, dim);
    if (rc != SFE_OK) return rc;
    SFE_CUDA(cudaMemcpyAsync(ids_host, d_ids, sizeof(int32_t) * out, cudaMemcpyDeviceToHost, ctx->stream));
    SFE_CUDA(cudaMemcpyAsync(dists_host, d_d, sizeof(float) * out, cudaMemcpyDeviceToHost, ctx->stream));
    SFE_CUDA(cudaStreamSynchronize(ctx->stream));
  }
  return SFE_OK;
}

int sfe_match_host(sfe_ctx *ctx, const float *ref_host, int n_ref, const float *in_host, int n_in, float max_dist,
                   int32_t *ids_host, float *dists_host) {
  return match_host(ctx, "sfe_match_host", ref_host, n_ref, in_host, n_in, 1, max_dist, ids_host, dists_host);
}

int sfe_match_knn_host(sfe_ctx *ctx, const float *ref_host, int n_ref, const float *in_host, int n_in, int knn,
                       float max_dist, int32_t *ids_host, float *dists_host) {
  return match_host(ctx, "sfe_match_knn_host", ref_host, n_ref, in_host, n_in, knn, max_dist, ids_host, dists_host);
}

int sfe_match_dim_host(sfe_ctx *ctx, const float *ref_host, int n_ref, const float *in_host, int n_in, int dim,
                       float max_dist, int32_t *ids_host, float *dists_host) {
  return match_host(ctx, "sfe_match_dim_host", ref_host, n_ref, in_host, n_in, 1, max_dist, ids_host, dists_host, dim);
}

int sfe_match_knn_dim_host(sfe_ctx *ctx, const float *ref_host, int n_ref, const float *in_host, int n_in, int dim,
                           int knn, float max_dist, int32_t *ids_host, float *dists_host) {
  return match_host(ctx, "sfe_match_knn_dim_host", ref_host, n_ref, in_host, n_in, knn, max_dist, ids_host, dists_host,
                    dim);
}

void sfe_icp_params_default(sfe_icp_params *p) {
  if (!p) return;
  p->matcher_max_dist = 10.0f;
  p->outlier_max_dist = 3.0f;
  p->trim_ratio = 0.8f;
  p->max_iterations = 40;
  p->min_diff_rot = 0.01f;
  p->min_diff_trans = 0.1f;
  p->smooth_length = 4;
  p->flags = 0;
  p->minimizer = 0;
  p->normals_knn = 5;
}

const char *sfe_icp_status_message(int status) {
  switch (status) {
    case SFE_ICP_SUCCESS: return "success";
    case SFE_ICP_NO_OUTLIER: return "no outlier to filter";
    case SFE_ICP_NO_POINT: return "ErrorMnimizer: no point to minimize";
    case SFE_ICP_NAN_ROT: return "abs rotation norm not a number";
    case SFE_ICP_NAN_TRANS: return "abs translation norm not a number";
    case SFE_ICP_NOT_RIGID: return "RigidTransformation: Error, rotation matrix is not orthogonal.";
    case SFE_ICP_EMPTY_REF: return "reference cloud is empty";
    case SFE_ICP_SKIPPED: return "not enough points";
    case SFE_ICP_TOO_LARGE: return "cloud exceeds the configured capacity";
    default: return "unknown ICP status";
  }
}

int sfe_icp_dev(sfe_ctx *ctx, const sfe_icp_params *prm, const float *src_pts_dev, const int32_t *src_off_dev,
                const float *tgt_pts_dev, const int32_t *tgt_off_dev, const int32_t *src_id_dev,
                const int32_t *tgt_id_dev, int n_problems, int ns_max, int nt_max, const float *guess_dev, float *T_dev,
                int32_t *iters_dev, int32_t *inliers_dev, int32_t *status_dev) {
  SFE_REQUIRE(ctx != nullptr, "sfe_icp_dev: null context");
  SFE_CUDA(cudaSetDevice(ctx->device));
  return icp_run(ctx, ctx->stream, prm,
                 {{src_pts_dev, src_off_dev, nullptr, ns_max}, {tgt_pts_dev, tgt_off_dev, nullptr, nt_max}, src_id_dev,
                  tgt_id_dev, n_problems, guess_dev, T_dev, iters_dev, inliers_dev, status_dev}, nullptr, 0, nullptr,
                 ctx->has_icp_filters ? &ctx->icp_filters : nullptr, ctx->has_icp_robust ? &ctx->icp_robust : nullptr);
}

int sfe_icp_set_filters(sfe_ctx *ctx, const sfe_icp_filters *filters) {
  SFE_REQUIRE(ctx != nullptr, "sfe_icp_set_filters: null context");
  if (filters) {
    const int rc = icp_filters_check(filters, "sfe_icp_set_filters");
    if (rc != SFE_OK) return rc;
    ctx->icp_filters = *filters;
  }
  ctx->has_icp_filters = filters != nullptr;
  return SFE_OK;
}

int sfe_icp_set_robust(sfe_ctx *ctx, const sfe_icp_robust *robust) {
  SFE_REQUIRE(ctx != nullptr, "sfe_icp_set_robust: null context");
  if (robust) {
    const int rc = icp_robust_check(robust, "sfe_icp_set_robust");
    if (rc != SFE_OK) return rc;
    ctx->icp_robust = *robust;
  }
  ctx->has_icp_robust = robust != nullptr;
  return SFE_OK;
}

int sfe_icp_host(sfe_ctx *ctx, const sfe_icp_params *prm, const float *src_host, int ns, const float *tgt_host, int nt,
                 const float *guess_host, int n_guesses, float *T_host, int32_t *iters_host, int32_t *inliers_host,
                 int32_t *status_host) {
  SFE_REQUIRE(ns >= 0 && nt >= 0 && n_guesses >= 0, "sfe_icp_host: negative size");
  if (n_guesses == 0) return SFE_OK;
  // one source / target pair: every guess is a problem on clouds 0 / 0
  const int32_t src_off[2] = {0, ns}, tgt_off[2] = {0, nt};
  std::vector<int32_t> zero((size_t)n_guesses, 0);
  return sfe_icp_batch_host(ctx, prm, src_host, src_off, 1, tgt_host, tgt_off, 1, zero.data(), zero.data(), n_guesses,
                            guess_host, T_host, iters_host, inliers_host, status_host);
}

// sfe_icp_batch_host and sfe_icp_batch_dim_host (`name` in messages): clouds of `dim` columns, (dim + 1)^2 guesses
static int icp_batch_host(sfe_ctx *ctx, const char *name, const sfe_icp_params *prm, const float *src_pts_host,
                          const int32_t *src_off_host, int n_src_clouds, const float *tgt_pts_host,
                          const int32_t *tgt_off_host, int n_tgt_clouds, const int32_t *src_id_host,
                          const int32_t *tgt_id_host, int n_problems, int dim, const float *guess_host, float *T_host,
                          int32_t *iters_host, int32_t *inliers_host, int32_t *status_host) {
  SFE_REQUIRE(ctx && prm, "%s: null context or parameters", name);
  SFE_REQUIRE(dim == 2 || dim == 3, "%s: points must have 2 or 3 columns (got %d)", name, dim);
  const sfe_icp_filters *filt = ctx->has_icp_filters ? &ctx->icp_filters : nullptr;
  const sfe_icp_robust *robust = ctx->has_icp_robust ? &ctx->icp_robust : nullptr;
  const int rc = icp_params_check(prm, dim, filt, name, robust);  // (before anything is copied)
  if (rc != SFE_OK) return rc;
  SFE_REQUIRE(n_src_clouds >= 1 && n_tgt_clouds >= 1 && n_problems >= 0, "%s: bad sizes", name);
  if (n_problems == 0) return SFE_OK;
  SFE_REQUIRE(src_off_host && tgt_off_host && src_id_host && tgt_id_host && guess_host && T_host && iters_host &&
                  inliers_host && status_host,
              "%s: null pointer", name);
  int ns_max = 0, nt_max = 0;
  for (int c = 0; c < n_src_clouds; ++c) {
    SFE_REQUIRE(src_off_host[c + 1] >= src_off_host[c], "%s: source offsets decrease at %d", name, c);
    ns_max = std::max(ns_max, src_off_host[c + 1] - src_off_host[c]);
  }
  for (int c = 0; c < n_tgt_clouds; ++c) {
    SFE_REQUIRE(tgt_off_host[c + 1] >= tgt_off_host[c], "%s: target offsets decrease at %d", name, c);
    nt_max = std::max(nt_max, tgt_off_host[c + 1] - tgt_off_host[c]);
  }
  SFE_REQUIRE(src_off_host[0] == 0 && tgt_off_host[0] == 0, "%s: offsets must start at 0", name);
  const int ns = src_off_host[n_src_clouds], nt = tgt_off_host[n_tgt_clouds];
  SFE_REQUIRE((src_pts_host || ns == 0) && (tgt_pts_host || nt == 0), "%s: null cloud pointer", name);
  for (int p = 0; p < n_problems; ++p)
    SFE_REQUIRE(src_id_host[p] >= 0 && src_id_host[p] < n_src_clouds && tgt_id_host[p] >= 0 &&
                    tgt_id_host[p] < n_tgt_clouds,
                "%s: problem %d names cloud %d / %d", name, p, src_id_host[p], tgt_id_host[p]);
  SFE_CUDA(cudaSetDevice(ctx->device));
  const size_t P = (size_t)n_problems, TS = (size_t)(dim + 1) * (dim + 1);
  Carver cv;
  for (int pass = 0; pass < 2; ++pass) {
    cv.off = 0;
    float *d_src = (float *)cv.take(sizeof(float) * dim * (size_t)(ns > 0 ? ns : 1));
    float *d_tgt = (float *)cv.take(sizeof(float) * dim * (size_t)(nt > 0 ? nt : 1));
    int32_t *d_soff = (int32_t *)cv.take(sizeof(int32_t) * (size_t)(n_src_clouds + 1));
    int32_t *d_toff = (int32_t *)cv.take(sizeof(int32_t) * (size_t)(n_tgt_clouds + 1));
    int32_t *d_ids = (int32_t *)cv.take(sizeof(int32_t) * 2 * P);
    float *d_guess = (float *)cv.take(sizeof(float) * TS * P);
    float *d_T = (float *)cv.take(sizeof(float) * TS * P);
    int32_t *d_res = (int32_t *)cv.take(sizeof(int32_t) * 3 * P);
    if (pass == 0) {
      int rc = ensure(ctx, ctx->stage_in[1], cv.off);
      if (rc != SFE_OK) return rc;
      cv.base = (char *)ctx->stage_in[1].ptr;
      continue;
    }
    if (ns > 0)
      SFE_CUDA(cudaMemcpyAsync(d_src, src_pts_host, sizeof(float) * dim * (size_t)ns, cudaMemcpyHostToDevice,
                               ctx->stream));
    if (nt > 0)
      SFE_CUDA(cudaMemcpyAsync(d_tgt, tgt_pts_host, sizeof(float) * dim * (size_t)nt, cudaMemcpyHostToDevice,
                               ctx->stream));
    SFE_CUDA(cudaMemcpyAsync(d_soff, src_off_host, sizeof(int32_t) * (size_t)(n_src_clouds + 1), cudaMemcpyHostToDevice,
                             ctx->stream));
    SFE_CUDA(cudaMemcpyAsync(d_toff, tgt_off_host, sizeof(int32_t) * (size_t)(n_tgt_clouds + 1), cudaMemcpyHostToDevice,
                             ctx->stream));
    SFE_CUDA(cudaMemcpyAsync(d_ids, src_id_host, sizeof(int32_t) * P, cudaMemcpyHostToDevice, ctx->stream));
    SFE_CUDA(cudaMemcpyAsync(d_ids + P, tgt_id_host, sizeof(int32_t) * P, cudaMemcpyHostToDevice, ctx->stream));
    SFE_CUDA(cudaMemcpyAsync(d_guess, guess_host, sizeof(float) * TS * P, cudaMemcpyHostToDevice, ctx->stream));
    IcpProblems pb{{d_src, d_soff, nullptr, ns_max}, {d_tgt, d_toff, nullptr, nt_max}, d_ids, d_ids + P, n_problems,
                   d_guess, d_T, d_res, d_res + P, d_res + 2 * P};
    pb.n_tgt_clouds = n_tgt_clouds, pb.n_src_clouds = n_src_clouds;
    int rc = dim == 3 ? icp3_run(ctx, ctx->stream, prm, pb, filt, robust)
                      : icp_run(ctx, ctx->stream, prm, pb, nullptr, 0, nullptr, filt, robust);
    if (rc != SFE_OK) return rc;
    SFE_CUDA(cudaMemcpyAsync(T_host, d_T, sizeof(float) * TS * P, cudaMemcpyDeviceToHost, ctx->stream));
    SFE_CUDA(cudaMemcpyAsync(iters_host, d_res, sizeof(int32_t) * P, cudaMemcpyDeviceToHost, ctx->stream));
    SFE_CUDA(cudaMemcpyAsync(inliers_host, d_res + P, sizeof(int32_t) * P, cudaMemcpyDeviceToHost, ctx->stream));
    SFE_CUDA(cudaMemcpyAsync(status_host, d_res + 2 * P, sizeof(int32_t) * P, cudaMemcpyDeviceToHost, ctx->stream));
    SFE_CUDA(cudaStreamSynchronize(ctx->stream));
  }
  return SFE_OK;
}

int sfe_icp_batch_host(sfe_ctx *ctx, const sfe_icp_params *prm, const float *src_pts_host, const int32_t *src_off_host,
                       int n_src_clouds, const float *tgt_pts_host, const int32_t *tgt_off_host, int n_tgt_clouds,
                       const int32_t *src_id_host, const int32_t *tgt_id_host, int n_problems, const float *guess_host,
                       float *T_host, int32_t *iters_host, int32_t *inliers_host, int32_t *status_host) {
  return icp_batch_host(ctx, "sfe_icp_batch_host", prm, src_pts_host, src_off_host, n_src_clouds, tgt_pts_host,
                        tgt_off_host, n_tgt_clouds, src_id_host, tgt_id_host, n_problems, 2, guess_host, T_host,
                        iters_host, inliers_host, status_host);
}

int sfe_icp_batch_dim_host(sfe_ctx *ctx, const sfe_icp_params *prm, const float *src_pts_host,
                           const int32_t *src_off_host, int n_src_clouds, const float *tgt_pts_host,
                           const int32_t *tgt_off_host, int n_tgt_clouds, const int32_t *src_id_host,
                           const int32_t *tgt_id_host, int n_problems, int dim, const float *guess_host, float *T_host,
                           int32_t *iters_host, int32_t *inliers_host, int32_t *status_host) {
  return icp_batch_host(ctx, "sfe_icp_batch_dim_host", prm, src_pts_host, src_off_host, n_src_clouds, tgt_pts_host,
                        tgt_off_host, n_tgt_clouds, src_id_host, tgt_id_host, n_problems, dim, guess_host, T_host,
                        iters_host, inliers_host, status_host);
}

int sfe_icp_dim_host(sfe_ctx *ctx, const sfe_icp_params *prm, const float *src_host, int ns, const float *tgt_host,
                     int nt, int dim, const float *guess_host, int n_guesses, float *T_host, int32_t *iters_host,
                     int32_t *inliers_host, int32_t *status_host) {
  SFE_REQUIRE(ns >= 0 && nt >= 0 && n_guesses >= 0, "sfe_icp_dim_host: negative size");
  if (n_guesses == 0) return SFE_OK;
  const int32_t src_off[2] = {0, ns}, tgt_off[2] = {0, nt};
  std::vector<int32_t> zero((size_t)n_guesses, 0);
  return icp_batch_host(ctx, "sfe_icp_dim_host", prm, src_host, src_off, 1, tgt_host, tgt_off, 1, zero.data(),
                        zero.data(), n_guesses, dim, guess_host, T_host, iters_host, inliers_host, status_host);
}

int sfe_icp_dim_dev(sfe_ctx *ctx, const sfe_icp_params *prm, const float *src_pts_dev, const int32_t *src_off_dev,
                    const float *tgt_pts_dev, const int32_t *tgt_off_dev, const int32_t *src_id_dev,
                    const int32_t *tgt_id_dev, int n_problems, int dim, int ns_max, int nt_max, const float *guess_dev,
                    float *T_dev, int32_t *iters_dev, int32_t *inliers_dev, int32_t *status_dev) {
  SFE_REQUIRE(ctx != nullptr && prm != nullptr, "sfe_icp_dim_dev: null context or parameters");
  SFE_REQUIRE(dim == 2 || dim == 3, "sfe_icp_dim_dev: points must have 2 or 3 columns (got %d)", dim);
  if (dim == 2)
    return sfe_icp_dev(ctx, prm, src_pts_dev, src_off_dev, tgt_pts_dev, tgt_off_dev, src_id_dev, tgt_id_dev, n_problems,
                       ns_max, nt_max, guess_dev, T_dev, iters_dev, inliers_dev, status_dev);
  SFE_CUDA(cudaSetDevice(ctx->device));
  return icp3_run(ctx, ctx->stream, prm,
                  {{src_pts_dev, src_off_dev, nullptr, ns_max}, {tgt_pts_dev, tgt_off_dev, nullptr, nt_max}, src_id_dev,
                   tgt_id_dev, n_problems, guess_dev, T_dev, iters_dev, inliers_dev, status_dev},
                  ctx->has_icp_filters ? &ctx->icp_filters : nullptr, ctx->has_icp_robust ? &ctx->icp_robust : nullptr);
}

int sfe_icp_cta_limit(sfe_ctx *ctx, int dim, int ns, int32_t *limit) {
  SFE_REQUIRE(ctx && limit, "sfe_icp_cta_limit: null pointer");
  SFE_CUDA(cudaSetDevice(ctx->device));
  int n;
  const int rc = icp_cta_limit(ctx, dim, ns, &n);
  if (rc == SFE_OK) *limit = n;
  return rc;
}

int sfe_icp_sampling_normals_dev(sfe_ctx *ctx, const float *pts_dev, const int32_t *off_dev, int n_clouds, int n_max,
                                 int knn, int method, float max_box, float *out_pts_dev, float *out_nrm_dev,
                                 int32_t *out_count_dev) {
  SFE_REQUIRE(ctx != nullptr, "sfe_icp_sampling_normals_dev: null context");
  SFE_REQUIRE(n_clouds >= 0 && n_max >= 0, "sfe_icp_sampling_normals_dev: negative sizes");
  if (n_clouds == 0) return SFE_OK;
  SFE_REQUIRE(pts_dev && off_dev && out_pts_dev && out_nrm_dev && out_count_dev,
              "sfe_icp_sampling_normals_dev: null pointer");
  sfe_icp_filters f = {-1.f, -1.f, 0, 1, {}, {}};
  f.reference[0] = {SFE_ICP_DATA_SAMPLING_NORMALS, method, max_box};
  sfe_icp_params prm;
  sfe_icp_params_default(&prm);
  prm.normals_knn = knn;
  int rc = icp_params_check(&prm, 2, &f, "sfe_icp_sampling_normals_dev");
  if (rc != SFE_OK) return rc;
  SFE_CUDA(cudaSetDevice(ctx->device));
  size_t bytes;
  if ((rc = sampling_normals_ws(n_clouds, n_max, knn, &bytes)) != SFE_OK) return rc;
  const size_t off_bytes = (sizeof(int) * (size_t)(n_clouds + 1) + 255) & ~size_t(255);
  if ((rc = ensure(ctx, ctx->scratch[SCR_ICP_FILTER], off_bytes + bytes, ctx->stream)) != SFE_OK) return rc;
  char *base = (char *)ctx->scratch[SCR_ICP_FILTER].ptr;
  return sampling_normals_run(ctx, ctx->stream, {pts_dev, off_dev, nullptr, n_max}, n_clouds, knn, method, max_box,
                              base + off_bytes, out_pts_dev, (int *)base, out_count_dev, (float2 *)out_nrm_dev);
}

int sfe_icp_surface_normals_dev(sfe_ctx *ctx, const float *pts_dev, const int32_t *off_dev, int n_clouds, int n_max,
                                int knn, float *out_nrm_dev) {
  SFE_REQUIRE(ctx != nullptr, "sfe_icp_surface_normals_dev: null context");
  SFE_REQUIRE(n_clouds >= 0 && n_max >= 0, "sfe_icp_surface_normals_dev: negative sizes");
  SFE_REQUIRE(knn >= 3 && knn <= GRID_KNN_MAX, "sfe_icp_surface_normals_dev: knn %d (3..%d)", knn, GRID_KNN_MAX);
  if (n_clouds == 0 || n_max == 0) return SFE_OK;
  SFE_REQUIRE(pts_dev && off_dev && out_nrm_dev, "sfe_icp_surface_normals_dev: null pointer");
  SFE_CUDA(cudaSetDevice(ctx->device));
  size_t bytes;
  int rc = surface_normals_ws(n_clouds, n_max, &bytes);
  if (rc != SFE_OK) return rc;
  if ((rc = ensure(ctx, ctx->scratch[SCR_ICP_FILTER], bytes > 0 ? bytes : 1, ctx->stream)) != SFE_OK) return rc;
  return surface_normals_run(ctx, ctx->stream, {pts_dev, off_dev, nullptr, n_max}, n_clouds, knn,
                             ctx->scratch[SCR_ICP_FILTER].ptr, (float2 *)out_nrm_dev);
}

int sfe_icp_source_limit(sfe_ctx *ctx, const sfe_icp_params *prm, int dim, int32_t *limit) {
  SFE_REQUIRE(dim == 2 || dim == 3, "sfe_icp_source_limit: points must have 2 or 3 columns (got %d)", dim);
  SFE_REQUIRE(ctx && prm && limit, "sfe_icp_source_limit: null pointer");
  SFE_CUDA(cudaSetDevice(ctx->device));
  int n;
  const int rc = icp_source_limit(ctx, prm, dim, ctx->has_icp_filters ? &ctx->icp_filters : nullptr, &n,
                                  ctx->has_icp_robust ? &ctx->icp_robust : nullptr);
  if (rc == SFE_OK) *limit = n;
  return rc;
}

}  // extern "C"
