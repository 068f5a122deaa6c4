// Global-initialisation cost (SURVEY row N2): occupancy grid of a target cloud + scoring of candidate poses.
// Replaces the closure of SLAM.get_matching_cost_subroutine1 (slam.py:461-570) that scipy.shgo evaluates
// 50-500+ times per keyframe (slam.py:683-701, 943-961).  The grid lives on the device as a bit-plane
// (1 bit per 0.05 m cell: a 60 m x 60 m target is ~190 KB, resident in L1/L2), the dilation is done by
// stamping the structuring element around every target point, and K candidate transforms are scored by
// one launch.
#include "common.cuh"

using namespace sfe;

struct sfe_costmap {
  int device;
  int rows, cols, wpr;  // wpr = 32-bit words per grid row
  float xmin, ymin, res;
  uint32_t *bits;       // device [rows][wpr]
  float *src;           // device copy of the closure's source cloud
  int n_src, src_cap;
  float *tf;            // device staging for transforms / costs of the host entry point
  int32_t *cost;
  int tf_cap;
};

namespace {

// cell index along one axis exactly like numpy on float32 arrays: int32(round((v - vmin) / resolution))
__device__ __forceinline__ float cell_f(const float v, const float vmin, const float res) {
  return rintf(__fdiv_rn(__fsub_rn(v, vmin), res));
}

constexpr int GI_THREADS = 256;

// one thread per (target point, structuring-element row)
__global__ void __launch_bounds__(GI_THREADS) costmap_stamp_kernel(const float *__restrict__ pts, const int n,
                                                                    const int *__restrict__ se_lo,
                                                                    const int *__restrict__ se_hi, const int hs,
                                                                    const sfe_costmap cm) {
  const int k = 2 * hs + 1;
  const long long gid = (long long)blockIdx.x * GI_THREADS + threadIdx.x;
  if (gid >= (long long)n * k) return;
  const int i = (int)(gid / k), j = (int)(gid % k);
  const float2 p = reinterpret_cast<const float2 *>(pts)[i];
  const float rf = cell_f(p.y, cm.ymin, cm.res), cf = cell_f(p.x, cm.xmin, cm.res);
  if (!(rf == rf) || !(cf == cf)) return;
  // np.clip(r, 0, rows - 1) on the int32 cast (slam.py:518-519)
  const int r = (int)fminf(fmaxf(rf, 0.f), (float)(cm.rows - 1));
  const int c = (int)fminf(fmaxf(cf, 0.f), (float)(cm.cols - 1));
  // dst(x, y) = max over SE offsets (dx, dy) of src(x + dx, y + dy): a lit source cell lights (c - dx, r - dy)
  const int lo = se_lo[j], hi = se_hi[j];
  if (lo >= hi) return;
  const int rr = r - (j - hs);
  if (rr < 0 || rr >= cm.rows) return;
  int c0 = c - (hi - 1 - hs), c1 = c - (lo - hs) + 1;  // [c0, c1)
  c0 = max(c0, 0), c1 = min(c1, cm.cols);
  if (c0 >= c1) return;
  uint32_t *row = cm.bits + (size_t)rr * cm.wpr;
  for (int w = c0 >> 5; w <= (c1 - 1) >> 5; ++w) {
    const int b0 = max(c0 - (w << 5), 0), b1 = min(c1 - (w << 5), 32);  // bits [b0, b1) of word w
    const uint32_t m = (b1 - b0 == 32) ? 0xffffffffu : (((1u << (b1 - b0)) - 1u) << b0);
    atomicOr(&row[w], m);
  }
}

__global__ void __launch_bounds__(GI_THREADS) costmap_expand_kernel(const sfe_costmap cm, uint8_t *__restrict__ out) {
  const long long gid = (long long)blockIdx.x * GI_THREADS + threadIdx.x;
  if (gid >= (long long)cm.rows * cm.cols) return;
  const int r = (int)(gid / cm.cols), c = (int)(gid % cm.cols);
  out[gid] = ((cm.bits[(size_t)r * cm.wpr + (c >> 5)] >> (c & 31)) & 1u) ? 255 : 0;
}

// W warps of a CTA share one candidate (W = 1, 2, 4 or 8; 8 / W candidates per CTA).  Every lane walks the
// source cloud with stride 32 * W: transform, round to the cell, test the bit.
template <int W>
__global__ void __launch_bounds__(GI_THREADS) costmap_score_kernel(const sfe_costmap cm, const float *__restrict__ src,
                                                                   const int n_src, const float *__restrict__ tf,
                                                                   const int n_cand, int32_t *__restrict__ cost) {
  constexpr int CPB = (GI_THREADS / 32) / W;  // candidates per CTA
  __shared__ int acc[CPB];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int slot = warp / W, part = warp % W;
  const int k = blockIdx.x * CPB + slot;
  if (tid < CPB) acc[tid] = 0;
  __syncthreads();
  if (k < n_cand) {
    const float r00 = tf[k * 6 + 0], r01 = tf[k * 6 + 1], r10 = tf[k * 6 + 2], r11 = tf[k * 6 + 3];
    const float tx = tf[k * 6 + 4], ty = tf[k * 6 + 5];
    const float rows_f = (float)cm.rows, cols_f = (float)cm.cols;
    int cnt = 0;
    for (int i = part * 32 + lane; i < n_src; i += 32 * W) {
      const float2 p = __ldg(reinterpret_cast<const float2 *>(src) + i);
      // Keyframe.transform_points (slam_objects.py:195-198): points.dot(R.T) + t in float32
      const float x = __fadd_rn(fmaf(p.y, r01, __fmul_rn(p.x, r00)), tx);
      const float y = __fadd_rn(fmaf(p.y, r11, __fmul_rn(p.x, r10)), ty);
      const float rf = cell_f(y, cm.ymin, cm.res), cf = cell_f(x, cm.xmin, cm.res);
      if (rf >= 0.f && rf < rows_f && cf >= 0.f && cf < cols_f) {  // `inside` (slam.py:558-563); NaN fails
        const int r = (int)rf, c = (int)cf;
        cnt += (__ldg(&cm.bits[(size_t)r * cm.wpr + (c >> 5)]) >> (c & 31)) & 1u;
      }
    }
    cnt = __reduce_add_sync(0xffffffffu, cnt);
    if (lane == 0) {
      if (W == 1)
        acc[slot] = cnt;
      else
        atomicAdd(&acc[slot], cnt);
    }
  }
  __syncthreads();
  if (tid < CPB && blockIdx.x * CPB + tid < n_cand) cost[blockIdx.x * CPB + tid] = -acc[tid];
}

int score_launch(sfe_ctx *ctx, cudaStream_t st, const sfe_costmap *cm, const float *src, int n_src, const float *tf,
                 int K, int32_t *cost) {
  // few candidates: spread each over more warps so that the launch still fills the machine
  const int sm = ctx->sm_count;
  int W = 1;
  while (W < 8 && (long long)K * W < 8LL * 4 * sm) W *= 2;
#define SFE_GI(W_) \
  costmap_score_kernel<W_><<<(K + (8 / W_) - 1) / (8 / W_), GI_THREADS, 0, st>>>(*cm, src, n_src, tf, K, cost)
  if (W == 1) SFE_GI(1); else if (W == 2) SFE_GI(2); else if (W == 4) SFE_GI(4); else SFE_GI(8);
#undef SFE_GI
  ctx->launches++;
  SFE_CUDA(cudaGetLastError());
  return SFE_OK;
}

}  // namespace

extern "C" {

int sfe_costmap_create(sfe_ctx *ctx, const float *target_xy_host, int n_target, float xmin, float ymin,
                       float resolution, int rows, int cols, int dilate_hs, const int32_t *se_lo,
                       const int32_t *se_hi, sfe_costmap **out) {
  SFE_REQUIRE(ctx && out, "sfe_costmap_create: null context / output");
  SFE_REQUIRE(n_target >= 0 && (target_xy_host || n_target == 0), "sfe_costmap_create: bad target cloud");
  SFE_REQUIRE(rows > 0 && cols > 0 && (long long)rows * cols <= (1LL << 31), "sfe_costmap_create: bad grid size %d x %d",
              rows, cols);
  SFE_REQUIRE(resolution > 0.f, "sfe_costmap_create: resolution must be positive");
  SFE_REQUIRE(dilate_hs >= 0 && dilate_hs <= 4096 && se_lo && se_hi, "sfe_costmap_create: bad structuring element");
  SFE_CUDA(cudaSetDevice(ctx->device));
  sfe_costmap *cm = new sfe_costmap();
  cm->device = ctx->device;
  cm->rows = rows, cm->cols = cols, cm->wpr = (cols + 31) / 32;
  cm->xmin = xmin, cm->ymin = ymin, cm->res = resolution;
  cm->bits = nullptr, cm->src = nullptr, cm->tf = nullptr, cm->cost = nullptr;
  cm->n_src = cm->src_cap = cm->tf_cap = 0;
  const size_t bytes = sizeof(uint32_t) * (size_t)rows * cm->wpr;
  const int k = 2 * dilate_hs + 1;
  float *d_pts = nullptr;
  int *d_se = nullptr;
  cudaError_t e = cudaMalloc(&cm->bits, bytes);
  if (e == cudaSuccess) e = cudaMemsetAsync(cm->bits, 0, bytes, ctx->stream);
  if (e == cudaSuccess && n_target > 0) {
    e = cudaMalloc(&d_pts, sizeof(float) * 2 * (size_t)n_target);
    if (e == cudaSuccess) e = cudaMalloc(&d_se, sizeof(int) * 2 * (size_t)k);
    if (e == cudaSuccess)
      e = cudaMemcpyAsync(d_pts, target_xy_host, sizeof(float) * 2 * (size_t)n_target, cudaMemcpyHostToDevice, ctx->stream);
    if (e == cudaSuccess) e = cudaMemcpyAsync(d_se, se_lo, sizeof(int) * k, cudaMemcpyHostToDevice, ctx->stream);
    if (e == cudaSuccess) e = cudaMemcpyAsync(d_se + k, se_hi, sizeof(int) * k, cudaMemcpyHostToDevice, ctx->stream);
    if (e == cudaSuccess) {
      const long long work = (long long)n_target * k;
      costmap_stamp_kernel<<<(unsigned)((work + GI_THREADS - 1) / GI_THREADS), GI_THREADS, 0, ctx->stream>>>(
          d_pts, n_target, d_se, d_se + k, dilate_hs, *cm);
      ctx->launches++;
      e = cudaGetLastError();
    }
  }
  if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);  // the host arrays may go away after return
  cudaFree(d_pts);
  cudaFree(d_se);
  if (e != cudaSuccess) {
    set_error("sfe_costmap_create: %s", cudaGetErrorString(e));
    cudaFree(cm->bits);
    delete cm;
    return SFE_ERR_CUDA;
  }
  *out = cm;
  return SFE_OK;
}

void sfe_costmap_destroy(sfe_costmap *cm) {
  if (!cm) return;
  cudaSetDevice(cm->device);
  cudaFree(cm->bits);
  cudaFree(cm->src);
  cudaFree(cm->tf);
  cudaFree(cm->cost);
  delete cm;
}

int sfe_costmap_grid_host(sfe_ctx *ctx, const sfe_costmap *cm, uint8_t *grid_host) {
  SFE_REQUIRE(ctx && cm && grid_host, "sfe_costmap_grid_host: null argument");
  SFE_CUDA(cudaSetDevice(ctx->device));
  const size_t n = (size_t)cm->rows * cm->cols;
  int rc = ensure(ctx, ctx->stage_out[0], n);
  if (rc != SFE_OK) return rc;
  uint8_t *d = (uint8_t *)ctx->stage_out[0].ptr;
  costmap_expand_kernel<<<(unsigned)((n + GI_THREADS - 1) / GI_THREADS), GI_THREADS, 0, ctx->stream>>>(*cm, d);
  ctx->launches++;
  SFE_CUDA(cudaGetLastError());
  SFE_CUDA(cudaMemcpyAsync(grid_host, d, n, cudaMemcpyDeviceToHost, ctx->stream));
  SFE_CUDA(cudaStreamSynchronize(ctx->stream));
  return SFE_OK;
}

int sfe_costmap_set_source_host(sfe_ctx *ctx, sfe_costmap *cm, const float *source_xy_host, int n_source) {
  SFE_REQUIRE(ctx && cm, "sfe_costmap_set_source_host: null argument");
  SFE_REQUIRE(n_source >= 0 && (source_xy_host || n_source == 0), "sfe_costmap_set_source_host: bad source cloud");
  SFE_CUDA(cudaSetDevice(ctx->device));
  if (n_source > cm->src_cap) {
    SFE_CUDA(cudaStreamSynchronize(ctx->stream));
    cudaFree(cm->src);
    cm->src = nullptr, cm->src_cap = 0;
    SFE_CUDA(cudaMalloc(&cm->src, sizeof(float) * 2 * (size_t)n_source));
    cm->src_cap = n_source;
  }
  cm->n_src = n_source;
  if (n_source > 0) {
    SFE_CUDA(cudaMemcpyAsync(cm->src, source_xy_host, sizeof(float) * 2 * (size_t)n_source, cudaMemcpyHostToDevice,
                             ctx->stream));
    SFE_CUDA(cudaStreamSynchronize(ctx->stream));
  }
  return SFE_OK;
}

int sfe_costmap_score_dev(sfe_ctx *ctx, const sfe_costmap *cm, const float *source_xy_dev, int n_source,
                          const float *transforms_dev, int n_candidates, int32_t *cost_dev) {
  SFE_REQUIRE(ctx && cm, "sfe_costmap_score_dev: null argument");
  SFE_REQUIRE(n_source >= 0 && n_candidates >= 0, "sfe_costmap_score_dev: negative count");
  if (n_candidates == 0) return SFE_OK;
  SFE_REQUIRE((source_xy_dev || n_source == 0) && transforms_dev && cost_dev, "sfe_costmap_score_dev: null pointer");
  SFE_CUDA(cudaSetDevice(ctx->device));
  return score_launch(ctx, ctx->stream, cm, source_xy_dev, n_source, transforms_dev, n_candidates, cost_dev);
}

int sfe_costmap_score_host(sfe_ctx *ctx, const sfe_costmap *cm_c, const float *transforms_host, int n_candidates,
                           int32_t *cost_host) {
  SFE_REQUIRE(ctx && cm_c, "sfe_costmap_score_host: null argument");
  SFE_REQUIRE(n_candidates >= 0, "sfe_costmap_score_host: negative count");
  if (n_candidates == 0) return SFE_OK;
  SFE_REQUIRE(transforms_host && cost_host, "sfe_costmap_score_host: null pointer");
  SFE_CUDA(cudaSetDevice(ctx->device));
  sfe_costmap *cm = const_cast<sfe_costmap *>(cm_c);  // staging buffers grow on demand
  if (n_candidates <= 64) {
    // A handful of poses (scipy.shgo asks for one at a time): no copies at all -- the kernel reads the transforms
    // from and writes the costs to pinned host memory, so one evaluation is a launch and a stream synchronise.
    const size_t tf_bytes = sizeof(float) * 6 * 64;
    int rc = ensure_pinned(ctx, tf_bytes + sizeof(int32_t) * 64);
    if (rc != SFE_OK) return rc;
    float *h_tf = (float *)ctx->pinned;
    int32_t *h_cost = (int32_t *)((char *)ctx->pinned + tf_bytes);
    memcpy(h_tf, transforms_host, sizeof(float) * 6 * (size_t)n_candidates);
    rc = score_launch(ctx, ctx->stream, cm, cm->src, cm->n_src, h_tf, n_candidates, h_cost);
    if (rc != SFE_OK) return rc;
    SFE_CUDA(cudaStreamSynchronize(ctx->stream));
    memcpy(cost_host, h_cost, sizeof(int32_t) * (size_t)n_candidates);
    return SFE_OK;
  }
  if (n_candidates > cm->tf_cap) {
    SFE_CUDA(cudaStreamSynchronize(ctx->stream));
    cudaFree(cm->tf);
    cudaFree(cm->cost);
    cm->tf = nullptr, cm->cost = nullptr, cm->tf_cap = 0;
    SFE_CUDA(cudaMalloc(&cm->tf, sizeof(float) * 6 * (size_t)n_candidates));
    SFE_CUDA(cudaMalloc(&cm->cost, sizeof(int32_t) * (size_t)n_candidates));
    cm->tf_cap = n_candidates;
  }
  SFE_CUDA(cudaMemcpyAsync(cm->tf, transforms_host, sizeof(float) * 6 * (size_t)n_candidates, cudaMemcpyHostToDevice,
                           ctx->stream));
  int rc = score_launch(ctx, ctx->stream, cm, cm->src, cm->n_src, cm->tf, n_candidates, cm->cost);
  if (rc != SFE_OK) return rc;
  SFE_CUDA(cudaMemcpyAsync(cost_host, cm->cost, sizeof(int32_t) * (size_t)n_candidates, cudaMemcpyDeviceToHost,
                           ctx->stream));
  SFE_CUDA(cudaStreamSynchronize(ctx->stream));
  return SFE_OK;
}

}  // extern "C"
