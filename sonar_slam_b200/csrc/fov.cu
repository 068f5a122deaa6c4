// Field-of-view pre-filter of loop-closure targets (SURVEY.md 8(f) row N3).
//
// SLAM.initialize_nonsequential_scan_matching, bruce_slam/src/bruce_slam/slam.py:878-899: the accumulated target
// cloud (global frame) is cut down to the points that at least one source keyframe could have seen, with the
// sensor's range and aperture inflated by five standard deviations of that keyframe's pose:
//     local  = Keyframe.transform_points(target_points, pose.inverse())          (float32, slam_objects.py:178-198)
//     ranges = np.linalg.norm(local, axis=1);  bearings = np.arctan2(local[:,1], local[:,0])      (float32)
//     sel   |= (ranges < range_bound) & (abs(bearings) < bearing_bound)          (bounds are float64 scalars)
// One thread per target point loops over the K source keyframes (K = nssm source_frames, a handful); the float32
// expressions are numpy's: the dot product as fma(y, r01, x * r00) + tx, the norm as sqrt(x*x + y*y) with the two
// products rounded separately, atan2 in float32; the comparisons promote to double like numpy does for a float64
// scalar bound.
#include "common.cuh"

namespace sfe {

__global__ void __launch_bounds__(256)
    fov_select_kernel(const float *__restrict__ pts, int n, const float *__restrict__ invT /* [K][6] */,
                      const double *__restrict__ range_bound, const double *__restrict__ bearing_bound, int K,
                      uint8_t *__restrict__ sel) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float x = pts[2 * (size_t)i], y = pts[2 * (size_t)i + 1];
  bool keep = false;
  for (int k = 0; k < K && !keep; ++k) {
    const float *T = invT + 6 * k;  // r00 r01 r10 r11 tx ty
    const float lx = __fadd_rn(__fmaf_rn(y, T[1], __fmul_rn(x, T[0])), T[4]);
    const float ly = __fadd_rn(__fmaf_rn(y, T[3], __fmul_rn(x, T[2])), T[5]);
    const float range = sqrtf(__fadd_rn(__fmul_rn(lx, lx), __fmul_rn(ly, ly)));
    const float bearing = atan2f(ly, lx);
    keep = ((double)range < range_bound[k]) && ((double)fabsf(bearing) < bearing_bound[k]);
  }
  sel[i] = keep ? 1 : 0;
}

static int fov_select_run(sfe_ctx *ctx, cudaStream_t st, const float *pts, int n, const float *invT, const double *rb,
                          const double *bb, int K, uint8_t *sel) {
  SFE_REQUIRE(ctx, "fov_select: null context");
  SFE_REQUIRE(n >= 0 && K >= 0, "fov_select: negative sizes");
  if (n == 0) return SFE_OK;
  SFE_REQUIRE(pts && sel && (K == 0 || (invT && rb && bb)), "fov_select: null pointer");
  fov_select_kernel<<<(n + 255) / 256, 256, 0, st>>>(pts, n, invT, rb, bb, K, sel);
  SFE_CUDA(cudaGetLastError());
  ctx->launches++;
  return SFE_OK;
}

}  // namespace sfe

using namespace sfe;

extern "C" {

int sfe_fov_select_dev(sfe_ctx *ctx, const float *pts_dev, int n, const float *inv_T_dev, const double *range_bound_dev,
                       const double *bearing_bound_dev, int n_frames, uint8_t *sel_dev) {
  SFE_REQUIRE(ctx != nullptr, "sfe_fov_select_dev: null context");
  SFE_CUDA(cudaSetDevice(ctx->device));
  return fov_select_run(ctx, ctx->stream, pts_dev, n, inv_T_dev, range_bound_dev, bearing_bound_dev, n_frames, sel_dev);
}

int sfe_fov_select_host(sfe_ctx *ctx, const float *pts_host, int n, const float *inv_T_host, const double *range_bound_host,
                        const double *bearing_bound_host, int n_frames, uint8_t *sel_host) {
  SFE_REQUIRE(ctx != nullptr, "sfe_fov_select_host: null context");
  SFE_REQUIRE(n >= 0 && n_frames >= 0, "sfe_fov_select_host: negative sizes");
  if (n == 0) return SFE_OK;
  SFE_REQUIRE(pts_host && sel_host && (n_frames == 0 || (inv_T_host && range_bound_host && bearing_bound_host)),
              "sfe_fov_select_host: null pointer");
  SFE_CUDA(cudaSetDevice(ctx->device));
  int rc;
  const size_t kb = (size_t)(n_frames > 0 ? n_frames : 1);
  if ((rc = ensure(ctx, ctx->stage_in[0], sizeof(float) * 2 * (size_t)n)) != SFE_OK) return rc;
  if ((rc = ensure(ctx, ctx->stage_in[1], kb * (6 * sizeof(float) + 2 * sizeof(double)) + 64)) != SFE_OK) return rc;
  if ((rc = ensure(ctx, ctx->stage_out[0], (size_t)n)) != SFE_OK) return rc;
  char *small = (char *)ctx->stage_in[1].ptr;  // [range_bound K doubles][bearing_bound K doubles][invT K*6 floats]
  double *rb = (double *)small, *bb = rb + kb;
  float *invT = (float *)(bb + kb);
  SFE_CUDA(cudaMemcpyAsync(ctx->stage_in[0].ptr, pts_host, sizeof(float) * 2 * (size_t)n, cudaMemcpyHostToDevice, ctx->stream));
  if (n_frames > 0) {
    SFE_CUDA(cudaMemcpyAsync(rb, range_bound_host, sizeof(double) * n_frames, cudaMemcpyHostToDevice, ctx->stream));
    SFE_CUDA(cudaMemcpyAsync(bb, bearing_bound_host, sizeof(double) * n_frames, cudaMemcpyHostToDevice, ctx->stream));
    SFE_CUDA(cudaMemcpyAsync(invT, inv_T_host, sizeof(float) * 6 * n_frames, cudaMemcpyHostToDevice, ctx->stream));
  }
  rc = fov_select_run(ctx, ctx->stream, (const float *)ctx->stage_in[0].ptr, n, invT, rb, bb, n_frames,
                      (uint8_t *)ctx->stage_out[0].ptr);
  if (rc != SFE_OK) return rc;
  SFE_CUDA(cudaMemcpyAsync(sel_host, ctx->stage_out[0].ptr, (size_t)n, cudaMemcpyDeviceToHost, ctx->stream));
  SFE_CUDA(cudaStreamSynchronize(ctx->stream));
  return SFE_OK;
}

}  // extern "C"
