// Batched per-keyframe front end: polar frames -> CFAR -> Cartesian cloud -> filters -> sequential
// scan matching against the window of previous frames, one C-ABI call per batch.
//
// This is the GPU form of what the reference does one message at a time in
// FeatureExtraction.callback (feature_extraction.py:196-252) followed, per keyframe, by
// SLAM.add_sequential_scan_matching (slam.py:718-837): source = the new frame's cloud, target =
// get_points(previous `window` frames, expressed in the previous frame) (slam.py:632-633,229-292:
// Keyframe.transform_points + pcl.downsample), guess = odometry between the two poses, then
// pcl.ICP.compute.  The pose-graph side (ISAM2) stays on the CPU and consumes the SE(2) results.
// Frames of one batch are independent given their odometry poses, which is what lets a backlog of
// keyframes be matched in parallel (and sharded over GPUs by the caller).
//
// Device layout: every per-frame cloud lives at a fixed stride (`cap_points` rows) with a count
// array, so all stages run without packing or host round trips; the host flavour overlaps the
// host->device copy of frame chunk k+1 with the kernels of chunk k on two streams.
#include <algorithm>
#include <cub/block/block_scan.cuh>
#include <functional>
#include <vector>

#include "stages.cuh"
#include "stream_decode.cuh"

namespace sfe {
// Small ICP size class of the front end (icp_run), from the problem sizes of bench.py's 4096-frame bag
// (tools/icp_sizes.py): sources after the filters mean 359, max 639 points; window submaps after the 0.5 m thinning
// (the ICP target) mean 406, max 779.  The class takes every frame of that bag: a second launch that holds only a
// few frames costs a full problem latency at its tail.  The source cap has no margin over the bag's largest source
// (639): above 5 points per thread (640 for 128 threads, icp.cu: ICP_SMALL_MULT) a problem leaves the one-pass path, so a
// larger cap would only admit problems that take the slower pruned path.  The target cap keeps 3 % over the bag's
// largest target (779): at 640 / 800 points a 128-thread CTA needs 27.4 KB of shared memory, which with the 1 KB the
// driver reserves per CTA lets an H100 SM (228 KB) hold 8 of them (810 is the largest target that does), and the
// class runs icp_kernel's 64-register instantiation (IcpClass::dense), so 8 problems are in flight per SM (7 at the
// former 640 / 896 class with 72 registers; DESIGN.md section 4).
constexpr int FE_ICP_SMALL_SRC = 640, FE_ICP_SMALL_TGT = 800;
// (the class is sized for 128-thread CTAs, which icp_run's CTA-size rule gives sources of up to 640 points)
static_assert(FE_ICP_SMALL_SRC <= 640, "the small ICP class must stay within icp_run's 128-thread CTAs");
// icp_run's class list (a problem takes the first class it fits; the capacity class takes the rest)
static const IcpClass FE_ICP_CLASSES[] = {{FE_ICP_SMALL_SRC, FE_ICP_SMALL_TGT, true}};
constexpr int FE_ICP_N_CLASSES = sizeof(FE_ICP_CLASSES) / sizeof(FE_ICP_CLASSES[0]);
// Size classes of the cloud filters (cloud.cu: two launches by cloud size).  Config-4 replay: 3-5 k raw Cartesian
// points per frame, ~580 after the voxel filter, ~400 after the outlier filter, window submaps <= 1.8 k raw points.
// The outlier filter and the submap down-sampling gain from a small-cloud class (chosen on the replay; not
// re-measured on H100).
constexpr int FE_RO_SPLIT = 1024, FE_SUBMAP_SPLIT = 2048;
// Frame class of the per-frame down-sampling (cloud.cu: downsample_frame_kernel), from the raw clouds of bench.py's
// 4096-frame bag (tools/ds_sizes.py): mean 3378, p99.9 5602, max 5647 points.  6144 leaves a 9 % margin over the
// largest; larger clouds take the capacity launch.  At 6144 points the frame kernel needs 97 KB of dynamic shared
// memory (16 bytes per point: the sorted points are staged there), so an H100 SM holds 2 of its 512-thread CTAs.
constexpr int FE_DS_FRAME = 6144;

// T_ab = pose_a^-1 * pose_b as float32 3x3 (gtsam Pose2::between, then matrix().astype(float32)).
// Evaluated on the host in double (libm), so the float32 matrices the kernels see are the ones a
// Python caller would compute.  Rotation as gtsam forms it: Rot2 holds (cos, sin) and between() multiplies
// r_a^-1 * r_b, i.e. c = ca*cb + sa*sb, s = ca*sb - sa*cb (not cos/sin of the angle difference; the two differ by
// ~1e-16, which matters only on a float32 rounding boundary); translation = r_a.unrotate(t_b - t_a).
static void pose_between(const double *a, const double *b, float *T) {
  const double ca = cos(a[2]), sa = sin(a[2]), cb = cos(b[2]), sb = sin(b[2]);
  const double dx = b[0] - a[0], dy = b[1] - a[1];
  const double x = ca * dx + sa * dy, y = -sa * dx + ca * dy;
  const double c = ca * cb + sa * sb, s = ca * sb - sa * cb;
  T[0] = (float)c, T[1] = (float)-s, T[2] = (float)x;
  T[3] = (float)s, T[4] = (float)c, T[5] = (float)y;
  T[6] = 0.f, T[7] = 0.f, T[8] = 1.f;
}

// A6: the keyframe cloud as SLAM holds it.  The feature node publishes xyz = [p0, 0, p1]
// (feature_extraction.py:182); SLAM reads np.c_[x, -z] = (p0, -p1) (slam_ros.py:169-170).  Negation is exact, so
// flipping the float32 cloud after the filters equals what the reference's float32 message round trip gives.
__global__ void flip_lateral_kernel(float *__restrict__ xy, const int32_t *__restrict__ cnt, int cap, int n) {
  const int f = blockIdx.x;
  if (f >= n) return;
  const int k = min(cnt[f], cap);
  float *p = xy + 2 * (size_t)f * cap;
  for (int i = threadIdx.x; i < k; i += blockDim.x) p[2 * i + 1] = -p[2 * i + 1];
}

// offsets helper: off[i] = i * stride
__global__ void fill_offsets_kernel(int32_t *off, int n, int stride) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i <= n) off[i] = i * stride;
}

// Packed clouds (sfe_frontend_set_clouds), step 1: the exclusive scan of the clouds' sizes of frames [f0, f0 + n),
// off[f + 1] = off[f] + min(cnt[f], cap), continuing from off[f0] (which an earlier chunk's scan wrote; f0 = 0 starts
// at 0).  One CTA: a call has at most max_frames frames, a few tiles.
constexpr int FE_SCAN_THREADS = 256;
__global__ void __launch_bounds__(FE_SCAN_THREADS)
    cloud_offsets_kernel(const int32_t *__restrict__ cnt, int cap, int f0, int n, int64_t *__restrict__ off) {
  using Scan = cub::BlockScan<int64_t, FE_SCAN_THREADS>;
  __shared__ typename Scan::TempStorage tmp;
  int64_t base = f0 == 0 ? 0 : off[f0];
  if (f0 == 0 && threadIdx.x == 0) off[0] = 0;
  for (int t0 = 0; t0 < n; t0 += FE_SCAN_THREADS) {
    const int i = t0 + threadIdx.x;
    int64_t incl, tile;
    Scan(tmp).InclusiveSum(i < n ? (int64_t)min(cnt[f0 + i], cap) : 0, incl, tile);
    if (i < n) off[f0 + 1 + i] = base + incl;
    base += tile;
    __syncthreads();  // tmp is reused by the next tile
  }
}

// Step 2: frame f's cloud (min(cnt[f], cap) points at its slot of `clouds`) to dst + 2 (off[f] - off[f0]), for the
// frames [f0, f0 + n), one CTA each; points at or past `limit` (numbered like off) are not written.
__global__ void __launch_bounds__(256)
    gather_clouds_kernel(const float *__restrict__ clouds, const int32_t *__restrict__ cnt, int cap,
                         const int64_t *__restrict__ off, int f0, int64_t limit, float *__restrict__ dst) {
  const int f = f0 + blockIdx.x;
  const int64_t o = off[f];
  const int m = 2 * (int)max((int64_t)0, min((int64_t)min(cnt[f], cap), limit - o));
  const float *src = clouds + 2 * (size_t)f * cap;
  float *out = dst + 2 * (o - off[f0]);
  for (int i = threadIdx.x; i < m; i += blockDim.x) out[i] = src[i];
}

// The scan match turned off (sfe_frontend_set_scan_match): the results icp_run gives a problem it skips, without
// the problem -- TOO_LARGE where the raw Cartesian cloud overflowed its cap, SKIPPED elsewhere.
__global__ void skip_match_kernel(const int32_t *__restrict__ raw_cnt, int cap, int n, float *__restrict__ T,
                                  int32_t *__restrict__ iters, int32_t *__restrict__ inliers,
                                  int32_t *__restrict__ status) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  for (int q = 0; q < 9; ++q) T[9 * (size_t)i + q] = (q % 4 == 0) ? 1.f : 0.f;
  iters[i] = 0, inliers[i] = 0;
  status[i] = raw_cnt[i] > cap ? SFE_ICP_TOO_LARGE : SFE_ICP_SKIPPED;
}

// Target assembly (slam.py:229-292 without the final downsample): for frame i gather the clouds of frames
// i-window .. i-1, each moved into frame (i-1)'s coordinates with Keyframe.transform_points
// (slam_objects.py:178-198: float32 points @ R^T + t), concatenated oldest first.  rel[i][w] is the
// float32 transform of window slot w (frame i-window+w), rel[i][window] the ICP guess.  One CTA per frame.
// Frames of the PREVIOUS call kept on the device (sfe_frontend_set_carry): `carry_n` clouds in carry_xy / carry_cnt
// precede frame 0 of this batch, so virtual frame u = carry_n + (batch index).
__global__ void __launch_bounds__(256)
    assemble_targets_kernel(const float *__restrict__ clouds, const int32_t *__restrict__ counts, int cap,
                            const float *__restrict__ rel, int f0, int F, int window, float *__restrict__ tgt,
                            int32_t *__restrict__ tgt_count, int tgt_cap, float *__restrict__ guess,
                            const float *__restrict__ carry_xy, const int32_t *__restrict__ carry_cnt, int carry_n) {
  const int i = f0 + blockIdx.x;  // frames [f0, F) of the batch
  if (i >= F) return;
  const float *myrel = rel + (size_t)i * (window + 1) * 9;
  if (threadIdx.x < 9) guess[9 * (size_t)i + threadIdx.x] = myrel[window * 9 + threadIdx.x];
  float *out = tgt + 2 * (size_t)i * tgt_cap;
  int base = 0;
  for (int w = 0; w < window; ++w) {
    const int u = i + carry_n - window + w;  // virtual index of the window frame
    if (u < 0) continue;
    const float *T = myrel + w * 9;
    const float t0 = T[0], t1 = T[1], t2 = T[2], t3 = T[3], t4 = T[4], t5 = T[5];
    const bool carried = u < carry_n;
    const int n = min(carried ? carry_cnt[u] : counts[u - carry_n], cap);
    const float *src = carried ? carry_xy + 2 * (size_t)u * cap : clouds + 2 * (size_t)(u - carry_n) * cap;
    for (int j = threadIdx.x; j < n && base + j < tgt_cap; j += blockDim.x) {
      const float x = src[2 * j], y = src[2 * j + 1];
      // numpy's float32 `points.dot(R.T) + t` (slam_objects.py:196): fma(y, r01, x * r00) + tx -- the same
      // convention as the costmap kernels (globalinit.cu), pinned against numpy in tests/test_oracle_globalinit.py
      out[2 * (base + j)] = __fadd_rn(__fmaf_rn(y, t1, __fmul_rn(x, t0)), t2);
      out[2 * (base + j) + 1] = __fadd_rn(__fmaf_rn(y, t4, __fmul_rn(x, t3)), t5);
    }
    base = min(base + n, tgt_cap);
  }
  if (threadIdx.x == 0) tgt_count[i] = base;
}

// A maximal run of consecutive frames of one geometry within a call: frames [f0, f0 + n) of geometry g.  Its polar
// frames lie at `frames`, packed at the geometry's natural stride R_g * B_g, and its bit planes likewise from the
// bit-plane slot of frame f0 on, so a run never needs more than its own n slots and the CFAR and Cartesian-point
// launchers serve it as they serve a batch of the creation geometry.  A call without per-frame geometry is one run of
// geometry 0, whose natural stride is the slot's.
struct GeoRun {
  int f0, n, g;
  const uint8_t *frames;
};

}  // namespace sfe

using namespace sfe;

struct sfe_frontend {
  sfe_ctx *ctx = nullptr;
  const sfe_maps *maps = nullptr;
  sfe_frontend_params p = {};
  int max_frames = 0;
  // geometries (sfe_frontend_add_geometry; geo[0] = maps), the runs of the current call, and for the compressed
  // flavours each frame's expected R x B
  const sfe_maps *geo[SFE_FE_MAX_GEOMETRIES] = {};
  int n_geo = 1;
  std::vector<GeoRun> runs;
  std::vector<int32_t> frame_shape;
  // device buffers (sized for max_frames)
  uint8_t *frames = nullptr;      // [max_frames][R][B]: the host flavours' frames, run_dev_geometry's packed runs
  uint32_t *bits = nullptr;       // [max_frames][R][wpr]
  int32_t *ij = nullptr;          // [max_frames][cap][2]
  float *xy_a = nullptr, *xy_b = nullptr;  // [max_frames][cap][2] ping-pong
  int32_t *idx = nullptr;         // [max_frames][cap]
  int32_t *cnt_a = nullptr, *cnt_b = nullptr, *cnt_c = nullptr;
  int32_t *off_pts = nullptr, *off_tgt = nullptr;
  float *tgt_a = nullptr, *tgt_b = nullptr;  // [max_frames][window*cap][2]
  int32_t *tgt_idx = nullptr, *tcnt_a = nullptr, *tcnt_b = nullptr;
  float *rel = nullptr;           // [max_frames][window+1][9] relative transforms (window slots, then the guess)
  float *rel_host[2] = {};        // pinned staging of the same, double-buffered (no stream sync per call)
  cudaEvent_t ev_rel[2] = {};
  int rel_turn = 0;
  float *guess = nullptr, *T = nullptr;
  int32_t *iters = nullptr, *inliers = nullptr, *status = nullptr;
  // continuation across calls: the last `window` clouds (+ host poses) of the previous call
  int carry_on = 0, carry_n = 0;
  float *carry_xy = nullptr;       // [window][cap][2]
  int32_t *carry_cnt = nullptr;    // [window]
  double *carry_poses = nullptr;   // host [window][3]
  cudaStream_t copy_stream = nullptr;
  cudaEvent_t ev_copy[2] = {}, ev_done = nullptr;
  // feature images (sfe_frontend_set_feature_images)
  uint8_t img_lut[256 * 3] = {};
  uint8_t *img_dst = nullptr;      // null: off
  int img_dst_host = 0;
  uint8_t *img_stage[2] = {};      // host flavours: a chunk's images [frames][rows][cols][3] each
  size_t img_stage_bytes = 0;
  cudaStream_t img_stream = nullptr;  // copies the images out, next to the frame copies of copy_stream
  cudaEvent_t ev_img_ready[2] = {}, ev_img_copied[2] = {};
  // packed clouds (sfe_frontend_set_clouds): the caller's destination and offsets; the device-side offsets and their
  // pinned copy of the host flavours, and the events that hand each chunk's clouds to copy_stream (allocated on first
  // use)
  float *cloud_dst = nullptr;      // null: off
  int64_t cloud_capacity = 0;
  int64_t *cloud_offsets = nullptr;
  int cloud_on_host = 0;
  int64_t *cloud_off = nullptr, *cloud_off_host = nullptr;  // [max_frames + 1]
  cudaEvent_t ev_cloud[2] = {};
  int scan_match = 1;  // sfe_frontend_set_scan_match
  sfe_icp_filters icp_filters = {};  // sfe_frontend_set_icp_filters
  bool has_icp_filters = false;
  sfe_icp_robust icp_robust = {};  // sfe_frontend_set_icp_robust
  bool has_icp_robust = false;
  StageTimer timer;  // optional per-stage timing, on ctx->stream
};

extern "C" {

void sfe_frontend_params_default(sfe_frontend_params *p) {
  if (!p) return;
  memset(p, 0, sizeof(*p));
  p->R = 512, p->B = 512;
  p->cfar_alg = SFE_CFAR_SOCA, p->train_hs = 20, p->guard_hs = 5, p->rank = 10;
  p->tau = 2.749063720096473;  // CFAR(40, 10, 0.1, 10).threshold_factor_SOCA
  p->gate_enable = 1, p->gate_threshold = 65.0;
  p->resolution = 0.5f;
  p->outlier_radius = 1.0, p->outlier_min_points = 5;
  p->window = 3;
  p->submap_resolution = 0.5f;
  p->min_points = 50;
  sfe_icp_params_default(&p->icp);
  p->cap_points = 8192;
  p->cap_source = 1024, p->cap_target = 3072;
  p->flip_lateral = 1;
}

#define FE_ALLOC(ptr, bytes)                                                        \
  do {                                                                              \
    cudaError_t e_ = cudaMalloc((void **)&(ptr), (bytes));                          \
    if (e_ != cudaSuccess) {                                                        \
      sfe::set_error("sfe_frontend_create: cudaMalloc(%zu) failed: %s", (size_t)(bytes), cudaGetErrorString(e_)); \
      sfe_frontend_destroy(fe);                                                     \
      return SFE_ERR_CUDA;                                                          \
    }                                                                               \
  } while (0)

int sfe_frontend_create(sfe_ctx *ctx, const sfe_maps *maps, const sfe_frontend_params *params, int max_frames,
                        sfe_frontend **out) {
  SFE_REQUIRE(ctx && maps && params && out, "sfe_frontend_create: null argument");
  *out = nullptr;
  SFE_REQUIRE(max_frames > 0, "sfe_frontend_create: max_frames must be positive");
  SFE_REQUIRE(params->R == maps->R && params->B == maps->B, "sfe_frontend_create: polar shape %dx%d differs from the maps' %dx%d",
              params->R, params->B, maps->R, maps->B);
  SFE_REQUIRE(params->cap_points > 0 && params->window >= 1 && params->window <= 16, "sfe_frontend_create: bad capacity/window");
  SFE_REQUIRE(params->cap_source > 0 && params->cap_target > 0 && params->cap_source <= 65535 && params->cap_target <= 65535,
              "sfe_frontend_create: cap_source / cap_target must be in [1, 65535]");
  SFE_CUDA(cudaSetDevice(ctx->device));
  sfe_frontend *fe = new sfe_frontend();
  fe->ctx = ctx, fe->maps = maps, fe->p = *params, fe->max_frames = max_frames;
  fe->geo[0] = maps;
  const size_t F = max_frames, cap = params->cap_points, tcap = (size_t)params->window * cap;
  const size_t wpr = (params->B + 31) / 32;
  FE_ALLOC(fe->frames, F * params->R * params->B);
  FE_ALLOC(fe->bits, F * params->R * wpr * 4);
  FE_ALLOC(fe->ij, F * cap * 2 * 4);
  FE_ALLOC(fe->xy_a, F * cap * 2 * 4);
  FE_ALLOC(fe->xy_b, F * cap * 2 * 4);
  FE_ALLOC(fe->idx, F * cap * 4);
  FE_ALLOC(fe->cnt_a, F * 4);
  FE_ALLOC(fe->cnt_b, F * 4);
  FE_ALLOC(fe->cnt_c, F * 4);
  FE_ALLOC(fe->off_pts, (F + 1) * 4);
  FE_ALLOC(fe->off_tgt, (F + 1) * 4);
  FE_ALLOC(fe->tgt_a, F * tcap * 2 * 4);
  FE_ALLOC(fe->tgt_b, F * tcap * 2 * 4);
  FE_ALLOC(fe->tgt_idx, F * tcap * 4);
  FE_ALLOC(fe->tcnt_a, F * 4);
  FE_ALLOC(fe->tcnt_b, F * 4);
  FE_ALLOC(fe->rel, F * (params->window + 1) * 9 * 4);
  for (int k = 0; k < 2; ++k)
    if (cudaMallocHost((void **)&fe->rel_host[k], F * (params->window + 1) * 9 * 4) != cudaSuccess ||
        cudaEventCreateWithFlags(&fe->ev_rel[k], cudaEventDisableTiming) != cudaSuccess) {
      sfe::set_error("sfe_frontend_create: pinned staging allocation failed");
      sfe_frontend_destroy(fe);
      return SFE_ERR_CUDA;
    }
  FE_ALLOC(fe->carry_xy, (size_t)params->window * cap * 2 * 4);
  FE_ALLOC(fe->carry_cnt, (size_t)params->window * 4);
  fe->carry_poses = new double[3 * (size_t)params->window]();
  FE_ALLOC(fe->guess, F * 9 * 4);
  FE_ALLOC(fe->T, F * 9 * 4);
  FE_ALLOC(fe->iters, F * 4);
  FE_ALLOC(fe->inliers, F * 4);
  FE_ALLOC(fe->status, F * 4);
  cudaError_t e = cudaStreamCreateWithFlags(&fe->copy_stream, cudaStreamNonBlocking);
  if (e == cudaSuccess) e = cudaEventCreateWithFlags(&fe->ev_copy[0], cudaEventDisableTiming);
  if (e == cudaSuccess) e = cudaEventCreateWithFlags(&fe->ev_copy[1], cudaEventDisableTiming);
  if (e == cudaSuccess) e = cudaEventCreateWithFlags(&fe->ev_done, cudaEventDisableTiming);
  if (e != cudaSuccess) {
    sfe::set_error("sfe_frontend_create: %s", cudaGetErrorString(e));
    sfe_frontend_destroy(fe);
    return SFE_ERR_CUDA;
  }
  fill_offsets_kernel<<<(max_frames + 256) / 256, 256, 0, ctx->stream>>>(fe->off_pts, max_frames, (int)cap);
  fill_offsets_kernel<<<(max_frames + 256) / 256, 256, 0, ctx->stream>>>(fe->off_tgt, max_frames, (int)tcap);
  SFE_CUDA(cudaGetLastError());
  ctx->launches += 2;
  *out = fe;
  return SFE_OK;
}

void sfe_frontend_destroy(sfe_frontend *fe) {
  if (!fe) return;
  cudaSetDevice(fe->ctx->device);
  cudaStreamSynchronize(fe->ctx->stream);
  void *bufs[] = {fe->frames, fe->bits, fe->ij, fe->xy_a, fe->xy_b, fe->idx, fe->cnt_a, fe->cnt_b, fe->cnt_c,
                  fe->off_pts, fe->off_tgt, fe->tgt_a, fe->tgt_b, fe->tgt_idx, fe->tcnt_a, fe->tcnt_b, fe->rel,
                  fe->guess, fe->T, fe->iters, fe->inliers, fe->status, fe->carry_xy, fe->carry_cnt, fe->cloud_off};
  for (void *b : bufs)
    if (b) cudaFree(b);
  delete[] fe->carry_poses;
  if (fe->cloud_off_host) cudaFreeHost(fe->cloud_off_host);
  for (cudaEvent_t ev : fe->ev_cloud)
    if (ev) cudaEventDestroy(ev);
  for (int k = 0; k < 2; ++k) {
    if (fe->rel_host[k]) cudaFreeHost(fe->rel_host[k]);
    if (fe->ev_rel[k]) cudaEventDestroy(fe->ev_rel[k]);
  }
  if (fe->copy_stream) cudaStreamDestroy(fe->copy_stream);
  for (auto &ev : fe->ev_copy)
    if (ev) cudaEventDestroy(ev);
  if (fe->ev_done) cudaEventDestroy(fe->ev_done);
  if (fe->img_stream) {
    cudaStreamSynchronize(fe->img_stream);
    cudaStreamDestroy(fe->img_stream);
  }
  for (int k = 0; k < 2; ++k) {
    if (fe->img_stage[k]) cudaFree(fe->img_stage[k]);
    if (fe->ev_img_ready[k]) cudaEventDestroy(fe->ev_img_ready[k]);
    if (fe->ev_img_copied[k]) cudaEventDestroy(fe->ev_img_copied[k]);
  }
  delete fe;
}

// Feature images of the host flavours, of geometry m (a call with images has one).  fe_images_begin checks the
// destination and sizes the staging buffers; fe_render_chunk renders frames [f0, f0 + n) (on the device by now, at
// `frames`) into staging buffer k & 1 and copies them out on img_stream; the render of chunk k waits for the copy-out of
// chunk k - 2, which used the same buffer.
static int fe_images_begin(sfe_frontend *fe, const sfe_maps *m, int n_frames, int chunk_frames, const char *what) {
  if (!fe->img_dst) return SFE_OK;
  SFE_REQUIRE(fe->img_dst_host, "%s: feature images are set to go to device memory; this flavour writes them to host "
              "memory (sfe_frontend_set_feature_images with dst_is_host != 0)", what);
  const size_t ib = (size_t)m->rows * m->cols * 3, want = (size_t)std::min(chunk_frames, n_frames) * ib;
  if (fe->img_stage_bytes >= want) return SFE_OK;
  if (!fe->img_stream) {
    SFE_CUDA(cudaStreamCreateWithFlags(&fe->img_stream, cudaStreamNonBlocking));
    for (int k = 0; k < 2; ++k) {
      SFE_CUDA(cudaEventCreateWithFlags(&fe->ev_img_ready[k], cudaEventDisableTiming));
      SFE_CUDA(cudaEventCreateWithFlags(&fe->ev_img_copied[k], cudaEventDisableTiming));
    }
  }
  SFE_CUDA(cudaStreamSynchronize(fe->ctx->stream));
  SFE_CUDA(cudaStreamSynchronize(fe->img_stream));
  fe->img_stage_bytes = 0;
  for (int k = 0; k < 2; ++k) {
    if (fe->img_stage[k]) SFE_CUDA(cudaFree(fe->img_stage[k]));
    fe->img_stage[k] = nullptr;
  }
  for (int k = 0; k < 2; ++k) SFE_CUDA(cudaMalloc((void **)&fe->img_stage[k], want));
  fe->img_stage_bytes = want;
  return SFE_OK;
}

static int fe_render_chunk(sfe_frontend *fe, const sfe_maps *m, const uint8_t *frames, int f0, int n, int k,
                           const char *what) {
  if (!fe->img_dst) return SFE_OK;
  sfe_ctx *ctx = fe->ctx;
  const size_t ib = (size_t)m->rows * m->cols * 3;
  uint8_t *stage = fe->img_stage[k & 1];
  SFE_CUDA(cudaStreamWaitEvent(ctx->stream, fe->ev_img_copied[k & 1], 0));
  int rc = feature_image_run(ctx, ctx->stream, m, frames, n, fe->img_lut, stage, what);
  if (rc != SFE_OK) return rc;
  SFE_CUDA(cudaEventRecord(fe->ev_img_ready[k & 1], ctx->stream));
  SFE_CUDA(cudaStreamWaitEvent(fe->img_stream, fe->ev_img_ready[k & 1], 0));
  SFE_CUDA(cudaMemcpyAsync(fe->img_dst + (size_t)f0 * ib, stage, (size_t)n * ib, cudaMemcpyDeviceToHost,
                           fe->img_stream));
  SFE_CUDA(cudaEventRecord(fe->ev_img_copied[k & 1], fe->img_stream));
  return SFE_OK;
}

// A host flavour returns only after the image and cloud copies it enqueued have landed, on every path.
struct CopiesDrained {
  const sfe_frontend *fe;
  ~CopiesDrained() {
    if (fe->img_dst && fe->img_stream) cudaStreamSynchronize(fe->img_stream);
    if (fe->cloud_dst) cudaStreamSynchronize(fe->copy_stream);
  }
};

// window transforms + guesses from the odometry poses (host, double), uploaded as float32.  With carried frames the
// pose sequence is (carried poses ++ this batch's poses): frame i of the batch is virtual frame v = carry_n + i, its
// reference is virtual frame v - 1 and its window the virtual frames v - window .. v - 1.
static int fe_upload_poses(sfe_frontend *fe, const double *poses, int n) {
  const int W = fe->p.window, C = fe->carry_n;
  const int turn = fe->rel_turn ^= 1;
  SFE_CUDA(cudaEventSynchronize(fe->ev_rel[turn]));  // the copy that last used this staging buffer (two calls ago)
  float *stage = fe->rel_host[turn];
  auto pose_of = [&](int v) { return v < C ? fe->carry_poses + 3 * (size_t)v : poses + 3 * (size_t)(v - C); };
  for (int i = 0; i < n; ++i) {
    float *r = stage + (size_t)i * (W + 1) * 9;
    const int v = C + i;
    for (int w = 0; w < W; ++w) {
      const int u = v - W + w;
      if (u >= 0 && v > 0)
        pose_between(pose_of(v - 1), pose_of(u), r + w * 9);
      else
        for (int q = 0; q < 9; ++q) r[w * 9 + q] = (q % 4 == 0) ? 1.f : 0.f;
    }
    if (v > 0)
      pose_between(pose_of(v - 1), pose_of(v), r + W * 9);
    else
      for (int q = 0; q < 9; ++q) r[W * 9 + q] = (q % 4 == 0) ? 1.f : 0.f;
  }
  SFE_CUDA(cudaMemcpyAsync(fe->rel, stage, sizeof(float) * 9 * (size_t)n * (W + 1), cudaMemcpyHostToDevice,
                           fe->ctx->stream));
  SFE_CUDA(cudaEventRecord(fe->ev_rel[turn], fe->ctx->stream));
  return SFE_OK;
}

// The runs of a call's frames (geometry: one id per frame, or null: every frame geometry 0), after checking every id;
// each run's `frames` is set by the caller.  Nothing touches the device.
static int fe_geometry_runs(sfe_frontend *fe, const int32_t *geometry, int n, const char *what) {
  fe->runs.clear();
  for (int i = 0; i < n; ++i) {
    const int g = geometry ? geometry[i] : 0;
    SFE_REQUIRE(g >= 0 && g < fe->n_geo, "%s: frame %d has geometry id %d; this front end has geometries 0 .. %d "
                "(sfe_frontend_add_geometry)", what, i, g, fe->n_geo - 1);
    if (!fe->runs.empty() && fe->runs.back().g == g)
      fe->runs.back().n++;
    else
      fe->runs.push_back({i, 1, g, nullptr});
  }
  SFE_REQUIRE(!fe->img_dst || fe->runs.size() <= 1, "%s: feature images are set, but the frames of this call have "
              "more than one geometry (%d runs), whose images differ in size; run each geometry's frames in calls of "
              "their own or turn the images off", what, (int)fe->runs.size());
  return SFE_OK;
}

static size_t fe_geo_bytes(const sfe_frontend *fe, int g) { return (size_t)fe->geo[g]->R * fe->geo[g]->B; }

// polar frame i of run r
static const uint8_t *fe_run_frame(const sfe_frontend *fe, const GeoRun &r, int i) {
  return r.frames + (size_t)(i - r.f0) * fe_geo_bytes(fe, r.g);
}

// the place of frame i of run r in the front end's frame buffer (where the host flavours copy or decode it)
static uint8_t *fe_slot_frame(const sfe_frontend *fe, const GeoRun &r, int i) {
  return fe->frames + (size_t)r.f0 * fe->p.R * fe->p.B + (size_t)(i - r.f0) * fe_geo_bytes(fe, r.g);
}

// fn(run, a, m) for the frames [a, a + m) of every run inside frames [f0, f0 + n), in frame order
static int fe_for_pieces(const sfe_frontend *fe, int f0, int n,
                         const std::function<int(const GeoRun &, int, int)> &fn) {
  auto r = std::partition_point(fe->runs.begin(), fe->runs.end(), [&](const GeoRun &q) { return q.f0 + q.n <= f0; });
  for (; r != fe->runs.end() && r->f0 < f0 + n; ++r) {
    const int a = std::max(r->f0, f0), b = std::min(r->f0 + r->n, f0 + n);
    const int rc = fn(*r, a, b - a);
    if (rc != SFE_OK) return rc;
  }
  return SFE_OK;
}

static const float *fe_cloud(const sfe_frontend *fe, const int32_t **cnt);

// stages 1-2 on frames [f0, f0+n) of run r: CFAR (bit plane) -> Cartesian points, with the run's geometry
static int fe_polar(sfe_frontend *fe, const GeoRun &r, int f0, int n) {
  sfe_ctx *ctx = fe->ctx;
  cudaStream_t st = ctx->stream;
  const sfe_frontend_params &p = fe->p;
  const sfe_maps *m = fe->geo[r.g];
  const size_t cap = p.cap_points, wpr = (m->B + 31) / 32;
  uint32_t *bits = fe->bits + (size_t)r.f0 * p.R * ((p.B + 31) / 32) + (size_t)(f0 - r.f0) * m->R * wpr;
  fe->timer.tic(st, SFE_FE_CFAR);
  int rc = cfar_run(ctx, st, fe_run_frame(fe, r, f0), SFE_U8, n, m->R, m->B, p.cfar_alg, p.train_hs, p.guard_hs, p.rank,
                    p.tau, p.gate_enable, p.gate_threshold, nullptr, nullptr, bits);
  fe->timer.toc(st);
  if (rc != SFE_OK) return rc;
  fe->timer.tic(st, SFE_FE_CART);
  rc = cart_points_run(ctx, st, m, nullptr, bits, n, (int)cap, fe->ij + (size_t)f0 * cap * 2,
                       fe->xy_a + (size_t)f0 * cap * 2, fe->cnt_a + f0);
  fe->timer.toc(st);
  return rc;
}

// stages 1-3 on frames [f0, f0+n): CFAR (bit plane) -> Cartesian points once per run of one geometry, then
// downsample -> outlier removal over all n frames.
// Final per-frame clouds end in xy_a / cnt_c (or wherever the last enabled filter wrote; see cloud()).
static int fe_features(sfe_frontend *fe, int f0, int n) {
  sfe_ctx *ctx = fe->ctx;
  cudaStream_t st = ctx->stream;
  const sfe_frontend_params &p = fe->p;
  const size_t cap = p.cap_points;
  int rc = fe_for_pieces(fe, f0, n, [&](const GeoRun &r, int a, int m) { return fe_polar(fe, r, a, m); });
  if (rc != SFE_OK) return rc;
  // feature_extraction.py:241-249
  const float *cur = fe->xy_a;
  const int32_t *cur_cnt = fe->cnt_a;
  if (p.resolution > 0.f) {
    fe->timer.tic(st, SFE_FE_DOWNSAMPLE);
    rc = downsample_run(ctx, st, {cur, fe->off_pts + f0, cur_cnt + f0, (int)cap}, n, 2, p.resolution, fe->xy_b, fe->idx,
                        fe->cnt_b + f0, FE_DS_FRAME, SCR_CLOUD, WORK_DS);
    fe->timer.toc(st);
    if (rc != SFE_OK) return rc;
    cur = fe->xy_b, cur_cnt = fe->cnt_b;
  }
  if (p.outlier_min_points > 1) {
    float *dst = (cur == fe->xy_a) ? fe->xy_b : fe->xy_a;
    fe->timer.tic(st, SFE_FE_OUTLIER);
    rc = remove_outlier_run(ctx, st, {cur, fe->off_pts + f0, cur_cnt + f0, (int)cap}, n, 2, p.outlier_radius,
                            p.outlier_min_points, dst, fe->idx, fe->cnt_c + f0, FE_RO_SPLIT);
    fe->timer.toc(st);
    if (rc != SFE_OK) return rc;
  }
  if (p.flip_lateral) {
    const int32_t *cnt;
    float *cloud = const_cast<float *>(fe_cloud(fe, &cnt));
    fe->timer.tic(st, SFE_FE_OUTLIER);
    flip_lateral_kernel<<<n, 128, 0, st>>>(cloud + 2 * (size_t)f0 * cap, cnt + f0, (int)cap, n);
    fe->timer.toc(st);
    SFE_CUDA(cudaGetLastError());
    ctx->launches++;
  }
  return SFE_OK;
}

static const float *fe_cloud(const sfe_frontend *fe, const int32_t **cnt) {
  const sfe_frontend_params &p = fe->p;
  const bool ds = p.resolution > 0.f, ro = p.outlier_min_points > 1;
  if (ro) {
    *cnt = fe->cnt_c;
    return ds ? fe->xy_a : fe->xy_b;
  }
  if (ds) {
    *cnt = fe->cnt_b;
    return fe->xy_b;
  }
  *cnt = fe->cnt_a;
  return fe->xy_a;
}

// stage 4-5 on frames [f0, f0+n): targets from the window of previous frames (which may precede f0), then ICP
static int fe_match(sfe_frontend *fe, int f0, int n) {
  sfe_ctx *ctx = fe->ctx;
  cudaStream_t st = ctx->stream;
  const sfe_frontend_params &p = fe->p;
  const int cap = p.cap_points, tcap = p.window * cap;
  if (!fe->scan_match) {
    skip_match_kernel<<<(n + 255) / 256, 256, 0, st>>>(fe->cnt_a + f0, cap, n, fe->T + 9 * (size_t)f0, fe->iters + f0,
                                                       fe->inliers + f0, fe->status + f0);
    SFE_CUDA(cudaGetLastError());
    ctx->launches++;
    return SFE_OK;
  }
  const int32_t *cnt;
  const float *cloud = fe_cloud(fe, &cnt);
  fe->timer.tic(st, SFE_FE_SUBMAP);
  assemble_targets_kernel<<<n, 256, 0, st>>>(cloud, cnt, cap, fe->rel, f0, f0 + n, p.window, fe->tgt_a, fe->tcnt_a,
                                             tcap, fe->guess, fe->carry_xy, fe->carry_cnt, fe->carry_n);
  SFE_CUDA(cudaGetLastError());
  ctx->launches++;
  const float *tgt = fe->tgt_a;
  const int32_t *tcnt = fe->tcnt_a;
  if (p.submap_resolution > 0.f) {
    int rc = downsample_run(ctx, st, {fe->tgt_a, fe->off_tgt + f0, fe->tcnt_a + f0, tcap}, n, 2, p.submap_resolution,
                            fe->tgt_b, fe->tgt_idx, fe->tcnt_b + f0, FE_SUBMAP_SPLIT, SCR_CLOUD, WORK_DS);
    if (rc != SFE_OK) return rc;
    tgt = fe->tgt_b, tcnt = fe->tcnt_b;
  }
  fe->timer.toc(st);
  fe->timer.tic(st, SFE_FE_ICP);
  IcpProblems pb{};
  pb.src = {cloud, fe->off_pts + f0, cnt + f0, p.cap_source};
  pb.tgt = {tgt, fe->off_tgt + f0, tcnt + f0, p.cap_target};
  pb.P = n, pb.min_points = p.min_points;
  pb.raw_cnt = fe->cnt_a + f0, pb.raw_cap = cap;  // the source's Cartesian points before the filters
  pb.guess = fe->guess + 9 * (size_t)f0, pb.T_out = fe->T + 9 * (size_t)f0;
  pb.iters = fe->iters + f0, pb.inliers = fe->inliers + f0, pb.status = fe->status + f0;
  const int rc = icp_run(ctx, st, &p.icp, pb, FE_ICP_CLASSES, FE_ICP_N_CLASSES, nullptr,
                         fe->has_icp_filters ? &fe->icp_filters : nullptr,
                         fe->has_icp_robust ? &fe->icp_robust : nullptr);
  fe->timer.toc(st);
  return rc;
}

// After a batch: the carried window becomes the last `window` frames of (carried ++ batch), stream-ordered after
// the batch's matching (which still reads the old carried clouds).  Slots move towards the front, in ascending
// order, so no frame is overwritten before it has been moved.
static int fe_update_carry(sfe_frontend *fe, cudaStream_t st, const double *poses, int n) {
  if (!fe->carry_on) return SFE_OK;
  const int W = fe->p.window, C = fe->carry_n, total = C + n, keep = total < W ? total : W;
  const size_t cap = fe->p.cap_points, cbytes = cap * 2 * sizeof(float);
  const int32_t *cnt;
  const float *cloud = fe_cloud(fe, &cnt);
  for (int j = 0; j < keep; ++j) {
    const int v = total - keep + j;
    if (v < C) {
      if (v != j) {
        SFE_CUDA(cudaMemcpyAsync(fe->carry_xy + (size_t)j * cap * 2, fe->carry_xy + (size_t)v * cap * 2, cbytes,
                                 cudaMemcpyDeviceToDevice, st));
        SFE_CUDA(cudaMemcpyAsync(fe->carry_cnt + j, fe->carry_cnt + v, 4, cudaMemcpyDeviceToDevice, st));
        memcpy(fe->carry_poses + 3 * (size_t)j, fe->carry_poses + 3 * (size_t)v, 3 * sizeof(double));
      }
    } else {
      const size_t b = (size_t)(v - C);
      SFE_CUDA(cudaMemcpyAsync(fe->carry_xy + (size_t)j * cap * 2, cloud + b * cap * 2, cbytes, cudaMemcpyDeviceToDevice,
                               st));
      SFE_CUDA(cudaMemcpyAsync(fe->carry_cnt + j, cnt + b, 4, cudaMemcpyDeviceToDevice, st));
      memcpy(fe->carry_poses + 3 * (size_t)j, poses + 3 * b, 3 * sizeof(double));
    }
  }
  fe->carry_n = keep;
  return SFE_OK;
}

// Packed clouds of the host flavours (sfe_frontend_set_clouds).  fe_clouds_chunk packs the clouds of chunk k = frames
// [f0, f0 + n), once its filters ran, into that chunk's own slots of the filter buffer that does not hold the final
// clouds (fe_cloud_stage: its content there is dead by then, and nothing writes those slots again before the call
// returns), and copies the chunk's offsets into the pinned copy.  fe_clouds_out waits for both, then copies the points
// that fit the capacity to the caller on copy_stream, next to the kernels of the chunks after it.
struct CloudChunk {
  int f0 = 0, n = 0, k = 0;
};

static float *fe_cloud_stage(sfe_frontend *fe) {
  const int32_t *cnt;
  return fe_cloud(fe, &cnt) == fe->xy_a ? fe->xy_b : fe->xy_a;
}

static int fe_clouds_chunk(sfe_frontend *fe, int f0, int n, int k) {
  if (!fe->cloud_dst) return SFE_OK;
  sfe_ctx *ctx = fe->ctx;
  const int cap = fe->p.cap_points;
  const int32_t *cnt;
  const float *cloud = fe_cloud(fe, &cnt);
  cloud_offsets_kernel<<<1, FE_SCAN_THREADS, 0, ctx->stream>>>(cnt, cap, f0, n, fe->cloud_off);
  gather_clouds_kernel<<<n, 256, 0, ctx->stream>>>(cloud, cnt, cap, fe->cloud_off, f0, INT64_MAX,
                                                   fe_cloud_stage(fe) + 2 * (size_t)f0 * cap);
  SFE_CUDA(cudaGetLastError());
  ctx->launches += 2;
  SFE_CUDA(cudaMemcpyAsync(fe->cloud_off_host + f0, fe->cloud_off + f0, sizeof(int64_t) * (n + 1),
                           cudaMemcpyDeviceToHost, ctx->stream));
  SFE_CUDA(cudaEventRecord(fe->ev_cloud[k & 1], ctx->stream));
  return SFE_OK;
}

static int fe_clouds_out(sfe_frontend *fe, const CloudChunk &c) {
  if (!fe->cloud_dst || c.n == 0) return SFE_OK;
  SFE_CUDA(cudaEventSynchronize(fe->ev_cloud[c.k & 1]));
  const int64_t a = fe->cloud_off_host[c.f0], b = std::min(fe->cloud_off_host[c.f0 + c.n], fe->cloud_capacity);
  if (b > a)
    SFE_CUDA(cudaMemcpyAsync(fe->cloud_dst + 2 * a, fe_cloud_stage(fe) + 2 * (size_t)c.f0 * fe->p.cap_points,
                             2 * sizeof(float) * (b - a), cudaMemcpyDeviceToHost, fe->copy_stream));
  return SFE_OK;
}

static int fe_clouds_check(const sfe_frontend *fe, int64_t total, const char *what) {
  if (total <= fe->cloud_capacity) return SFE_OK;
  set_error("%s: the clouds of this call need %lld points; the destination holds %lld (sfe_frontend_set_clouds)", what,
            (long long)total, (long long)fe->cloud_capacity);
  return SFE_ERR_CAPACITY;
}

// the end of a host flavour's clouds: every copy has landed, the offsets go to the caller, the capacity is checked
static int fe_clouds_finish(sfe_frontend *fe, int n_frames, const char *what) {
  if (!fe->cloud_dst) return SFE_OK;
  SFE_CUDA(cudaStreamSynchronize(fe->copy_stream));
  memcpy(fe->cloud_offsets, fe->cloud_off_host, sizeof(int64_t) * (n_frames + 1));
  return fe_clouds_check(fe, fe->cloud_off_host[n_frames], what);
}

// run_dev's clouds: one scan and one gather over the call's frames straight into the caller's device buffers, then
// the wait for the total
static int fe_clouds_dev(sfe_frontend *fe, int n_frames, const char *what) {
  if (!fe->cloud_dst) return SFE_OK;
  sfe_ctx *ctx = fe->ctx;
  const int cap = fe->p.cap_points;
  const int32_t *cnt;
  const float *cloud = fe_cloud(fe, &cnt);
  cloud_offsets_kernel<<<1, FE_SCAN_THREADS, 0, ctx->stream>>>(cnt, cap, 0, n_frames, fe->cloud_offsets);
  gather_clouds_kernel<<<n_frames, 256, 0, ctx->stream>>>(cloud, cnt, cap, fe->cloud_offsets, 0, fe->cloud_capacity,
                                                          fe->cloud_dst);
  SFE_CUDA(cudaGetLastError());
  ctx->launches += 2;
  SFE_CUDA(cudaMemcpyAsync(fe->cloud_off_host, fe->cloud_offsets + n_frames, sizeof(int64_t), cudaMemcpyDeviceToHost,
                           ctx->stream));
  SFE_CUDA(cudaStreamSynchronize(ctx->stream));
  return fe_clouds_check(fe, fe->cloud_off_host[0], what);
}

// the destination kind a flavour writes to, checked before any device work
static int fe_clouds_args(const sfe_frontend *fe, bool host_flavour, const char *what) {
  SFE_REQUIRE(!fe->cloud_dst || (fe->cloud_on_host != 0) == host_flavour, "%s: clouds are set to go to %s memory; "
              "this flavour writes them to %s memory (sfe_frontend_set_clouds with on_host %s)", what,
              fe->cloud_on_host ? "host" : "device", host_flavour ? "host" : "device", host_flavour ? "!= 0" : "= 0");
  return SFE_OK;
}

int sfe_frontend_set_carry(sfe_frontend *fe, int enable) {
  SFE_REQUIRE(fe != nullptr, "sfe_frontend_set_carry: null handle");
  fe->carry_on = enable != 0;
  if (!fe->carry_on) fe->carry_n = 0;
  return SFE_OK;
}

int sfe_frontend_add_geometry(sfe_frontend *fe, const sfe_maps *maps, int *geometry_id) {
  SFE_REQUIRE(fe && maps && geometry_id, "sfe_frontend_add_geometry: null argument");
  SFE_REQUIRE(fe->n_geo < SFE_FE_MAX_GEOMETRIES, "sfe_frontend_add_geometry: the front end already has %d geometries, "
              "the most it takes (SFE_FE_MAX_GEOMETRIES)", fe->n_geo);
  SFE_REQUIRE(maps->R <= fe->p.R && maps->B <= fe->p.B, "sfe_frontend_add_geometry: polar shape %dx%d does not fit "
              "the front end's %dx%d frame slots (create it with the largest R and B the geometries need)", maps->R,
              maps->B, fe->p.R, fe->p.B);
  SFE_REQUIRE(maps->device == fe->ctx->device, "sfe_frontend_add_geometry: the maps live on device %d, the front end "
              "on device %d", maps->device, fe->ctx->device);
  fe->geo[fe->n_geo] = maps;
  *geometry_id = fe->n_geo++;
  return SFE_OK;
}

int sfe_frontend_set_feature_images(sfe_frontend *fe, const uint8_t *lut_bgr_host, uint8_t *dst, int dst_is_host) {
  SFE_REQUIRE(fe != nullptr, "sfe_frontend_set_feature_images: null handle");
  SFE_REQUIRE(dst == nullptr || lut_bgr_host != nullptr, "sfe_frontend_set_feature_images: null colour table");
  if (dst) memcpy(fe->img_lut, lut_bgr_host, sizeof(fe->img_lut));
  fe->img_dst = dst;
  fe->img_dst_host = dst_is_host != 0;
  return SFE_OK;
}

int sfe_frontend_set_clouds(sfe_frontend *fe, float *dst, int64_t capacity_points, int64_t *offsets, int on_host) {
  SFE_REQUIRE(fe != nullptr, "sfe_frontend_set_clouds: null handle");
  if (dst) {
    SFE_REQUIRE(offsets != nullptr, "sfe_frontend_set_clouds: null offsets");
    SFE_REQUIRE(capacity_points >= 0, "sfe_frontend_set_clouds: negative capacity %lld", (long long)capacity_points);
    SFE_CUDA(cudaSetDevice(fe->ctx->device));
    const size_t bytes = sizeof(int64_t) * (fe->max_frames + 1);
    if (!fe->cloud_off) SFE_CUDA(cudaMalloc((void **)&fe->cloud_off, bytes));
    if (!fe->cloud_off_host) SFE_CUDA(cudaMallocHost((void **)&fe->cloud_off_host, bytes));
    for (cudaEvent_t &ev : fe->ev_cloud)
      if (!ev) SFE_CUDA(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
  }
  fe->cloud_dst = dst;
  fe->cloud_capacity = capacity_points;
  fe->cloud_offsets = offsets;
  fe->cloud_on_host = on_host != 0;
  return SFE_OK;
}

int sfe_frontend_set_scan_match(sfe_frontend *fe, int enable) {
  SFE_REQUIRE(fe != nullptr, "sfe_frontend_set_scan_match: null handle");
  fe->scan_match = enable != 0;
  return SFE_OK;
}

int sfe_frontend_set_icp_filters(sfe_frontend *fe, const sfe_icp_filters *filters) {
  SFE_REQUIRE(fe != nullptr, "sfe_frontend_set_icp_filters: null handle");
  if (filters) {
    const int rc = icp_filters_check(filters, "sfe_frontend_set_icp_filters");
    if (rc != SFE_OK) return rc;
    fe->icp_filters = *filters;
  }
  fe->has_icp_filters = filters != nullptr;
  return SFE_OK;
}

int sfe_frontend_set_icp_robust(sfe_frontend *fe, const sfe_icp_robust *robust) {
  SFE_REQUIRE(fe != nullptr, "sfe_frontend_set_icp_robust: null handle");
  if (robust) {
    const int rc = icp_robust_check(robust, "sfe_frontend_set_icp_robust");
    if (rc != SFE_OK) return rc;
    fe->icp_robust = *robust;
  }
  fe->has_icp_robust = robust != nullptr;
  return SFE_OK;
}

int sfe_frontend_set_timing(sfe_frontend *fe, int enable) {
  SFE_REQUIRE(fe != nullptr, "sfe_frontend_set_timing: null handle");
  fe->timer.reset(enable != 0);
  return SFE_OK;
}

int sfe_frontend_get_timing(sfe_frontend *fe, double *stage_ms, int64_t *stage_calls) {
  SFE_REQUIRE(fe && stage_ms, "sfe_frontend_get_timing: null argument");
  SFE_CUDA(cudaSetDevice(fe->ctx->device));
  return fe->timer.collect(fe->ctx->stream, SFE_FE_STAGES, stage_ms, stage_calls);
}

}  // extern "C"

// `after` waits for what has been enqueued on `before` so far
static int fe_order(cudaStream_t before, cudaEvent_t ev, cudaStream_t after) {
  SFE_CUDA(cudaEventRecord(ev, before));
  SFE_CUDA(cudaStreamWaitEvent(after, ev, 0));
  return SFE_OK;
}

// feature images of chunk [f0, f0 + n) of a host flavour (the call has one run when images are on)
static int fe_render_host_chunk(sfe_frontend *fe, int f0, int n, int k, const char *what) {
  if (!fe->img_dst) return SFE_OK;
  const GeoRun &r = fe->runs[0];
  return fe_render_chunk(fe, fe->geo[r.g], fe_run_frame(fe, r, f0), f0, n, k, what);
}

// What a host flavour's call returns in host memory (npoints may be null)
struct HostResults {
  float *T;
  int32_t *iters, *inliers, *status, *npoints;
};

// The end of a host flavour: the last chunk's clouds go out (a call whose clouds overflow stops here, its carried window
// as it was), the carried window moves on, the results go to the host and the call waits for them.
static int fe_host_finish(sfe_frontend *fe, const CloudChunk &last, const double *poses_host, int n_frames,
                          const HostResults &out, const char *what) {
  sfe_ctx *ctx = fe->ctx;
  int rc = fe_clouds_out(fe, last);
  if (rc == SFE_OK) rc = fe_clouds_finish(fe, n_frames, what);
  if (rc == SFE_OK) rc = fe_update_carry(fe, ctx->stream, poses_host, n_frames);
  if (rc != SFE_OK) return rc;
  SFE_CUDA(cudaMemcpyAsync(out.T, fe->T, sizeof(float) * 9 * (size_t)n_frames, cudaMemcpyDeviceToHost, ctx->stream));
  SFE_CUDA(cudaMemcpyAsync(out.iters, fe->iters, 4 * (size_t)n_frames, cudaMemcpyDeviceToHost, ctx->stream));
  SFE_CUDA(cudaMemcpyAsync(out.inliers, fe->inliers, 4 * (size_t)n_frames, cudaMemcpyDeviceToHost, ctx->stream));
  SFE_CUDA(cudaMemcpyAsync(out.status, fe->status, 4 * (size_t)n_frames, cudaMemcpyDeviceToHost, ctx->stream));
  if (out.npoints) {
    const int32_t *cnt;
    fe_cloud(fe, &cnt);
    SFE_CUDA(cudaMemcpyAsync(out.npoints, cnt, 4 * (size_t)n_frames, cudaMemcpyDeviceToHost, ctx->stream));
  }
  SFE_CUDA(cudaStreamSynchronize(ctx->stream));
  return SFE_OK;
}

// The checks every host flavour makes first, before its own and before any device work: null arguments (inputs_ok:
// those of the flavour's frame inputs), the frame count, the clouds' destination and the geometry runs.
static int fe_host_args(sfe_frontend *fe, bool inputs_ok, const int32_t *geometry, const double *poses_host,
                        int n_frames, const HostResults &out, const char *what) {
  SFE_REQUIRE(fe && inputs_ok && poses_host && out.T && out.iters && out.inliers && out.status, "%s: null argument",
              what);
  SFE_REQUIRE(n_frames >= 0 && n_frames <= fe->max_frames, "%s: %d frames exceed max_frames %d", what, n_frames,
              fe->max_frames);
  int rc = fe_clouds_args(fe, true, what);
  if (rc == SFE_OK) rc = fe_geometry_runs(fe, geometry, n_frames, what);
  return rc;
}

// How a host flavour's frames get into their slots of fe->frames.  begin(chunk_frames) runs once the call has its
// device, chunk size and image staging, before the pose upload: the flavour's last checks and its set-up.
// stage(f0, n, k), if set, enqueues chunk k = frames [f0, f0 + n) into its slots one chunk ahead; ready(f0, n, k)
// makes chunk k usable on ctx->stream.
struct HostFrames {
  std::function<int(int)> begin;
  std::function<int(int, int, int)> stage, ready;
};

// The chunk loop of every host flavour.  A flavour that stages ahead has chunk k+1 staged before chunk k is waited for,
// so its decode runs next to the kernels of chunk k.  Once chunk k is ready its feature images, feature stages, clouds
// and scan match are enqueued (its window reaches back only into chunks already processed), and the clouds of chunk
// k-1 go out.
static int fe_run_host(sfe_frontend *fe, const HostFrames &in, const double *poses_host, int n_frames,
                       int chunk_frames, const HostResults &out, const char *what) {
  if (n_frames == 0) return SFE_OK;
  // the device, the default chunk size, every run's place in fe->frames, the feature-image staging (of the call's one
  // geometry)
  SFE_CUDA(cudaSetDevice(fe->ctx->device));
  if (chunk_frames <= 0) chunk_frames = 256;
  for (GeoRun &r : fe->runs) r.frames = fe->frames + (size_t)r.f0 * fe->p.R * fe->p.B;
  int rc = fe_images_begin(fe, fe->geo[fe->runs[0].g], n_frames, chunk_frames, what);
  if (rc != SFE_OK) return rc;
  CopiesDrained drained{fe};
  rc = in.begin(chunk_frames);
  if (rc == SFE_OK) rc = fe_upload_poses(fe, poses_host, n_frames);
  if (rc == SFE_OK && in.stage) rc = in.stage(0, std::min(chunk_frames, n_frames), 0);
  int k = 0;
  CloudChunk prev;
  for (int f0 = 0; rc == SFE_OK && f0 < n_frames; f0 += chunk_frames, ++k) {
    const int n = std::min(chunk_frames, n_frames - f0), next = f0 + chunk_frames;
    if (in.stage && next < n_frames) rc = in.stage(next, std::min(chunk_frames, n_frames - next), k + 1);
    if (rc == SFE_OK) rc = in.ready(f0, n, k);
    if (rc == SFE_OK) rc = fe_render_host_chunk(fe, f0, n, k, what);
    if (rc == SFE_OK) rc = fe_features(fe, f0, n);
    if (rc == SFE_OK) rc = fe_clouds_chunk(fe, f0, n, k);
    if (rc == SFE_OK) rc = fe_match(fe, f0, n);
    if (rc == SFE_OK) rc = fe_clouds_out(fe, prev);
    prev = {f0, n, k};
  }
  if (rc != SFE_OK) return rc;
  return fe_host_finish(fe, prev, poses_host, n_frames, out, what);
}

// sfe_frontend_run_host[_geometry]: frame i at bytes + offsets[i] with its geometry's size (offsets and geometry null:
// bytes + i * R * B, geometry 0).  Chunks of frames stream in on the copy stream, run by run into their places in
// fe->frames, while the kernels of the chunk before run.
static int fe_run_raw_host(sfe_frontend *fe, const uint8_t *bytes, const int64_t *offsets, const int32_t *geometry,
                           const double *poses_host, int n_frames, int chunk_frames, const HostResults &out,
                           const char *what) {
  int rc = fe_host_args(fe, bytes && (!geometry || offsets), geometry, poses_host, n_frames, out, what);
  if (rc != SFE_OK) return rc;
  if (offsets) {
    SFE_REQUIRE(offsets_ok(offsets, n_frames), "%s: offsets must be non-decreasing", what);
    for (int i = 0; i < n_frames; ++i) {
      const sfe_maps *m = fe->geo[geometry[i]];
      SFE_REQUIRE(offsets[i + 1] - offsets[i] == (int64_t)m->R * m->B, "%s: frame %d has %lld bytes; its geometry %d "
                  "takes %d x %d = %lld", what, i, (long long)(offsets[i + 1] - offsets[i]), geometry[i], m->R, m->B,
                  (long long)m->R * m->B);
    }
  }
  const size_t fbytes = (size_t)fe->p.R * fe->p.B;
  HostFrames in;
  // the copies into fe->frames come after earlier work on ctx->stream that may still read it (the frames
  // sfe_frontend_run_dev_geometry packs there)
  in.begin = [&](int) { return fe_order(fe->ctx->stream, fe->ev_done, fe->copy_stream); };
  // No stage ahead: chunk k is copied only once the kernels of chunk k-1 are enqueued.  A copy from pageable host
  // memory returns only when its bytes are staged, so a copy issued a chunk ahead would hold back those kernels.
  in.ready = [&](int f0, int n, int k) -> int {
    const int r = fe_for_pieces(fe, f0, n, [&](const GeoRun &run, int a, int m) {
      const size_t src = offsets ? (size_t)offsets[a] : (size_t)a * fbytes;
      const size_t len = offsets ? (size_t)(offsets[a + m] - offsets[a]) : (size_t)m * fbytes;
      SFE_CUDA(cudaMemcpyAsync(fe_slot_frame(fe, run, a), bytes + src, len, cudaMemcpyHostToDevice, fe->copy_stream));
      return SFE_OK;
    });
    if (r != SFE_OK) return r;
    SFE_CUDA(cudaEventRecord(fe->ev_copy[k & 1], fe->copy_stream));
    SFE_CUDA(cudaStreamWaitEvent(fe->ctx->stream, fe->ev_copy[k & 1], 0));
    return SFE_OK;
  };
  return fe_run_host(fe, in, poses_host, n_frames, chunk_frames, out, what);
}

// The raw-frame copy of sfe_frontend_run_host replaced by the copy of the compressed bytes and the decode into
// fe->frames.  The host waits for chunk k's decode status once chunk k+1 is decoding, so the wait overlaps device work;
// the front-end stages of a chunk are enqueued only once its frames decoded.  geometry: one id per frame, or null
// (every frame geometry 0, R x B).
static int fe_run_compressed_host(sfe_frontend *fe, StreamDecoder *(*decoder)(sfe_ctx *), const uint8_t *bytes,
                                  const int64_t *offsets, const int32_t *geometry, const double *poses_host,
                                  int n_frames, int chunk_frames, const HostResults &out, const char *what) {
  int rc = fe_host_args(fe, bytes && offsets, geometry, poses_host, n_frames, out, what);
  if (rc != SFE_OK) return rc;
  SFE_REQUIRE(offsets_ok(offsets, n_frames), "%s: offsets must be non-decreasing", what);
  const int32_t *shape = nullptr;  // each frame's R x B, checked by the decoder
  if (geometry) {
    fe->frame_shape.resize(2 * (size_t)n_frames);
    for (int i = 0; i < n_frames; ++i)
      fe->frame_shape[2 * i] = fe->geo[geometry[i]]->R, fe->frame_shape[2 * i + 1] = fe->geo[geometry[i]]->B;
    shape = fe->frame_shape.data();
  }
  sfe_ctx *ctx = fe->ctx;
  StreamDecoder *dec = nullptr;
  int32_t *st_host = nullptr;       // each frame's decode status, read back chunk by chunk
  const int32_t *st_dev = nullptr;
  auto reject = [&](int i, int status) {
    if (geometry)
      set_error("%s: frame %d (geometry %d, %d x %d): %s", what, i, geometry[i], shape[2 * i], shape[2 * i + 1],
                dec->message(status));
    else
      set_error("%s: frame %d: %s", what, i, dec->message(status));
    return SFE_ERR_ARG;
  };
  HostFrames in;
  in.begin = [&](int chunk_frames) -> int {
    dec = decoder(ctx);
    dec->parse(bytes, offsets, n_frames, fe->p.R, fe->p.B, shape);
    for (int i = 0; i < n_frames; ++i)
      if (dec->frame_status(i) != 0) return reject(i, dec->frame_status(i));
    int r = dec->reserve(ctx, chunk_frames, 0);
    if (r == SFE_OK) r = ensure_pinned(ctx, 4 * (size_t)n_frames);
    st_host = static_cast<int32_t *>(ctx->pinned);
    st_dev = static_cast<const int32_t *>(dec->status.ptr);
    return r;
  };
  in.stage = [&](int f0, int n, int k) -> int {
    // a decode_chunk takes frames of one shape: a chunk that crosses a geometry change decodes run by run, each part
    // into its place in its run (every part is a subset of the chunk, which reserve() sized the decoder for)
    const int r = fe_for_pieces(fe, f0, n, [&](const GeoRun &run, int a, int m) {
      return dec->decode_chunk(ctx, a, m, fe_slot_frame(fe, run, a));
    });
    if (r != SFE_OK) return r;
    SFE_CUDA(cudaMemcpyAsync(st_host + f0, st_dev + f0, 4 * (size_t)n, cudaMemcpyDeviceToHost, ctx->stream));
    SFE_CUDA(cudaEventRecord(fe->ev_copy[k & 1], ctx->stream));
    return SFE_OK;
  };
  in.ready = [&](int f0, int n, int k) -> int {
    SFE_CUDA(cudaEventSynchronize(fe->ev_copy[k & 1]));
    for (int i = f0; i < f0 + n; ++i)
      if (st_host[i] != 0) {
        SFE_CUDA(cudaStreamSynchronize(ctx->stream));
        return reject(i, st_host[i]);
      }
    return SFE_OK;
  };
  return fe_run_host(fe, in, poses_host, n_frames, chunk_frames, out, what);
}

// sfe_frontend_run_dev[_geometry]; geometry: one id per frame, or null (every frame geometry 0)
static int fe_run_dev(sfe_frontend *fe, const uint8_t *frames_dev, const int32_t *geometry, const double *poses_host,
                      int n_frames, const char *what) {
  SFE_REQUIRE(fe && frames_dev && poses_host, "%s: null argument", what);
  SFE_REQUIRE(n_frames >= 0 && n_frames <= fe->max_frames, "%s: %d frames exceed max_frames %d", what, n_frames,
              fe->max_frames);
  SFE_REQUIRE(!fe->img_dst || !fe->img_dst_host, "%s: feature images are set to go to host memory; this flavour "
              "writes them to device memory (sfe_frontend_set_feature_images with dst_is_host = 0)", what);
  int rc = fe_clouds_args(fe, false, what);
  if (rc == SFE_OK) rc = fe_geometry_runs(fe, geometry, n_frames, what);
  if (rc != SFE_OK || n_frames == 0) return rc;
  sfe_ctx *ctx = fe->ctx;
  SFE_CUDA(cudaSetDevice(ctx->device));
  rc = fe_upload_poses(fe, poses_host, n_frames);
  if (rc != SFE_OK) return rc;
  // a run of a geometry smaller than the slots is packed into fe->frames at its natural stride, one copy per run (a
  // run of one frame, or of a geometry that fills its slots, is read where it is)
  const size_t fbytes = (size_t)fe->p.R * fe->p.B;
  for (GeoRun &r : fe->runs) {
    const size_t gb = fe_geo_bytes(fe, r.g);
    r.frames = frames_dev + (size_t)r.f0 * fbytes;
    if (gb == fbytes || r.n == 1) continue;
    uint8_t *dst = fe_slot_frame(fe, r, r.f0);
    SFE_CUDA(cudaMemcpy2DAsync(dst, gb, r.frames, fbytes, gb, r.n, cudaMemcpyDeviceToDevice, ctx->stream));
    r.frames = dst;
  }
  if (fe->img_dst) {  // (one run)
    const GeoRun &r = fe->runs[0];
    rc = feature_image_run(ctx, ctx->stream, fe->geo[r.g], r.frames, n_frames, fe->img_lut, fe->img_dst, what);
    if (rc != SFE_OK) return rc;
  }
  rc = fe_features(fe, 0, n_frames);
  if (rc == SFE_OK) rc = fe_match(fe, 0, n_frames);
  // a call whose clouds overflow leaves the carried window as it was
  if (rc == SFE_OK) rc = fe_clouds_dev(fe, n_frames, what);
  if (rc != SFE_OK) return rc;
  return fe_update_carry(fe, ctx->stream, poses_host, n_frames);
}

extern "C" {

int sfe_frontend_icp_dev(sfe_ctx *ctx, const sfe_icp_params *prm, const float *src_pts_dev, const int32_t *src_off_dev,
                         const float *tgt_pts_dev, const int32_t *tgt_off_dev, int n_problems, int ns_max, int nt_max,
                         const float *guess_dev, float *T_dev, int32_t *iters_dev, int32_t *inliers_dev,
                         int32_t *status_dev, int32_t *class_dev) {
  SFE_REQUIRE(ctx != nullptr, "sfe_frontend_icp_dev: null context");
  SFE_CUDA(cudaSetDevice(ctx->device));
  IcpProblems pb{{src_pts_dev, src_off_dev, nullptr, ns_max}, {tgt_pts_dev, tgt_off_dev, nullptr, nt_max}, nullptr,
                 nullptr, n_problems, guess_dev, T_dev, iters_dev, inliers_dev, status_dev};
  return icp_run(ctx, ctx->stream, prm, pb, FE_ICP_CLASSES, FE_ICP_N_CLASSES, class_dev,
                 ctx->has_icp_filters ? &ctx->icp_filters : nullptr, ctx->has_icp_robust ? &ctx->icp_robust : nullptr);
}

int sfe_frontend_run_dev(sfe_frontend *fe, const uint8_t *frames_dev, const double *poses_host, int n_frames) {
  return fe_run_dev(fe, frames_dev, nullptr, poses_host, n_frames, "sfe_frontend_run_dev");
}

int sfe_frontend_run_dev_geometry(sfe_frontend *fe, const uint8_t *frames_dev, const int32_t *geometry,
                                  const double *poses_host, int n_frames) {
  SFE_REQUIRE(geometry != nullptr, "sfe_frontend_run_dev_geometry: null geometry");
  return fe_run_dev(fe, frames_dev, geometry, poses_host, n_frames, "sfe_frontend_run_dev_geometry");
}

int sfe_frontend_results_dev(const sfe_frontend *fe, const float **T, const int32_t **iters, const int32_t **inliers,
                             const int32_t **status, const float **cloud_xy, const int32_t **cloud_count,
                             int32_t *cloud_stride) {
  SFE_REQUIRE(fe != nullptr, "sfe_frontend_results_dev: null handle");
  if (T) *T = fe->T;
  if (iters) *iters = fe->iters;
  if (inliers) *inliers = fe->inliers;
  if (status) *status = fe->status;
  const int32_t *cnt;
  const float *cloud = fe_cloud(fe, &cnt);
  if (cloud_xy) *cloud_xy = cloud;
  if (cloud_count) *cloud_count = cnt;
  if (cloud_stride) *cloud_stride = fe->p.cap_points;
  return SFE_OK;
}

int sfe_frontend_run_host(sfe_frontend *fe, const uint8_t *frames_host, const double *poses_host, int n_frames,
                          int chunk_frames, float *T_host, int32_t *iters_host, int32_t *inliers_host,
                          int32_t *status_host, int32_t *npoints_host) {
  return fe_run_raw_host(fe, frames_host, nullptr, nullptr, poses_host, n_frames, chunk_frames,
                         {T_host, iters_host, inliers_host, status_host, npoints_host}, "sfe_frontend_run_host");
}

int sfe_frontend_run_host_geometry(sfe_frontend *fe, const uint8_t *bytes, const int64_t *offsets,
                                   const int32_t *geometry, const double *poses_host, int n_frames, int chunk_frames,
                                   float *T_host, int32_t *iters_host, int32_t *inliers_host, int32_t *status_host,
                                   int32_t *npoints_host) {
  SFE_REQUIRE(offsets && geometry, "sfe_frontend_run_host_geometry: null offsets / geometry");
  return fe_run_raw_host(fe, bytes, offsets, geometry, poses_host, n_frames, chunk_frames,
                         {T_host, iters_host, inliers_host, status_host, npoints_host},
                         "sfe_frontend_run_host_geometry");
}

int sfe_frontend_run_jpeg_host(sfe_frontend *fe, const uint8_t *bytes, const int64_t *offsets, const double *poses_host,
                               int n_frames, int chunk_frames, float *T_host, int32_t *iters_host,
                               int32_t *inliers_host, int32_t *status_host, int32_t *npoints_host) {
  return fe_run_compressed_host(fe, jpeg_decoder, bytes, offsets, nullptr, poses_host, n_frames, chunk_frames,
                                {T_host, iters_host, inliers_host, status_host, npoints_host},
                                "sfe_frontend_run_jpeg_host");
}

int sfe_frontend_run_png_host(sfe_frontend *fe, const uint8_t *bytes, const int64_t *offsets, const double *poses_host,
                              int n_frames, int chunk_frames, float *T_host, int32_t *iters_host, int32_t *inliers_host,
                              int32_t *status_host, int32_t *npoints_host) {
  return fe_run_compressed_host(fe, png_decoder, bytes, offsets, nullptr, poses_host, n_frames, chunk_frames,
                                {T_host, iters_host, inliers_host, status_host, npoints_host},
                                "sfe_frontend_run_png_host");
}

int sfe_frontend_run_jpeg_host_geometry(sfe_frontend *fe, const uint8_t *bytes, const int64_t *offsets,
                                        const int32_t *geometry, const double *poses_host, int n_frames,
                                        int chunk_frames, float *T_host, int32_t *iters_host, int32_t *inliers_host,
                                        int32_t *status_host, int32_t *npoints_host) {
  SFE_REQUIRE(geometry != nullptr, "sfe_frontend_run_jpeg_host_geometry: null geometry");
  return fe_run_compressed_host(fe, jpeg_decoder, bytes, offsets, geometry, poses_host, n_frames, chunk_frames,
                                {T_host, iters_host, inliers_host, status_host, npoints_host},
                                "sfe_frontend_run_jpeg_host_geometry");
}

int sfe_frontend_run_png_host_geometry(sfe_frontend *fe, const uint8_t *bytes, const int64_t *offsets,
                                       const int32_t *geometry, const double *poses_host, int n_frames,
                                       int chunk_frames, float *T_host, int32_t *iters_host, int32_t *inliers_host,
                                       int32_t *status_host, int32_t *npoints_host) {
  SFE_REQUIRE(geometry != nullptr, "sfe_frontend_run_png_host_geometry: null geometry");
  return fe_run_compressed_host(fe, png_decoder, bytes, offsets, geometry, poses_host, n_frames, chunk_frames,
                                {T_host, iters_host, inliers_host, status_host, npoints_host},
                                "sfe_frontend_run_png_host_geometry");
}

}  // extern "C"
