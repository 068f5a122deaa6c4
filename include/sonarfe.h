/* libsonarfe -- H100 (sm_90a) sonar front end: CFAR detector, polar->Cartesian
 * feature cloud, cloud filters, ICP scan matcher.
 *
 * C ABI that replaces the two pybind11 modules of jake3991/sonar-SLAM's
 * bruce_slam package on its per-keyframe hot path:
 *
 *     bruce_slam.cfar   bruce_slam/src/bruce_slam/cpp/cfar.cpp:194-204
 *     bruce_slam.pcl    bruce_slam/src/bruce_slam/cpp/pcl.cpp:176-214
 *
 * plus the numeric body of FeatureExtraction.callback that sits between them
 * (bruce_slam/src/bruce_slam/feature_extraction.py:223-249).  Plain pointers and
 * sizes only.  Every function returns SFE_OK (0) or a negative SFE_ERR_* code and
 * never throws; sfe_last_error() gives the thread's last message.
 *
 * Pointer suffixes:  *_dev  = device memory on the context's GPU (asynchronous on
 * the context's stream; call sfe_sync() or synchronise the stream yourself),
 * *_host = ordinary host memory (the call copies in/out and returns when done).
 * There is no CPU fallback: every entry point runs CUDA kernels.
 */
#ifndef SONARFE_H_
#define SONARFE_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SFE_VERSION 202 /* round 2: + sfe_fov_select_*, sfe_frontend_set_carry, sfe_frontend_params.flip_lateral, sfe_icp_params.flags bit 1;
                            201: + sfe_icp_params.minimizer / normals_knn (point-to-plane, icp.yaml:18-19);
                            202: - sfe_frontend_set_overlap (run_dev runs every stage over the whole batch); later
                                 additions that change no existing entry point: sfe_match_dim_*, sfe_match_knn_dim_*,
                                 sfe_downsample_cta_limit, dim = 3 in sfe_downsample_dev / _host, sfe_icp_dim_dev,
                                 sfe_icp_dim_host, sfe_icp_batch_dim_host, sfe_icp_cta_limit, sfe_icp_source_limit,
                                 SFE_ICP_DATA_OCTREE and SFE_ICP_DATA_VOXEL (new sfe_icp_data_filter kinds; both structs
                                 keep their sizes), sfe_ctx_set_grid_sms, sfe_ctx_occupancy, sfe_icp_robust with
                                 sfe_icp_set_robust and sfe_frontend_set_icp_robust, SFE_ICP_DATA_SAMPLING_NORMALS (a
                                 new sfe_icp_data_filter kind; both structs keep their sizes) with
                                 sfe_icp_sampling_normals_dev, SFE_ICP_DATA_NORMALS and SFE_ICP_DATA_SHADOW (new
                                 sfe_icp_data_filter kinds, reading side; both structs keep their sizes) with
                                 sfe_icp_surface_normals_dev */

#if defined(__GNUC__)
#define SFE_API __attribute__((visibility("default")))
#else
#define SFE_API
#endif

enum {
  SFE_OK = 0,
  SFE_ERR_ARG = -1,      /* bad argument (shape, dtype code, null pointer ...) */
  SFE_ERR_CUDA = -2,     /* a CUDA runtime/driver call failed                  */
  SFE_ERR_CAPACITY = -3, /* a caller-provided output buffer was too small      */
  SFE_ERR_UNSUPPORTED = -4
};

/* CFAR variants, in the order of cfar.cpp:194-204 */
enum { SFE_CFAR_CA = 0, SFE_CFAR_SOCA = 1, SFE_CFAR_GOCA = 2, SFE_CFAR_OS = 3 };
/* image element types */
enum { SFE_U8 = 0, SFE_F32 = 1 };

typedef struct sfe_ctx sfe_ctx; /* one GPU + one stream + scratch memory; not thread-safe */

SFE_API int sfe_version(void);
SFE_API const char *sfe_last_error(void);

/* Create a context on `device`.  own_stream != 0: the library creates its own
 * non-blocking stream (cuda_stream is ignored).  own_stream == 0: all work is enqueued
 * on the caller's cudaStream_t `cuda_stream` (NULL = the legacy default stream; pass
 * e.g. torch's current stream). */
SFE_API int sfe_ctx_create(int device, void *cuda_stream, int own_stream, sfe_ctx **out);
SFE_API void sfe_ctx_destroy(sfe_ctx *ctx);
SFE_API int sfe_sync(sfe_ctx *ctx);
/* blocking device -> host copy on the context's stream (for callers without a CUDA runtime binding) */
SFE_API int sfe_copy_to_host(sfe_ctx *ctx, void *dst_host, const void *src_dev, uint64_t bytes);
/* number of kernels this context has launched so far (bench.py: gpu_launches) */
SFE_API uint64_t sfe_launch_count(const sfe_ctx *ctx);
/* For tests: the number of SMs this context sizes its persistent launches for.  sms >= 1 sets it to min(sms, the
 * device's SM count), sms <= 0 restores the device's count; *effective (may be NULL) receives the value now in force.
 * Every persistent or grid-stride launch (Cartesian points, down-sample, outlier removal, match, ICP and the front
 * end's stages) then runs that many SMs' worth of CTAs, so each CTA takes more work items in a row.  Results must not
 * change.  The other uses of the count move with it and are claimed not to change results either: the Cartesian
 * points' dense variants (F >= 2 * and 4 * the count), the costmap's warps per candidate and the PNG front end's
 * chunk_frames.  Size classes (the ICP class split, source and one-CTA limits, the front end's classes) do not read
 * it.  Not for concurrent use with other calls on the context. */
SFE_API int sfe_ctx_set_grid_sms(sfe_ctx *ctx, int sms, int32_t *effective);
/* For tests: the CTAs per SM of the persistent one-CTA launch configurations (kernel, threads, dynamic shared memory)
 * this context has sized so far, in the order it first sized them; the context keeps the last 16.  Entry k:
 * threads[k], smem[k] (bytes) and per_sm[k]; *n receives the number of entries, at most `capacity` are written.  A
 * capped launch (sfe_ctx_set_grid_sms) runs sms * per_sm CTAs. */
SFE_API int sfe_ctx_occupancy(const sfe_ctx *ctx, int32_t *threads, int32_t *smem, int32_t *per_sm, int capacity,
                              int32_t *n);

/* ------------------------------------------------------------------ CFAR
 * Replaces cfar::{ca,soca,goca,os} (cfar.cpp:10,30,53,76) and, with a non-NULL
 * thr pointer, cfar::{ca2,soca2,goca2,os2} (cfar.cpp:98,120,145,170), batched
 * over `n_frames` images [n_frames][R][B] (range bins x beams, beams contiguous).
 * The detection window runs along R for every beam, exactly as in the reference:
 * `train_hs` leading + `train_hs` lagging training cells separated from the cell
 * under test by `guard_hs` guard cells on each side; the first and last
 * train_hs+guard_hs rows of the mask are 0.
 *
 *   dtype        SFE_U8 or SFE_F32.  The reference takes float32 (pybind converts
 *                the node's uint8 image); uint8 is accepted directly and gives the
 *                same result as converting first.
 *   k, tau       OS rank (0-based, < 2*train_hs; ignored otherwise), threshold factor
 *   gate_enable / gate_threshold
 *                fuses the node's `peaks &= img > threshold`
 *                (feature_extraction.py:224) into the detector when gate_enable != 0
 *   mask         uint8 0/1, [n_frames][R][B]                     (may be NULL)
 *   thr          float32 threshold image, [n_frames][R][B]       (may be NULL)
 *   bits         the same mask as a bit plane: uint32 [n_frames][R][ceil(B/32)],
 *                bit (b & 31) of word b >> 5 is beam b             (may be NULL)
 * Results are bit-identical to the reference for every float32 input, integer
 * valued or not (non-integer tiles are re-done with the reference's sequential
 * float32 accumulation order).
 */
SFE_API int sfe_cfar_dev(sfe_ctx *ctx, const void *img_dev, int dtype, int n_frames, int R, int B, int alg,
                 int train_hs, int guard_hs, int k, double tau, int gate_enable, double gate_threshold,
                 uint8_t *mask_dev, float *thr_dev, uint32_t *bits_dev);
SFE_API int sfe_cfar_host(sfe_ctx *ctx, const void *img_host, int dtype, int n_frames, int R, int B, int alg,
                  int train_hs, int guard_hs, int k, double tau, int gate_enable, double gate_threshold,
                  uint8_t *mask_host, float *thr_host);

/* ------------------------------------------------------------------ polar -> Cartesian cloud
 * Replaces feature_extraction.py:231-238: cv2.remap(mask, map_x, map_y, INTER_LINEAR),
 * np.nonzero, pixel -> metres.  `sfe_maps` holds, on the device, the per-geometry sampling
 * table derived from the float32 maps that generate_map_xy builds (feature_extraction.py:134-173;
 * the maps themselves stay host-side Python).  R x B = polar image (range bins x beams),
 * rows x cols = Cartesian image, width/height = its extent in metres (self.width, self.height).
 */
typedef struct sfe_maps sfe_maps;
SFE_API int sfe_maps_create(sfe_ctx *ctx, const float *map_x_host, const float *map_y_host, int rows, int cols, int R,
                            int B, double width, double height, sfe_maps **out);
/* Diagnostic, host only (no context, no GPU): the inverse lists sfe_maps_create uploads -- for every polar cell
 * the Cartesian pixels the detection-driven kernel tests when that cell is a detection -- as a CSR structure:
 * off_out [R*B + 1], idx_out [*n_entries] pixel indices (row * cols + col).  A pixel is listed under the smallest
 * set of its taps that every firing configuration must light (see featx.cu: build_inverse_lists).  Returns
 * SFE_ERR_CAPACITY (with *n_entries set) when idx_capacity is too small. */
SFE_API int sfe_maps_inverse_lists_host(const float *map_x_host, const float *map_y_host, int rows, int cols, int R,
                                        int B, int32_t *off_out, int32_t *idx_out, int64_t idx_capacity,
                                        int64_t *n_entries);
SFE_API void sfe_maps_destroy(sfe_maps *maps);

/* For each of n_frames polar 0/1 masks (bytes [n_frames][R][B], or the bit plane written by
 * sfe_cfar_dev -- pass exactly one, the other NULL) emit the non-zero Cartesian pixels in row-major
 * order: ij[f][i] = (row, col) int32 (np.nonzero order), xy[f][i] = (y_forward_m, x_lateral_m)
 * float32 = float32(points) of feature_extraction.py:238, count[f] = number found.  At most
 * `capacity` points per frame are written (count still reports the true number). */
SFE_API int sfe_cart_points_dev(sfe_ctx *ctx, const sfe_maps *maps, const uint8_t *mask_dev, const uint32_t *bits_dev,
                                int n_frames, int capacity, int32_t *ij_dev, float *xy_dev, int32_t *count_dev);
/* Host-buffer flavour (byte masks); returns SFE_ERR_CAPACITY if a frame overflowed `capacity`. */
SFE_API int sfe_cart_points_host(sfe_ctx *ctx, const sfe_maps *maps, const uint8_t *mask_host, int n_frames,
                                 int capacity, int32_t *ij_host, float *xy_host, int32_t *count_host);

/* ------------------------------------------------------------------ feature image
 * feature_extraction.py:226-228: cv2.applyColorMap(cv2.remap(img, map_x, map_y, INTER_LINEAR), COLORMAP_JET), the
 * bgr8 image the reference publishes on its feature-image topic, for n_frames uint8 polar frames [n][R][B] of the maps'
 * geometry.  Output: uint8 [n][rows][cols][3], B, G, R = lut_bgr[v] where v is cv2.remap's 8-bit value (fixed-point
 * bilinear on 1/32-px coordinates, constant-0 border; NaN, infinite or |map * 32| >= 1e9 coordinates give 0), bit for
 * bit.  lut_bgr_host: uint8 [256][3] in HOST memory (COLORMAP_JET: sonar_slam_b200.feature_image.JET).
 * Device flavour: asynchronous on the context's stream.  Host flavour: copies the frames in and the images out in
 * chunks overlapped with the kernel and returns when the images are in out_host. */
SFE_API int sfe_feature_image_dev(sfe_ctx *ctx, const sfe_maps *maps, const uint8_t *frames_dev, int n_frames,
                                  const uint8_t *lut_bgr_host, uint8_t *out_dev);
SFE_API int sfe_feature_image_host(sfe_ctx *ctx, const sfe_maps *maps, const uint8_t *frames_host, int n_frames,
                                   const uint8_t *lut_bgr_host, uint8_t *out_host);

/* ------------------------------------------------------------------ point-cloud filters
 * Clouds are packed: pts [total][dim] float32 (dim = 2: x,y; dim = 3: x,y,z),
 * off [n_clouds + 1] int32 offsets (cloud c = rows off[c] .. off[c+1]-1), n_max = largest cloud.
 * Results are compacted in place of each cloud: out_pts rows off[c] .. off[c]+out_count[c]-1, and
 * out_idx gives, for every surviving point, its row inside its input cloud.
 *
 * sfe_downsample_*      bruce_slam.pcl.downsample (pcl.cpp:128-159): libpointmatcher
 *                       OctreeGridDataPointsFilter{maxSizeByNode = resolution, samplingMethod = 3}:
 *                       quadtree on the cloud's bounding square, one medoid per leaf, leaves in
 *                       depth-first order.  The two-argument overload (points + descriptors,
 *                       pcl.cpp:143) is served by gathering descriptors with out_idx.
 *                       Any cloud size is accepted: clouds that fit one CTA's shared memory
 *                       (13 880 points on an H100) run one CTA each; larger ones (whole maps)
 *                       run in the same call on a grid-wide path (radix sort of path keys,
 *                       medoid sums one thread per member), with the same results.  A call
 *                       with a cloud above that limit takes at most 65 535 clouds and
 *                       n_clouds * n_max slots (at most 2^31 - 1); its workspace holds 48 bytes
 *                       per slot.  Trees stop at 15 levels (16 km at a 0.5 m resolution).
 *                       dim = 3 (libpointmatcher's 3-D Octree): an octree on the bounding cube
 *                       (half-size = the largest half-extent, children by x, y, z > centre), the
 *                       3-D medoid sum; the one-CTA limit is lower (24 bytes per point of shared
 *                       memory instead of 16), the grid-wide workspace 52 bytes per slot.
 * sfe_remove_outlier_*  bruce_slam.pcl.remove_outlier (pcl.cpp:54-74): PCL RadiusOutlierRemoval:
 *                       keep a point iff at least min_points OTHER points lie within `radius`;
 *                       input order is preserved.
 *                       Any cloud size is accepted: clouds that fit one CTA's shared memory
 *                       (24 445 points on an H100) run one CTA each; larger ones (whole maps) run
 *                       in the same call in a map class (the map grid of sfe_match_dev in global
 *                       memory, one thread per point), with the same results.  A call with a cloud
 *                       above that limit takes at most 65 535 clouds and n_clouds * n_max slots
 *                       (at most 2^31 - 1); its workspace holds 48 bytes per slot, a cell table of
 *                       6 bytes per n_max point and 28 bytes per cloud, and CUB's temporary storage.
 */
SFE_API int sfe_downsample_dev(sfe_ctx *ctx, const float *pts_dev, const int32_t *off_dev, int n_clouds, int dim,
                               int n_max, float resolution, float *out_pts_dev, int32_t *out_idx_dev,
                               int32_t *out_count_dev);
SFE_API int sfe_remove_outlier_dev(sfe_ctx *ctx, const float *pts_dev, const int32_t *off_dev, int n_clouds, int dim,
                                   int n_max, double radius, int min_points, float *out_pts_dev,
                                   int32_t *out_idx_dev, int32_t *out_count_dev);
/* the batched front end's per-frame down-sample: clouds of up to frame_points points in a launch laid out for them,
 * larger ones in a launch laid out for n_max (at most 65 535; layouts above the one-CTA shared-memory limit keep
 * their workspace in global memory, 16 bytes per point per SM); cnt_dev (optional) holds the clouds' point counts, else
 * off_dev[c + 1] - off_dev[c].  2-column clouds only.  Same results as sfe_downsample_dev. */
SFE_API int sfe_downsample_frames_dev(sfe_ctx *ctx, const float *pts_dev, const int32_t *off_dev,
                                      const int32_t *cnt_dev, int n_clouds, int n_max, int frame_points,
                                      float resolution, float *out_pts_dev, int32_t *out_idx_dev,
                                      int32_t *out_count_dev);
/* *limit = the largest cloud of `dim` columns that sfe_downsample_* runs in one CTA on this context's device (larger
 * clouds take the grid-wide path) */
SFE_API int sfe_downsample_cta_limit(sfe_ctx *ctx, int dim, int32_t *limit);
/* single-cloud host flavours: n points in, *n_out points out (out buffers hold n entries) */
SFE_API int sfe_downsample_host(sfe_ctx *ctx, const float *pts_host, int n, int dim, float resolution,
                                float *out_pts_host, int32_t *out_idx_host, int32_t *n_out);
SFE_API int sfe_remove_outlier_host(sfe_ctx *ctx, const float *pts_host, int n, int dim, double radius,
                                    int min_points, float *out_pts_host, int32_t *out_idx_host, int32_t *n_out);

/* ------------------------------------------------------------------ nearest-neighbour match
 * bruce_slam.pcl.match(ref, in, knn = 1, max_dist) (pcl.cpp:161-174; libpointmatcher KDTreeMatcher):
 * for every query point the index of the nearest reference point and the SQUARED float32 distance;
 * no reference point within max_dist -> id -1, dist +inf; ties -> lowest reference index.
 * Batched over n_pairs (ref cloud p, query cloud p), both packed [total][2] with CSR offsets;
 * ids / dists are indexed like the query points.
 * References of any size: those that fit one CTA's shared memory (24 k points on an H100) run one CTA per pair; larger
 * ones (whole maps) are sorted once into a grid in global memory and searched by the whole device, with the same
 * results.  Their workspace holds 40 bytes for each of n_pairs * n_ref_max slot points (at most 2^31 - 1), 6 bytes
 * per n_ref_max point of cell table per pair, and CUB's temporary storage. */
SFE_API int sfe_match_dev(sfe_ctx *ctx, const float *ref_pts_dev, const int32_t *ref_off_dev, const float *in_pts_dev,
                          const int32_t *in_off_dev, int n_pairs, int n_ref_max, float max_dist, int32_t *ids_dev,
                          float *dists_dev);
SFE_API int sfe_match_host(sfe_ctx *ctx, const float *ref_host, int n_ref, const float *in_host, int n_in,
                           float max_dist, int32_t *ids_host, float *dists_host);
/* k nearest neighbours, knn = 1 .. 16 (libnabo's exact k-NN search with a radius, as KDTreeMatcher runs it): for every
 * query point the knn reference points nearest to it among those with squared float32 distance <= max_dist^2 (the
 * radius test and distance expression above), in ascending squared distance, ties -> lower reference index.  Row j
 * of ids / dists holds every query's j-th neighbour: ids / dists are [knn][total query points] (for one pair the
 * binding's [knn, N]); slots with no neighbour left hold id -1, dist +inf.  Row 0 is sfe_match_*'s result, and rows
 * 0 .. k-1 do not depend on knn >= k.  knn = 1 runs sfe_match_*'s kernels; knn outside 1 .. 16 is SFE_ERR_ARG.
 * References that fit one CTA's shared memory next to the 6 * 512 * knn bytes of the per-thread lists run one CTA per
 * pair (24.1 k points at knn 2 down to 18.7 k at knn 16 on an H100); larger ones go to the map grids, whose workspace is
 * sfe_match_dev's. */
SFE_API int sfe_match_knn_dev(sfe_ctx *ctx, const float *ref_pts_dev, const int32_t *ref_off_dev,
                              const float *in_pts_dev, const int32_t *in_off_dev, int n_pairs, int n_ref_max, int knn,
                              float max_dist, int32_t *ids_dev, float *dists_dev);
SFE_API int sfe_match_knn_host(sfe_ctx *ctx, const float *ref_host, int n_ref, const float *in_host, int n_in, int knn,
                               float max_dist, int32_t *ids_host, float *dists_host);
/* sfe_match_* and sfe_match_knn_* for clouds of `dim` columns (2: the calls above, same kernels and results; 3: x, y, z
 * in both clouds).  3-D: squared float32 distance (dx*dx + dy*dy) + dz*dz, every other rule as above; the search runs on
 * a grid of x, y (exact: the 3-D distance is never below the xy one), so a reference tall in z over a small xy
 * footprint is searched column by column.  The one-CTA / map-grid split is sfe_match_knn_*'s at every knn (its lists
 * included at knn = 1); the map grids' workspace is sfe_match_dev's.  dim outside 2 .. 3 is SFE_ERR_ARG. */
SFE_API int sfe_match_dim_dev(sfe_ctx *ctx, const float *ref_pts_dev, const int32_t *ref_off_dev,
                              const float *in_pts_dev, const int32_t *in_off_dev, int n_pairs, int dim, int n_ref_max,
                              float max_dist, int32_t *ids_dev, float *dists_dev);
SFE_API int sfe_match_dim_host(sfe_ctx *ctx, const float *ref_host, int n_ref, const float *in_host, int n_in, int dim,
                               float max_dist, int32_t *ids_host, float *dists_host);
SFE_API int sfe_match_knn_dim_dev(sfe_ctx *ctx, const float *ref_pts_dev, const int32_t *ref_off_dev,
                                  const float *in_pts_dev, const int32_t *in_off_dev, int n_pairs, int dim,
                                  int n_ref_max, int knn, float max_dist, int32_t *ids_dev, float *dists_dev);
SFE_API int sfe_match_knn_dim_host(sfe_ctx *ctx, const float *ref_host, int n_ref, const float *in_host, int n_in,
                                   int dim, int knn, float max_dist, int32_t *ids_host, float *dists_host);

/* ------------------------------------------------------------------ ICP scan matcher
 * bruce_slam.pcl.ICP (pcl.cpp:185-213): libpointmatcher PointMatcher<float>::ICP configured by
 * bruce_slam/config/icp.yaml.  The struct carries what that YAML sets; sfe_icp_params_default()
 * fills in the shipped values (the host side parses the YAML, see bruce_slam/pcl.py). */
typedef struct {
  float matcher_max_dist; /* KDTreeMatcher maxDist                      icp.yaml:9   10.0 */
  float outlier_max_dist; /* MaxDistOutlierFilter maxDist (<= 0: off)   icp.yaml:13   3.0 */
  float trim_ratio;       /* TrimmedDistOutlierFilter ratio (< 0: off)  icp.yaml:15   0.8 */
  int max_iterations;     /* CounterTransformationChecker               icp.yaml:24    40 */
  float min_diff_rot;     /* DifferentialTransformationChecker          icp.yaml:26  0.01 */
  float min_diff_trans;   /*                                            icp.yaml:27   0.1 */
  int smooth_length;      /* (0: differential checker off; <= 15)        icp.yaml:28     4 */
  int flags;              /* bit 0: MaxDist filter compares squared distance with maxDist itself
                             bit 1: accumulate the sums over points (reference mean, pair means, cross-covariance) in
                                    float64, order-independent.  DEFAULT (bit clear): every such sum is a SEQUENTIAL
                                    float32 sum in point order, the accumulation order of the CPU oracle
                                    (oracle/icp_ref.c) -- results are bit-identical to it.  The float64 mode is
                                    closer to exact arithmetic, but differs from the float32 chain by
                                    up to ~2e-3 m on ill-conditioned scans (tests/test_icp_parity_gpu.py). */
  int minimizer;          /* errorMinimizer: 0 PointToPointErrorMinimizer (shipped, icp.yaml:20)
                             1 PointToPlaneErrorMinimizer force2D (the alternative the YAML keeps commented out,
                               icp.yaml:18-19): per iteration the 3x3 normal equations of sum ((R q + t - r).n)^2
                               linearised in (theta, tx, ty), solved by Cholesky; the step is Rotation2D(theta), (tx, ty) */
  int normals_knn;        /* point-to-plane only: the reference's normals, as a SurfaceNormalDataPointsFilter{knn}
                             in referenceDataPointsFilters would attach them (libpointmatcher default 5; 3..16):
                             smaller-eigenvalue direction of the covariance of each point's knn nearest reference
                             points (itself included).  With an SFE_ICP_DATA_SAMPLING_NORMALS reference filter (either
                             minimizer): that filter's knn, the largest box (3..64), and its normals replace these */
} sfe_icp_params;
SFE_API void sfe_icp_params_default(sfe_icp_params *p);

/* per-problem status (ICP.compute returns the text as its message, pcl.cpp:203-211) */
enum {
  SFE_ICP_SUCCESS = 0,      /* "success" */
  SFE_ICP_NO_OUTLIER = 1,   /* ConvergenceError "no outlier to filter" (no source point has a match) */
  SFE_ICP_NO_POINT = 2,     /* ConvergenceError "ErrorMnimizer: no point to minimize" */
  SFE_ICP_NAN_ROT = 3,      /* ConvergenceError "abs rotation norm not a number" */
  SFE_ICP_NAN_TRANS = 4,    /* ConvergenceError "abs translation norm not a number" */
  SFE_ICP_NOT_RIGID = 5,    /* TransformationError: the initial guess is not a rigid transform */
  SFE_ICP_EMPTY_REF = 6,    /* the target cloud is empty */
  SFE_ICP_SKIPPED = 7,      /* front-end pipeline only: fewer than min_points source/target points (slam.py:654-663),
                               or the scan match is off (sfe_frontend_set_scan_match) */
  SFE_ICP_TOO_LARGE = 8     /* front-end pipeline only: a cloud exceeded the configured capacity */
};
SFE_API const char *sfe_icp_status_message(int status);

/* Solve n_problems scan matches.  Problem p aligns source cloud src_id[p] to target cloud tgt_id[p]
 * (ids NULL: cloud p) from the initial guess guess[p] (3x3 row-major float32, as ICP.compute's third
 * argument); clouds packed [total][2] with CSR offsets, ns_max / nt_max = largest source / target.
 * Outputs per problem: T (3x3 row-major; = guess when status != 0, like pcl.cpp:207-210), iterations
 * made, inlier count of the last iteration (pairs with non-zero weight), status.
 * Targets of any size: the problems whose target fits one CTA's shared memory next to the sources (22 k points
 * next to 1 500-point sources on an H100) run as before; the others read their target from a map grid built once
 * per distinct target cloud in global memory (mean, normals and grid computed once, not per guess), with the same
 * results.  Map workspace: 40 bytes (48 point-to-plane) for each of slots * nt_max slot points (at most 2^31 - 1),
 * 6 bytes per nt_max point of cell table per slot, 28 bytes per problem and CUB's temporary storage; slots =
 * n_problems for sfe_icp_dev, min(n_problems, n_tgt_clouds) for the host flavours.
 * Sources of any size: sources of up to sfe_icp_source_limit points (about 8 400 on an H100, 27 bytes of shared memory
 * per point) run in the shared-memory layouts as before.  Larger ones take the global-source class: persistent
 * 512-thread CTAs that keep the per-source-point arrays in a slice of global workspace (29 bytes per ns_max point,
 * 256-byte aligned) and read every target, small or large, from a map grid.  As many CTAs run as fit the SMs and a
 * fixed 512 MiB for all slices together, at least one; a source whose one slice exceeds 512 MiB (about 18 million
 * points) is SFE_ERR_UNSUPPORTED, and nothing is launched.  A call whose targets all fit one CTA next to its sources
 * still runs in that CTA.  Results are the same in every class. */
SFE_API int sfe_icp_dev(sfe_ctx *ctx, const sfe_icp_params *prm, const float *src_pts_dev, const int32_t *src_off_dev,
                        const float *tgt_pts_dev, const int32_t *tgt_off_dev, const int32_t *src_id_dev,
                        const int32_t *tgt_id_dev, int n_problems, int ns_max, int nt_max, const float *guess_dev,
                        float *T_dev, int32_t *iters_dev, int32_t *inliers_dev, int32_t *status_dev);
/* sfe_icp_dev (problem p: clouds p / p) through the batched front end's size classes: each class its own launch,
 * problems largest first; same results.  class_dev (device [2 * n_problems] or NULL): class_dev[p] = the class that
 * solved problem p (the front end's classes in order, the capacity launch last), class_dev[n_problems + p] = its place in that
 * class's work list. */
SFE_API int sfe_frontend_icp_dev(sfe_ctx *ctx, const sfe_icp_params *prm, const float *src_pts_dev,
                                 const int32_t *src_off_dev, const float *tgt_pts_dev, const int32_t *tgt_off_dev,
                                 int n_problems, int ns_max, int nt_max, const float *guess_dev, float *T_dev,
                                 int32_t *iters_dev, int32_t *inliers_dev, int32_t *status_dev, int32_t *class_dev);
/* One source / target pair from host memory, n_guesses initial guesses (1 = ICP.compute; >1 = the
 * loop of SLAM.compute_icp_with_cov, slam.py:346-358, run as one batch). */
SFE_API int sfe_icp_host(sfe_ctx *ctx, const sfe_icp_params *prm, const float *src_host, int ns, const float *tgt_host,
                         int nt, const float *guess_host, int n_guesses, float *T_host, int32_t *iters_host,
                         int32_t *inliers_host, int32_t *status_host);
/* Host-buffer flavour of sfe_icp_dev: packed clouds with CSR offsets (src_off [n_src_clouds + 1], tgt_off
 * [n_tgt_clouds + 1]) and per-problem src_id / tgt_id, all in host memory, so that the guesses of many loop-closure
 * candidates (each its own cloud pair) go out in one launch.  ns_max / nt_max are taken from the offsets.  Clouds of
 * any size, as sfe_icp_dev: sources above sfe_icp_source_limit take the global-source class and its workspace. */
SFE_API int sfe_icp_batch_host(sfe_ctx *ctx, const sfe_icp_params *prm, const float *src_pts_host,
                               const int32_t *src_off_host, int n_src_clouds, const float *tgt_pts_host,
                               const int32_t *tgt_off_host, int n_tgt_clouds, const int32_t *src_id_host,
                               const int32_t *tgt_id_host, int n_problems, const float *guess_host, float *T_host,
                               int32_t *iters_host, int32_t *inliers_host, int32_t *status_host);

/* More of libpointmatcher's ICP modules than sfe_icp_params carries: distance data filters on the reading (source) and
 * reference (target) clouds, and the MinDist / MedianDist outlier filters.
 *   data filters   applied once per problem before the iterations, in the listed order; the survivors keep their
 *                  input order.  Reading filters see the source in its input frame (before the guess), reference
 *                  filters the target in its input frame (before centring: mean, grid and normals come from the
 *                  survivors).  SFE_ICP_DATA_MAX_DIST {dim, dist}: dim -1 keeps sqrtf(x*x + y*y) < |dist|, dim 0 / 1
 *                  keeps coordinate < dist; SFE_ICP_DATA_MIN_DIST the mirror (> |dist|, coordinate > dist).
 *                  SFE_ICP_DATA_OCTREE {dim, dist}: OctreeGridDataPointsFilter with maxSizeByNode = dist (finite, > 0)
 *                  and samplingMethod = dim -- the quadtree of sfe_downsample_dev (bounding square, stable 4-way
 *                  partition, split while 2 * radius > dist and more than one point, at most 15 levels), one point
 *                  per leaf in depth-first leaf order: 0 the leaf's first (lowest-index) member, 2 its centroid
 *                  (float32 sequential sums of x and y in member order, each divided by the member count), 3 its
 *                  medoid (as sfe_downsample_dev).  Later filters and the iterations see the leaf order.
 *                  SFE_ICP_DATA_VOXEL {dim, dist}: VoxelGridDataPointsFilter with vSizeX = vSizeY = dist (finite, > 0)
 *                  and useCentroid = dim (1; 0 is not supported) -- per axis minB = min / dist, maxB = max / dist,
 *                  numDiv = 1 + (unsigned)(maxB - minB); point p lies in voxel (unsigned)floorf(x / dist - minBX) +
 *                  (unsigned)floorf(y / dist - minBY) * numDivX; the first point of every voxel is kept, in point
 *                  order, holding the voxel's centroid (float32 sequential sums from the first point's coordinates in
 *                  point order, each divided by (float)count).  A cloud whose numDivX * numDivY does not fit 32 bits
 *                  (or whose bounds are not finite) makes the call SFE_ERR_UNSUPPORTED after the filter stages and
 *                  before any ICP launch (the grid spans the cloud the filter receives, known on the device only;
 *                  the call waits for the stages to check).
 *                  SFE_ICP_DATA_SAMPLING_NORMALS {dim, dist}: SamplingSurfaceNormalDataPointsFilter with samplingMethod
 *                  = dim (1, or 0 for ratio 1) and maxBoxDim = dist (>= 0, +inf allowed); knn = sfe_icp_params.
 *                  normals_knn (3..64).  Reference side only, and only as its last filter.  The cloud is split into
 *                  boxes of at most knn points by median cuts (root bounds: the cloud's min and max; a range of more
 *                  than knn points is cut on the axis of its bounds' larger extent, x on a tie, its first count -
 *                  count / 2 points in (coordinate, index) order going left, the cut value being the next point's
 *                  coordinate); a box whose own points span more than maxBoxDim on an axis is dropped; every other box
 *                  gets the normal of its points in index order (the closed form of the knn normals above, over k
 *                  points); samplingMethod 1 keeps its lowest-index point moved to the box's float32 centroid, 0 keeps
 *                  all its points.  Kept points stay in index order, each with its box's normal, which point-to-plane
 *                  then reads instead of computing normals.
 *                  SFE_ICP_DATA_NORMALS {dim}: SurfaceNormalDataPointsFilter with knn = dim (3..16) on the reading
 *                  (reading side only, at most once per chain): every point gets the knn normal above, computed on the
 *                  cloud this filter receives, centred on its mean (sequential float32 sum / n).  The points do not
 *                  change.  Only distance filters and SFE_ICP_DATA_SHADOW may follow it; each survivor keeps its
 *                  normal.  The normals are dropped after the reading chain.
 *                  SFE_ICP_DATA_SHADOW {dist}: ShadowDataPointsFilter with eps = dist (finite, radians; reading side
 *                  only, after an SFE_ICP_DATA_NORMALS): keeps a point p (as the filter receives it, in the reading's
 *                  input frame) with normal n iff |n^ . p^| > sinf(eps), where v^ = v / sqrtf(v.v) when v.v > 0, else
 *                  v, the dot nx * px + ny * py, all float32 and nothing contracted; sinf is the host C library's.
 *                  It drops points whose surface runs along the line of sight from the sensor at the origin.
 *                  A target the filters empty is SFE_ICP_EMPTY_REF; a source they empty ends as an empty source does:
 *                  SFE_ICP_NO_OUTLIER with a quantile filter (trim_ratio or median_factor) on, else SFE_ICP_NO_POINT.
 *   min_dist       MinDistOutlierFilter minDist (< 0: off): keep pairs with d^2 > minDist^2 (sfe_icp_params.flags
 *                  bit 0: d^2 > minDist, as for MaxDist)
 *   median_factor  MedianDistOutlierFilter factor (< 0: off): keep d^2 <= factor * median, median = element
 *                  floor(n_finite * 0.5) of the ascending finite squared distances (no finite one: SFE_ICP_NO_OUTLIER)
 * Outlier weights are the product over the chain (with sfe_icp_params' MaxDist and TrimmedDist). */
enum { SFE_ICP_DATA_MAX_DIST = 1, SFE_ICP_DATA_MIN_DIST = 2, SFE_ICP_DATA_OCTREE = 3, SFE_ICP_DATA_VOXEL = 4,
       SFE_ICP_DATA_SAMPLING_NORMALS = 5, SFE_ICP_DATA_NORMALS = 6, SFE_ICP_DATA_SHADOW = 7,
       SFE_ICP_MAX_DATA_FILTERS = 4 };
typedef struct {
  int kind;   /* SFE_ICP_DATA_MAX_DIST, SFE_ICP_DATA_MIN_DIST, SFE_ICP_DATA_OCTREE, SFE_ICP_DATA_VOXEL,
                 SFE_ICP_DATA_SAMPLING_NORMALS, SFE_ICP_DATA_NORMALS or SFE_ICP_DATA_SHADOW */
  int dim;    /* distance filters: -1 radial, 0 x, 1 y; octree: the sampling method, 0, 2 or 3; voxel: useCentroid, 1;
                 sampling normals: samplingMethod, 0 or 1; normals: knn, 3..16; shadow: unused */
  float dist; /* distance filters: the distance; octree: maxSizeByNode; voxel: vSize; sampling normals: maxBoxDim;
                 normals: unused; shadow: eps (radians) */
} sfe_icp_data_filter;
typedef struct {
  float min_dist;
  float median_factor;
  int n_reading, n_reference; /* 0 .. SFE_ICP_MAX_DATA_FILTERS */
  sfe_icp_data_filter reading[SFE_ICP_MAX_DATA_FILTERS], reference[SFE_ICP_MAX_DATA_FILTERS];
} sfe_icp_filters;
/* sfe_icp_dev, sfe_icp_host and sfe_icp_batch_host for clouds of `dim` columns; guesses and results are (dim + 1)^2
 * row-major float32.  dim 2: the calls above, same launches and results.  dim 3: x, y, z in both clouds, libpointmatcher's
 * 3-D point-to-point chain (oracle/icp3_ref.c): exact 3-D nearest neighbours ((dx*dx + dy*dy) + dz*dz, ties to the lower
 * index, on a grid of x, y), the MaxDist and Trimmed weights, R = U V^T from a float32 restatement of Eigen's JacobiSVD of
 * the 3x3 cross-covariance with the reflection fix (a planar cloud whose 2-D fit would be a reflection gets a rotation
 * that flips z), Counter and Differential checkers on quaternions.  Same statuses and messages.  Targets above
 * sfe_icp_cta_limit(ctx, 3, ns_max) read map grids (sfe_icp_dev's workspace, plus 4 bytes per slot point).  Sources of
 * any size, as for dim 2: above sfe_icp_source_limit(ctx, prm, 3) (about 11 000 points on an H100) the global-source
 * class keeps reading, dist and match in global memory (20 bytes per ns_max point per CTA, two 256-thread CTAs per SM,
 * all slices within 512 MiB) and reads every target from a map grid.  dim 3 with
 * minimizer 1, flags bit 1 or ICP filters set on ctx is SFE_ERR_UNSUPPORTED, and nothing is launched; dim outside
 * 2 .. 3 is SFE_ERR_ARG. */
SFE_API int sfe_icp_dim_dev(sfe_ctx *ctx, const sfe_icp_params *prm, const float *src_pts_dev,
                            const int32_t *src_off_dev, const float *tgt_pts_dev, const int32_t *tgt_off_dev,
                            const int32_t *src_id_dev, const int32_t *tgt_id_dev, int n_problems, int dim, int ns_max,
                            int nt_max, const float *guess_dev, float *T_dev, int32_t *iters_dev, int32_t *inliers_dev,
                            int32_t *status_dev);
SFE_API int sfe_icp_dim_host(sfe_ctx *ctx, const sfe_icp_params *prm, const float *src_host, int ns,
                             const float *tgt_host, int nt, int dim, const float *guess_host, int n_guesses,
                             float *T_host, int32_t *iters_host, int32_t *inliers_host, int32_t *status_host);
SFE_API int sfe_icp_batch_dim_host(sfe_ctx *ctx, const sfe_icp_params *prm, const float *src_pts_host,
                                   const int32_t *src_off_host, int n_src_clouds, const float *tgt_pts_host,
                                   const int32_t *tgt_off_host, int n_tgt_clouds, const int32_t *src_id_host,
                                   const int32_t *tgt_id_host, int n_problems, int dim, const float *guess_host,
                                   float *T_host, int32_t *iters_host, int32_t *inliers_host, int32_t *status_host);
/* *limit = the largest target of `dim` columns that sfe_icp_dim_* solves in one CTA next to sources of ns points on this
 * context's device (dim 2: the shipped point-to-point chain without filters); larger targets take the map class */
SFE_API int sfe_icp_cta_limit(sfe_ctx *ctx, int dim, int ns, int32_t *limit);
/* *limit = the largest source of `dim` columns that sfe_icp_dev / sfe_icp_dim_* / the host flavours solve in their
 * shared-memory layouts next to targets of any size, for the settings prm and the ICP filters set on ctx, on this
 * context's device.  Larger sources take the global-source class (sfe_icp_dev), unless every target of the call fits
 * one CTA next to them (sfe_icp_cta_limit).  Settings the chain does not run are reported as by sfe_icp_dim_dev; dim
 * outside 2 .. 3 and null pointers are SFE_ERR_ARG. */
SFE_API int sfe_icp_source_limit(sfe_ctx *ctx, const sfe_icp_params *prm, int dim, int32_t *limit);
/* The SFE_ICP_DATA_SAMPLING_NORMALS stage of an ICP call alone, on n_clouds 2-D clouds packed with CSR offsets (device
 * memory; clouds of up to n_max points): cloud c's kept points, in index order, at out_pts_dev + 2 * c * n_max, their
 * boxes' normals at the same place of out_nrm_dev, their number in out_count_dev[c].  knn 3..64, method 0 or 1,
 * max_box >= 0 (+inf allowed).  Clouds of up to 4 096 points take one CTA each, larger ones the grid-wide path. */
SFE_API int sfe_icp_sampling_normals_dev(sfe_ctx *ctx, const float *pts_dev, const int32_t *off_dev, int n_clouds,
                                         int n_max, int knn, int method, float max_box, float *out_pts_dev,
                                         float *out_nrm_dev, int32_t *out_count_dev);
/* The SFE_ICP_DATA_NORMALS stage alone: the knn normal (knn 3..16) of every point of n_clouds 2-D clouds packed with CSR
 * offsets (device memory; clouds of up to n_max points; larger ones are not read), written in point order to
 * out_nrm_dev, laid out as the points (cloud c's point i at 2 * (off_dev[c] + i)).  Clouds of up to 4 096 points take
 * one CTA each with their grid in shared memory; larger ones are sorted into grids in global memory (sfe_icp_dev's map
 * grid workspace). */
SFE_API int sfe_icp_surface_normals_dev(sfe_ctx *ctx, const float *pts_dev, const int32_t *off_dev, int n_clouds,
                                        int n_max, int knn, float *out_nrm_dev);

/* The filters later sfe_icp_dev / _host / _batch_host and sfe_frontend_icp_dev calls on ctx apply (copied; NULL: none,
 * the default).  Checked here: no NaN, kind and dim known, an octree's maxSizeByNode and a voxel filter's vSize finite and
 * positive, counts in range, SFE_ICP_DATA_NORMALS and SFE_ICP_DATA_SHADOW on the reading only, SHADOW after a NORMALS
 * with a finite eps, only distance filters and SHADOW after a NORMALS; SFE_ERR_ARG leaves the setting as it was. */
SFE_API int sfe_icp_set_filters(sfe_ctx *ctx, const sfe_icp_filters *filters);

/* libpointmatcher's RobustOutlierFilter with scaleEstimator none / fixed (scale 1) and point2point residuals: a soft
 * M-estimator weight for every matched pair, from its squared distance e2 (the value MaxDist compares) and k = tuning,
 * k2 = k * k, all float32 with IEEE-rounded division and sqrt and nothing contracted:
 *   SFE_ICP_ROBUST_CAUCHY  1 / (1 + e2 / k2)              SFE_ICP_ROBUST_WELSCH  (float)exp((double)(-(e2 / k2)))
 *   SFE_ICP_ROBUST_SC      e2 >= k ? 4k2 / (k + e2)^2 : 1  SFE_ICP_ROBUST_GM      k2 / (k + e2)^2
 *   SFE_ICP_ROBUST_TUKEY   e2 >= k2 ? 0 : (1 - e2 / k2)^2  SFE_ICP_ROBUST_HUBER   e2 >= k2 ? k / sqrt(e2) : 1
 *   SFE_ICP_ROBUST_L1      1 / sqrt(e2)
 * and 0 where e2 >= approximation (+inf: no cut-off).  A pair's weight is the product with the 0 / 1 weights of the
 * other outlier filters (MaxDist, Trimmed, MinDist, Median): the robust weight where they keep the pair, else 0 -- NaN
 * for an L1 weight of inf (e2 == 0).  Pairs of non-zero weight are kept (inliers); the point-to-point minimiser takes
 * weighted means (sum w p) * (1 / sum w) and the cross-covariance sum (w (r - mean_r)) (p - mean_p)^T, the
 * point-to-plane one A = sum (w F) F^T and b = -sum (w F) ((q - r).n); every sum sequential in point order
 * (oracle/robust_ref.c).  2-D clouds only, float32 sums only (flags bit 1 is SFE_ERR_UNSUPPORTED with a robust filter).
 * The point-to-plane minimiser keeps its sum scratch apart from the distances, 2.5 KB more shared memory per CTA. */
enum { SFE_ICP_ROBUST_CAUCHY = 1, SFE_ICP_ROBUST_WELSCH = 2, SFE_ICP_ROBUST_SC = 3, SFE_ICP_ROBUST_GM = 4,
       SFE_ICP_ROBUST_TUKEY = 5, SFE_ICP_ROBUST_HUBER = 6, SFE_ICP_ROBUST_L1 = 7 };
typedef struct {
  int fct;             /* SFE_ICP_ROBUST_* */
  float tuning;        /* k: finite and positive */
  float approximation; /* weight 0 where e2 >= approximation; not NaN; +inf: no cut-off */
} sfe_icp_robust;
/* The RobustOutlierFilter later sfe_icp_dev / _host / _batch_host / sfe_icp_source_limit and sfe_frontend_icp_dev
 * calls on ctx apply (copied; NULL: none, the default).  Checked here: fct known, tuning finite and positive,
 * approximation not NaN; SFE_ERR_ARG leaves the setting as it was.  dim 3 calls with it set are SFE_ERR_UNSUPPORTED. */
SFE_API int sfe_icp_set_robust(sfe_ctx *ctx, const sfe_icp_robust *robust);

/* ------------------------------------------------------------------ robust covariance of ICP samples (row N1)
 * SLAM.compute_icp_with_cov, slam.py:365-371: MinCovDet(store_precision=False, support_fraction=0.8).fit(samples),
 * batched over n_problems candidates.  The algorithm is scikit-learn 1.9's (sklearn/covariance/_robust_covariance.py:
 * fast_mcd for n_samples <= 500, then MinCovDet.correct_covariance and reweight_covariance); releases before the
 * _consistency_factor correction reweight differently and are not what this computes.  See csrc/mcd.cu.
 *   samples      double [P][32][3], rows 0 .. n[p]-1 used (x, y, theta)
 *   n            int32 [P]; n > 32 is SFE_ERR_UNSUPPORTED (host flavour) or status SFE_MCD_UNSUPPORTED (device)
 *   subsets      int8 [P][30][32]: the 30 random trial supports, first h = int(0.8 n) entries used -- what
 *                np.random.permutation(n)[:h] gives for each of sklearn's 30 trials, in order
 *   c_support_host  double [33], ALWAYS host memory: entry n = _consistency_factor(3, int(0.8 n) / n)
 *   c_reweight   _consistency_factor(3, 0.975);  chi2_cut = chi2(3).isf(0.025)  (computed by the caller with scipy)
 *   flags        SFE_MCD_FLOAT32: the samples are float32 values and numpy's float32 arithmetic applies where
 *                sklearn keeps that dtype (the location mean, X - location); compute_icp_with_cov's samples are float32
 * Outputs per problem: location [3] and covariance [3][3] as MinCovDet leaves location_ / covariance_ (NaN unless
 * status is SFE_MCD_OK), raw_support / support as bit masks (bit i = sample i), status SFE_MCD_*. */
enum { SFE_MCD_TRIALS = 30, SFE_MCD_MAX_SAMPLES = 32, SFE_MCD_FLOAT32 = 1 };
enum {
  SFE_MCD_OK = 0,
  SFE_MCD_TOO_FEW = 1,     /* n < 5: "Too few samples for covariance computation" (slam.py:361-363) */
  SFE_MCD_ZERO_COV = 2,    /* correct_covariance's ValueError: "Failed to calculate covariance" (slam.py:365-371) */
  SFE_MCD_UNSUPPORTED = 3, /* n > 32 */
  SFE_MCD_BAD_SUBSET = 4   /* a trial support does not name h distinct rows below n */
};
SFE_API int sfe_mincovdet_dev(sfe_ctx *ctx, const double *samples_dev, const int32_t *n_dev, const int8_t *subsets_dev,
                              int n_problems, const double *c_support_host, double c_reweight, double chi2_cut,
                              int flags, double *location_dev, double *covariance_dev, uint32_t *raw_support_dev,
                              uint32_t *support_dev, int32_t *status_dev);
SFE_API int sfe_mincovdet_host(sfe_ctx *ctx, const double *samples_host, const int32_t *n_host,
                               const int8_t *subsets_host, int n_problems, const double *c_support_host,
                               double c_reweight, double chi2_cut, int flags, double *location_host,
                               double *covariance_host, uint32_t *raw_support_host, uint32_t *support_host,
                               int32_t *status_host);

/* ------------------------------------------------------------------ batched per-keyframe front end
 * One call for a backlog of frames: FeatureExtraction.callback (feature_extraction.py:196-252)
 * for every frame, then for every frame i the sequential scan match of SLAM
 * (slam.py:607-633,718-776): source = cloud i, target = clouds of frames i-window .. i-1 moved into
 * frame i-1 with the odometry poses and voxel-down-sampled (get_points, slam.py:229-292),
 * guess = between(pose[i-1], pose[i]), then ICP.  Frame 0 of a batch has no target (status
 * SFE_ICP_SKIPPED), frames 1 .. window-1 use the frames available.  Pose-graph optimisation is not
 * part of this library: the SE(2) results feed the caller's (CPU) ISAM2.
 */
typedef struct {
  int R, B;                 /* polar image: range bins x beams (must equal the maps') */
  int cfar_alg, train_hs, guard_hs, rank; /* feature.yaml CFAR/{alg, Ntc/2, Ngc/2, rank} */
  double tau;               /* threshold factor of that variant (CFAR.py:71-121, computed by the host) */
  int gate_enable;          /* feature.yaml filter/threshold: `peaks &= img > threshold` */
  double gate_threshold;
  float resolution;         /* feature.yaml filter/resolution (<= 0: no down-sampling) */
  double outlier_radius;    /* feature.yaml filter/radius */
  int outlier_min_points;   /* feature.yaml filter/min_points (<= 1: no outlier removal) */
  int window;               /* slam.yaml ssm/target_frames (3) */
  float submap_resolution;  /* slam.yaml point_resolution (0.5; <= 0: no down-sampling of the target) */
  int min_points;           /* slam.yaml ssm/min_points (50) */
  sfe_icp_params icp;
  int cap_points;           /* capacity (rows) reserved per frame for its Cartesian cloud; a frame with more
                               detections is truncated and reported as SFE_ICP_TOO_LARGE */
  int cap_source, cap_target; /* largest source / target cloud the scan matcher accepts */
  int flip_lateral;         /* != 0 (default 1, the reference's behaviour): the cloud SLAM matches on is
                               (forward, -lateral).  FeatureExtraction publishes points as xyz = [p0, 0, p1]
                               (feature_extraction.py:182) and the SLAM node reads them back as
                               np.c_[x, -z] = (p0, -p1) (slam_ros.py:169-170), so every keyframe cloud -- scan-match
                               source, window submap, and the clouds sfe_frontend_results_dev exposes -- has its
                               lateral coordinate negated AFTER the feature filters.  0 keeps
                               FeatureExtraction.callback's own (p0, p1) convention. */
} sfe_frontend_params;
SFE_API void sfe_frontend_params_default(sfe_frontend_params *p);

typedef struct sfe_frontend sfe_frontend;
SFE_API int sfe_frontend_create(sfe_ctx *ctx, const sfe_maps *maps, const sfe_frontend_params *params,
                                int max_frames, sfe_frontend **out);
SFE_API void sfe_frontend_destroy(sfe_frontend *fe);
/* frames: uint8 [n_frames][R][B]; poses: float64 [n_frames][3] = odometry (x, y, theta) of every
 * frame in a common frame, always in HOST memory (24 B per frame).  Device flavour: frames already in
 * device memory, asynchronous, results stay on the device
 * (sfe_frontend_results_dev).  Host flavour: copies frames in chunks of `chunk_frames` (<= 0: 256)
 * overlapped with the kernels, copies the results back and returns when they are there:
 * T [n][9] (row-major 3x3, source -> previous frame), iterations, inliers, status (SFE_ICP_*),
 * npoints (size of every frame's filtered cloud; may be NULL). */
SFE_API int sfe_frontend_run_dev(sfe_frontend *fe, const uint8_t *frames_dev, const double *poses_host, int n_frames);
SFE_API int sfe_frontend_results_dev(const sfe_frontend *fe, const float **T, const int32_t **iters,
                                     const int32_t **inliers, const int32_t **status, const float **cloud_xy,
                                     const int32_t **cloud_count, int32_t *cloud_stride);
/* Continuation across calls (SURVEY 8(f) N3: the window submap stays resident on the device).  With carry enabled,
 * every call keeps the clouds and odometry poses of its last `window` frames on the device, and the next call on
 * this handle continues the sequence: its first frames are matched against the carried frames (frame 0 included),
 * exactly as if the batches had been one call -- a replay can be fed in pieces of any size without a cold window at
 * every seam.  enable = 0 (the default) drops the carried frames: every call starts cold (frame 0 SFE_ICP_SKIPPED). */
SFE_API int sfe_frontend_set_carry(sfe_frontend *fe, int enable);
/* Feature images from the front end.  With dst != NULL, every later run call on this handle also writes frame i's
 * feature image (as sfe_feature_image_dev, table lut_bgr_host, copied by this call) to dst + i * rows * cols * 3.
 * sfe_frontend_run_dev needs dst in device memory (dst_is_host = 0; asynchronous like the rest of the call);
 * sfe_frontend_run_host / _run_jpeg_host / _run_png_host need it in host memory (dst_is_host != 0): each chunk is
 * rendered as soon as its frames are on the device, into a double-buffered device staging area (chunk_frames images,
 * allocated on first use) that is copied out while later chunks compute, and the call returns after the last image has
 * landed.  Pinned host memory lets the copies run asynchronously.  dst = NULL (the default) turns it off.  The numeric
 * results are the same with and without images. */
SFE_API int sfe_frontend_set_feature_images(sfe_frontend *fe, const uint8_t *lut_bgr_host, uint8_t *dst,
                                            int dst_is_host);
/* Optional per-stage device timing (CUDA events on the context's stream around every stage's kernels).
 * get_timing synchronises, adds the intervals recorded since the last call to running totals and
 * returns the totals: stage_ms[SFE_FE_STAGES], stage_calls[SFE_FE_STAGES] (may be NULL). */
enum { SFE_FE_CFAR = 0, SFE_FE_CART = 1, SFE_FE_DOWNSAMPLE = 2, SFE_FE_OUTLIER = 3, SFE_FE_SUBMAP = 4,
       SFE_FE_ICP = 5, SFE_FE_STAGES = 6 };
SFE_API int sfe_frontend_set_timing(sfe_frontend *fe, int enable);
SFE_API int sfe_frontend_get_timing(sfe_frontend *fe, double *stage_ms, int64_t *stage_calls);
SFE_API int sfe_frontend_run_host(sfe_frontend *fe, const uint8_t *frames_host, const double *poses_host,
                                  int n_frames, int chunk_frames, float *T_host, int32_t *iters_host,
                                  int32_t *inliers_host, int32_t *status_host, int32_t *npoints_host);
/* Every frame's filtered cloud, packed.  With dst != NULL, every later run call on this handle (all flavours) also
 * writes the clouds of its frames one after another: frame i's cloud is dst[offsets[i] .. offsets[i + 1]) as float32
 * (x, y) pairs, in the front end's flip_lateral convention (1: SLAM's (x, -z); 0: FeatureExtraction.callback's
 * (p0, p1)), the points those of sfe_frontend_results_dev's strided clouds; offsets int64 [n_frames + 1], offsets[0] =
 * 0.  Both live in host memory (on_host != 0) for the host, geometry, JPEG and PNG flavours and in device memory
 * (on_host = 0) for sfe_frontend_run_dev[_geometry]; a call of the other kind is rejected before any device work.
 * The host flavours copy each chunk's clouds out while later chunks compute; run_dev writes them on the device and then
 * waits for the call to finish, to check the capacity.  A call whose clouds need more than capacity_points points fails
 * with SFE_ERR_CAPACITY, its message stating the total needed: offsets is filled all the same, no point is written
 * past the capacity, the other outputs are unspecified and the carried window (sfe_frontend_set_carry) stays as it
 * was, so a retry with a larger buffer continues the sequence.  dst = NULL (the default) turns it off; the other
 * results are the same with and without clouds. */
SFE_API int sfe_frontend_set_clouds(sfe_frontend *fe, float *dst, int64_t capacity_points, int64_t *offsets,
                                    int on_host);
/* enable = 0: every run flavour computes the clouds only.  The window submaps and ICP are not launched; every frame's
 * status is SFE_ICP_SKIPPED (SFE_ICP_TOO_LARGE where its Cartesian cloud overflowed cap_points), T the identity,
 * iterations and inliers 0.  With carry on the carried window still advances, so turning the scan match back on
 * continues the sequence.  enable != 0: the default. */
SFE_API int sfe_frontend_set_scan_match(sfe_frontend *fe, int enable);
/* The ICP filters (sfe_icp_filters) of this front end's scan match, from the next run call on (copied; NULL: none, the
 * default).  The reading filters see each frame's cloud, the reference filters its window submap; the min_points test
 * still counts the clouds before the filters (slam.py checks them before ICP runs). */
SFE_API int sfe_frontend_set_icp_filters(sfe_frontend *fe, const sfe_icp_filters *filters);
/* The RobustOutlierFilter (sfe_icp_robust) of this front end's scan match, from the next run call on (copied; NULL:
 * none, the default); checked as by sfe_icp_set_robust. */
SFE_API int sfe_frontend_set_icp_robust(sfe_frontend *fe, const sfe_icp_robust *robust);
/* Several sonar geometries in one front end: a bag whose range setting changes (num_ranges, range_resolution, beam
 * count) is fed as one sequence, and the first frames after a change are matched against the keyframes before it, as
 * the reference's window of metric keyframe clouds does (slam.py:632-633).
 *
 * sfe_frontend_add_geometry registers `maps` as a further geometry and returns its id; the creation maps are geometry
 * 0.  The geometry must fit the frame slots the front end was created with (maps->R <= params.R, maps->B <= params.B);
 * nothing is reallocated.  The front end keeps `maps` referenced (it does not own it).  At most
 * SFE_FE_MAX_GEOMETRIES geometries, the creation maps included.
 *
 * The *_geometry run flavours take one geometry id per frame (geometry, int32 [n_frames], HOST memory), checked before
 * any device work; otherwise they are the flavours above, carry and schedule included.  The feature stages (CFAR,
 * Cartesian points) run once per maximal run of consecutive frames of one geometry; everything after the Cartesian
 * points runs over the whole batch (or chunk) as before.
 *   _run_dev_geometry:  frame i of geometry g occupies the first R_g * B_g bytes of its slot, frames_dev + i * R * B,
 *                       row-major [R_g][B_g].
 *   _run_host_geometry: frames packed as the compressed flavours pack streams: frame i = bytes[offsets[i] ..
 *                       offsets[i + 1]), exactly R_g * B_g bytes (offsets int64 [n_frames + 1]).
 *   _run_jpeg_host_geometry / _run_png_host_geometry: every stream must decode to its own geometry's R_g x B_g.
 * Feature images (sfe_frontend_set_feature_images) need every frame of a call in one geometry; they then have that
 * geometry's rows x cols.  A call whose frames have more than one geometry is rejected while images are set. */
enum { SFE_FE_MAX_GEOMETRIES = 8 };
SFE_API int sfe_frontend_add_geometry(sfe_frontend *fe, const sfe_maps *maps, int *geometry_id);
SFE_API int sfe_frontend_run_dev_geometry(sfe_frontend *fe, const uint8_t *frames_dev, const int32_t *geometry,
                                          const double *poses_host, int n_frames);
SFE_API int sfe_frontend_run_host_geometry(sfe_frontend *fe, const uint8_t *bytes, const int64_t *offsets,
                                           const int32_t *geometry, const double *poses_host, int n_frames,
                                           int chunk_frames, float *T_host, int32_t *iters_host,
                                           int32_t *inliers_host, int32_t *status_host, int32_t *npoints_host);

/* ------------------------------------------------------------------ global-initialisation cost (next row N2)
 * SLAM.get_matching_cost_subroutine1 (slam.py:461-570), the function scipy.shgo minimises in
 * initialize_sequential_scan_matching (slam.py:683-701) and initialize_nonsequential_scan_matching
 * (slam.py:943-961): an occupancy grid of the target cloud at `resolution` (= point_noise / 10), dilated by an
 * elliptical structuring element, and for a candidate transform the NEGATED number of transformed source points
 * that land on an occupied cell.
 *
 * The grid geometry is computed by the caller exactly like slam.py:507-512 (xmin/ymin = cloud minimum minus
 * 2 * point_noise as float32; rows/cols = lengths of the two np.arange calls).  Cell of a point (slam.py:516-517,
 * 556-557), all in float32 like numpy:  r = int(rint((y - ymin) / resolution)), c = int(rint((x - xmin) / resolution)),
 * target cells clipped into the grid, source cells outside the grid not counted.  The structuring element is
 * passed as one column span [se_lo[j], se_hi[j]) per row j of the (2 * dilate_hs + 1)^2 kernel (empty row: lo >= hi)
 * -- for cv2.getStructuringElement(MORPH_ELLIPSE, ...) the caller evaluates OpenCV's span formula (slam.py:523-527).
 * A candidate transform is 6 floats {r00, r01, r10, r11, tx, ty} = sample_transform.matrix().astype(float32)
 * (slam_objects.py:195); points move as x' = fma(y, r01, x * r00) + tx (what numpy's float32 dot does).  */
typedef struct sfe_costmap sfe_costmap;
SFE_API int sfe_costmap_create(sfe_ctx *ctx, const float *target_xy_host, int n_target, float xmin, float ymin,
                               float resolution, int rows, int cols, int dilate_hs, const int32_t *se_lo,
                               const int32_t *se_hi, sfe_costmap **out);
SFE_API void sfe_costmap_destroy(sfe_costmap *cm);
/* the dilated grid as the reference holds it: uint8 [rows][cols], 0 or 255 */
SFE_API int sfe_costmap_grid_host(sfe_ctx *ctx, const sfe_costmap *cm, uint8_t *grid_host);
/* source cloud of the closure (kept on the device between evaluations) */
SFE_API int sfe_costmap_set_source_host(sfe_ctx *ctx, sfe_costmap *cm, const float *source_xy_host, int n_source);
/* cost[k] = -(number of source points on occupied cells under transform k); K candidates in one launch */
SFE_API int sfe_costmap_score_host(sfe_ctx *ctx, const sfe_costmap *cm, const float *transforms_host, int n_candidates,
                                   int32_t *cost_host);
/* device flavour: source cloud, transforms and costs in device memory, asynchronous on the context's stream */
SFE_API int sfe_costmap_score_dev(sfe_ctx *ctx, const sfe_costmap *cm, const float *source_xy_dev, int n_source,
                                  const float *transforms_dev, int n_candidates, int32_t *cost_dev);

/* ------------------------------------------------------------------ loop-closure target pre-filter (next row N3)
 * SLAM.initialize_nonsequential_scan_matching, slam.py:878-899: keep the points of the accumulated target cloud that
 * lie inside the field of view of at least one of the n_frames source keyframes, range and aperture inflated by the
 * keyframe's pose uncertainty.  Per source keyframe k the caller passes (computed on the host exactly like
 * slam.py:883-888):
 *   inv_T[k]          6 floats {r00, r01, r10, r11, tx, ty} of pose.inverse().matrix().astype(float32)
 *                     (Keyframe.transform_points, slam_objects.py:195)
 *   range_bound[k]    translation_std * 5.0 + oculus.max_range                       (float64)
 *   bearing_bound[k]  rotation_std * 5.0 + oculus.horizontal_aperture * 0.5          (float64)
 * pts: float32 [n][2] (global frame); sel[i] = 1 iff for some k the point moved into keyframe k's frame has
 * float32 norm < range_bound[k] and |float32 atan2| < bearing_bound[k]  (the `sel |= sel_i` loop, slam.py:879-895). */
SFE_API int sfe_fov_select_dev(sfe_ctx *ctx, const float *pts_dev, int n, const float *inv_T_dev,
                               const double *range_bound_dev, const double *bearing_bound_dev, int n_frames,
                               uint8_t *sel_dev);
SFE_API int sfe_fov_select_host(sfe_ctx *ctx, const float *pts_host, int n, const float *inv_T_host,
                                const double *range_bound_host, const double *bearing_bound_host, int n_frames,
                                uint8_t *sel_host);

/* ------------------------------------------------------------------ resident keyframe map (row N3)
 * SLAM.get_points (slam.py:229-292) without re-sending the map: the keyframe clouds are stored once on the device, in
 * local coordinates, and every call assembles the requested keyframes under that call's poses and down-samples the
 * result like bruce_slam.pcl.downsample (sfe_downsample_*), with the same results as the host lines
 *     np.concatenate([transform_points(kf.points, pose) (, key)]) -> pcl.downsample(points (, keys), resolution)
 * Poses are not stored: the caller computes each entry's transform on the host, as get_points does.
 *
 * A map belongs to the context it was created with (its stream runs every call) and is destroyed before it.  Its arena
 * of float32 (x, y) points starts with room for `initial_points` (0: 65 536) and doubles when an append needs more,
 * keeping the stored clouds (device-to-device copy on the context's stream).  Clouds get consecutive slot ids from 0 in
 * append order; the map holds at most 2^31 - 2 points.
 *
 * Appends (slots_host int32 [n_clouds] receives the slot ids assigned; may be NULL):
 *   _append_host  points float32 [sum counts][2] packed in cloud order, counts int32 [n_clouds] (>= 0), host memory;
 *                 returns when the points are on the device.
 *   _append_dev   clouds already on the device in sfe_frontend_results_dev's layout: cloud c = cloud_count_dev[c]
 *                 points at cloud_xy_dev + 2 * c * cloud_stride (a count above cloud_stride keeps cloud_stride points,
 *                 as the front end's window assembly does).  The counts are read back (one small copy) and returned in
 *                 counts_host int32 [n_clouds] (may be NULL).
 * Assemble: n_entries entries (all in HOST memory: they index the map's host-side table) of
 *     slots_host      int32 [K]     the cloud of entry k (repeats allowed)
 *     keys_host       float32 [K]   the key every point of entry k carries (NULL when no keys are requested)
 *     transforms_host float32 [K][6] {r00, r01, r10, r11, tx, ty} = that entry's pose.matrix().astype(float32)
 *                     (Keyframe.transform_points, slam_objects.py:195); points move as x' = fma(y, r01, x * r00) + tx
 * The entries' points, moved, form one cloud in entry order (N = sum of the entries' counts, at most 2^31 - 2); it is
 * down-sampled at `resolution` (> 0): out_pts float32 [M][2], with out_keys non-NULL out_keys float32 [M] (the key of
 * the entry each kept point came from), n_out = M.  The outputs must hold `capacity` >= N rows (else SFE_ERR_CAPACITY).
 * Bad slots, negative counts, totals above the limit and a non-positive resolution are rejected before any device
 * work.  Workspace, kept with the map between calls: 12 bytes per assembled point (16 with keys; the host flavour 8 (12)
 * more for its device-side outputs) and 36 bytes per entry (the uploaded table), plus the down-sample's own (48 bytes
 * per point above the one-CTA limit, in the context).
 *   _assemble_dev   outputs in device memory, asynchronous on the context's stream.
 *   _assemble_host  outputs in host memory (only the M kept rows are copied back); returns when they are there. */
typedef struct sfe_keyframe_map sfe_keyframe_map;
SFE_API int sfe_keyframe_map_create(sfe_ctx *ctx, int initial_points, sfe_keyframe_map **out);
SFE_API void sfe_keyframe_map_destroy(sfe_keyframe_map *km);
SFE_API int sfe_keyframe_map_size(const sfe_keyframe_map *km, int *n_clouds, int64_t *n_points);
SFE_API int sfe_keyframe_map_append_host(sfe_keyframe_map *km, const float *pts_host, const int32_t *counts_host,
                                         int n_clouds, int32_t *slots_host);
SFE_API int sfe_keyframe_map_append_dev(sfe_keyframe_map *km, const float *cloud_xy_dev, const int32_t *cloud_count_dev,
                                        int cloud_stride, int n_clouds, int32_t *slots_host, int32_t *counts_host);
SFE_API int sfe_keyframe_map_assemble_dev(sfe_keyframe_map *km, const int32_t *slots_host, const float *keys_host,
                                          const float *transforms_host, int n_entries, float resolution, int capacity,
                                          float *out_pts_dev, float *out_keys_dev, int32_t *n_out_dev);
SFE_API int sfe_keyframe_map_assemble_host(sfe_keyframe_map *km, const int32_t *slots_host, const float *keys_host,
                                           const float *transforms_host, int n_entries, float resolution, int capacity,
                                           float *out_pts_host, float *out_keys_host, int32_t *n_out);

/* ------------------------------------------------------------------ compressed pings (row N4)
 * feature_extraction.py:210-213 (compressed_images: True): cv2.cvtColor(cv2.imdecode(buf, IMREAD_COLOR), BGR2GRAY),
 * i.e. libjpeg-turbo's default decompression (JDCT_ISLOW, fancy upsampling) followed by OpenCV's fixed-point
 * BGR -> gray.  The decoder reproduces that uint8 frame bit for bit for the streams it accepts:
 *   baseline / extended sequential Huffman (SOF0, SOF1), 8-bit samples, one interleaved scan;
 *   1 component, or 3 components that libjpeg-turbo takes as YCbCr (JFIF marker, ids 1/2/3, Adobe transform 1);
 *   sampling 4:4:4, 4:2:2 (luma 2x1), 4:2:0 (luma 2x2); any restart interval; 8- and 16-bit DQT tables;
 *   tables that differ from frame to frame; APPn / COM segments are skipped.
 * Everything else gets a per-stream status (sfe_jpeg_status_message names the reason); PNG stays on the host path.
 * Streams are packed: stream i = bytes[offsets[i] .. offsets[i+1]), offsets int64 [n + 1].  See csrc/jpeg.cu. */
enum {
  SFE_JPEG_OK = 0,
  SFE_JPEG_NOT_JPEG = 1,     /* no SOI marker (PNG, random bytes ...) */
  SFE_JPEG_TRUNCATED = 2,    /* the headers end before the start of scan */
  SFE_JPEG_PROGRESSIVE = 3,
  SFE_JPEG_LOSSLESS = 4,
  SFE_JPEG_ARITHMETIC = 5,
  SFE_JPEG_PRECISION = 6,    /* sample precision other than 8 (12-bit) */
  SFE_JPEG_SAMPLING = 7,     /* 4:1:1, 4:4:0 and other factors */
  SFE_JPEG_COLORSPACE = 8,   /* CMYK / YCCK, 2 components, RGB (Adobe transform 0, R/G/B ids) */
  SFE_JPEG_ORIENTATION = 9,  /* EXIF orientation other than 1: imdecode would rotate the image */
  SFE_JPEG_SIZE = 10,        /* decoders only: frame size differs from the call's R x B */
  SFE_JPEG_CORRUPT = 11,     /* decoders only: invalid Huffman code, run past coefficient 63, data ending before the
                                last MCU of a segment (libjpeg-turbo pads such data with zeros and warns), missing or
                                out-of-sequence RSTn.  Data after a segment's last MCU is skipped, as libjpeg-turbo
                                skips it */
  SFE_JPEG_BAD_HEADER = 12   /* malformed tables, multi-scan or partial scans, hierarchical mode */
};
/* sampling codes of sfe_jpeg_inspect_host */
enum { SFE_JPEG_GRAY = 0, SFE_JPEG_444 = 1, SFE_JPEG_422 = 2, SFE_JPEG_420 = 3, SFE_JPEG_INFO = 6 };
SFE_API const char *sfe_jpeg_status_message(int status);
/* Headers only, no context, no GPU.  info int32 [n][SFE_JPEG_INFO]: status, height, width, components, sampling code
 * (-1 unless status is SFE_JPEG_OK), restart interval (MCUs; 0 = none). */
SFE_API int sfe_jpeg_inspect_host(const uint8_t *bytes, const int64_t *offsets, int n, int32_t *info);
/* Decode n streams into uint8 [n][R][B] frames (host memory / device memory of the context's GPU).  Headers are
 * parsed on the host; the entropy-coded bytes go in chunk by chunk on a copy stream, overlapped with decoding, and
 * device scratch is bounded by the chunk.  status_host int32 [n]: SFE_JPEG_*; a frame whose status is not
 * SFE_JPEG_OK is written as zeros.  Both return when the frames and statuses are there. */
SFE_API int sfe_jpeg_decode_host(sfe_ctx *ctx, const uint8_t *bytes, const int64_t *offsets, int n, int R, int B,
                                 uint8_t *out_host, int32_t *status_host);
SFE_API int sfe_jpeg_decode_to_dev(sfe_ctx *ctx, const uint8_t *bytes_host, const int64_t *offsets_host, int n, int R,
                                   int B, uint8_t *out_dev, int32_t *status_host);
/* Diagnostic: the dequantised coefficient blocks the IDCT consumes, int32 [n][cap_blocks][64] in natural order, blocks
 * in decode (MCU) order, zeros after a frame's last block and for frames whose status is not SFE_JPEG_OK.
 * SFE_ERR_CAPACITY when a frame has more than cap_blocks blocks. */
/* Optional per-stage device timing of the decoders (CUDA events on the context's stream around the kernels of every
 * chunk).  get_timing synchronises, adds the intervals recorded since the last call to running totals and returns them:
 * stage_ms[SFE_JPEG_STAGES], stage_calls[SFE_JPEG_STAGES] (may be NULL). */
enum { SFE_JPEG_T_UNSTUFF = 0, SFE_JPEG_T_ENTROPY = 1, SFE_JPEG_T_PIXELS = 2 /* IDCT + colour */, SFE_JPEG_STAGES = 3 };
SFE_API int sfe_jpeg_set_timing(sfe_ctx *ctx, int enable);
SFE_API int sfe_jpeg_get_timing(sfe_ctx *ctx, double *stage_ms, int64_t *stage_calls);
SFE_API int sfe_jpeg_coefficients_host(sfe_ctx *ctx, const uint8_t *bytes, const int64_t *offsets, int n, int R, int B,
                                       int cap_blocks, int32_t *coef_host, int32_t *status_host);
/* sfe_frontend_run_host with compressed pings: the copy of raw frames is replaced by the copy of the streams' bytes
 * and the decode into the front end's frame buffer.  Carry, chunking and results are those of sfe_frontend_run_host.
 * A stream that is rejected (checked for all n before any work) or fails to decode makes the call return
 * SFE_ERR_ARG naming the first such frame, before any front-end stage runs on its chunk. */
SFE_API int sfe_frontend_run_jpeg_host(sfe_frontend *fe, const uint8_t *bytes, const int64_t *offsets,
                                       const double *poses_host, int n_frames, int chunk_frames, float *T_host,
                                       int32_t *iters_host, int32_t *inliers_host, int32_t *status_host,
                                       int32_t *npoints_host);

/* PNG pings: the same cv2.imdecode(IMREAD_COLOR) + BGR2GRAY frame, bit for bit, for the streams a ping encoder
 * writes: IHDR with bit depth 8, colour type 0 (gray) or 2 (truecolour), no interlace; any number of IDAT chunks;
 * stored, fixed and dynamic deflate blocks with any window; the five row filters.  Ancillary chunks are ignored as
 * libpng ignores them.  Gray samples are the image; truecolour goes through OpenCV 4.x's BGR2GRAY.  Everything else
 * gets a per-stream status.  Inflated data past the last row is skipped (libpng warns "Too much image data") but must
 * still be valid deflate with a matching Adler-32.  Streams are packed as for JPEG.  See csrc/png.cu. */
enum {
  SFE_PNG_OK = 0,
  SFE_PNG_NOT_PNG = 1,      /* no PNG signature (JPEG, random bytes ...) */
  SFE_PNG_TRUNCATED = 2,    /* the chunk list ends before IEND */
  SFE_PNG_BAD_HEADER = 3,   /* malformed IHDR (or its CRC), no IDAT, IDATs not consecutive, unknown critical chunk,
                               PLTE after IDAT, width or height 0 or above libpng's 1000000 limit */
  SFE_PNG_DEPTH = 4,        /* bit depth other than 8 */
  SFE_PNG_COLORTYPE = 5,    /* palette, gray + alpha, RGBA */
  SFE_PNG_INTERLACED = 6,   /* Adam7 */
  SFE_PNG_ORIENTATION = 7,  /* eXIf orientation other than 1: imdecode would rotate the image */
  SFE_PNG_ANIMATED = 8,     /* acTL chunk (APNG) */
  SFE_PNG_SIZE = 9,         /* decoders only: frame size differs from the call's R x B */
  SFE_PNG_CORRUPT = 10      /* decoders only: IDAT CRC, zlib header, invalid deflate (reserved block type, stored
                               LEN / NLEN, bad code lengths, invalid symbol, distance beyond the output or the
                               declared window), Adler-32, filter byte above 4, too little image data */
};
enum { SFE_PNG_INFO = 5 };
SFE_API const char *sfe_png_status_message(int status);
/* Chunk list only, no context, no GPU.  info int32 [n][SFE_PNG_INFO]: status, height, width, colour type, number of
 * IDAT chunks (geometry as far as the IHDR could be read, else 0). */
SFE_API int sfe_png_inspect_host(const uint8_t *bytes, const int64_t *offsets, int n, int32_t *info);
/* As sfe_jpeg_decode_host / _to_dev: uint8 [n][R][B] frames, status_host int32 [n] SFE_PNG_*; a frame whose status is
 * not SFE_PNG_OK is written as zeros. */
SFE_API int sfe_png_decode_host(sfe_ctx *ctx, const uint8_t *bytes, const int64_t *offsets, int n, int R, int B,
                                uint8_t *out_host, int32_t *status_host);
SFE_API int sfe_png_decode_to_dev(sfe_ctx *ctx, const uint8_t *bytes_host, const int64_t *offsets_host, int n, int R,
                                  int B, uint8_t *out_dev, int32_t *status_host);
/* Per-stage device timing, as sfe_jpeg_set_timing / _get_timing. */
enum { SFE_PNG_T_CHECK = 0 /* IDAT CRC + gather */, SFE_PNG_T_INFLATE = 1, SFE_PNG_T_UNFILTER = 2 /* + gray, Adler */,
       SFE_PNG_STAGES = 3 };
SFE_API int sfe_png_set_timing(sfe_ctx *ctx, int enable);
SFE_API int sfe_png_get_timing(sfe_ctx *ctx, double *stage_ms, int64_t *stage_calls);
/* sfe_frontend_run_jpeg_host with PNG streams. */
SFE_API int sfe_frontend_run_png_host(sfe_frontend *fe, const uint8_t *bytes, const int64_t *offsets,
                                      const double *poses_host, int n_frames, int chunk_frames, float *T_host,
                                      int32_t *iters_host, int32_t *inliers_host, int32_t *status_host,
                                      int32_t *npoints_host);
/* The compressed flavours with one geometry id per frame (sfe_frontend_add_geometry). */
SFE_API int sfe_frontend_run_jpeg_host_geometry(sfe_frontend *fe, const uint8_t *bytes, const int64_t *offsets,
                                                const int32_t *geometry, const double *poses_host, int n_frames,
                                                int chunk_frames, float *T_host, int32_t *iters_host,
                                                int32_t *inliers_host, int32_t *status_host, int32_t *npoints_host);
SFE_API int sfe_frontend_run_png_host_geometry(sfe_frontend *fe, const uint8_t *bytes, const int64_t *offsets,
                                               const int32_t *geometry, const double *poses_host, int n_frames,
                                               int chunk_frames, float *T_host, int32_t *iters_host,
                                               int32_t *inliers_host, int32_t *status_host, int32_t *npoints_host);

#ifdef __cplusplus
}
#endif
#endif /* SONARFE_H_ */
