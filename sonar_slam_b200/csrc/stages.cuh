// Stage launchers shared by the C entry points and the batched front end (pipeline.cu).  Each one checks its
// arguments, then enqueues all of its work -- launches, memsets, scratch growth -- on `st` and nowhere else, so a
// caller may run stages on streams of its own.  Returns an SFE_* code.
#pragma once
#include "common.cuh"

namespace sfe {

// A batch of 2-D point clouds packed row-wise: cloud c starts at row off[c] of pts.  Its point count is cnt[c] or,
// with cnt null, off[c + 1] - off[c].  n_max bounds every count and sizes the launches.
struct PackedClouds {
  const float *pts;
  const int *off;
  const int *cnt;
  int n_max;
};

// P scan-matching problems: problem p moves source src_id[p] onto target tgt_id[p] (null ids: cloud p) from
// guess[p].  Problems whose source or target has fewer than min_points points are skipped; with raw_cnt, a source
// whose raw cloud had more than raw_cap points is reported too large.
struct IcpProblems {
  PackedClouds src, tgt;
  const int *src_id, *tgt_id;
  int P;
  const float *guess;  // [P][9] row-major 3x3
  float *T_out;        // [P][9]
  int *iters, *inliers, *status;
  int min_points;
  const int *raw_cnt;
  int raw_cap;
  int n_tgt_clouds;  // number of target clouds when the caller knows it (bounds the map grids, icp.cu), else 0
  int n_src_clouds;  // number of source clouds when the caller knows it (the data filters run once per cloud), else 0
};

int cfar_run(sfe_ctx *ctx, cudaStream_t st, const void *img, int dtype, int F, int R, int B, int alg, int T, int G,
             int k, double tau, int gate_on, double gate, uint8_t *mask, float *thr, uint32_t *bits);
int cart_points_run(sfe_ctx *ctx, cudaStream_t st, const sfe_maps *m, const uint8_t *mask, const uint32_t *bits, int F,
                    int cap, int32_t *ij, float *xy, int32_t *count);
int feature_image_run(sfe_ctx *ctx, cudaStream_t st, const sfe_maps *m, const uint8_t *frames, int F,
                      const uint8_t *lut_bgr, uint8_t *out, const char *what);  // what: the caller, for errors
// n_split > 0: two launches of the one-CTA kernel by cloud size (cloud.cu; n_max at most 65 535 points),
// DS_ANY_SIZE: clouds of any size (one-CTA kernel up to the device's limit, grid-wide path above it).  slot: scratch
// buffer, counter: work counter (WORK_*) of the one-CTA launches.  sampler: the point every leaf keeps, numbered as
// libpointmatcher's samplingMethod -- DS_MEDOID (pcl.downsample), or, for 2-D clouds with DS_ANY_SIZE, DS_FIRST (the
// leaf's lowest-index member) and DS_CENTROID (float32 sequential means); out_idx then names the leaf's first member.
constexpr int DS_ANY_SIZE = -1;
enum { DS_FIRST = 0, DS_CENTROID = 2, DS_MEDOID = 3 };
int downsample_run(sfe_ctx *ctx, cudaStream_t st, const PackedClouds &in, int n_clouds, int dim, float resolution,
                   float *out_pts, int32_t *out_idx, int32_t *out_count, int n_split, int slot, int counter,
                   int sampler = DS_MEDOID);
// VoxelGridDataPointsFilter (vSize, useCentroid) on every 2-D cloud of `in` (clouds above in.n_max points are not read):
// the first point of every voxel, in point order, holding its voxel's centroid, at out_off[c]; out_count[c] its number.
// A cloud whose voxel index would not fit 32 bits sets *overflow (device) to 1.  Workspace: scratch[SCR_DS_GRID].
int voxel_filter_run(sfe_ctx *ctx, cudaStream_t st, const PackedClouds &in, int n_clouds, float vsize, float *out_pts,
                     int *out_off, int *out_count, int *overflow);
// SamplingSurfaceNormalDataPointsFilter {knn, samplingMethod `method` (0: every point, 1: one per box), maxBoxDim
// `max_box`} on every 2-D cloud of `in` (statement oracle/sampling_normal_ref.c; clouds above in.n_max points are not
// read): the kept points in index order at c * n_max of out_pts, their box's normal at the same place of out_nrm,
// out_off[c] = c * n_max, out_count[c] their number.  ws: sampling_normals_ws(n_clouds, in.n_max, knn) bytes.
int sampling_normals_ws(int n_clouds, int n_max, int knn, size_t *bytes);
int sampling_normals_run(sfe_ctx *ctx, cudaStream_t st, const PackedClouds &in, int n_clouds, int knn, int method,
                         float max_box, void *ws, float *out_pts, int *out_off, int *out_count, float2 *out_nrm);
// SurfaceNormalDataPointsFilter {knn 3..16} on every 2-D cloud of `in` (statement oracle/shadow_ref.c; clouds above
// in.n_max points are not read): the knn normal of point i of cloud c, computed on the cloud centred on its mean, at
// out_nrm[in.off[c] + i].  Clouds of up to 4 096 points take one CTA each, larger ones map grids (map_build, in
// scratch[SCR_MAP]).  ws: surface_normals_ws(n_clouds, in.n_max) bytes.
int surface_normals_ws(int n_clouds, int n_max, size_t *bytes);
int surface_normals_run(sfe_ctx *ctx, cudaStream_t st, const PackedClouds &in, int n_clouds, int knn, void *ws,
                        float2 *out_nrm);
// the largest cloud of `dim` columns (2 or 3) downsample_run's one-CTA kernel lays out in shared memory on this device
int downsample_cta_limit(const sfe_ctx *ctx, int *limit, int dim);
// n_split > 0: two launches by cloud size (front end), 0: clouds of any size (one-CTA kernel up to the device's limit,
// the map class above it)
int remove_outlier_run(sfe_ctx *ctx, cudaStream_t st, const PackedClouds &in, int n_clouds, int dim, double radius,
                       int min_points, float *out_pts, int32_t *out_idx, int32_t *out_count, int n_split);
// One size class of icp_run: problems whose source has at most ns and whose target at most nt points, solved in a
// launch laid out for that size.  dense: 128-thread CTAs take icp_kernel's 64-register instantiation, for layouts that
// fit 8 CTAs per SM (more problems in flight; the one-pass iteration is latency-bound).
struct IcpClass {
  int ns, nt;
  bool dense;
};
constexpr int ICP_MAX_CLASSES = 3;  // classes an icp_run call may list (the capacity class comes on top)
// n_classes > 0: every problem goes to the first listed class it fits, the others to a capacity class laid out for
// src.n_max x tgt.n_max; one launch per class, the widest first, each taking its problems largest first from a list
// built on the device (icp.cu).  n_classes 0: launches that partition the problems -- in-CTA, the map class for the
// targets one CTA does not hold, the global-source class for the sources no shared-memory layout holds -- each problem
// solved and written by exactly one of them (icp.cu's icp_split_run).  class_of (device [P], may be null; classes only): receives
// every problem's class (0 .. n_classes, the capacity class last) and, in class_of[P + p], its place in that class's
// list.
// filt (may be null): sfe_icp_filters -- data filters run into scratch once per cloud before the launches (distance
// filters compacted, octree filters through downsample_run), and the outlier filters in icp_kernel's FILT
// instantiations; min_points then counts the clouds before the data filters.  robust (may be null): the
// RobustOutlierFilter, in icp_kernel's ROBUST instantiations (which are FILT ones).
int icp_run(sfe_ctx *ctx, cudaStream_t st, const sfe_icp_params *prm, const IcpProblems &pb, const IcpClass *classes,
            int n_classes, int *class_of = nullptr, const sfe_icp_filters *filt = nullptr,
            const sfe_icp_robust *robust = nullptr);
// SFE_OK, or SFE_ERR_ARG with a message naming `what`: NaN, unknown kind, dim outside -1 .. 1, counts out of range
int icp_filters_check(const sfe_icp_filters *f, const char *what);
// SFE_OK, or SFE_ERR_ARG with a message naming `what`: unknown robustFct, tuning not finite and positive, NaN
// approximation
int icp_robust_check(const sfe_icp_robust *r, const char *what);
// SFE_OK, or an error with a message naming `what`: the settings prm, the filters filt and the robust filter robust
// (both may be null) that icp_run (dim 2) or icp3_run (dim 3) does not solve.  The 3-D chain refuses point-to-plane,
// float64 accumulation, filters and the robust filter; the 2-D one a robust filter with float64 accumulation
// (SFE_ERR_UNSUPPORTED).
int icp_params_check(const sfe_icp_params *prm, int dim, const sfe_icp_filters *filt, const char *what,
                     const sfe_icp_robust *robust = nullptr);
// icp_run on [x, y, z] clouds (icp3.cuh; statement oracle/icp3_ref.c): guess and T_out are [P][16] row-major 4x4,
// point-to-point with float32 sums only; no counts, classes or filters (icp_params_check).  The same launch split as
// icp_run without classes: targets above icp_cta_limit(ctx, 3, ns) read map grids, sources above icp_source_limit take
// the global-source class, with the same results.
int icp3_run(sfe_ctx *ctx, cudaStream_t st, const sfe_icp_params *prm, const IcpProblems &pb,
             const sfe_icp_filters *filt = nullptr, const sfe_icp_robust *robust = nullptr);
// *limit = the largest target of `dim` columns that icp_run (dim 2: shipped point-to-point chain, no filters) or
// icp3_run (dim 3) solves in one CTA next to sources of ns points; larger targets take the map class
int icp_cta_limit(const sfe_ctx *ctx, int dim, int ns, int *limit);
// *limit = the largest source of `dim` columns that icp_run / icp3_run solve in their shared-memory layouts next to
// targets of any size, for the settings prm, filt and robust (may be null); larger sources take the global-source class
int icp_source_limit(const sfe_ctx *ctx, const sfe_icp_params *prm, int dim, const sfe_icp_filters *filt, int *limit,
                     const sfe_icp_robust *robust = nullptr);
// nearest neighbour in reference cloud p of every point of input cloud p; no counts, in.n_max is not used; references
// of any size (the map class above one CTA's limit)
int match_run(sfe_ctx *ctx, cudaStream_t st, const PackedClouds &ref, const PackedClouds &in, int P, float max_dist,
              int32_t *ids, float *dists);
// the knn (1 .. GRID_KNN_MAX) nearest reference points of every input point: ids / dists [knn][in.off[P]], neighbour j
// of every point in row j; knn 1 of 2-D clouds is match_run.  dim 3: [x, y, z] rows in both clouds.
int match_knn_run(sfe_ctx *ctx, cudaStream_t st, const PackedClouds &ref, const PackedClouds &in, int P, int knn,
                  float max_dist, int32_t *ids, float *dists, int dim = 2);

// One map grid: a cloud too large for a one-CTA layout, built once per call in global memory (map_build).
struct MapGrid {
  float mean[2];  // cloud mean (icp_kernel's sequential float32 sum; 0 when the grid is not centred)
  float bbox[4];  // bounding box of the centred points
  float ox, oy, cell, inv_cell;
  int nx, ny, n, pad;
};

// What the map-class kernels read of map_build's grids: problem p's target is the grid in slot slot[p] (map_grid_view)
struct MapArgs {
  const int *slot;
  const MapGrid *grid;
  const float2 *pts;
  const int *cstart;
  const int *orig;
  const float2 *nrm;
  int cell_cap;
};

struct MapWs {  // device pointers into scratch[SCR_MAP]
  int *slot;       // [P] slot of every problem, -1: not in the map class
  int *n_slots;    // [1]
  int *slot_tgt;   // [slot_cap] cloud of every slot
  MapGrid *grid;   // [slot_cap]
  float2 *pts;     // [slot_cap * nt_max] (centred) x, y sorted by (slot, cell, index); padding at the end
  int *orig;       // [slot_cap * nt_max] sorted position -> index in the slot's cloud
  int *cstart;     // [slot_cap][cell_cap]: absolute position in pts of every cell's first point, entry nx * ny = end
  float2 *nrm;     // [slot_cap * nt_max] point-to-plane only
  int cell_cap;
  MapArgs args() const { return {slot, grid, pts, cstart, orig, nrm, cell_cap}; }
};

// Map grids (map_grid.cu) of the clouds with more than `limit` points among those that P problems name (problem p:
// cloud tgt_id[p], or p with tgt_id null); slot_cap bounds the number of distinct such clouds.  Points are read from
// t.pts with a stride of `dim` floats (x, y first).  center: points centred on the cloud's mean (seq: icp_kernel's
// sequential float32 sum, else a float64 sum); knn > 0: point-to-plane normals too; given_nrm (laid out as t.pts, 2-D):
// those normals instead, gathered to the sorted positions.
int map_build(sfe_ctx *ctx, cudaStream_t st, const PackedClouds &t, int dim, const int *tgt_id, int P, int limit,
              int slot_cap, bool center, bool seq, int knn, MapWs &w, const float2 *given_nrm = nullptr);

// Measurement build (-DSFE_MAP_CLASS_ALL, tools/build_map_class_variant.sh): downsample_run, remove_outlier_run,
// icp_run and match_run dispatch with a one-CTA limit of 0, so every non-empty cloud takes the large-cloud path and can
// be compared with the one-CTA kernel on clouds both hold.
#ifdef SFE_MAP_CLASS_ALL
constexpr bool MAP_CLASS_ALL = true;
#else
constexpr bool MAP_CLASS_ALL = false;
#endif

}  // namespace sfe
