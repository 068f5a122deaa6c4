/* TEST INFRASTRUCTURE ONLY (oracle/). Not part of the product path.
 *
 * The point-cloud helpers of oracle/cloud_ref.c and oracle/knn_ref.c on [x, y, z] clouds, which the reference's pybind
 * module accepts whenever a matrix has three columns (bruce_slam/src/bruce_slam/cpp/pcl.cpp:18-50, fromEigen builds an
 * x, y, z DataPoints).  The arithmetic lives in libpointmatcher / libnabo, not vendored here: **parity unpinned**, as for
 * the 2-D restatements.  Built with -ffp-contract=off: every float32 product and sum is rounded separately.
 *
 * Conventions restated
 *   downsample3  libpointmatcher's Octree_<T,3> with the medoid sampler: octree over the bounding CUBE (centre = bbox
 *                middle per axis, min + extent * 0.5 in float32 as cloud_ref.c's quadtree; half-size = the largest of
 *                the three half-extents); a node is split while 2*radius > resolution AND it holds more than one point;
 *                child id bit0 = (x > cx), bit1 = (y > cy), bit2 = (z > cz), children visited in index order after a
 *                stable 8-way partition; every non-empty leaf yields its medoid = the first minimum of the float32
 *                sequential sum of sqrtf((dx*dx + dy*dy) + dz*dz) over its members; output in visiting order.  No
 *                depth limit.
 *   match3       squared distance (dx*dx + dy*dy) + dz*dz in float32; a reference point counts when dist <= maxDist^2;
 *                no neighbour -> id -1, dist +inf; ties -> lower reference index (orc_match_brute3, knn 1).
 *   match_knn3   the k nearest under the same rule, ascending (distance, index), layout [knn][n_in] with -1 / +inf in
 *                the slots past the neighbours found (orc_match_knn3; row 0 = orc_match_brute3).
 */
#include <float.h>
#include <math.h>
#include <stddef.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

typedef struct {
  const float *pts;
  int *out;
  int n_out;
  float max_size;
} ds_ctx;

/* orc_match_brute on [x, y, z] clouds (ref [n_ref][3], in [n_in][3]) */
void orc_match_brute3(const float *ref, int n_ref, const float *in, int n_in, float max_dist, int32_t *ids,
                      float *dists) {
  const float max_d2 = max_dist * max_dist;
  for (int i = 0; i < n_in; ++i) {
    int best = -1;
    float bd = INFINITY;
    for (int j = 0; j < n_ref; ++j) {
      const float dx = in[3 * i] - ref[3 * j], dy = in[3 * i + 1] - ref[3 * j + 1], dz = in[3 * i + 2] - ref[3 * j + 2];
      const float d2 = (dx * dx + dy * dy) + dz * dz;
      if (d2 < bd) bd = d2, best = j;
    }
    if (best >= 0 && !(bd <= max_d2)) best = -1;
    ids[i] = best;
    dists[i] = best >= 0 ? bd : INFINITY;
  }
}

/* orc_match_knn on [x, y, z] clouds (ref [n_ref][3], in [n_in][3]): squared distance (dx*dx + dy*dy) + dz*dz in
 * float32, every other convention as above */
void orc_match_knn3(const float *ref, int n_ref, const float *in, int n_in, int knn, float max_dist, int32_t *ids,
                    float *dists) {
  const float max_d2 = max_dist * max_dist;
  if (knn < 1) return;
  for (int i = 0; i < n_in; ++i) {
    int k = 0;
    for (int j = 0; j < n_ref; ++j) {
      const float dx = in[3 * i] - ref[3 * j], dy = in[3 * i + 1] - ref[3 * j + 1], dz = in[3 * i + 2] - ref[3 * j + 2];
      const float d2 = (dx * dx + dy * dy) + dz * dz;
      if (!(d2 <= max_d2) || !(d2 < INFINITY)) continue;
      if (k == knn && !(d2 < dists[(size_t)(knn - 1) * n_in + i])) continue;
      int at = k < knn ? k++ : knn - 1;
      while (at > 0 && d2 < dists[(size_t)(at - 1) * n_in + i]) {
        dists[(size_t)at * n_in + i] = dists[(size_t)(at - 1) * n_in + i];
        ids[(size_t)at * n_in + i] = ids[(size_t)(at - 1) * n_in + i];
        --at;
      }
      dists[(size_t)at * n_in + i] = d2;
      ids[(size_t)at * n_in + i] = j;
    }
    for (; k < knn; ++k) ids[(size_t)k * n_in + i] = -1, dists[(size_t)k * n_in + i] = INFINITY;
  }
}

/* ------------------------------------------------------------------ downsample3 (octree medoid) */
static void ds3_leaf(ds_ctx *c, const int *idx, int n) {
  float best = FLT_MAX;
  int med = 0;
  for (int a = 0; a < n; ++a) {
    const float *pa = c->pts + 3 * (size_t)idx[a];
    float acc = 0.f;
    for (int b = 0; b < n; ++b) {
      const float *pb = c->pts + 3 * (size_t)idx[b];
      const float dx = pa[0] - pb[0], dy = pa[1] - pb[1], dz = pa[2] - pb[2];
      acc += sqrtf((dx * dx + dy * dy) + dz * dz);
    }
    if (acc < best) best = acc, med = a;
  }
  c->out[c->n_out++] = idx[med];
}

static int ds3_child(const float *p, float cx, float cy, float cz) {
  return (p[0] > cx ? 1 : 0) | (p[1] > cy ? 2 : 0) | (p[2] > cz ? 4 : 0);
}

static void ds3_build(ds_ctx *c, int *idx, int n, float cx, float cy, float cz, float radius, int *scratch) {
  if (n == 0) return;
  if (((double)radius * 2.0 <= (double)c->max_size) || n <= 1) {
    ds3_leaf(c, idx, n);
    return;
  }
  /* stable 8-way partition by child id */
  int cnt[8] = {0}, off[9], cur[8];
  for (int i = 0; i < n; ++i) cnt[ds3_child(c->pts + 3 * (size_t)idx[i], cx, cy, cz)]++;
  off[0] = 0;
  for (int k = 0; k < 8; ++k) off[k + 1] = off[k] + cnt[k], cur[k] = off[k];
  for (int i = 0; i < n; ++i) scratch[cur[ds3_child(c->pts + 3 * (size_t)idx[i], cx, cy, cz)]++] = idx[i];
  memcpy(idx, scratch, sizeof(int) * (size_t)n);
  const float hr = radius * 0.5f;
  for (int k = 0; k < 8; ++k) {
    const float ncx = cx + ((k & 1) ? hr : -hr), ncy = cy + ((k & 2) ? hr : -hr), ncz = cz + ((k & 4) ? hr : -hr);
    ds3_build(c, idx + off[k], cnt[k], ncx, ncy, ncz, hr, scratch + off[k]);
  }
}

/* pts [n][3]; out_idx[n] <- indices of the kept points in output order; returns their number */
int orc_downsample3(const float *pts, int n, float resolution, int32_t *out_idx) {
  if (n == 0) return 0;
  float mn[3] = {pts[0], pts[1], pts[2]}, mx[3] = {pts[0], pts[1], pts[2]};
  for (int i = 1; i < n; ++i)
    for (int d = 0; d < 3; ++d) {
      const float v = pts[3 * (size_t)i + d];
      if (v < mn[d]) mn[d] = v;
      if (v > mx[d]) mx[d] = v;
    }
  float ext[3], ctr[3], radius = 0.f;
  for (int d = 0; d < 3; ++d) {
    ext[d] = mx[d] - mn[d];
    ctr[d] = mn[d] + ext[d] * 0.5f;
    if (radius < ext[d] * 0.5f) radius = ext[d] * 0.5f;
  }
  int *idx = (int *)malloc(sizeof(int) * (size_t)n), *scratch = (int *)malloc(sizeof(int) * (size_t)n);
  for (int i = 0; i < n; ++i) idx[i] = i;
  ds_ctx c = {pts, (int *)out_idx, 0, resolution};
  ds3_build(&c, idx, n, ctr[0], ctr[1], ctr[2], radius, scratch);
  free(idx);
  free(scratch);
  return c.n_out;
}
