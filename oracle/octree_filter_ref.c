/* TEST INFRASTRUCTURE ONLY (oracle/). Not part of the product path.
 *
 * libpointmatcher's OctreeGridDataPointsFilter as an ICP data filter (2-D clouds), and the ICP data-filter chains that
 * mix it with the distance filters of icp_filters_ref.c (which this file includes, with icp_ref.c under it).
 *
 *   OctreeGridDataPointsFilter {maxSizeByNode, samplingMethod}   (kind 3 of orc_data_filter: dim = samplingMethod,
 *   dist = maxSizeByNode > 0)
 *     tree     the quadtree of cloud_ref.c's orc_downsample: the cloud's bounding SQUARE (centre = bbox middle,
 *              half-size = larger half-extent); a node is split while 2*radius > maxSizeByNode AND it holds more than
 *              one point AND it lies less than 15 levels below the root; stable 4-way partition by bit0 = (x > cx),
 *              bit1 = (y > cy); children visited in index order; every non-empty leaf yields one point, in visiting
 *              (depth-first) order.
 *     samplers 0: the leaf's first member (the stable partition makes it its lowest input index);
 *              2: the centroid -- float32 sequential sums of x and of y in member order, each divided once by
 *                 (float)n;
 *              3: the medoid -- the member minimising the float32 sequential sum of Euclidean distances to all
 *                 members, first one on ties (orc_downsample's rule).
 *   the chain  the filters of one cloud run in their listed order, each on what the one before left: the distance
 *              filters keep their survivors in order, the octree emits its leaves' points.  Later filters, and the
 *              iterations' sequential sums, see the octree's leaf order.
 *
 * Unpinned choices (upstream source not at hand; parity stays "unpinned" like the rest of ICP):
 *   - the first-point sampler's member and the centroid's summation order and single division, as stated above;
 *   - maxPointByNode is ignored once maxSizeByNode > 0 (as we recall, upstream's constructor then sets the point bound
 *     to 1), and buildParallel does not change the result;
 *   - the 15-level cut: the depth the device's path keys hold (DS_MAX_DEPTH); a node at that depth is a leaf whatever
 *     its size.  orc_downsample keeps its uncut tree;
 *   - samplingMethod 1 (random) and the point-count criterion (no maxSizeByNode) are not restated.
 *
 * Everything else -- the ICP loop, the distance and outlier filters -- is icp_filters_ref.c's: orc_icp_chain filters
 * both clouds with orc_chain_filters and hands the results to orc_icp_filtered with no data filter left.
 */
#include <float.h>
#include <limits.h>

#include "icp_filters_ref.c"

enum { ORC_DATA_OCTREE = 3, ORC_OCT_FIRST = 0, ORC_OCT_CENTROID = 2, ORC_OCT_MEDOID = 3, ORC_OCT_MAX_DEPTH = 15 };

typedef struct {
  const float *pts;
  float *out; /* [n_out][2] the kept point of every leaf */
  int n_out;
  float max_size;
  int sampler;
  int max_depth;
} oct_ctx;

static void oct_leaf(oct_ctx *c, const int *idx, int n) {
  float px, py;
  if (c->sampler == ORC_OCT_CENTROID) {
    float sx = 0.f, sy = 0.f;
    for (int a = 0; a < n; ++a) sx += c->pts[2 * idx[a]], sy += c->pts[2 * idx[a] + 1];
    px = sx / (float)n, py = sy / (float)n;
  } else {
    int keep = 0;
    if (c->sampler == ORC_OCT_MEDOID) {
      float best = FLT_MAX;
      for (int a = 0; a < n; ++a) {
        const float ax = c->pts[2 * idx[a]], ay = c->pts[2 * idx[a] + 1];
        float acc = 0.f;
        for (int b = 0; b < n; ++b) {
          const float dx = ax - c->pts[2 * idx[b]], dy = ay - c->pts[2 * idx[b] + 1];
          acc += sqrtf(dx * dx + dy * dy);
        }
        if (acc < best) best = acc, keep = a;
      }
    }
    px = c->pts[2 * idx[keep]], py = c->pts[2 * idx[keep] + 1];
  }
  c->out[2 * c->n_out] = px, c->out[2 * c->n_out + 1] = py;
  ++c->n_out;
}

static void oct_build(oct_ctx *c, int *idx, int n, float cx, float cy, float radius, int *scratch, int depth) {
  if (n == 0) return;
  if (((double)radius * 2.0 <= (double)c->max_size) || n <= 1 || depth >= c->max_depth) {
    oct_leaf(c, idx, n);
    return;
  }
  int cnt[4] = {0, 0, 0, 0};
  for (int i = 0; i < n; ++i) cnt[(c->pts[2 * idx[i]] > cx ? 1 : 0) | (c->pts[2 * idx[i] + 1] > cy ? 2 : 0)]++;
  const int off[5] = {0, cnt[0], cnt[0] + cnt[1], cnt[0] + cnt[1] + cnt[2], n};
  int cur[4] = {off[0], off[1], off[2], off[3]};
  for (int i = 0; i < n; ++i)
    scratch[cur[(c->pts[2 * idx[i]] > cx ? 1 : 0) | (c->pts[2 * idx[i] + 1] > cy ? 2 : 0)]++] = idx[i];
  memcpy(idx, scratch, sizeof(int) * (size_t)n);
  const float hr = radius * 0.5f;
  for (int k = 0; k < 4; ++k)
    oct_build(c, idx + off[k], cnt[k], cx + ((k & 1) ? hr : -hr), cy + ((k & 2) ? hr : -hr), hr, scratch + off[k],
              depth + 1);
}

/* the filter on pts [n][2] -> out [n][2] in leaf order; max_depth: the cut (ORC_OCT_MAX_DEPTH in an ICP chain, INT_MAX:
 * none); returns the number of points kept */
int orc_octree_filter_depth(const float *pts, int n, float max_size, int sampler, int max_depth, float *out) {
  if (n == 0) return 0;
  float minx = pts[0], maxx = pts[0], miny = pts[1], maxy = pts[1];
  for (int i = 1; i < n; ++i) {
    const float x = pts[2 * i], y = pts[2 * i + 1];
    if (x < minx) minx = x;
    if (x > maxx) maxx = x;
    if (y < miny) miny = y;
    if (y > maxy) maxy = y;
  }
  const float rx = maxx - minx, ry = maxy - miny;
  const float cx = minx + rx * 0.5f, cy = miny + ry * 0.5f;
  float radius = rx;
  if (radius < ry) radius = ry;
  radius *= 0.5f;
  int *idx = (int *)malloc(sizeof(int) * (size_t)n), *scratch = (int *)malloc(sizeof(int) * (size_t)n);
  for (int i = 0; i < n; ++i) idx[i] = i;
  oct_ctx c = {pts, out, 0, max_size, sampler, max_depth};
  oct_build(&c, idx, n, cx, cy, radius, scratch, 0);
  free(idx);
  free(scratch);
  return c.n_out;
}

int orc_octree_filter(const float *pts, int n, float max_size, int sampler, float *out) {
  return orc_octree_filter_depth(pts, n, max_size, sampler, ORC_OCT_MAX_DEPTH, out);
}

/* the chain f[0 .. n) on pts [n_in][2] -> out [n_in][2], one filter after the other; returns the points left */
int orc_chain_filters(const orc_data_filter *f, int n, const float *pts, int n_in, float *out) {
  int m = n_in;
  memcpy(out, pts, sizeof(float) * 2 * (size_t)n_in);
  float *in = (float *)malloc(sizeof(float) * 2 * (size_t)(n_in > 0 ? n_in : 1));
  for (int k = 0; k < n; ++k) {
    memcpy(in, out, sizeof(float) * 2 * (size_t)m);
    m = f[k].kind == ORC_DATA_OCTREE ? orc_octree_filter(in, m, f[k].dist, f[k].dim, out)
                                     : orc_data_filters(&f[k], 1, in, m, out);
  }
  free(in);
  return m;
}

/* orc_icp_filtered with the chains of flt run by orc_chain_filters (octree filters included) */
int orc_icp_chain(const float *src_in, int ns_in, const float *tgt_in, int nt_in, const float *guess,
                  const orc_icp_params *prm, const orc_icp_filters *flt, float *T_out, int *iters_out,
                  int *inliers_out) {
  float *src = (float *)malloc(sizeof(float) * 2 * (size_t)(ns_in > 0 ? ns_in : 1));
  float *tgt = (float *)malloc(sizeof(float) * 2 * (size_t)(nt_in > 0 ? nt_in : 1));
  const int ns = orc_chain_filters(flt->reading, flt->n_reading, src_in, ns_in, src);
  const int nt = orc_chain_filters(flt->reference, flt->n_reference, tgt_in, nt_in, tgt);
  orc_icp_filters rest = *flt;
  rest.n_reading = rest.n_reference = 0;
  const int st = orc_icp_filtered(src, ns, tgt, nt, guess, prm, &rest, T_out, iters_out, inliers_out);
  free(src), free(tgt);
  return st;
}
