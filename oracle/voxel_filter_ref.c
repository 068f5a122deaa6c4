/* TEST INFRASTRUCTURE ONLY (oracle/). Not part of the product path.
 *
 * libpointmatcher's VoxelGridDataPointsFilter as an ICP data filter (2-D clouds), and the ICP data-filter chains that
 * mix it with the octree and distance filters of octree_filter_ref.c (which this file includes, with
 * icp_filters_ref.c and icp_ref.c under it).
 *
 *   VoxelGridDataPointsFilter {vSizeX = vSizeY = vSize, useCentroid = 1}   (kind 4 of orc_data_filter: dim =
 *   useCentroid, dist = vSize > 0), VoxelGridDataPointsFilter::inPlaceFilter on a 2-D cloud:
 *     1. minB = min(x) / vSize and maxB = max(x) / vSize in float32, the same for y; numDivX = 1 + (unsigned)(maxBX -
 *        minBX), likewise numDivY.
 *     2. for every point p in point order: i = (unsigned)floorf(x_p / vSize - minBX), j likewise, idx = i + j *
 *        numDivX; the first point of a voxel becomes its firstPoint, and the voxel counts its points.
 *     3. every point that is not its voxel's first point, in point order, adds its x and y into the first point's
 *        coordinates (float32, sequential, starting from the first point's own value); each first point is then
 *        divided by (float)numPoints.
 *     4. the first points are kept in ascending index order (upstream's std::sort of pointsToKeep): the output is the
 *        first point of every voxel, in input order, holding its voxel's centroid.
 *   the chain  the filters of one cloud run in their listed order, each on what the one before left.
 *
 * Unpinned choices (upstream source not at hand; parity stays "unpinned" like the rest of ICP):
 *   - the float32 evaluation of the bounds, of numDiv as 1 + (unsigned)(maxB - minB) and of the voxel coordinates as
 *     floorf(x / vSize - minB), in that order of operations;
 *   - the centroid's summation order (point order, into the first point) and its single division per axis;
 *   - the output order (first points in input order);
 *   - vSizeX == vSizeY only (vSizeZ is moot on 2-D clouds); useCentroid 0 (the voxel centre) is not restated;
 *     averageExistingDescriptors is moot (an ICP reading has no descriptors);
 *   - a cloud whose numDivX * numDivY does not fit 32 bits (upstream's unsigned index would wrap, undefined there),
 *     or whose bounds are not finite, is reported: orc_voxel_filter returns -1.
 */
#include "octree_filter_ref.c"

enum { ORC_DATA_VOXEL = 4 };

typedef struct {
  unsigned idx;
  int p;
} vox_pair;

static int vox_cmp(const void *a, const void *b) {
  const vox_pair *x = (const vox_pair *)a, *y = (const vox_pair *)b;
  if (x->idx != y->idx) return x->idx < y->idx ? -1 : 1;
  return (x->p > y->p) - (x->p < y->p);
}

/* the filter on pts [n][2] -> out [n][2]; returns the number of points kept, or -1 when the voxel index would not fit
 * 32 bits */
int orc_voxel_filter(const float *pts, int n, float vsize, float *out) {
  if (n == 0) return 0;
  float minx = pts[0], maxx = pts[0], miny = pts[1], maxy = pts[1];
  for (int i = 1; i < n; ++i) {
    const float x = pts[2 * i], y = pts[2 * i + 1];
    if (x < minx) minx = x;
    if (x > maxx) maxx = x;
    if (y < miny) miny = y;
    if (y > maxy) maxy = y;
  }
  const float minbx = minx / vsize, minby = miny / vsize;
  const float dx = maxx / vsize - minbx, dy = maxy / vsize - minby;
  if (!(dx < 4294967296.f && dy < 4294967296.f)) return -1;
  const unsigned long long ndx = 1ull + (unsigned)dx, ndy = 1ull + (unsigned)dy;
  if (ndx * ndy > 0xffffffffull) return -1;
  /* the voxel table as (idx, p) pairs sorted by voxel, then point: a voxel's first point heads its run (a table of
   * numDivX * numDivY entries would not fit memory at small sizes) */
  vox_pair *v = (vox_pair *)malloc(sizeof(vox_pair) * (size_t)n);
  float *acc = (float *)malloc(sizeof(float) * 2 * (size_t)n);
  char *keep = (char *)calloc((size_t)n, 1);
  if (!v || !acc || !keep) abort();
  for (int p = 0; p < n; ++p) {
    const unsigned i = (unsigned)floorf(pts[2 * p] / vsize - minbx);
    const unsigned j = (unsigned)floorf(pts[2 * p + 1] / vsize - minby);
    v[p].idx = i + j * (unsigned)ndx, v[p].p = p;
  }
  qsort(v, (size_t)n, sizeof(vox_pair), vox_cmp);
  for (int a = 0; a < n;) {
    int e = a + 1;
    while (e < n && v[e].idx == v[a].idx) ++e;
    const int f = v[a].p;
    float sx = pts[2 * f], sy = pts[2 * f + 1];
    for (int q = a + 1; q < e; ++q) sx += pts[2 * v[q].p], sy += pts[2 * v[q].p + 1];
    acc[2 * f] = sx / (float)(e - a), acc[2 * f + 1] = sy / (float)(e - a);
    keep[f] = 1;
    a = e;
  }
  int m = 0;
  for (int p = 0; p < n; ++p)
    if (keep[p]) out[2 * m] = acc[2 * p], out[2 * m + 1] = acc[2 * p + 1], ++m;
  free(v), free(acc), free(keep);
  return m;
}

/* the chain f[0 .. n) on pts [n_in][2] -> out [n_in][2] (octree, voxel and distance filters); returns the points
 * left, or -1 when a voxel filter's index would not fit 32 bits */
int orc_chain_filters_voxel(const orc_data_filter *f, int n, const float *pts, int n_in, float *out) {
  int m = n_in;
  memcpy(out, pts, sizeof(float) * 2 * (size_t)n_in);
  float *in = (float *)malloc(sizeof(float) * 2 * (size_t)(n_in > 0 ? n_in : 1));
  for (int k = 0; k < n && m >= 0; ++k) {
    memcpy(in, out, sizeof(float) * 2 * (size_t)m);
    m = f[k].kind == ORC_DATA_VOXEL    ? orc_voxel_filter(in, m, f[k].dist, out)
        : f[k].kind == ORC_DATA_OCTREE ? orc_octree_filter(in, m, f[k].dist, f[k].dim, out)
                                       : orc_data_filters(&f[k], 1, in, m, out);
  }
  free(in);
  return m;
}

/* orc_icp_chain with chains that may hold voxel filters; -1 when a voxel filter's index would not fit 32 bits */
int orc_icp_chain_voxel(const float *src_in, int ns_in, const float *tgt_in, int nt_in, const float *guess,
                        const orc_icp_params *prm, const orc_icp_filters *flt, float *T_out, int *iters_out,
                        int *inliers_out) {
  float *src = (float *)malloc(sizeof(float) * 2 * (size_t)(ns_in > 0 ? ns_in : 1));
  float *tgt = (float *)malloc(sizeof(float) * 2 * (size_t)(nt_in > 0 ? nt_in : 1));
  const int ns = orc_chain_filters_voxel(flt->reading, flt->n_reading, src_in, ns_in, src);
  const int nt = orc_chain_filters_voxel(flt->reference, flt->n_reference, tgt_in, nt_in, tgt);
  int st = -1;
  if (ns >= 0 && nt >= 0) {
    orc_icp_filters rest = *flt;
    rest.n_reading = rest.n_reference = 0;
    st = orc_icp_filtered(src, ns, tgt, nt, guess, prm, &rest, T_out, iters_out, inliers_out);
  }
  free(src), free(tgt);
  return st;
}
