/* TEST INFRASTRUCTURE ONLY (oracle/). Not part of the product path.
 *
 * libpointmatcher's SurfaceNormalDataPointsFilter and ShadowDataPointsFilter on the reading (source) cloud (2-D clouds),
 * restated from the published filters (the library is not available here, so parity stays "unpinned" like the rest of
 * ICP), and the whole ICP chain with them: the reading chain below, then orc_icp_sampling of sampling_normal_ref.c
 * (included here) with the filtered source -- its reference chain and its iterations.
 *
 *   SurfaceNormalDataPointsFilter {knn, epsilon 0, keepNormals 1}   (kind 6 of orc_data_filter: dim = knn, 3 .. 16)
 *     every point of the cloud the filter receives gets orc_surface_normals' normal: its knn nearest points (itself
 *     included; brute force, ascending squared float32 distance, ties to the lower index), the closed form of icp_ref.c,
 *     computed on the cloud centred on its mean (sequential float32 sums in point order, each divided by (float)n).
 *     The points do not change.
 *   ShadowDataPointsFilter {eps}   (kind 7: dist = eps, radians)
 *     keeps point p (as the filter receives it: the reading's input frame, the sensor at the origin) with normal n iff
 *     |n^ . p^| > sinf(eps), v^ = v / sqrtf(v.v) when v.v > 0 else v (Eigen's normalized()), the dot nx*px + ny*py;
 *     float32, nothing contracted, sinf the C library's (the device library calls the same one on the host).
 *   the chain  filters before the normals run as in voxel_filter_ref.c; after it only the distance filters and the
 *     shadow filter (per-point tests), the survivors keeping their input order and their normals.  The normals are
 *     dropped after the reading chain.
 *
 * Unpinned choices (upstream source not at hand):
 *   - the normals on the centred cloud (upstream does not centre; the difference is rounding-level).  This is the rule
 *     the reference normals follow, so the device computes both with one piece of code at every cloud size;
 *   - orc_surface_normals' closed form in place of upstream's Eigen eigen-solver (the shadow test does not depend on
 *     the normal's sign);
 *   - keepDensities, keepEigenValues, keepEigenVectors and keepMatchedIds have no consumer here.
 */
#include "sampling_normal_ref.c"

enum { ORC_DATA_NORMALS = 6, ORC_DATA_SHADOW = 7 };

/* the reading normals of pts [n][2] -> nrm [n][2] */
void orc_reading_normals(const float *pts, int n, int knn, float *nrm) {
  if (n <= 0) return;
  float sx = 0.f, sy = 0.f;
  for (int i = 0; i < n; ++i) sx += pts[2 * i], sy += pts[2 * i + 1];
  const float mx = sx / (float)n, my = sy / (float)n;
  float *c = (float *)malloc(sizeof(float) * 2 * (size_t)n);
  for (int i = 0; i < n; ++i) c[2 * i] = pts[2 * i] - mx, c[2 * i + 1] = pts[2 * i + 1] - my;
  orc_surface_normals(c, n, knn, nrm);
  free(c);
}

/* the shadow test of one point with its normal, against sin_eps = sinf(eps) */
int orc_shadow_keep(float x, float y, float nx, float ny, float sin_eps) {
  const float nn = nx * nx + ny * ny, pp = x * x + y * y;
  if (nn > 0.f) {
    const float l = sqrtf(nn);
    nx = nx / l, ny = ny / l;
  }
  if (pp > 0.f) {
    const float l = sqrtf(pp);
    x = x / l, y = y / l;
  }
  return fabsf(nx * x + ny * y) > sin_eps;
}

float orc_sinf(float x) { return sinf(x); }

/* the reading chain f[0 .. n) on pts [n_in][2] -> out [n_in][2]; returns the points left, or -1 as
 * orc_chain_filters_voxel */
int orc_chain_filters_shadow(const orc_data_filter *f, int n, const float *pts, int n_in, float *out) {
  int at = -1;
  for (int k = 0; k < n; ++k)
    if (f[k].kind == ORC_DATA_NORMALS) at = k;
  if (at < 0) return orc_chain_filters_voxel(f, n, pts, n_in, out);
  int m = orc_chain_filters_voxel(f, at, pts, n_in, out);
  if (m < 0) return m;
  float *nrm = (float *)malloc(sizeof(float) * 2 * (size_t)(m > 0 ? m : 1));
  orc_reading_normals(out, m, f[at].dim, nrm);
  int kept = 0;
  for (int i = 0; i < m; ++i) {
    const float x = out[2 * i], y = out[2 * i + 1];
    int keep = 1;
    for (int k = at + 1; k < n && keep; ++k)
      keep = f[k].kind == ORC_DATA_SHADOW ? orc_shadow_keep(x, y, nrm[2 * i], nrm[2 * i + 1], sinf(f[k].dist))
                                          : data_keep(&f[k], x, y);
    if (keep) out[2 * kept] = x, out[2 * kept + 1] = y, ++kept;
  }
  free(nrm);
  return kept;
}

/* The whole chain: the reading chain above, then orc_icp_sampling (the reference chain, the iterations) with no
 * reading filter left.  Returns the ICP status, or -1 when a voxel filter's index would not fit 32 bits. */
int orc_icp_shadow(const float *src_in, int ns_in, const float *tgt_in, int nt_in, const float *guess,
                   const orc_icp_params *prm, const orc_icp_filters *flt, const orc_robust *rob, float *T_out,
                   int *iters_out, int *inliers_out) {
  float *src = (float *)malloc(sizeof(float) * 2 * (size_t)(ns_in > 0 ? ns_in : 1));
  const int ns = orc_chain_filters_shadow(flt->reading, flt->n_reading, src_in, ns_in, src);
  int st = -1;
  if (ns >= 0) {
    orc_icp_filters rest = *flt;
    rest.n_reading = 0;
    st = orc_icp_sampling(src, ns, tgt_in, nt_in, guess, prm, &rest, rob, T_out, iters_out, inliers_out);
  }
  free(src);
  return st;
}
