/* TEST INFRASTRUCTURE ONLY (oracle/). Not part of the product path.
 *
 * libpointmatcher's SamplingSurfaceNormalDataPointsFilter as the last reference data filter (2-D clouds), restated from
 * the published algorithm (the library is not available here, so parity stays "unpinned" like the rest of ICP), and
 * the whole ICP chain with it: the data filters of voxel_filter_ref.c (which robust_ref.c, included here, includes),
 * then the iterations of robust_ref.c with the filter's normals in place of orc_surface_normals.
 *
 *   SamplingSurfaceNormalDataPointsFilter {knn, samplingMethod, ratio, maxBoxDim, keepNormals}   (kind 5 of
 *   orc_data_filter: dim = samplingMethod, dist = maxBoxDim; knn = orc_icp_params.normals_knn, 3 .. 64)
 *     partition  build(first, last, minV, maxV) over the cloud's points, the root bounds being the cloud's
 *                coordinate-wise min and max:
 *                  count = last - first <= knn: the range is a box;
 *                  else cutDim = argmax(maxV - minV) (float32 differences; a tie goes to x, Eigen's maxCoeff),
 *                  leftCount = count - count / 2, the range is ordered so that its first leftCount points are the
 *                  smallest on cutDim, cutVal = cutDim coordinate of the point at first + leftCount, and the halves
 *                  recurse with maxV[cutDim] = cutVal (left) and minV[cutDim] = cutVal (right).
 *     per box    (fuseRange) of k points, taken in ascending original index:
 *                  boxDim = max(max x - min x, max y - min y) over the box's own points; boxDim > maxBoxDim drops the
 *                  box and all its points;
 *                  normal = orc_surface_normals' closed form on the k points (mean = sum / k, C = sum / k, C == 0
 *                  gives (0, 0));
 *                  samplingMethod 1: one point, the member of lowest original index, moved to the box centroid
 *                  (float32 sequential sums in ascending index, each divided by (float)k -- the normal's mean);
 *                  samplingMethod 0 (ratio 1): every member, each with its box's normal.
 *     output     the kept points in ascending original index, each with its box's normal.
 *   the chain  the reference filters before it run as in voxel_filter_ref.c, in the input frame; this filter then
 *     runs on what they left, still in the input frame, and the ICP loop centres the reference on the survivors'
 *     mean afterwards.  Point-to-plane reads the filter's normals (they do not depend on that translation);
 *     point-to-point ignores them.
 *
 * Unpinned choices (upstream source not at hand):
 *   - the order inside a range: points compare by (coordinate, original index), coordinates as float32 values
 *     (-0 == +0).  Upstream's std::nth_element leaves tied points on either side; this is one outcome it may produce,
 *     and it makes results reproducible on clouds with ties (sonar clouds come off a pixel lattice);
 *   - the normal of orc_surface_normals in place of upstream's Eigen eigen-solver (one normal formula serves the
 *     whole project; the fit does not depend on the normal's sign);
 *   - samplingMethod 1 keeps the lowest-index member (upstream: indices[first], whichever member nth_element left
 *     there), as the octree filter keeps its first (lowest-index) member;
 *   - samplingMethod 0 keeps a point when rand() / RAND_MAX < ratio: with ratio 1 every point is kept, where upstream
 *     would drop one whenever rand() == RAND_MAX.  Ratios below 1 (random sampling) are not restated;
 *   - averageExistingDescriptors, keepDensities, keepEigenValues and keepEigenVectors have no consumer here.
 */
#include "robust_ref.c"

enum { ORC_DATA_SAMPLING_NORMALS = 5 };

static float sn_coord(const float *pts, int i, int d) {
  const float v = pts[2 * i + d];
  return v == 0.f ? 0.f : v; /* -0 orders as +0 */
}

static void sn_sort(const float *pts, int *idx, int n, int d) { /* merge sort by (coordinate, index) */
  if (n < 2) return;
  const int h = n / 2;
  sn_sort(pts, idx, h, d);
  sn_sort(pts, idx + h, n - h, d);
  int *tmp = (int *)malloc(sizeof(int) * (size_t)n);
  int a = 0, b = h, k = 0;
  while (a < h && b < n) {
    const float va = sn_coord(pts, idx[a], d), vb = sn_coord(pts, idx[b], d);
    tmp[k++] = (va < vb || (va == vb && idx[a] < idx[b])) ? idx[a++] : idx[b++];
  }
  while (a < h) tmp[k++] = idx[a++];
  while (b < n) tmp[k++] = idx[b++];
  memcpy(idx, tmp, sizeof(int) * (size_t)n);
  free(tmp);
}

static int sn_cmp_int(const void *a, const void *b) { return (*(const int *)a > *(const int *)b) - (*(const int *)a < *(const int *)b); }

typedef struct {
  const float *pts;
  int knn, method;
  float max_box;
  char *keep;     /* [n] */
  float *val;     /* [n][2]: the kept point's coordinates */
  float *nrm;     /* [n][2] */
} sn_ctx;

static void sn_fuse(const sn_ctx *c, int *idx, int k) {
  qsort(idx, (size_t)k, sizeof(int), sn_cmp_int);
  const float *p = c->pts;
  float mnx = p[2 * idx[0]], mxx = mnx, mny = p[2 * idx[0] + 1], mxy = mny;
  for (int j = 1; j < k; ++j) {
    const float x = p[2 * idx[j]], y = p[2 * idx[j] + 1];
    if (x < mnx) mnx = x;
    if (x > mxx) mxx = x;
    if (y < mny) mny = y;
    if (y > mxy) mxy = y;
  }
  const float ex = mxx - mnx, ey = mxy - mny, box = ex > ey ? ex : ey;
  if (box > c->max_box) return;
  /* orc_surface_normals' closed form on the members in ascending index */
  float *q = (float *)malloc(sizeof(float) * 2 * (size_t)k);
  for (int j = 0; j < k; ++j) q[2 * j] = p[2 * idx[j]], q[2 * j + 1] = p[2 * idx[j] + 1];
  float sx = 0.f, sy = 0.f;
  for (int j = 0; j < k; ++j) sx += q[2 * j], sy += q[2 * j + 1];
  const float kf = (float)k, mx = sx / kf, my = sy / kf;
  float a = 0.f, b = 0.f, cc = 0.f;
  for (int j = 0; j < k; ++j) {
    const float ux = q[2 * j] - mx, uy = q[2 * j + 1] - my;
    a += ux * ux, b += ux * uy, cc += uy * uy;
  }
  a /= kf, b /= kf, cc /= kf;
  float nx = 0.f, ny = 0.f;
  if (a != 0.f || b != 0.f || cc != 0.f) {
    const float d = 0.5f * (a - cc), r = sqrtf(d * d + b * b);
    if (r == 0.f) {
      nx = 1.f, ny = 0.f;
    } else {
      const float ux = d >= 0.f ? r + d : b, uy = d >= 0.f ? b : r - d;
      const float len = sqrtf(ux * ux + uy * uy);
      nx = -(uy / len), ny = ux / len;
    }
  }
  free(q);
  for (int j = 0; j < (c->method == 1 ? 1 : k); ++j) {
    const int i = idx[j];
    c->keep[i] = 1;
    c->val[2 * i] = c->method == 1 ? mx : p[2 * i], c->val[2 * i + 1] = c->method == 1 ? my : p[2 * i + 1];
    c->nrm[2 * i] = nx, c->nrm[2 * i + 1] = ny;
  }
}

static void sn_build(const sn_ctx *c, int *idx, int count, float minx, float miny, float maxx, float maxy) {
  if (count <= c->knn) {
    if (count > 0) sn_fuse(c, idx, count);
    return;
  }
  const int d = (maxy - miny) > (maxx - minx) ? 1 : 0;
  const int left = count - count / 2;
  sn_sort(c->pts, idx, count, d);
  const float cut = c->pts[2 * idx[left] + d];
  if (d == 0) {
    sn_build(c, idx, left, minx, miny, cut, maxy);
    sn_build(c, idx + left, count - left, cut, miny, maxx, maxy);
  } else {
    sn_build(c, idx, left, minx, miny, maxx, cut);
    sn_build(c, idx + left, count - left, minx, cut, maxx, maxy);
  }
}

/* the filter on pts [n][2] -> out [n][2] and nrm_out [n][2] (kept points in ascending index, each with its box's
 * normal); returns the number of points kept */
int orc_sampling_normals(const float *pts, int n, int knn, int method, float max_box, float *out, float *nrm_out) {
  if (n <= 0) return 0;
  sn_ctx c = {pts, knn, method, max_box, (char *)calloc((size_t)n, 1), (float *)malloc(sizeof(float) * 2 * (size_t)n),
              (float *)malloc(sizeof(float) * 2 * (size_t)n)};
  int *idx = (int *)malloc(sizeof(int) * (size_t)n);
  float minx = pts[0], maxx = pts[0], miny = pts[1], maxy = pts[1];
  for (int i = 0; i < n; ++i) {
    idx[i] = i;
    const float x = pts[2 * i], y = pts[2 * i + 1];
    if (x < minx) minx = x;
    if (x > maxx) maxx = x;
    if (y < miny) miny = y;
    if (y > maxy) maxy = y;
  }
  sn_build(&c, idx, n, minx, miny, maxx, maxy);
  int m = 0;
  for (int i = 0; i < n; ++i)
    if (c.keep[i]) {
      out[2 * m] = c.val[2 * i], out[2 * m + 1] = c.val[2 * i + 1];
      nrm_out[2 * m] = c.nrm[2 * i], nrm_out[2 * m + 1] = c.nrm[2 * i + 1];
      ++m;
    }
  free(c.keep), free(c.val), free(c.nrm), free(idx);
  return m;
}

/* a reference chain that may end with the filter: the filters before it (orc_chain_filters_voxel), then it.  nrm_out
 * receives the normals when it ran (*has_nrm = 1).  Returns the points left, or -1 as orc_chain_filters_voxel. */
int orc_chain_filters_sampling(const orc_data_filter *f, int n, const float *pts, int n_in, int knn, float *out,
                               float *nrm_out, int *has_nrm) {
  const int sn = n > 0 && f[n - 1].kind == ORC_DATA_SAMPLING_NORMALS;
  *has_nrm = sn;
  if (!sn) return orc_chain_filters_voxel(f, n, pts, n_in, out);
  float *tmp = (float *)malloc(sizeof(float) * 2 * (size_t)(n_in > 0 ? n_in : 1));
  int m = orc_chain_filters_voxel(f, n - 1, pts, n_in, tmp);
  if (m >= 0) m = orc_sampling_normals(tmp, m, knn, f[n - 1].dim, f[n - 1].dist, out, nrm_out);
  free(tmp);
  return m;
}

/* orc_icp_robust_loop with the reference's normals given (nrm, [nt][2]) instead of orc_surface_normals'; with every
 * weight 1 its sums are icp_filters_ref.c's term for term, as robust_ref.c states */
static int orc_icp_given_normals_loop(const float *src, int ns, const float *tgt, const float *nrm, int nt,
                                      const float *guess, const orc_icp_params *prm, const orc_icp_filters *flt,
                                      const orc_robust *rob, float *T_out, int *iters_out, int *inliers_out) {
  const int use_min = flt->min_dist >= 0.f, use_med = flt->median_factor >= 0.f, use_rob = rob && rob->fct != 0;
  const float min_d2 = (prm->flags & 1) ? flt->min_dist : flt->min_dist * flt->min_dist;
  memcpy(T_out, guess, 9 * sizeof(float));
  *iters_out = 0;
  *inliers_out = 0;
  if (nt <= 0) return ORC_ICP_EMPTY_REF;
  {
    const float det = guess[0] * guess[4] - guess[1] * guess[3];
    if (fabsf(1.0f - det) > 0.001f || det != det) return ORC_ICP_NOT_RIGID;
  }
  float sx = 0.f, sy = 0.f;
  for (int i = 0; i < nt; ++i) sx += tgt[2 * i], sy += tgt[2 * i + 1];
  const float mx = sx / (float)nt, my = sy / (float)nt;
  float *ref = (float *)malloc(sizeof(float) * 2 * (size_t)nt);
  for (int i = 0; i < nt; ++i) ref[2 * i] = tgt[2 * i] - mx, ref[2 * i + 1] = tgt[2 * i + 1] - my;
  nn_grid *grid = nn_grid_build(ref, nt);
  const float *normals = nrm;
  const float Tmean[9] = {1, 0, mx, 0, 1, my, 0, 0, 1}, Tmean_inv[9] = {1, 0, -mx, 0, 1, -my, 0, 0, 1};
  float T0[9];
  mat3_mul(Tmean_inv, guess, T0);
  const size_t nb = (size_t)(ns > 0 ? ns : 1);
  float *reading = (float *)malloc(sizeof(float) * 2 * nb);
  for (int i = 0; i < ns; ++i) {
    const float x = src[2 * i], y = src[2 * i + 1];
    reading[2 * i] = (T0[0] * x + T0[1] * y) + T0[2];
    reading[2 * i + 1] = (T0[3] * x + T0[4] * y) + T0[5];
  }
  float *step = (float *)malloc(sizeof(float) * 2 * nb);
  float *dist = (float *)malloc(sizeof(float) * nb);
  float *wt = (float *)malloc(sizeof(float) * nb);
  float *sorted = (float *)malloc(sizeof(float) * nb);
  int *match = (int *)malloc(sizeof(int) * nb);

  float Ti[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
  const float max_d2 = prm->matcher_max_dist * prm->matcher_max_dist;
  const float out_d2 = (prm->flags & 1) ? prm->outlier_max_dist : prm->outlier_max_dist * prm->outlier_max_dist;
  enum { HMAX = 64 };
  float hq_w[HMAX], hq_z[HMAX], ht_x[HMAX], ht_y[HMAX];
  int hn = 0;
  const int smooth = prm->smooth_length > HMAX - 1 ? HMAX - 1 : prm->smooth_length;
  rot_to_quat(Ti, &hq_w[0], &hq_z[0]);
  ht_x[0] = Ti[2], ht_y[0] = Ti[5];
  hn = 1;

  int status = ORC_ICP_OK, iterate = 1, count = 0, inliers = 0;
  while (iterate) {
    for (int i = 0; i < ns; ++i) {
      const float x = reading[2 * i], y = reading[2 * i + 1];
      step[2 * i] = (Ti[0] * x + Ti[1] * y) + Ti[2];
      step[2 * i + 1] = (Ti[3] * x + Ti[4] * y) + Ti[5];
    }
    int n_fin = 0;
    for (int i = 0; i < ns; ++i) {
      match[i] = nn_grid_query(grid, step[2 * i], step[2 * i + 1], max_d2, &dist[i]);
      if (match[i] >= 0) sorted[n_fin++] = dist[i];
    }
    float limit = INFINITY, med_limit = INFINITY;
    if (prm->trim_ratio >= 0.f || use_med) {
      if (n_fin == 0) {
        status = ORC_ICP_NO_OUTLIER;
        break;
      }
      if (prm->trim_ratio >= 0.f) limit = quantile_of(sorted, n_fin, prm->trim_ratio);
      if (use_med) med_limit = flt->median_factor * quantile_of(sorted, n_fin, 0.5f);
    }
    int n_keep = 0;
    float sw = 0.f, srx = 0.f, sry = 0.f, sfx = 0.f, sfy = 0.f;
    for (int i = 0; i < ns; ++i) {
      if (match[i] < 0) continue;
      int keep = 1;
      if (prm->outlier_max_dist > 0.f) keep = keep && (dist[i] <= out_d2);
      if (prm->trim_ratio >= 0.f) keep = keep && (dist[i] <= limit);
      if (use_min) keep = keep && (dist[i] > min_d2);
      if (use_med) keep = keep && (dist[i] <= med_limit);
      const float w = use_rob ? (float)keep * orc_robust_weight(rob, dist[i]) : (float)keep;
      if (w == 0.f) {
        match[i] = -1;
        continue;
      }
      wt[i] = w;
      ++n_keep;
      sw += w;
      srx += w * step[2 * i], sry += w * step[2 * i + 1];
      sfx += w * ref[2 * match[i]], sfy += w * ref[2 * match[i] + 1];
    }
    if (n_keep == 0) {
      status = ORC_ICP_NO_POINT;
      break;
    }
    inliers = n_keep;
    float dT[9];
    if (prm->minimizer == 1) {
      float A[6] = {0, 0, 0, 0, 0, 0}, bb[3] = {0, 0, 0}, x[3];
      for (int i = 0; i < ns; ++i) {
        if (match[i] < 0) continue;
        const float w = wt[i];
        const float qx = step[2 * i], qy = step[2 * i + 1];
        const float nx = normals[2 * match[i]], ny = normals[2 * match[i] + 1];
        const float cr = qx * ny - qy * nx;
        const float dp = (qx - ref[2 * match[i]]) * nx + (qy - ref[2 * match[i] + 1]) * ny;
        const float wc = w * cr, wx = w * nx, wy = w * ny;
        A[0] += wc * cr, A[1] += wc * nx, A[2] += wc * ny, A[3] += wx * nx, A[4] += wx * ny, A[5] += wy * ny;
        bb[0] += wc * dp, bb[1] += wx * dp, bb[2] += wy * dp;
      }
      bb[0] = -bb[0], bb[1] = -bb[1], bb[2] = -bb[2];
      solve_llt3(A, bb, x);
      const float c = (float)cos((double)x[0]), s = (float)sin((double)x[0]);
      const float d[9] = {c, -s, x[1], s, c, x[2], 0, 0, 1};
      memcpy(dT, d, sizeof(d));
    } else {
      const float winv = 1.0f / sw;
      const float mrx = srx * winv, mry = sry * winv, mfx = sfx * winv, mfy = sfy * winv;
      float m00 = 0.f, m01 = 0.f, m10 = 0.f, m11 = 0.f;
      for (int i = 0; i < ns; ++i) {
        if (match[i] < 0) continue;
        const float w = wt[i];
        const float px = step[2 * i] - mrx, py = step[2 * i + 1] - mry;
        const float qx = w * (ref[2 * match[i]] - mfx), qy = w * (ref[2 * match[i] + 1] - mfy);
        m00 += qx * px, m01 += qx * py, m10 += qy * px, m11 += qy * py;
      }
      const float a = m00 + m11, b = m10 - m01;
      const float h = sqrtf(a * a + b * b);
      float c = 1.f, s = 0.f;
      if (h > 0.f) c = a / h, s = b / h;
      const float tx = mfx - (c * mrx + (-s) * mry), ty = mfy - (s * mrx + c * mry);
      const float d[9] = {c, -s, tx, s, c, ty, 0, 0, 1};
      memcpy(dT, d, sizeof(d));
    }
    mat3_mul(dT, Ti, Ti);

    ++count;
    int counter_stop = 0;
    if (count >= prm->max_iterations) iterate = 0, counter_stop = 1;
    if (!counter_stop && smooth > 0) {
      if (hn == HMAX) {
        memmove(hq_w, hq_w + 1, sizeof(float) * (HMAX - 1));
        memmove(hq_z, hq_z + 1, sizeof(float) * (HMAX - 1));
        memmove(ht_x, ht_x + 1, sizeof(float) * (HMAX - 1));
        memmove(ht_y, ht_y + 1, sizeof(float) * (HMAX - 1));
        hn = HMAX - 1;
      }
      rot_to_quat(Ti, &hq_w[hn], &hq_z[hn]);
      ht_x[hn] = Ti[2], ht_y[hn] = Ti[5];
      ++hn;
      float vr = 0.f, vt = 0.f;
      if (hn > smooth) {
        for (int i = hn - 1; i >= hn - smooth; --i) {
          const float dw = hq_w[i] * hq_w[i - 1] + hq_z[i] * hq_z[i - 1];
          const float dz = hq_z[i] * hq_w[i - 1] - hq_w[i] * hq_z[i - 1];
          vr += fabsf(2.0f * atan2f(fabsf(dz), fabsf(dw)));
          const float ex = ht_x[i] - ht_x[i - 1], ey = ht_y[i] - ht_y[i - 1];
          vt += fabsf(sqrtf(ex * ex + ey * ey));
        }
        vr /= (float)smooth;
        vt /= (float)smooth;
        if (vr < prm->min_diff_rot && vt < prm->min_diff_trans) iterate = 0;
      }
      if (vr != vr) {
        status = ORC_ICP_NAN_ROT;
        break;
      }
      if (vt != vt) {
        status = ORC_ICP_NAN_TRANS;
        break;
      }
    }
  }
  *iters_out = count;
  *inliers_out = inliers;
  if (status == ORC_ICP_OK) {
    float tmp[9];
    mat3_mul(Tmean, Ti, tmp);
    mat3_mul(tmp, T0, T_out);
  }
  nn_grid_free(grid);
  free(ref), free(reading), free(step), free(dist), free(wt), free(sorted), free(match);
  return status;
}

/* The whole chain with the filter as the last reference filter: data filters, the filter, then the iterations with
 * its normals.  Without the filter this is orc_icp_robust.  Returns the ICP status, or -1 as orc_icp_robust. */
int orc_icp_sampling(const float *src_in, int ns_in, const float *tgt_in, int nt_in, const float *guess,
                     const orc_icp_params *prm, const orc_icp_filters *flt, const orc_robust *rob, float *T_out,
                     int *iters_out, int *inliers_out) {
  const size_t nsb = (size_t)(ns_in > 0 ? ns_in : 1), ntb = (size_t)(nt_in > 0 ? nt_in : 1);
  float *src = (float *)malloc(sizeof(float) * 2 * nsb);
  float *tgt = (float *)malloc(sizeof(float) * 2 * ntb);
  float *nrm = (float *)malloc(sizeof(float) * 2 * ntb);
  int has_nrm = 0, st = -1;
  const int ns = orc_chain_filters_voxel(flt->reading, flt->n_reading, src_in, ns_in, src);
  const int nt = orc_chain_filters_sampling(flt->reference, flt->n_reference, tgt_in, nt_in, prm->normals_knn, tgt,
                                            nrm, &has_nrm);
  if (ns >= 0 && nt >= 0) {
    if (!has_nrm)
      st = orc_icp_robust_loop(src, ns, tgt, nt, guess, prm, flt, rob, T_out, iters_out, inliers_out);
    else
      st = orc_icp_given_normals_loop(src, ns, tgt, nrm, nt, guess, prm, flt, rob, T_out, iters_out, inliers_out);
  }
  free(src), free(tgt), free(nrm);
  return st;
}
