/* TEST INFRASTRUCTURE ONLY (oracle/). Not part of the product path.
 *
 * libpointmatcher's RobustOutlierFilter (OutlierFiltersImpl::RobustOutlierFilter, restated from memory of
 * RobustOutlierFilter.cpp; the library is not available here, so parity stays "unpinned" like the rest of ICP) on 2-D
 * clouds, after the data-filter chains of voxel_filter_ref.c (which this file includes, with octree_filter_ref.c,
 * icp_filters_ref.c and icp_ref.c under it): the whole chain runs -- data filters, then the weighted iterations.
 *
 *   RobustOutlierFilter {robustFct, tuning = k, approximation, scaleEstimator none | fixed, distanceType point2point}
 *     e2 = the pair's squared float32 distance (the value MaxDist compares), k2 = k * k (float32):
 *       1 cauchy   1 / (1 + e2 / k2)
 *       2 welsch   (float)exp((double)(-(e2 / k2)))
 *       3 sc       e2 >= k ? (4 * k2) / ((k + e2) * (k + e2)) : 1
 *       4 gm       k2 / ((k + e2) * (k + e2))
 *       5 tukey    e2 >= k2 ? 0 : (1 - e2 / k2) * (1 - e2 / k2)
 *       6 huber    e2 >= k2 ? k / sqrtf(e2) : 1
 *       7 L1       1 / sqrtf(e2)
 *     then 0 where e2 >= approximation (+inf: no cut-off).  Division and sqrtf are IEEE-rounded, nothing is contracted
 *     (-ffp-contract=off), and the only exp is the float64 one rounded to float32 (as Rotation2D's cos / sin).
 *   the chain  a pair's weight is the product of every outlier filter's weight, in YAML order (OutlierFiltersImpl::
 *     compute).  MaxDist, Trimmed, MinDist and Median give 0 or 1, and a robust weight is never negative, so the order
 *     does not change the product: it is the robust weight where the others keep the pair, and 0 * w where one drops
 *     it -- 0, or NaN for w = inf (L1 at e2 == 0), as upstream.
 *   kept pairs  a matched pair whose weight is not 0 (NaN included); `inliers` is their number, and none at all is
 *     "no point to minimize".
 *   minimisers (sequential float32 sums in point order over the kept pairs, w the pair's weight):
 *     point-to-point  W = sum w;  mean_read = (sum (w * p)) * (1 / W), mean_ref likewise;  M = sum ((w * r~) * p~)
 *                     for r~ = r - mean_ref, p~ = p - mean_read (m00 = (w * r~x) * p~x, ...);  then icp_ref.c's fit.
 *     point-to-plane  wF = w * F (elementwise) for F = (c, n.x, n.y);  A = sum wF F^T (a00 = (w * c) * c, ...),
 *                     b = -sum wF ((q - r).n);  then icp_ref.c's Cholesky solve.
 *   With every weight 1 these are icp_ref.c's sums term for term (W counts the kept pairs exactly below 2^24), so
 *   orc_icp_robust with a Huber k2 above every kept e2 equals orc_icp_chain_voxel bit for bit.
 *
 * Unpinned choices (upstream source not at hand):
 *   - the float32 form of every weight above (k2 rounded once; 4 * k2 before the division; the square of a sum as a
 *     product of two equal factors), and `sc` comparing e2 with k, not k2;
 *   - the cut-off as e2 >= approximation, applied after the weight function;
 *   - the weighting order inside the sums: (w * coordinate) for the means, (w * r~) * p~ and (w * F_i) * F_j;
 *   - scaleEstimator none / fixed as scale 1 (the tuning is k itself); nbIterationForScale is moot then.  mad, berg,
 *     student and point2plane residuals are not restated.
 */
#include "voxel_filter_ref.c"

enum { ORC_ROBUST_CAUCHY = 1, ORC_ROBUST_WELSCH = 2, ORC_ROBUST_SC = 3, ORC_ROBUST_GM = 4, ORC_ROBUST_TUKEY = 5,
       ORC_ROBUST_HUBER = 6, ORC_ROBUST_L1 = 7 };

typedef struct {
  int fct;             /* ORC_ROBUST_*; 0: no RobustOutlierFilter */
  float tuning;        /* k */
  float approximation; /* weight 0 where e2 >= approximation; +inf: no cut-off */
} orc_robust;

float orc_robust_weight(const orc_robust *r, float e2) {
  const float k = r->tuning, k2 = k * k;
  float w;
  switch (r->fct) {
    case ORC_ROBUST_CAUCHY: w = 1.0f / (1.0f + e2 / k2); break;
    case ORC_ROBUST_WELSCH: w = (float)exp((double)(-(e2 / k2))); break;
    case ORC_ROBUST_SC: {
      const float s = k + e2;
      w = e2 >= k ? (4.0f * k2) / (s * s) : 1.0f;
      break;
    }
    case ORC_ROBUST_GM: {
      const float s = k + e2;
      w = k2 / (s * s);
      break;
    }
    case ORC_ROBUST_TUKEY: {
      const float u = 1.0f - e2 / k2;
      w = e2 >= k2 ? 0.0f : u * u;
      break;
    }
    case ORC_ROBUST_HUBER: w = e2 >= k2 ? k / sqrtf(e2) : 1.0f; break;
    case ORC_ROBUST_L1: w = 1.0f / sqrtf(e2); break;
    default: w = 1.0f; break;
  }
  if (e2 >= r->approximation) w = 0.0f;
  return w;
}

/* the weights of n squared distances (for the tests) */
void orc_robust_weights(const orc_robust *r, const float *e2, int n, float *w) {
  for (int i = 0; i < n; ++i) w[i] = orc_robust_weight(r, e2[i]);
}

static int orc_icp_robust_loop(const float *src, int ns, const float *tgt, int nt, const float *guess,
                               const orc_icp_params *prm, const orc_icp_filters *flt, const orc_robust *rob,
                               float *T_out, int *iters_out, int *inliers_out) {
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
  float *normals = NULL;
  if (prm->minimizer == 1) {
    normals = (float *)malloc(sizeof(float) * 2 * (size_t)nt);
    orc_surface_normals(ref, nt, prm->normals_knn, normals);
  }
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
    /* weights: the 0/1 filters, times the robust weight; kept = matched and weight != 0 */
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
  free(ref), free(reading), free(step), free(dist), free(wt), free(sorted), free(match), free(normals);
  return status;
}

/* The whole chain: data filters (orc_chain_filters_voxel), then the weighted iterations.  rob may be NULL (no robust
 * filter).  Returns the ICP status, or -1 when a voxel filter's index would not fit 32 bits. */
int orc_icp_robust(const float *src_in, int ns_in, const float *tgt_in, int nt_in, const float *guess,
                   const orc_icp_params *prm, const orc_icp_filters *flt, const orc_robust *rob, float *T_out,
                   int *iters_out, int *inliers_out) {
  float *src = (float *)malloc(sizeof(float) * 2 * (size_t)(ns_in > 0 ? ns_in : 1));
  float *tgt = (float *)malloc(sizeof(float) * 2 * (size_t)(nt_in > 0 ? nt_in : 1));
  const int ns = orc_chain_filters_voxel(flt->reading, flt->n_reading, src_in, ns_in, src);
  const int nt = orc_chain_filters_voxel(flt->reference, flt->n_reference, tgt_in, nt_in, tgt);
  int st = -1;
  if (ns >= 0 && nt >= 0) st = orc_icp_robust_loop(src, ns, tgt, nt, guess, prm, flt, rob, T_out, iters_out, inliers_out);
  free(src), free(tgt);
  return st;
}
