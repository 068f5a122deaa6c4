/* TEST INFRASTRUCTURE ONLY (oracle/). Not part of the product path.
 *
 * The ICP restatement of icp_ref.c with libpointmatcher's distance data filters and two more outlier filters
 * (DataPointsFiltersImpl / OutlierFiltersImpl at d478ef2e, restated; the library is not available here, so this
 * stays "parity unpinned" like the rest of ICP):
 *
 *   data filters (once per problem, before the iterations; survivors keep their input order, like setColFrom):
 *     MaxDistDataPointsFilter {dim, maxDist}   dim -1: keep sqrtf(x*x + y*y) < |maxDist|; dim 0 / 1: keep coord < maxDist
 *     MinDistDataPointsFilter {dim, minDist}   dim -1: keep sqrtf(x*x + y*y) > |minDist|; dim 0 / 1: keep coord > minDist
 *     reading filters run on the source in its input frame, before the initial guess is applied; reference filters
 *     on the target in its input frame, before it is centred: mean, grid and normals come from the survivors only.
 *     A target the filters empty is an empty target (ORC_ICP_EMPTY_REF).  A source they empty reaches the status
 *     libpointmatcher's chain reaches with no matches: "no outlier to filter" when a quantile filter (Trimmed or
 *     Median) is on, else "no point to minimize"; 0 iterations either way.
 *   outlier filters (every filter sees all matches; the weights are the product over the chain):
 *     MinDistOutlierFilter {minDist}           keep d2 > minDist^2 (flags bit 0: d2 > minDist, as for MaxDist)
 *     MedianDistOutlierFilter {factor}         median = element floor(float(n_finite) * 0.5) of the ascending finite
 *                                              distances (getDistsQuantile(0.5)); keep d2 <= factor * median (float32
 *                                              product); no finite distance: "no outlier to filter", as for Trimmed
 *
 * Unpinned choices (upstream source not at hand):
 *   - strict `<` / `>` in the data filters and strict `>` in MinDist; non-strict `<=` in Median (as MaxDist / Trimmed);
 *   - |dist| for the radial data filters, the signed value for the per-axis ones;
 *   - the radial norm as sqrtf of the unfused float32 x*x + y*y (the squared norm against dist^2 can differ at a tie).
 *
 * Everything else -- the loop, its float32 expressions, the sequential sums -- is icp_ref.c's, which this file
 * includes; with no filter set, orc_icp_filtered equals orc_icp bit for bit (tests/test_icp_filters_cpu.py).
 */
#include "icp_ref.c"

enum { ORC_DATA_MAX_DIST = 1, ORC_DATA_MIN_DIST = 2, ORC_MAX_DATA_FILTERS = 4 };

typedef struct {
  int kind; /* 0 none, ORC_DATA_MAX_DIST, ORC_DATA_MIN_DIST */
  int dim;  /* -1 radial, 0 x, 1 y */
  float dist;
} orc_data_filter;

typedef struct {
  float min_dist;      /* MinDistOutlierFilter minDist; < 0 off */
  float median_factor; /* MedianDistOutlierFilter factor; < 0 off */
  int n_reading, n_reference;
  orc_data_filter reading[ORC_MAX_DATA_FILTERS], reference[ORC_MAX_DATA_FILTERS];
} orc_icp_filters;

static int data_keep(const orc_data_filter *f, float x, float y) {
  if (f->dim < 0) {
    const float r = sqrtf(x * x + y * y);
    return f->kind == ORC_DATA_MAX_DIST ? r < fabsf(f->dist) : r > fabsf(f->dist);
  }
  const float v = f->dim == 0 ? x : y;
  return f->kind == ORC_DATA_MAX_DIST ? v < f->dist : v > f->dist;
}

/* the chain of n filters on pts[n_in][2] -> out (survivors in input order); returns their number */
int orc_data_filters(const orc_data_filter *f, int n, const float *pts, int n_in, float *out) {
  int m = 0;
  for (int i = 0; i < n_in; ++i) {
    int keep = 1;
    for (int k = 0; k < n && keep; ++k) keep = data_keep(&f[k], pts[2 * i], pts[2 * i + 1]);
    if (keep) out[2 * m] = pts[2 * i], out[2 * m + 1] = pts[2 * i + 1], ++m;
  }
  return m;
}

static float quantile_of(float *sorted, int n_fin, float q) { /* getDistsQuantile(q), q in [0, 1] */
  if (q == 1.0f) {
    float m = sorted[0];
    for (int i = 1; i < n_fin; ++i)
      if (sorted[i] > m) m = sorted[i];
    return m;
  }
  qsort(sorted, (size_t)n_fin, sizeof(float), cmp_f);
  return sorted[(size_t)((float)n_fin * q)];
}

int orc_icp_filtered(const float *src_in, int ns_in, const float *tgt_in, int nt_in, const float *guess,
                     const orc_icp_params *prm, const orc_icp_filters *flt, float *T_out, int *iters_out,
                     int *inliers_out) {
  float *src = (float *)malloc(sizeof(float) * 2 * (size_t)(ns_in > 0 ? ns_in : 1));
  float *tgt = (float *)malloc(sizeof(float) * 2 * (size_t)(nt_in > 0 ? nt_in : 1));
  const int ns = orc_data_filters(flt->reading, flt->n_reading, src_in, ns_in, src);
  const int nt = orc_data_filters(flt->reference, flt->n_reference, tgt_in, nt_in, tgt);
  const int use_min = flt->min_dist >= 0.f, use_med = flt->median_factor >= 0.f;
  const float min_d2 = (prm->flags & 1) ? flt->min_dist : flt->min_dist * flt->min_dist;

  memcpy(T_out, guess, 9 * sizeof(float));
  *iters_out = 0;
  *inliers_out = 0;
  if (nt <= 0) {
    free(src), free(tgt);
    return ORC_ICP_EMPTY_REF;
  }
  {
    const float det = guess[0] * guess[4] - guess[1] * guess[3];
    if (fabsf(1.0f - det) > 0.001f || det != det) {
      free(src), free(tgt);
      return ORC_ICP_NOT_RIGID;
    }
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
    /* the quantile filters, each on all matches */
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
    float srx = 0.f, sry = 0.f, sfx = 0.f, sfy = 0.f;
    for (int i = 0; i < ns; ++i) {
      int keep = match[i] >= 0;
      if (prm->outlier_max_dist > 0.f) keep = keep && (dist[i] <= out_d2);
      if (prm->trim_ratio >= 0.f) keep = keep && (dist[i] <= limit);
      if (use_min) keep = keep && (dist[i] > min_d2);
      if (use_med) keep = keep && (dist[i] <= med_limit);
      if (!keep) {
        match[i] = -1;
        continue;
      }
      ++n_keep;
      srx += step[2 * i], sry += step[2 * i + 1];
      sfx += ref[2 * match[i]], sfy += ref[2 * match[i] + 1];
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
        const float qx = step[2 * i], qy = step[2 * i + 1];
        const float nx = normals[2 * match[i]], ny = normals[2 * match[i] + 1];
        const float cr = qx * ny - qy * nx;
        const float dp = (qx - ref[2 * match[i]]) * nx + (qy - ref[2 * match[i] + 1]) * ny;
        A[0] += cr * cr, A[1] += cr * nx, A[2] += cr * ny, A[3] += nx * nx, A[4] += nx * ny, A[5] += ny * ny;
        bb[0] += cr * dp, bb[1] += nx * dp, bb[2] += ny * dp;
      }
      bb[0] = -bb[0], bb[1] = -bb[1], bb[2] = -bb[2];
      solve_llt3(A, bb, x);
      const float c = (float)cos((double)x[0]), s = (float)sin((double)x[0]);
      const float d[9] = {c, -s, x[1], s, c, x[2], 0, 0, 1};
      memcpy(dT, d, sizeof(d));
    } else {
      const float winv = 1.0f / (float)n_keep;
      const float mrx = srx * winv, mry = sry * winv, mfx = sfx * winv, mfy = sfy * winv;
      float m00 = 0.f, m01 = 0.f, m10 = 0.f, m11 = 0.f;
      for (int i = 0; i < ns; ++i) {
        if (match[i] < 0) continue;
        const float px = step[2 * i] - mrx, py = step[2 * i + 1] - mry;
        const float qx = ref[2 * match[i]] - mfx, qy = ref[2 * match[i] + 1] - mfy;
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
  free(ref), free(reading), free(step), free(dist), free(sorted), free(match), free(normals), free(src), free(tgt);
  return status;
}
