/* TEST INFRASTRUCTURE ONLY (oracle/). Not part of the product path.
 *
 * CPU restatement of `bruce_slam.pcl.ICP.compute` on [x, y, z] clouds with a 4x4 guess: the reference's pybind module
 * builds 3-D DataPoints whenever a matrix has three columns (bruce_slam/src/bruce_slam/cpp/pcl.cpp:18-50) and
 * libpointmatcher's PointMatcher<float>::ICP then runs its 3-D chain (pcl.cpp:198-212).  The chain is the shipped
 * icp.yaml, point-to-point only:
 *     matcher            KDTreeMatcher  knn 1, epsilon 0, maxDist
 *     outlierFilters     MaxDistOutlierFilter x TrimmedDistOutlierFilter (flags bit 0: raw MaxDist compare)
 *     errorMinimizer     PointToPointErrorMinimizer (R = U V^T from a JacobiSVD of the 3x3 cross-covariance)
 *     checkers           Counter + Differential (quaternion angular distance, 3-vector translation step)
 * libpointmatcher, libnabo and Eigen are not vendored and not installed: **parity unpinned**, as for the 2-D
 * restatement (oracle/icp_ref.c, which this file mirrors step for step).  Every float32 product and sum is rounded
 * separately (-ffp-contract=off); every sum over points is a sequential float32 sum in point order.
 *
 * Steps
 *  0. target empty -> status 6.  Guess check (RigidTransformation::checkParameters): d = det of the guess's top-left
 *     3x3 in Eigen's cofactor order (det3 below: (m00 (m11 m22 - m12 m21) - m01 (m10 m22 - m12 m20)) + m02 (m10 m21 -
 *     m11 m20)); |1 - d| > 0.001 or d NaN -> status 5.
 *  1. reference centred on its mean (sequential sums in point order, sum / n); reading <- (T_mean^-1 T_init) reading,
 *     once.  Transforms apply as ((r00 x + r01 y) + r02 z) + t; 4x4 products with k ascending.
 *  2. every iteration: step = T_iter reading; exact nearest reference point in 3-D, squared distance (dx*dx + dy*dy) +
 *     dz*dz, accepted when <= maxDist^2, ties to the lower index (nn3 below: a voxel grid, exact); MaxDist and Trimmed
 *     weights exactly as oracle/icp_ref.c; kept means (sum * (1 / n_keep)); M = sum (r - r_mean)(p - p_mean)^T, i.e.
 *     M[a][b] = sum over kept pairs of (ref_a - mean) * (step_b - mean), reference times reading^T as
 *     PointToPointErrorMinimizer::compute_in_place forms it.
 *  3. R = U V^T from svd3 (Eigen's JacobiSVD<Matrix3f>, restated below); det(R) < 0 (det3 order): row 2 of V^T negated
 *     and R recomputed (Sorkine's fix, as upstream).  t = mean_ref - R mean_read; T_iter <- [R t] T_iter.
 *  4. Counter, then Differential: Eigen's rotation-matrix -> quaternion conversion (trace branch when
 *     (m00 + m11) + m22 > 0, else the largest-diagonal branch), angular distance 2 atan2(|vec(q_i conj(q_{i-1}))|,
 *     |w|) with Eigen's generic quaternion product and |vec| = sqrtf((x*x + y*y) + z*z); translation step
 *     sqrtf((dx*dx + dy*dy) + dz*dz); both averaged over the last smoothLength steps.  NaN -> status 3 / 4.
 *  5. result T_mean T_iter T_0 (status 0), else the guess.
 *
 * Modelling choices (the device kernel, icp3.cu, makes the same ones)
 *  - svd3: the matrix is divided by its largest |coefficient| (zero: by 1); sweeps over (p, q) = (1, 0), (2, 0),
 *    (2, 1) while |w_pq| or |w_qp| exceeds max(FLT_MIN, (2 FLT_EPSILON) maxDiag), maxDiag updated after every
 *    rotation; the loop ends after a sweep that rotated nothing, or after SVD3_MAX_SWEEPS (32) sweeps (Eigen has no
 *    cap; 3x3 float matrices settle in a handful).  Rotations are applied coefficient by coefficient, x' = c x + s y,
 *    y' = (-s) x + c y, and skipped when c == 1 and s == 0 (Eigen's apply_rotation_in_the_plane).  Negative diagonal
 *    entries negate the column of U; the singular values are multiplied back by the scale and sorted descending
 *    (first maximum wins; the sort stops at a zero maximum), columns of U and V swapped with them.
 *  - A non-finite M (Eigen: InvalidInput, U and V never computed) gives R = I; t is formed as usual, so a NaN mean ends
 *    the run through the Differential checker (status 4), as the 2-D closed form's fallback does.
 *  - U V^T and the recomputed product are 3x3 products with k ascending.
 *  - Planar clouds (z = 0 everywhere): a 2-D cross-covariance with a negative determinant makes det(U V^T) < 0 only
 *    through the zero third singular value, and the fix flips the z axis: the result is a proper 3-D rotation with
 *    R[2][2] = -1, not the 2-D closed form's answer.  libpointmatcher's 3-D chain does the same.
 */
#include <float.h>
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

typedef struct { /* = orc_icp_params of oracle/icp_ref.c (minimizer and normals_knn unused: point-to-point only) */
  float matcher_max_dist;
  float outlier_max_dist;
  float trim_ratio;
  int max_iterations;
  float min_diff_rot;
  float min_diff_trans;
  int smooth_length;
  int flags;
  int minimizer;
  int normals_knn;
} orc_icp_params;

enum { ORC_ICP_OK = 0, ORC_ICP_NO_OUTLIER = 1, ORC_ICP_NO_POINT = 2, ORC_ICP_NAN_ROT = 3, ORC_ICP_NAN_TRANS = 4,
       ORC_ICP_NOT_RIGID = 5, ORC_ICP_EMPTY_REF = 6 };

#define SVD3_MAX_SWEEPS 32

/* determinant of the 3x3 at m with row stride s, Eigen's cofactor order */
float orc_det3(const float *m, int s) {
  const float a = m[0] * (m[s + 1] * m[2 * s + 2] - m[s + 2] * m[2 * s + 1]);
  const float b = m[1] * (m[s] * m[2 * s + 2] - m[s + 2] * m[2 * s]);
  const float c = m[2] * (m[s] * m[2 * s + 1] - m[s + 1] * m[2 * s]);
  return (a - b) + c;
}

/* x' = c x + s y, y' = (-s) x + c y over three coefficient pairs x[k * st], y[k * st] */
static void rot_pair(float *x, float *y, int st, float c, float s) {
  if (c == 1.0f && s == 0.0f) return;
  for (int k = 0; k < 3; ++k) {
    const float xi = x[k * st], yi = y[k * st];
    x[k * st] = c * xi + s * yi;
    y[k * st] = (-s) * xi + c * yi;
  }
}

/* Eigen's JacobiSVD<Matrix3f> (full U and V) on row-major A.  Returns the sweeps made, or -1 for a non-finite A
 * (U = V = I, S = NaN). */
int orc_svd3(const float *A, float *U, float *S, float *V) {
  float scale = 0.f;
  int finite = 1;
  for (int k = 0; k < 9; ++k) {
    const float a = fabsf(A[k]);
    if (!(a <= FLT_MAX)) finite = 0;
    else if (a > scale) scale = a;
  }
  for (int k = 0; k < 9; ++k) U[k] = V[k] = (k % 4 == 0) ? 1.f : 0.f;
  if (!finite) {
    S[0] = S[1] = S[2] = NAN;
    return -1;
  }
  if (scale == 0.f) scale = 1.f;
  float W[9];
  for (int k = 0; k < 9; ++k) W[k] = A[k] / scale;
  float max_diag = fabsf(W[0]);
  if (fabsf(W[4]) > max_diag) max_diag = fabsf(W[4]);
  if (fabsf(W[8]) > max_diag) max_diag = fabsf(W[8]);
  int sweeps = 0, finished = 0;
  while (!finished && sweeps < SVD3_MAX_SWEEPS) {
    finished = 1;
    ++sweeps;
    for (int p = 1; p < 3; ++p)
      for (int q = 0; q < p; ++q) {
        const float pm = (2.0f * FLT_EPSILON) * max_diag, thr = FLT_MIN < pm ? pm : FLT_MIN;
        if (!(fabsf(W[p * 3 + q]) > thr || fabsf(W[q * 3 + p]) > thr)) continue;
        finished = 0;
        /* real_2x2_jacobi_svd: rot1 makes the block symmetric, then makeJacobi */
        const float m00 = W[p * 3 + p], m01 = W[p * 3 + q], m10 = W[q * 3 + p], m11 = W[q * 3 + q];
        const float t = m00 + m11, d = m10 - m01;
        float c1 = 1.f, s1 = 0.f;
        if (!(fabsf(d) < FLT_MIN)) {
          const float u = t / d, tmp = sqrtf(1.0f + u * u);
          s1 = 1.0f / tmp;
          c1 = u / tmp;
        }
        float n00 = m00, n01 = m01, n11 = m11;
        if (!(c1 == 1.0f && s1 == 0.0f)) {
          n00 = c1 * m00 + s1 * m10;
          n01 = c1 * m01 + s1 * m11;
          n11 = (-s1) * m01 + c1 * m11;
        }
        float cr = 1.f, sr = 0.f;
        const float deno = 2.0f * fabsf(n01);
        if (!(deno < FLT_MIN)) {
          const float tau = (n00 - n11) / deno, w = sqrtf(tau * tau + 1.0f);
          const float tt = tau > 0.f ? 1.0f / (tau + w) : 1.0f / (tau - w);
          const float sign_t = tt > 0.f ? 1.0f : -1.0f, n = 1.0f / sqrtf(tt * tt + 1.0f);
          sr = (((-sign_t) * (n01 / fabsf(n01))) * fabsf(tt)) * n;
          cr = n;
        }
        /* j_left = rot1 * j_right^T */
        const float cl = c1 * cr - s1 * (-sr), sl = c1 * (-sr) + s1 * cr;
        rot_pair(W + p * 3, W + q * 3, 1, cl, sl); /* W.applyOnTheLeft(p, q, j_left): rows */
        rot_pair(U + p, U + q, 3, cl, sl);         /* U.applyOnTheRight(p, q, j_left^T): columns */
        rot_pair(W + p, W + q, 3, cr, -sr);        /* W.applyOnTheRight(p, q, j_right) */
        rot_pair(V + p, V + q, 3, cr, -sr);        /* V.applyOnTheRight(p, q, j_right) */
        const float dp = fabsf(W[p * 3 + p]), dq = fabsf(W[q * 3 + q]), dm = dp < dq ? dq : dp;
        if (max_diag < dm) max_diag = dm;
      }
  }
  for (int i = 0; i < 3; ++i) {
    const float a = W[i * 3 + i];
    S[i] = fabsf(a);
    if (a < 0.f)
      for (int k = 0; k < 3; ++k) U[k * 3 + i] = -U[k * 3 + i];
  }
  for (int i = 0; i < 3; ++i) S[i] = S[i] * scale;
  for (int i = 0; i < 3; ++i) {
    int pos = i;
    for (int j = i + 1; j < 3; ++j)
      if (S[j] > S[pos]) pos = j;
    if (S[pos] == 0.f) break;
    if (pos != i) {
      float tmp = S[i];
      S[i] = S[pos], S[pos] = tmp;
      for (int k = 0; k < 3; ++k) {
        tmp = U[k * 3 + i], U[k * 3 + i] = U[k * 3 + pos], U[k * 3 + pos] = tmp;
        tmp = V[k * 3 + i], V[k * 3 + i] = V[k * 3 + pos], V[k * 3 + pos] = tmp;
      }
    }
  }
  return sweeps;
}

/* R = U V^T with Sorkine's reflection fix.  Returns 1 when the fix was applied, 0 when not, -1 for a non-finite M
 * (R = I). */
int orc_rot3(const float *M, float *R) {
  float U[9], S[3], V[9];
  if (orc_svd3(M, U, S, V) < 0) {
    for (int k = 0; k < 9; ++k) R[k] = (k % 4 == 0) ? 1.f : 0.f;
    return -1;
  }
  float Vt[9];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) Vt[i * 3 + j] = V[j * 3 + i];
  int fixed = 0;
  for (int pass = 0; pass < 2; ++pass) {
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j)
        R[i * 3 + j] = (U[i * 3 + 0] * Vt[0 * 3 + j] + U[i * 3 + 1] * Vt[1 * 3 + j]) + U[i * 3 + 2] * Vt[2 * 3 + j];
    if (pass == 1 || !(orc_det3(R, 3) < 0.f)) break;
    for (int j = 0; j < 3; ++j) Vt[2 * 3 + j] = -Vt[2 * 3 + j];
    fixed = 1;
  }
  return fixed;
}

/* Eigen's rotation-matrix -> quaternion conversion of the 3x3 at m (row stride s): q = (w, x, y, z) */
void orc_quat3(const float *m, int s, float *q) {
#define M_(i, j) m[(i) * s + (j)]
  float t = (M_(0, 0) + M_(1, 1)) + M_(2, 2);
  if (t > 0.f) {
    t = sqrtf(t + 1.0f);
    q[0] = 0.5f * t;
    t = 0.5f / t;
    q[1] = (M_(2, 1) - M_(1, 2)) * t;
    q[2] = (M_(0, 2) - M_(2, 0)) * t;
    q[3] = (M_(1, 0) - M_(0, 1)) * t;
  } else {
    int i = 0;
    if (M_(1, 1) > M_(0, 0)) i = 1;
    if (M_(2, 2) > M_(i, i)) i = 2;
    const int j = (i + 1) % 3, k = (j + 1) % 3;
    t = sqrtf(((M_(i, i) - M_(j, j)) - M_(k, k)) + 1.0f);
    q[1 + i] = 0.5f * t;
    t = 0.5f / t;
    q[0] = (M_(k, j) - M_(j, k)) * t;
    q[1 + j] = (M_(j, i) + M_(i, j)) * t;
    q[1 + k] = (M_(k, i) + M_(i, k)) * t;
  }
#undef M_
}

/* Eigen's angularDistance(a, b) = 2 atan2(|vec(a conj(b))|, |w(a conj(b))|) */
float orc_angular_distance3(const float *a, const float *b) {
  const float bw = b[0], bx = -b[1], by = -b[2], bz = -b[3];
  const float dw = ((a[0] * bw - a[1] * bx) - a[2] * by) - a[3] * bz;
  const float dx = ((a[0] * bx + a[1] * bw) + a[2] * bz) - a[3] * by;
  const float dy = ((a[0] * by + a[2] * bw) + a[3] * bx) - a[1] * bz;
  const float dz = ((a[0] * bz + a[3] * bw) + a[1] * by) - a[2] * bx;
  return 2.0f * atan2f(sqrtf((dx * dx + dy * dy) + dz * dz), fabsf(dw));
}

/* 4x4 row-major products, k ascending */
static void mat4_mul(const float *a, const float *b, float *c) {
  float r[16];
  for (int i = 0; i < 4; ++i)
    for (int j = 0; j < 4; ++j)
      r[i * 4 + j] = ((a[i * 4 + 0] * b[0 * 4 + j] + a[i * 4 + 1] * b[1 * 4 + j]) + a[i * 4 + 2] * b[2 * 4 + j]) +
                     a[i * 4 + 3] * b[3 * 4 + j];
  memcpy(c, r, sizeof(r));
}

static void apply4(const float *T, const float *p, float *o) {
  for (int i = 0; i < 3; ++i) o[i] = ((T[i * 4 + 0] * p[0] + T[i * 4 + 1] * p[1]) + T[i * 4 + 2] * p[2]) + T[i * 4 + 3];
}

/* ------------------------------------------------------------------ exact 3-D nearest neighbour (voxel grid)
 * Points counting-sorted into cubic cells (index order inside a cell); a query scans shells of cells around its own
 * until the distance to everything outside the shells scanned (computed in double, shrunk far beyond float32
 * rounding) exceeds the best squared distance or maxDist^2.  Distances are the float32 (dx*dx + dy*dy) + dz*dz; ties
 * go to the lower index. */
typedef struct {
  const float *pts;
  int n, nc[3];
  double o[3], h, inv_h;
  int *start, *idx;
} nn3;

static int nn3_coord(const nn3 *g, double v, int d) {
  const double c = floor((v - g->o[d]) * g->inv_h);
  return c < 0.0 ? 0 : (c >= (double)g->nc[d] ? g->nc[d] - 1 : (int)c);
}

static int nn3_cell(const nn3 *g, const float *p) {
  return (nn3_coord(g, p[2], 2) * g->nc[1] + nn3_coord(g, p[1], 1)) * g->nc[0] + nn3_coord(g, p[0], 0);
}

static void nn3_build(nn3 *g, const float *pts, int n) {
  memset(g, 0, sizeof(*g));
  g->pts = pts, g->n = n;
  double mn[3] = {0, 0, 0}, mx[3] = {0, 0, 0};
  for (int i = 0; i < n; ++i)
    for (int d = 0; d < 3; ++d) {
      const double v = pts[3 * (size_t)i + d];
      if (i == 0 || v < mn[d]) mn[d] = v;
      if (i == 0 || v > mx[d]) mx[d] = v;
    }
  double e[3], emax = 0.0;
  for (int d = 0; d < 3; ++d) e[d] = mx[d] - mn[d], g->o[d] = mn[d], emax = e[d] > emax ? e[d] : emax;
  if (!(emax > 0.0)) emax = 1.0;
  double s[3] = {e[0], e[1], e[2]}; /* descending */
  for (int a = 0; a < 3; ++a)
    for (int b = a + 1; b < 3; ++b)
      if (s[b] > s[a]) { const double t = s[a]; s[a] = s[b], s[b] = t; }
  const double nn = n > 0 ? (double)n : 1.0, tiny = emax * 1e-3;
  double h = s[2] > tiny ? cbrt(s[0] * s[1] * s[2] / nn) : (s[1] > tiny ? sqrt(s[0] * s[1] / nn) : s[0] / nn);
  if (!(h > emax * 1e-6)) h = emax * 1e-6;
  for (;;) {
    double cells = 1.0;
    for (int d = 0; d < 3; ++d) cells *= floor(e[d] / h) + 1.0;
    if (cells <= 2.0 * nn + 64.0) break;
    h *= 1.5;
  }
  g->h = h, g->inv_h = 1.0 / h;
  for (int d = 0; d < 3; ++d) g->nc[d] = (int)floor(e[d] / h) + 1;
  const int ncells = g->nc[0] * g->nc[1] * g->nc[2];
  g->start = (int *)calloc((size_t)ncells + 1, sizeof(int));
  g->idx = (int *)malloc(sizeof(int) * (size_t)(n > 0 ? n : 1));
  int *cell = (int *)malloc(sizeof(int) * (size_t)(n > 0 ? n : 1));
  for (int i = 0; i < n; ++i) cell[i] = nn3_cell(g, pts + 3 * (size_t)i), g->start[cell[i] + 1]++;
  for (int c = 0; c < ncells; ++c) g->start[c + 1] += g->start[c];
  int *fill = (int *)malloc(sizeof(int) * (size_t)ncells);
  memcpy(fill, g->start, sizeof(int) * (size_t)ncells);
  for (int i = 0; i < n; ++i) g->idx[fill[cell[i]]++] = i;
  free(fill);
  free(cell);
}

static void nn3_free(nn3 *g) {
  free(g->start);
  free(g->idx);
}

static int nn3_query(const nn3 *g, const float *q, float max_d2, float *d2_out) {
  *d2_out = INFINITY;
  if (g->n <= 0 || !isfinite(q[0]) || !isfinite(q[1]) || !isfinite(q[2])) return -1;
  int c[3];
  for (int d = 0; d < 3; ++d) c[d] = nn3_coord(g, q[d], d);
  float best = INFINITY;
  int bi = -1;
  for (int k = 0;; ++k) {
    int lo[3], hi[3];
    for (int d = 0; d < 3; ++d) lo[d] = c[d] - k, hi[d] = c[d] + k;
    for (int z = lo[2] < 0 ? 0 : lo[2]; z <= hi[2] && z < g->nc[2]; ++z)
      for (int y = lo[1] < 0 ? 0 : lo[1]; y <= hi[1] && y < g->nc[1]; ++y) {
        /* a row on the shell's z or y face is scanned whole, any other row only at x = lo and x = hi */
        const int face = z == lo[2] || z == hi[2] || y == lo[1] || y == hi[1];
        for (int x = lo[0] < 0 ? 0 : lo[0]; x <= hi[0] && x < g->nc[0]; ++x) {
          if (!face && x != lo[0] && x != hi[0]) {
            if (hi[0] >= g->nc[0]) break;
            x = hi[0] - 1;
            continue;
          }
          const int cc = (z * g->nc[1] + y) * g->nc[0] + x;
          for (int s = g->start[cc]; s < g->start[cc + 1]; ++s) {
            const int j = g->idx[s];
            const float *t = g->pts + 3 * (size_t)j;
            const float dx = q[0] - t[0], dy = q[1] - t[1], dz = q[2] - t[2];
            const float d2 = (dx * dx + dy * dy) + dz * dz;
            if (d2 < best || (d2 == best && j < bi)) best = d2, bi = j;
          }
        }
      }
    double b = INFINITY;
    for (int d = 0; d < 3; ++d) {
      if (lo[d] > 0) { const double v = (double)q[d] - (g->o[d] + lo[d] * g->h); b = v < b ? v : b; }
      if (hi[d] < g->nc[d] - 1) { const double v = (g->o[d] + (hi[d] + 1) * g->h) - (double)q[d]; b = v < b ? v : b; }
    }
    if (b == INFINITY) break; /* the shells cover the grid */
    double bb = b - 1e-6 * g->h;
    bb = bb > 0.0 ? bb * bb * (1.0 - 1e-5) : 0.0;
    if (bb > (double)best || bb > (double)max_d2) break;
  }
  if (bi >= 0 && !(best <= max_d2)) return -1;
  if (bi >= 0) *d2_out = best;
  return bi;
}

/* pcl.match(ref, in, 1, max_dist) on [x, y, z] clouds through nn3 (cross-checked against orc_match_brute3) */
void orc_nn3_match(const float *ref, int n_ref, const float *in, int n_in, float max_dist, int32_t *ids, float *dists) {
  nn3 g;
  nn3_build(&g, ref, n_ref);
  const float max_d2 = max_dist * max_dist;
  for (int i = 0; i < n_in; ++i) ids[i] = nn3_query(&g, in + 3 * (size_t)i, max_d2, &dists[i]);
  nn3_free(&g);
}

static int cmp_f(const void *a, const void *b) {
  const float x = *(const float *)a, y = *(const float *)b;
  return (x > y) - (x < y);
}

int orc_icp3(const float *src, int ns, const float *tgt, int nt, const float *guess /* 4x4 row-major */,
             const orc_icp_params *prm, float *T_out, int *iters_out, int *inliers_out) {
  memcpy(T_out, guess, 16 * sizeof(float));
  *iters_out = 0;
  *inliers_out = 0;
  if (nt <= 0) return ORC_ICP_EMPTY_REF;
  {
    const float det = orc_det3(guess, 4);
    if (fabsf(1.0f - det) > 0.001f || det != det) return ORC_ICP_NOT_RIGID;
  }
  /* 1. centre the reference */
  float sx = 0.f, sy = 0.f, sz = 0.f;
  for (int i = 0; i < nt; ++i) sx += tgt[3 * i], sy += tgt[3 * i + 1], sz += tgt[3 * i + 2];
  const float mx = sx / (float)nt, my = sy / (float)nt, mz = sz / (float)nt;
  float *ref = (float *)malloc(sizeof(float) * 3 * (size_t)nt);
  for (int i = 0; i < nt; ++i) ref[3 * i] = tgt[3 * i] - mx, ref[3 * i + 1] = tgt[3 * i + 1] - my, ref[3 * i + 2] = tgt[3 * i + 2] - mz;
  nn3 grid;
  nn3_build(&grid, ref, nt);

  const float Tmean[16] = {1, 0, 0, mx, 0, 1, 0, my, 0, 0, 1, mz, 0, 0, 0, 1};
  const float Tmean_inv[16] = {1, 0, 0, -mx, 0, 1, 0, -my, 0, 0, 1, -mz, 0, 0, 0, 1};
  float T0[16];
  mat4_mul(Tmean_inv, guess, T0);
  const size_t nb = (size_t)(ns > 0 ? ns : 1);
  float *reading = (float *)malloc(sizeof(float) * 3 * nb), *step = (float *)malloc(sizeof(float) * 3 * nb);
  float *dist = (float *)malloc(sizeof(float) * nb), *sorted = (float *)malloc(sizeof(float) * nb);
  int *match = (int *)malloc(sizeof(int) * nb);
  for (int i = 0; i < ns; ++i) apply4(T0, src + 3 * i, reading + 3 * i);

  float Ti[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
  const float max_d2 = prm->matcher_max_dist * prm->matcher_max_dist;
  const float out_d2 = (prm->flags & 1) ? prm->outlier_max_dist : prm->outlier_max_dist * prm->outlier_max_dist;
  enum { HMAX = 64 };
  float hq[HMAX][4], ht[HMAX][3];
  const int smooth = prm->smooth_length > HMAX - 1 ? HMAX - 1 : prm->smooth_length;
  orc_quat3(Ti, 4, hq[0]);
  ht[0][0] = Ti[3], ht[0][1] = Ti[7], ht[0][2] = Ti[11];
  int hn = 1;

  int status = ORC_ICP_OK, iterate = 1, count = 0, inliers = 0;
  while (iterate) {
    for (int i = 0; i < ns; ++i) apply4(Ti, reading + 3 * i, step + 3 * i);
    int n_fin = 0;
    for (int i = 0; i < ns; ++i) {
      match[i] = nn3_query(&grid, step + 3 * i, max_d2, &dist[i]);
      if (match[i] >= 0) sorted[n_fin++] = dist[i];
    }
    float limit = INFINITY;
    if (prm->trim_ratio >= 0.f) {
      if (n_fin == 0) {
        status = ORC_ICP_NO_OUTLIER;
        break;
      }
      if (prm->trim_ratio == 1.0f) {
        limit = sorted[0];
        for (int i = 1; i < n_fin; ++i)
          if (sorted[i] > limit) limit = sorted[i];
      } else {
        qsort(sorted, (size_t)n_fin, sizeof(float), cmp_f);
        limit = sorted[(size_t)((float)n_fin * prm->trim_ratio)];
      }
    }
    int n_keep = 0;
    float sr[3] = {0.f, 0.f, 0.f}, sf[3] = {0.f, 0.f, 0.f};
    for (int i = 0; i < ns; ++i) {
      int keep = match[i] >= 0;
      if (prm->outlier_max_dist > 0.f) keep = keep && (dist[i] <= out_d2);
      if (prm->trim_ratio >= 0.f) keep = keep && (dist[i] <= limit);
      if (!keep) {
        match[i] = -1;
        continue;
      }
      ++n_keep;
      for (int d = 0; d < 3; ++d) sr[d] += step[3 * i + d], sf[d] += ref[3 * match[i] + d];
    }
    if (n_keep == 0) {
      status = ORC_ICP_NO_POINT;
      break;
    }
    inliers = n_keep;
    const float winv = 1.0f / (float)n_keep;
    float mr[3], mf[3];
    for (int d = 0; d < 3; ++d) mr[d] = sr[d] * winv, mf[d] = sf[d] * winv;
    float M[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
    for (int i = 0; i < ns; ++i) {
      if (match[i] < 0) continue;
      float p[3], r[3];
      for (int d = 0; d < 3; ++d) p[d] = step[3 * i + d] - mr[d], r[d] = ref[3 * match[i] + d] - mf[d];
      for (int a = 0; a < 3; ++a)
        for (int b = 0; b < 3; ++b) M[a * 3 + b] += r[a] * p[b];
    }
    float R[9];
    orc_rot3(M, R);
    float dT[16] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 1};
    for (int a = 0; a < 3; ++a) {
      for (int b = 0; b < 3; ++b) dT[a * 4 + b] = R[a * 3 + b];
      dT[a * 4 + 3] = mf[a] - ((R[a * 3 + 0] * mr[0] + R[a * 3 + 1] * mr[1]) + R[a * 3 + 2] * mr[2]);
    }
    mat4_mul(dT, Ti, Ti);

    ++count;
    int counter_stop = 0;
    if (count >= prm->max_iterations) iterate = 0, counter_stop = 1;
    if (!counter_stop && smooth > 0) {
      if (hn == HMAX) {
        memmove(hq, hq + 1, sizeof(hq[0]) * (HMAX - 1));
        memmove(ht, ht + 1, sizeof(ht[0]) * (HMAX - 1));
        hn = HMAX - 1;
      }
      orc_quat3(Ti, 4, hq[hn]);
      ht[hn][0] = Ti[3], ht[hn][1] = Ti[7], ht[hn][2] = Ti[11];
      ++hn;
      float vr = 0.f, vt = 0.f;
      if (hn > smooth) {
        for (int i = hn - 1; i >= hn - smooth; --i) {
          vr += fabsf(orc_angular_distance3(hq[i], hq[i - 1]));
          const float ex = ht[i][0] - ht[i - 1][0], ey = ht[i][1] - ht[i - 1][1], ez = ht[i][2] - ht[i - 1][2];
          vt += fabsf(sqrtf((ex * ex + ey * ey) + ez * ez));
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
    float tmp[16];
    mat4_mul(Tmean, Ti, tmp);
    mat4_mul(tmp, T0, T_out);
  }
  nn3_free(&grid);
  free(ref), free(reading), free(step), free(dist), free(sorted), free(match);
  return status;
}
