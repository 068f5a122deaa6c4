// Robust covariance of loop-closure ICP samples (SURVEY.md row N1): batched FastMCD.
//
// SLAM.compute_icp_with_cov, bruce_slam/src/bruce_slam/slam.py:365-371, fits
//     MinCovDet(store_precision=False, support_fraction=0.8).fit(sample_transforms)
// to the (x, y, theta) results of up to 30 ICP runs.  This is that fit, restated from the installed scikit-learn 1.9
// (sklearn/covariance/_robust_covariance.py) for n_samples <= 32, n_features = 3 -- the `n_samples <= 500` branch of
// fast_mcd -- and solved for many candidates at once:
//   stage 1   30 _c_step runs (remaining_iterations = 2) from the caller's random supports of h = int(0.8 n) rows;
//             the 10 with the smallest log-det survive (np.argsort; ties here go to the earlier trial)
//   stage 2   _c_step (remaining_iterations = 30) from each of those 10 (location, covariance) estimates, including
//             the extra first iteration such a run makes; the smallest log-det wins
//   fit       correct_covariance: ValueError when h < n and allclose(raw_covariance, 0) (atol 1e-8), else
//             dist /= _consistency_factor(3, h / n); reweight_covariance: rows with dist < chi2(3).isf(0.025), their
//             mean and biased covariance, the covariance times _consistency_factor(3, 0.975)
// _c_step is followed branch for branch: the loop condition `det < previous_det and remaining and not isinf(det)`,
// the isinf / allclose / "determinant has increased" / early-stop branches, and the final dist that uses the precision
// of the previous covariance.  Building blocks: the covariance is np.cov(X.T, bias=1) (centred sum of products times
// 1 / h); the log-det is fast_logdet (LU with partial pivoting, -inf unless the sign is positive); the precision is
// scipy.linalg.pinvh (symmetric eigendecomposition, eigenvalues with |s| <= 3 eps max|s| dropped); the support is the
// h smallest Mahalanobis distances, ties to the lower row index.
//
// dtype: numpy keeps float32 samples (what compute_icp_with_cov builds from float32 ICP transforms) in float32 where
// sklearn does not convert them: X_support.mean(0) is a sequential float32 sum divided in float32, and X - location is
// rounded to float32 before the float64 product with the precision.  np.cov and the determinant work in float64 either
// way.  SFE_MCD_FLOAT32 selects that arithmetic; without it every step is float64.  Means are sequential sums in row
// order: the random supports in the order drawn, every other support in ascending row order (numpy's argpartition
// order is its own; only the rounding of a mean depends on it).
//
// Layout: one CTA per problem, 10 warps; a warp runs one trial at a time with one lane per sample.  Every lane carries
// the same location / covariance / determinant (computed redundantly from the rows in shared memory), lanes only
// differ in their own row's distance.
#include <math_constants.h>

#include "common.cuh"

namespace sfe {

namespace {

constexpr int MCD_N = SFE_MCD_MAX_SAMPLES;  // 32: one warp lane per sample
constexpr int MCD_TRIALS = SFE_MCD_TRIALS;  // 30 random starts
constexpr int MCD_BEST = 10;                // survivors of stage 1
constexpr int MCD_WARPS = 10;
constexpr unsigned FULL = 0xffffffffu;

struct McdConst {
  double c_support[MCD_N + 1];  // _consistency_factor(3, int(0.8 n) / n), by n
  double c_reweight;            // _consistency_factor(3, 0.975)
  double chi2_cut;              // chi2(3).isf(0.025)
  int f32;
};

// covariance packed as xx xy xz yy yz zz
struct Est {
  double loc[3];
  double cov[6];
  double det;
  uint32_t mask;
};

__device__ __forceinline__ double cv(const double c[6], int i, int j) {
  const int a = i < j ? i : j, b = i < j ? j : i;
  return c[a == 0 ? b : a + b + 1];
}

// rows of a support mask in ascending order, into this warp's row list
__device__ __forceinline__ void rows_from_mask(int8_t *rows, uint32_t mask, int lane) {
  __syncwarp();
  if ((mask >> lane) & 1u) rows[__popc(mask & ((1u << lane) - 1u))] = (int8_t)lane;
  __syncwarp();
}

// location = X_support.mean(axis=0); covariance = np.cov(X_support.T, bias=1)
__device__ __forceinline__ void mean_cov(const double (*X)[3], const int8_t *rows, int cnt, bool f32, double loc[3], double cov[6]) {
  double m[3];
  if (f32) {
    float s[3] = {0.f, 0.f, 0.f};
    for (int k = 0; k < cnt; ++k) {
      const int r = rows[k];
#pragma unroll
      for (int c = 0; c < 3; ++c) s[c] = __fadd_rn(s[c], (float)X[r][c]);
    }
    double t[3] = {0.0, 0.0, 0.0};
    for (int k = 0; k < cnt; ++k) {
      const int r = rows[k];
#pragma unroll
      for (int c = 0; c < 3; ++c) t[c] = __dadd_rn(t[c], X[r][c]);
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) loc[c] = (double)__fdiv_rn(s[c], (float)cnt), m[c] = __ddiv_rn(t[c], (double)cnt);
  } else {
    double t[3] = {0.0, 0.0, 0.0};
    for (int k = 0; k < cnt; ++k) {
      const int r = rows[k];
#pragma unroll
      for (int c = 0; c < 3; ++c) t[c] = __dadd_rn(t[c], X[r][c]);
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) loc[c] = m[c] = __ddiv_rn(t[c], (double)cnt);
  }
  double acc[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
  for (int k = 0; k < cnt; ++k) {
    const int r = rows[k];
    const double a = X[r][0] - m[0], b = X[r][1] - m[1], c = X[r][2] - m[2];
    acc[0] += a * a, acc[1] += a * b, acc[2] += a * c, acc[3] += b * b, acc[4] += b * c, acc[5] += c * c;
  }
  const double inv = 1.0 / (double)cnt;
#pragma unroll
  for (int i = 0; i < 6; ++i) cov[i] = acc[i] * inv;
}

// fast_logdet: slogdet by LU with partial pivoting (first largest pivot), -inf unless the sign is positive
__device__ __forceinline__ double logdet3(const double c[6]) {
  double a[3][3];
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) a[i][j] = cv(c, i, j);
  int sign = 1;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    int p = k;
#pragma unroll
    for (int i = k + 1; i < 3; ++i)
      if (fabs(a[i][k]) > fabs(a[p][k])) p = i;
#pragma unroll
    for (int i = k + 1; i < 3; ++i)
      if (i == p) {
#pragma unroll
        for (int j = 0; j < 3; ++j) {
          const double t = a[k][j];
          a[k][j] = a[i][j], a[i][j] = t;
        }
        sign = -sign;
      }
    if (a[k][k] == 0.0) return -CUDART_INF;
#pragma unroll
    for (int i = k + 1; i < 3; ++i) {
      const double l = a[i][k] / a[k][k];
#pragma unroll
      for (int j = k + 1; j < 3; ++j) a[i][j] -= l * a[k][j];
    }
  }
  double ld = 0.0;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    if (a[k][k] < 0.0) sign = -sign;
    ld += log(fabs(a[k][k]));
  }
  return sign > 0 ? ld : -CUDART_INF;
}

// one cyclic-Jacobi rotation annihilating a[p][q] (r = the third index)
template <int P, int Q, int R>
__device__ __forceinline__ void jacobi_rot(double a[3][3], double v[3][3], int sweep) {
  const double apq = a[P][Q];
  if (apq == 0.0) return;
  const double g = 100.0 * fabs(apq);
  if (sweep > 3 && fabs(a[P][P]) + g == fabs(a[P][P]) && fabs(a[Q][Q]) + g == fabs(a[Q][Q])) {
    a[P][Q] = a[Q][P] = 0.0;
    return;
  }
  const double hd = a[Q][Q] - a[P][P];
  double t;
  if (fabs(hd) + g == fabs(hd)) {
    t = apq / hd;
  } else {
    const double theta = 0.5 * hd / apq;
    t = 1.0 / (fabs(theta) + sqrt(1.0 + theta * theta));
    if (theta < 0.0) t = -t;
  }
  const double c = 1.0 / sqrt(1.0 + t * t), s = t * c, tau = s / (1.0 + c);
  a[P][P] -= t * apq;
  a[Q][Q] += t * apq;
  a[P][Q] = a[Q][P] = 0.0;
  const double gr = a[R][P], hr = a[R][Q];
  a[R][P] = a[P][R] = gr - s * (hr + gr * tau);
  a[R][Q] = a[Q][R] = hr + s * (gr - hr * tau);
#pragma unroll
  for (int r = 0; r < 3; ++r) {
    const double gv = v[r][P], hv = v[r][Q];
    v[r][P] = gv - s * (hv + gv * tau);
    v[r][Q] = hv + s * (gv - hv * tau);
  }
}

// scipy.linalg.pinvh: B = sum over kept eigenpairs of (u_k / s_k) u_k^T, kept = |s| > max|s| * 3 * eps
__device__ __forceinline__ void pinvh3(const double c[6], double out[6]) {
  double a[3][3], v[3][3];
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) a[i][j] = cv(c, i, j), v[i][j] = i == j ? 1.0 : 0.0;
  for (int sweep = 0; sweep < 50; ++sweep) {
    if (a[0][1] == 0.0 && a[0][2] == 0.0 && a[1][2] == 0.0) break;
    jacobi_rot<0, 1, 2>(a, v, sweep);
    jacobi_rot<0, 2, 1>(a, v, sweep);
    jacobi_rot<1, 2, 0>(a, v, sweep);
  }
  const double s0 = a[0][0], s1 = a[1][1], s2 = a[2][2];
  const double cut = fmax(fabs(s0), fmax(fabs(s1), fabs(s2))) * (3.0 * 2.220446049250313e-16);
  const double w[3] = {fabs(s0) > cut ? 1.0 / s0 : 0.0, fabs(s1) > cut ? 1.0 / s1 : 0.0, fabs(s2) > cut ? 1.0 / s2 : 0.0};
  const bool keep[3] = {fabs(s0) > cut, fabs(s1) > cut, fabs(s2) > cut};
  int o = 0;
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = i; j < 3; ++j) {
      double b = 0.0;
#pragma unroll
      for (int k = 0; k < 3; ++k)
        if (keep[k]) b += (v[i][k] * w[k]) * v[j][k];
      out[o++] = b;
    }
}

// (np.dot(X - location, precision) * (X - location)).sum(axis=1) for this lane's row
__device__ __forceinline__ double mahal(const double x[3], const double loc[3], const double P[6], bool f32) {
  double d[3];
#pragma unroll
  for (int c = 0; c < 3; ++c) d[c] = f32 ? (double)__fsub_rn((float)x[c], (float)loc[c]) : x[c] - loc[c];
  double r = 0.0;
#pragma unroll
  for (int j = 0; j < 3; ++j) r += (d[0] * cv(P, 0, j) + d[1] * cv(P, 1, j) + d[2] * cv(P, 2, j)) * d[j];
  return r;
}

// the h rows of smallest distance (NaN sorts last, ties to the lower row)
__device__ __forceinline__ uint32_t select_h(double d, int lane, int n, int h) {
  const double dd = isnan(d) ? CUDART_INF : d;
  int rank = 0;
#pragma unroll
  for (int j = 0; j < MCD_N; ++j) {
    const double dj = __shfl_sync(FULL, dd, j);
    rank += (j < n && (dj < dd || (dj == dd && j < lane))) ? 1 : 0;
  }
  return __ballot_sync(FULL, lane < n && rank < h);
}

// np.allclose for two scalars (rtol 1e-5, atol 1e-8; infinities close only to themselves)
__device__ __forceinline__ bool allclose(double a, double b) {
  if (isinf(a) || isinf(b)) return a == b;
  return fabs(a - b) <= 1e-8 + 1e-5 * fabs(b);
}

// sklearn _c_step.  from_est: start from (e.loc, e.cov); otherwise from the h rows already in `rows`.
// Returns the estimate in e (uniform over the warp) and this lane's distance.
__device__ __forceinline__ double c_step(const double (*X)[3], int8_t *rows, int lane, int n, int h, bool f32, int remaining,
                         bool from_est, Est &e) {
  double x[3] = {0.0, 0.0, 0.0};
  if (lane < n) x[0] = X[lane][0], x[1] = X[lane][1], x[2] = X[lane][2];
  double prec[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
  double dist = CUDART_INF;
  if (from_est) {
    pinvh3(e.cov, prec);
    dist = mahal(x, e.loc, prec, f32);
    e.mask = select_h(dist, lane, n, h);
    rows_from_mask(rows, e.mask, lane);
  } else {
    e.mask = __reduce_or_sync(FULL, lane < h ? 1u << rows[lane] : 0u);
  }
  mean_cov(X, rows, h, f32, e.loc, e.cov);
  e.det = logdet3(e.cov);
  if (isinf(e.det)) pinvh3(e.cov, prec);
  Est prev = e;
  prev.det = CUDART_INF;
  double prev_dist = dist;
  while (e.det < prev.det && remaining > 0 && !isinf(e.det)) {
    prev = e;
    pinvh3(e.cov, prec);
    dist = mahal(x, e.loc, prec, f32);
    e.mask = select_h(dist, lane, n, h);
    rows_from_mask(rows, e.mask, lane);
    mean_cov(X, rows, h, f32, e.loc, e.cov);
    e.det = logdet3(e.cov);
    --remaining;
  }
  prev_dist = dist;
  dist = mahal(x, e.loc, prec, f32);
  // isinf(det) and allclose keep the current estimate; "determinant has increased" returns the previous one unless
  // the iterations ran out (the early-stop branch comes last and wins)
  if (!allclose(e.det, prev.det) && e.det > prev.det && remaining != 0) {
    e = prev;
    dist = prev_dist;
  }
  return dist;
}

__device__ __forceinline__ void write_empty(int p, int tid, int status, double *loc, double *cov, uint32_t *raw,
                                            uint32_t *sup, int32_t *st) {
  if (tid < 3) loc[3 * (size_t)p + tid] = CUDART_NAN;
  if (tid < 9) cov[9 * (size_t)p + tid] = CUDART_NAN;
  if (tid == 0) raw[p] = 0u, sup[p] = 0u, st[p] = status;
}

__global__ void __launch_bounds__(MCD_WARPS * 32, 1)
    mincovdet_kernel(const double *__restrict__ samples, const int32_t *__restrict__ n_arr,
                     const int8_t *__restrict__ subsets, McdConst k, double *__restrict__ loc_out,
                     double *__restrict__ cov_out, uint32_t *__restrict__ raw_out, uint32_t *__restrict__ sup_out,
                     int32_t *__restrict__ status_out) {
  __shared__ double X[MCD_N][3];
  __shared__ Est s1[MCD_TRIALS];
  __shared__ Est s2[MCD_BEST];
  __shared__ double d2[MCD_BEST][MCD_N];
  __shared__ int8_t rows[MCD_WARPS][MCD_N];
  __shared__ int order[MCD_BEST];
  __shared__ int bad;
  const int p = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int n = n_arr[p];
  if (n < 0 || n > MCD_N) return write_empty(p, tid, SFE_MCD_UNSUPPORTED, loc_out, cov_out, raw_out, sup_out, status_out);
  if (n < 5) return write_empty(p, tid, SFE_MCD_TOO_FEW, loc_out, cov_out, raw_out, sup_out, status_out);
  const int h = (int)(0.8 * (double)n);  // int(support_fraction * n_samples)
  const bool f32 = k.f32 != 0;
  const int8_t *sub = subsets + (size_t)p * MCD_TRIALS * MCD_N;
  if (tid == 0) bad = 0;
  if (tid < 3 * n) X[tid / 3][tid % 3] = samples[(size_t)p * MCD_N * 3 + tid];
  __syncthreads();
  // every random support must name h distinct rows of the problem
  for (int t = warp; t < MCD_TRIALS; t += MCD_WARPS) {
    const int r = lane < h ? sub[t * MCD_N + lane] : 0;
    const bool ok = r >= 0 && r < n;
    const uint32_t m = __reduce_or_sync(FULL, lane < h && ok ? 1u << r : 0u);
    const bool all_ok = __all_sync(FULL, ok);
    if (lane == 0 && (__popc(m) != h || !all_ok)) bad = 1;
  }
  __syncthreads();
  if (bad) return write_empty(p, tid, SFE_MCD_BAD_SUBSET, loc_out, cov_out, raw_out, sup_out, status_out);

  // stage 1: select_candidates(X, h, n_trials=30, select=10, n_iter=2)
  for (int t = warp; t < MCD_TRIALS; t += MCD_WARPS) {
    __syncwarp();
    if (lane < h) rows[warp][lane] = sub[t * MCD_N + lane];
    __syncwarp();
    Est e;
    c_step(X, rows[warp], lane, n, h, f32, 2, false, e);
    if (lane == 0) s1[t] = e;
  }
  __syncthreads();
  if (tid < MCD_TRIALS) {  // np.argsort(dets)[:10], equal dets in trial order
    const double dt = s1[tid].det;
    int rank = 0;
    for (int u = 0; u < MCD_TRIALS; ++u) rank += (s1[u].det < dt || (s1[u].det == dt && u < tid)) ? 1 : 0;
    if (rank < MCD_BEST) order[rank] = tid;
  }
  __syncthreads();
  // stage 2: select_candidates(X, h, n_trials=(locations_best, covariances_best), select=1)
  if (warp < MCD_BEST) {
    Est e = s1[order[warp]];
    const double d = c_step(X, rows[warp], lane, n, h, f32, 30, true, e);
    if (lane == 0) s2[warp] = e;
    d2[warp][lane] = d;
  }
  __syncthreads();
  if (warp != 0) return;
  int best = 0;
  for (int w = 1; w < MCD_BEST; ++w)
    if (s2[w].det < s2[best].det) best = w;
  const Est raw = s2[best];
  // MinCovDet.correct_covariance
  bool zero = h < n;
#pragma unroll
  for (int i = 0; i < 6; ++i) zero = zero && fabs(raw.cov[i]) <= 1e-8;
  if (zero) {
    if (lane < 3) loc_out[3 * (size_t)p + lane] = CUDART_NAN;
    if (lane < 9) cov_out[9 * (size_t)p + lane] = CUDART_NAN;
    if (lane == 0) raw_out[p] = raw.mask, sup_out[p] = 0u, status_out[p] = SFE_MCD_ZERO_COV;
    return;
  }
  const double dist = d2[best][lane] / k.c_support[n];
  // MinCovDet.reweight_covariance
  const uint32_t m = __ballot_sync(FULL, lane < n && dist < k.chi2_cut);
  rows_from_mask(rows[0], m, lane);
  double loc[3], cov[6];
  mean_cov(X, rows[0], __popc(m), f32, loc, cov);
#pragma unroll
  for (int i = 0; i < 9; ++i) {  // (compile-time register indices)
    if (lane == i && i < 3) loc_out[3 * (size_t)p + i] = loc[i];
    if (lane == i) cov_out[9 * (size_t)p + i] = cv(cov, i / 3, i % 3) * k.c_reweight;
  }
  if (lane == 0) raw_out[p] = raw.mask, sup_out[p] = m, status_out[p] = SFE_MCD_OK;
}

}  // namespace

static int mincovdet_run(sfe_ctx *ctx, cudaStream_t st, const double *samples, const int32_t *n, const int8_t *subsets,
                         int P, const double *c_support_host, double c_reweight, double chi2_cut, int flags,
                         double *location, double *covariance, uint32_t *raw_support, uint32_t *support,
                         int32_t *status) {
  SFE_REQUIRE(P >= 0, "sfe_mincovdet: negative problem count");
  SFE_REQUIRE((flags & ~SFE_MCD_FLOAT32) == 0, "sfe_mincovdet: unknown flags 0x%x", flags);
  if (P == 0) return SFE_OK;
  SFE_REQUIRE(samples && n && subsets && c_support_host && location && covariance && raw_support && support && status,
              "sfe_mincovdet: null pointer");
  McdConst k;
  memcpy(k.c_support, c_support_host, sizeof(k.c_support));
  k.c_reweight = c_reweight;
  k.chi2_cut = chi2_cut;
  k.f32 = (flags & SFE_MCD_FLOAT32) ? 1 : 0;
  mincovdet_kernel<<<P, MCD_WARPS * 32, 0, st>>>(samples, n, subsets, k, location, covariance, raw_support, support,
                                                  status);
  SFE_CUDA(cudaGetLastError());
  ctx->launches++;
  return SFE_OK;
}

}  // namespace sfe

using namespace sfe;

extern "C" {

int sfe_mincovdet_dev(sfe_ctx *ctx, const double *samples_dev, const int32_t *n_dev, const int8_t *subsets_dev,
                      int n_problems, const double *c_support_host, double c_reweight, double chi2_cut, int flags,
                      double *location_dev, double *covariance_dev, uint32_t *raw_support_dev, uint32_t *support_dev,
                      int32_t *status_dev) {
  SFE_REQUIRE(ctx != nullptr, "sfe_mincovdet_dev: null context");
  SFE_CUDA(cudaSetDevice(ctx->device));
  return mincovdet_run(ctx, ctx->stream, samples_dev, n_dev, subsets_dev, n_problems, c_support_host, c_reweight,
                       chi2_cut, flags, location_dev, covariance_dev, raw_support_dev, support_dev, status_dev);
}

int sfe_mincovdet_host(sfe_ctx *ctx, const double *samples_host, const int32_t *n_host, const int8_t *subsets_host,
                       int n_problems, const double *c_support_host, double c_reweight, double chi2_cut, int flags,
                       double *location_host, double *covariance_host, uint32_t *raw_support_host,
                       uint32_t *support_host, int32_t *status_host) {
  SFE_REQUIRE(ctx != nullptr, "sfe_mincovdet_host: null context");
  SFE_REQUIRE(n_problems >= 0, "sfe_mincovdet_host: negative problem count");
  if (n_problems == 0) return SFE_OK;
  SFE_REQUIRE(samples_host && n_host && subsets_host && location_host && covariance_host && raw_support_host &&
                  support_host && status_host,
              "sfe_mincovdet_host: null pointer");
  for (int p = 0; p < n_problems; ++p)
    if (n_host[p] > SFE_MCD_MAX_SAMPLES || n_host[p] < 0) {
      set_error("sfe_mincovdet_host: problem %d has %d samples; at most %d are supported", p, n_host[p],
                SFE_MCD_MAX_SAMPLES);
      return SFE_ERR_UNSUPPORTED;
    }
  SFE_CUDA(cudaSetDevice(ctx->device));
  const size_t P = (size_t)n_problems;
  const size_t b_x = sizeof(double) * 3 * MCD_N * P, b_n = sizeof(int32_t) * P, b_s = (size_t)MCD_TRIALS * MCD_N * P;
  const size_t b_loc = sizeof(double) * 3 * P, b_cov = sizeof(double) * 9 * P, b_m = sizeof(uint32_t) * P;
  int rc;
  if ((rc = ensure(ctx, ctx->stage_in[0], b_x + b_n + b_s + 512)) != SFE_OK) return rc;
  if ((rc = ensure(ctx, ctx->stage_out[0], b_loc + b_cov + 3 * b_m + 512)) != SFE_OK) return rc;
  char *in = (char *)ctx->stage_in[0].ptr, *out = (char *)ctx->stage_out[0].ptr;
  double *d_x = (double *)in;
  int32_t *d_n = (int32_t *)(in + b_x);
  int8_t *d_s = (int8_t *)(in + b_x + b_n);
  double *d_loc = (double *)out, *d_cov = (double *)(out + b_loc);
  uint32_t *d_raw = (uint32_t *)(out + b_loc + b_cov), *d_sup = d_raw + P;
  int32_t *d_st = (int32_t *)(d_sup + P);
  SFE_CUDA(cudaMemcpyAsync(d_x, samples_host, b_x, cudaMemcpyHostToDevice, ctx->stream));
  SFE_CUDA(cudaMemcpyAsync(d_n, n_host, b_n, cudaMemcpyHostToDevice, ctx->stream));
  SFE_CUDA(cudaMemcpyAsync(d_s, subsets_host, b_s, cudaMemcpyHostToDevice, ctx->stream));
  rc = mincovdet_run(ctx, ctx->stream, d_x, d_n, d_s, n_problems, c_support_host, c_reweight, chi2_cut, flags, d_loc,
                     d_cov, d_raw, d_sup, d_st);
  if (rc != SFE_OK) return rc;
  SFE_CUDA(cudaMemcpyAsync(location_host, d_loc, b_loc, cudaMemcpyDeviceToHost, ctx->stream));
  SFE_CUDA(cudaMemcpyAsync(covariance_host, d_cov, b_cov, cudaMemcpyDeviceToHost, ctx->stream));
  SFE_CUDA(cudaMemcpyAsync(raw_support_host, d_raw, b_m, cudaMemcpyDeviceToHost, ctx->stream));
  SFE_CUDA(cudaMemcpyAsync(support_host, d_sup, b_m, cudaMemcpyDeviceToHost, ctx->stream));
  SFE_CUDA(cudaMemcpyAsync(status_host, d_st, sizeof(int32_t) * P, cudaMemcpyDeviceToHost, ctx->stream));
  SFE_CUDA(cudaStreamSynchronize(ctx->stream));
  return SFE_OK;
}

}  // extern "C"
