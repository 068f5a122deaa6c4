// 3-D scan matcher (sm_90a): bruce_slam.pcl.ICP.compute on [x, y, z] clouds with 4x4 guesses, point-to-point.
// Included by icp.cu only, after its helpers (IcpBox, IcpShared, block_select_kth, block_total, seq_sum9_warp, the
// map-class arguments, pick_max_cells).  Algorithm statement and conventions: oracle/icp3_ref.c (same steps, same
// float32 expressions; every product, sum, quotient and square root below is an IEEE-rounded _rn operation, so no
// contraction differs from the oracle's -ffp-contract=off).
//
// One CTA solves one (source, target, guess) problem, persistent over the problem list from a work counter.  The
// target is centred on its mean and counting-sorted into grid.cuh's grid of x, y; z is kept by sorted position next
// to it (the iterations read the target many times: shared memory in the in-CTA class, global memory in the map
// class).  Every iteration: exact 3-D nearest neighbour of every source point (grid_knn_query3, knn 1: the xy rings
// bound the 3-D distance from below), MaxDist and Trimmed weights, the six means sums and the nine cross-covariance
// sums as sequential float32 sums in point order (seq_sum9_warp, warp 0), then the SVD, the update and the checkers
// on thread 0.  No pruned or seeded search: every point searches from scratch every iteration.
#include <cfloat>

namespace sfe {

constexpr int ICP3_THREADS = 256;
constexpr int ICP3_SCRATCH = 2 * 320;  // floats: seq_sum9_warp's two buffers
constexpr int ICP3_MAX_SWEEPS = 32;    // oracle/icp3_ref.c SVD3_MAX_SWEEPS

struct Icp3Batch {
  const float *src_pts;  // [total][3]
  const int *src_off;
  const float *tgt_pts;  // [total][3]
  const int *tgt_off;
  const int *src_id, *tgt_id;  // may be null (problem p uses cloud p)
  const float *guess;          // [P][16] row-major 4x4
  float *T_out;                // [P][16]
  int *iters, *inliers, *status;
  int P, ns_max, nt_max, max_cells;
  IcpBox box;  // the problems this launch takes (icp_takes)
  sfe_icp_params prm;
  uint16_t *orig_ws;     // in-CTA: [grid][nt_max] original index of every sorted position
  int *next;             // work counter, or null: CTA c takes problems c, c + gridDim.x, ...
  const float *map_z;    // map class: centred z of every map-grid position
  const float *map_zm;   // map class: z mean of every slot
  // global-source class (icp3_gsrc_kernel): CTA c keeps reading, dist and match at src_ws + c * src_ws_stride in global
  // memory
  unsigned char *src_ws;
  size_t src_ws_stride;
};

struct Icp3Shared {
  IcpShared s;  // status, iterate, count, inliers, the selection's histograms, block_total's partials, wred
  float Ti[16], T0[16], mean[3];
  float hq[ICP_HIST][4], ht[ICP_HIST][3];
  int item;  // work-counter broadcast
};

__device__ __forceinline__ void mat4_mul_rn(const float *a, const float *b, float *c) {
  float r[16];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j)
      r[i * 4 + j] = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(a[i * 4 + 0], b[0 * 4 + j]), __fmul_rn(a[i * 4 + 1], b[1 * 4 + j])),
                                         __fmul_rn(a[i * 4 + 2], b[2 * 4 + j])),
                               __fmul_rn(a[i * 4 + 3], b[3 * 4 + j]));
#pragma unroll
  for (int i = 0; i < 16; ++i) c[i] = r[i];
}

__device__ __forceinline__ float3 apply4_rn(const float *T, float x, float y, float z) {
  float3 o;
  o.x = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(T[0], x), __fmul_rn(T[1], y)), __fmul_rn(T[2], z)), T[3]);
  o.y = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(T[4], x), __fmul_rn(T[5], y)), __fmul_rn(T[6], z)), T[7]);
  o.z = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(T[8], x), __fmul_rn(T[9], y)), __fmul_rn(T[10], z)), T[11]);
  return o;
}

// determinant of the 3x3 at m (row stride S), Eigen's cofactor order (orc_det3)
template <int S>
__device__ __forceinline__ float det3_rn(const float *m) {
  const float a = __fmul_rn(m[0], __fsub_rn(__fmul_rn(m[S + 1], m[2 * S + 2]), __fmul_rn(m[S + 2], m[2 * S + 1])));
  const float b = __fmul_rn(m[1], __fsub_rn(__fmul_rn(m[S], m[2 * S + 2]), __fmul_rn(m[S + 2], m[2 * S])));
  const float c = __fmul_rn(m[2], __fsub_rn(__fmul_rn(m[S], m[2 * S + 1]), __fmul_rn(m[S + 1], m[2 * S])));
  return __fadd_rn(__fsub_rn(a, b), c);
}

// x' = c x + s y, y' = (-s) x + c y on coefficients x[k * ST], y[k * ST], k < 3; skipped for c == 1, s == 0
template <int ST>
__device__ __forceinline__ void rot_pair_rn(float *x, float *y, float c, float s) {
  if (c == 1.0f && s == 0.0f) return;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const float xi = x[k * ST], yi = y[k * ST];
    x[k * ST] = __fadd_rn(__fmul_rn(c, xi), __fmul_rn(s, yi));
    y[k * ST] = __fadd_rn(__fmul_rn(-s, xi), __fmul_rn(c, yi));
  }
}

// One Jacobi step of Eigen's JacobiSVD on the (P, Q) block of W (orc_svd3's loop body)
template <int P, int Q>
__device__ __forceinline__ bool svd3_step(float *W, float *U, float *V, float &max_diag) {
  const float pm = __fmul_rn(2.0f * FLT_EPSILON, max_diag), thr = FLT_MIN < pm ? pm : FLT_MIN;
  if (!(fabsf(W[P * 3 + Q]) > thr || fabsf(W[Q * 3 + P]) > thr)) return false;
  const float m00 = W[P * 3 + P], m01 = W[P * 3 + Q], m10 = W[Q * 3 + P], m11 = W[Q * 3 + Q];
  const float t = __fadd_rn(m00, m11), d = __fsub_rn(m10, m01);
  float c1 = 1.f, s1 = 0.f;
  if (!(fabsf(d) < FLT_MIN)) {
    const float u = __fdiv_rn(t, d), tmp = __fsqrt_rn(__fadd_rn(1.0f, __fmul_rn(u, u)));
    s1 = __fdiv_rn(1.0f, tmp);
    c1 = __fdiv_rn(u, tmp);
  }
  float n00 = m00, n01 = m01, n11 = m11;
  if (!(c1 == 1.0f && s1 == 0.0f)) {
    n00 = __fadd_rn(__fmul_rn(c1, m00), __fmul_rn(s1, m10));
    n01 = __fadd_rn(__fmul_rn(c1, m01), __fmul_rn(s1, m11));
    n11 = __fadd_rn(__fmul_rn(-s1, m01), __fmul_rn(c1, m11));
  }
  float cr = 1.f, sr = 0.f;
  const float deno = __fmul_rn(2.0f, fabsf(n01));
  if (!(deno < FLT_MIN)) {
    const float tau = __fdiv_rn(__fsub_rn(n00, n11), deno), w = __fsqrt_rn(__fadd_rn(__fmul_rn(tau, tau), 1.0f));
    const float tt = tau > 0.f ? __fdiv_rn(1.0f, __fadd_rn(tau, w)) : __fdiv_rn(1.0f, __fsub_rn(tau, w));
    const float sign_t = tt > 0.f ? 1.0f : -1.0f, n = __fdiv_rn(1.0f, __fsqrt_rn(__fadd_rn(__fmul_rn(tt, tt), 1.0f)));
    sr = __fmul_rn(__fmul_rn(__fmul_rn(-sign_t, __fdiv_rn(n01, fabsf(n01))), fabsf(tt)), n);
    cr = n;
  }
  const float cl = __fsub_rn(__fmul_rn(c1, cr), __fmul_rn(s1, -sr)), sl = __fadd_rn(__fmul_rn(c1, -sr), __fmul_rn(s1, cr));
  rot_pair_rn<1>(W + P * 3, W + Q * 3, cl, sl);
  rot_pair_rn<3>(U + P, U + Q, cl, sl);
  rot_pair_rn<3>(W + P, W + Q, cr, -sr);
  rot_pair_rn<3>(V + P, V + Q, cr, -sr);
  const float dp = fabsf(W[P * 3 + P]), dq = fabsf(W[Q * 3 + Q]), dm = dp < dq ? dq : dp;
  if (max_diag < dm) max_diag = dm;
  return true;
}

// R = U V^T of Eigen's JacobiSVD of M, with Sorkine's reflection fix (orc_rot3); a non-finite M gives R = I.
// One thread; kept out of line, so that its registers do not weigh on the search loops of the kernels.
__device__ __noinline__ void icp3_rotation(const float *M, float *R) {
  float scale = 0.f;
  bool finite = true;
#pragma unroll
  for (int k = 0; k < 9; ++k) {
    const float a = fabsf(M[k]);
    if (!(a <= FLT_MAX)) finite = false;
    else if (a > scale) scale = a;
  }
#pragma unroll
  for (int k = 0; k < 9; ++k) R[k] = (k % 4 == 0) ? 1.f : 0.f;
  if (!finite) return;
  if (scale == 0.f) scale = 1.f;
  float W[9], U[9], V[9], S[3];
#pragma unroll
  for (int k = 0; k < 9; ++k) W[k] = __fdiv_rn(M[k], scale), U[k] = V[k] = (k % 4 == 0) ? 1.f : 0.f;
  float max_diag = fmaxf(fmaxf(fabsf(W[0]), fabsf(W[4])), fabsf(W[8]));
  for (int sweep = 0; sweep < ICP3_MAX_SWEEPS; ++sweep) {
    bool rotated = svd3_step<1, 0>(W, U, V, max_diag);
    rotated |= svd3_step<2, 0>(W, U, V, max_diag);
    rotated |= svd3_step<2, 1>(W, U, V, max_diag);
    if (!rotated) break;
  }
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    const float a = W[i * 3 + i];
    S[i] = __fmul_rn(fabsf(a), scale);
    if (a < 0.f)
#pragma unroll
      for (int k = 0; k < 3; ++k) U[k * 3 + i] = -U[k * 3 + i];
  }
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    int pos = i;
#pragma unroll
    for (int j = i + 1; j < 3; ++j)
      if (S[j] > S[pos]) pos = j;
    if (S[pos] == 0.f) break;
    if (pos != i) {
#pragma unroll
      for (int j = i + 1; j < 3; ++j)
        if (j == pos) {
          float tmp = S[i];
          S[i] = S[j], S[j] = tmp;
#pragma unroll
          for (int k = 0; k < 3; ++k) {
            tmp = U[k * 3 + i], U[k * 3 + i] = U[k * 3 + j], U[k * 3 + j] = tmp;
            tmp = V[k * 3 + i], V[k * 3 + i] = V[k * 3 + j], V[k * 3 + j] = tmp;
          }
        }
    }
  }
  float Vt[9];
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) Vt[i * 3 + j] = V[j * 3 + i];
  auto product = [&]() {
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
      for (int j = 0; j < 3; ++j)
        R[i * 3 + j] = __fadd_rn(__fadd_rn(__fmul_rn(U[i * 3 + 0], Vt[0 * 3 + j]), __fmul_rn(U[i * 3 + 1], Vt[1 * 3 + j])),
                                 __fmul_rn(U[i * 3 + 2], Vt[2 * 3 + j]));
  };
  product();
  if (det3_rn<3>(R) < 0.f) {
#pragma unroll
    for (int j = 0; j < 3; ++j) Vt[2 * 3 + j] = -Vt[2 * 3 + j];
    product();
  }
}

// Eigen's rotation-matrix -> quaternion conversion of T's top-left 3x3 (orc_quat3): q = (w, x, y, z)
__device__ __forceinline__ void quat3_rn(const float *T, float *q) {
  auto m = [&](int i, int j) { return T[i * 4 + j]; };
  float t = __fadd_rn(__fadd_rn(m(0, 0), m(1, 1)), m(2, 2));
  if (t > 0.f) {
    t = __fsqrt_rn(__fadd_rn(t, 1.0f));
    q[0] = __fmul_rn(0.5f, t);
    t = __fdiv_rn(0.5f, t);
    q[1] = __fmul_rn(__fsub_rn(m(2, 1), m(1, 2)), t);
    q[2] = __fmul_rn(__fsub_rn(m(0, 2), m(2, 0)), t);
    q[3] = __fmul_rn(__fsub_rn(m(1, 0), m(0, 1)), t);
  } else {
    int i = 0;
    if (m(1, 1) > m(0, 0)) i = 1;
    if (m(2, 2) > m(i, i)) i = 2;
    const int j = (i + 1) % 3, k = (j + 1) % 3;
    t = __fsqrt_rn(__fadd_rn(__fsub_rn(__fsub_rn(m(i, i), m(j, j)), m(k, k)), 1.0f));
    q[1 + i] = __fmul_rn(0.5f, t);
    t = __fdiv_rn(0.5f, t);
    q[0] = __fmul_rn(__fsub_rn(m(k, j), m(j, k)), t);
    q[1 + j] = __fmul_rn(__fadd_rn(m(j, i), m(i, j)), t);
    q[1 + k] = __fmul_rn(__fadd_rn(m(k, i), m(i, k)), t);
  }
}

// Eigen's angularDistance(a, b) (orc_angular_distance3)
__device__ __forceinline__ float angular_distance3_rn(const float *a, const float *b) {
  const float bw = b[0], bx = -b[1], by = -b[2], bz = -b[3];
  const float dw = __fsub_rn(__fsub_rn(__fsub_rn(__fmul_rn(a[0], bw), __fmul_rn(a[1], bx)), __fmul_rn(a[2], by)), __fmul_rn(a[3], bz));
  const float dx = __fsub_rn(__fadd_rn(__fadd_rn(__fmul_rn(a[0], bx), __fmul_rn(a[1], bw)), __fmul_rn(a[2], bz)), __fmul_rn(a[3], by));
  const float dy = __fsub_rn(__fadd_rn(__fadd_rn(__fmul_rn(a[0], by), __fmul_rn(a[2], bw)), __fmul_rn(a[3], bx)), __fmul_rn(a[1], bz));
  const float dz = __fsub_rn(__fadd_rn(__fadd_rn(__fmul_rn(a[0], bz), __fmul_rn(a[3], bw)), __fmul_rn(a[1], by)), __fmul_rn(a[2], bx));
  const float nv = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz)));
  return __fmul_rn(2.0f, atan2f(nv, fabsf(dw)));
}

// Thread 0's step after the sums: rigid fit from the kept means and M, T_iter update, Counter then Differential.
__device__ __noinline__ void icp3_update(Icp3Shared &sh, const sfe_icp_params &prm, int smooth, int n_keep,
                                         const float *mr, const float *mf, const float *M) {
  float R[9];
  icp3_rotation(M, R);
  float dT[16] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 1.f};
#pragma unroll
  for (int a = 0; a < 3; ++a) {
#pragma unroll
    for (int c = 0; c < 3; ++c) dT[a * 4 + c] = R[a * 3 + c];
    dT[a * 4 + 3] = __fsub_rn(mf[a], __fadd_rn(__fadd_rn(__fmul_rn(R[a * 3 + 0], mr[0]), __fmul_rn(R[a * 3 + 1], mr[1])),
                                               __fmul_rn(R[a * 3 + 2], mr[2])));
  }
  float Tn[16];
  mat4_mul_rn(dT, sh.Ti, Tn);
#pragma unroll
  for (int i = 0; i < 16; ++i) sh.Ti[i] = Tn[i];
  sh.s.inliers = n_keep;
  const int count = ++sh.s.count;
  if (count >= prm.max_iterations) {
    sh.s.iterate = 0;
    return;
  }
  if (smooth <= 0) return;
  int hn = sh.s.hn;
  if (hn == ICP_HIST) {
    for (int i = 0; i + 1 < ICP_HIST; ++i) {
#pragma unroll
      for (int k = 0; k < 4; ++k) sh.hq[i][k] = sh.hq[i + 1][k];
#pragma unroll
      for (int k = 0; k < 3; ++k) sh.ht[i][k] = sh.ht[i + 1][k];
    }
    hn = ICP_HIST - 1;
  }
  quat3_rn(Tn, sh.hq[hn]);
  sh.ht[hn][0] = Tn[3], sh.ht[hn][1] = Tn[7], sh.ht[hn][2] = Tn[11];
  sh.s.hn = ++hn;
  float vr = 0.f, vt = 0.f;
  if (hn > smooth) {
    for (int i = hn - 1; i >= hn - smooth; --i) {
      vr = __fadd_rn(vr, fabsf(angular_distance3_rn(sh.hq[i], sh.hq[i - 1])));
      const float ex = __fsub_rn(sh.ht[i][0], sh.ht[i - 1][0]), ey = __fsub_rn(sh.ht[i][1], sh.ht[i - 1][1]);
      const float ez = __fsub_rn(sh.ht[i][2], sh.ht[i - 1][2]);
      vt = __fadd_rn(vt, fabsf(__fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(ex, ex), __fmul_rn(ey, ey)), __fmul_rn(ez, ez)))));
    }
    vr = __fdiv_rn(vr, (float)smooth);
    vt = __fdiv_rn(vt, (float)smooth);
    if (vr < prm.min_diff_rot && vt < prm.min_diff_trans) sh.s.iterate = 0;
  }
  if (vr != vr) sh.s.status = ICP_NAN_ROT;
  else if (vt != vt) sh.s.status = ICP_NAN_TRANS;
}

// The body of icp3_kernel (MAP false: the target's grid in shared memory), icp3_map_kernel (MAP true: map grids) and
// icp3_gsrc_kernel (MAP and GSRC: map grids, and sources too large for shared memory).
// Shared layout: [Icp3Shared][sorted float2 nt_max][z f32 nt_max][cells u32]  (MAP: none of these three)
//                [reading f32 3 ns_max][dist f32 ns_max][match Pos ns_max][seq_sum9_warp scratch]
// GSRC: [Icp3Shared][seq_sum9_warp scratch] in shared memory, [reading][dist][match] at the start of the CTA's slice of
// global workspace.
template <bool MAP, bool GSRC = false>
__device__ __forceinline__ void icp3_body(const Icp3Batch &b, const MapArgs &mp) {
  static_assert(MAP || !GSRC, "icp3_body: the global-source class reads its targets as map grids");
  extern __shared__ __align__(16) unsigned char smem_raw[];
  using Pos = std::conditional_t<MAP, int, uint16_t>;
  constexpr int NONE = MAP ? -1 : 0xffff;
  Icp3Shared &sh = *reinterpret_cast<Icp3Shared *>(smem_raw);
  size_t off = (sizeof(Icp3Shared) + 15) & ~size_t(15);
  float2 *sorted = reinterpret_cast<float2 *>(smem_raw + off);
  if constexpr (!MAP) off += sizeof(float2) * (size_t)b.nt_max;
  float *zs = reinterpret_cast<float *>(smem_raw + off);
  if constexpr (!MAP) off += sizeof(float) * (size_t)b.nt_max;
  uint32_t *cells = reinterpret_cast<uint32_t *>(smem_raw + off);
  if constexpr (!MAP) off += sizeof(uint32_t) * (size_t)((b.max_cells + 2) / 2 + 1);
  off = (off + 15) & ~size_t(15);
  unsigned char *src_base = smem_raw;  // where reading .. match start (GSRC: the CTA's slice, from 0)
  const size_t shared_end = off;
  if constexpr (GSRC) src_base = b.src_ws + (size_t)blockIdx.x * b.src_ws_stride, off = 0;
  float *reading = reinterpret_cast<float *>(src_base + off);
  off += sizeof(float) * 3 * (size_t)b.ns_max;
  float *dist = reinterpret_cast<float *>(src_base + off);
  off += sizeof(float) * (size_t)b.ns_max;
  Pos *match = reinterpret_cast<Pos *>(src_base + off);
  off += sizeof(Pos) * (size_t)b.ns_max;
  off = (off + 15) & ~size_t(15);
  if constexpr (GSRC) off = shared_end;  // (the scratch stays in shared memory)
  (void)shared_end;
  float *scratch = reinterpret_cast<float *>(smem_raw + off);

  const int tid = threadIdx.x, nthr = blockDim.x;
  int tot_phase = 0, sel_pass = 0;
  for (int h = tid; h < 3 * 256; h += nthr) (&sh.s.hist[0][0])[h] = 0;
  uint16_t *orig = MAP ? nullptr : b.orig_ws + (size_t)blockIdx.x * b.nt_max;
  const sfe_icp_params prm = b.prm;
  const float max_d2 = __fmul_rn(prm.matcher_max_dist, prm.matcher_max_dist);
  const float out_d2 = (prm.flags & 1) ? prm.outlier_max_dist : __fmul_rn(prm.outlier_max_dist, prm.outlier_max_dist);
  const int smooth = min(prm.smooth_length, ICP_HIST - 1);

  for (int p = blockIdx.x; p < b.P; p = b.next ? next_work_item(b.next, &sh.item) : p + (int)gridDim.x) {
    const int si = b.src_id ? b.src_id[p] : p, ti = b.tgt_id ? b.tgt_id[p] : p;
    const float *src = b.src_pts + 3 * (size_t)b.src_off[si];
    const int ns = b.src_off[si + 1] - b.src_off[si];
    const float *tgt = b.tgt_pts + 3 * (size_t)b.tgt_off[ti];
    const int nt = b.tgt_off[ti + 1] - b.tgt_off[ti];
    const float *guess = b.guess + 16 * (size_t)p;
    if (!icp_takes(b.box, ns, nt)) continue;  // another launch's
    __syncthreads();  // previous problem fully retired before shared state is reused

    if (tid == 0) {  // admission: failure leaves T = guess
      int st = ICP_OK;
      if (ns > b.ns_max || nt > b.nt_max) st = ICP_TOO_LARGE;
      else if (nt <= 0) st = ICP_EMPTY_REF;
      else if (!(fabsf(__fsub_rn(1.0f, det3_rn<4>(guess))) <= 0.001f)) st = ICP_NOT_RIGID;
      sh.s.status = st;
      sh.s.count = 0, sh.s.inliers = 0;
    }
    __syncthreads();
    if (sh.s.status != ICP_OK) {
      if (tid < 16) b.T_out[16 * (size_t)p + tid] = guess[tid];
      if (tid == 0) b.iters[p] = 0, b.inliers[p] = 0, b.status[p] = sh.s.status;
      continue;
    }

    // ---- 1. mean of the reference; the centred grid of x, y and the centred z by sorted position
    std::conditional_t<MAP, MapGridView, GridView> g;
    const float *zp;
    if constexpr (MAP) {
      const int ms = mp.slot[p];
      const MapGrid &mg = mp.grid[ms];
      if (tid == 0) sh.mean[0] = mg.mean[0], sh.mean[1] = mg.mean[1], sh.mean[2] = b.map_zm[ms];
      g = map_grid_view(mp, ms);
      sorted = const_cast<float2 *>(mp.pts);
      zp = b.map_z;
      __syncthreads();
    } else {
      if (tid < 96) {  // warps 0, 1, 2: x, y, z
        const float sum = seq_sum_warp_global(tgt + (tid >> 5), nt, 3);
        if ((tid & 31) == 0) sh.mean[tid >> 5] = __fdiv_rn(sum, (float)nt);
      }
      __syncthreads();
      const float mx = sh.mean[0], my = sh.mean[1];
      float bnd[4] = {INFINITY, INFINITY, -INFINITY, -INFINITY};  // bounding box of the centred x, y
      for (int i = tid; i < nt; i += nthr) {
        const float x = tgt[3 * i] - mx, y = tgt[3 * i + 1] - my;
        bnd[0] = fminf(bnd[0], x), bnd[1] = fminf(bnd[1], y), bnd[2] = fmaxf(bnd[2], x), bnd[3] = fmaxf(bnd[3], y);
      }
#pragma unroll
      for (int d = 16; d > 0; d >>= 1) {
        bnd[0] = fminf(bnd[0], __shfl_xor_sync(0xffffffffu, bnd[0], d));
        bnd[1] = fminf(bnd[1], __shfl_xor_sync(0xffffffffu, bnd[1], d));
        bnd[2] = fmaxf(bnd[2], __shfl_xor_sync(0xffffffffu, bnd[2], d));
        bnd[3] = fmaxf(bnd[3], __shfl_xor_sync(0xffffffffu, bnd[3], d));
      }
      if ((tid & 31) == 0)
#pragma unroll
        for (int k = 0; k < 4; ++k) sh.s.wred[(tid >> 5) * 4 + k] = bnd[k];
      __syncthreads();
      if (tid == 0) {
        for (int w = 1; w < (nthr >> 5); ++w) {
          bnd[0] = fminf(bnd[0], sh.s.wred[w * 4 + 0]), bnd[1] = fminf(bnd[1], sh.s.wred[w * 4 + 1]);
          bnd[2] = fmaxf(bnd[2], sh.s.wred[w * 4 + 2]), bnd[3] = fmaxf(bnd[3], sh.s.wred[w * 4 + 3]);
        }
#pragma unroll
        for (int k = 0; k < 4; ++k) sh.s.bbox[k] = bnd[k];
      }
      __syncthreads();
      grid_geometry(nt, sh.s.bbox[0], sh.s.bbox[1], sh.s.bbox[2], sh.s.bbox[3], 0.05f, g, b.max_cells);
      grid_build(tgt, 3, nt, mx, my, g, sorted, cells, orig, sh.s.scan);
      const float mz = sh.mean[2];
      for (int j = tid; j < nt; j += nthr) zs[j] = __fsub_rn(tgt[3 * (size_t)orig[j] + 2], mz);
      zp = zs;
      // (published by the barrier of step 2)
    }
    const float mx = sh.mean[0], my = sh.mean[1], mz = sh.mean[2];

    // ---- 2. reading into the centred frame; T_iter = I; checker history
    if (tid == 0) {
      const float Tinv[16] = {1.f, 0.f, 0.f, -mx, 0.f, 1.f, 0.f, -my, 0.f, 0.f, 1.f, -mz, 0.f, 0.f, 0.f, 1.f};
      float gs[16];
#pragma unroll
      for (int i = 0; i < 16; ++i) gs[i] = guess[i];
      mat4_mul_rn(Tinv, gs, sh.T0);
#pragma unroll
      for (int i = 0; i < 16; ++i) sh.Ti[i] = (i % 5 == 0) ? 1.f : 0.f;
      quat3_rn(sh.Ti, sh.hq[0]);
      sh.ht[0][0] = sh.ht[0][1] = sh.ht[0][2] = 0.f;
      sh.s.hn = 1;
      sh.s.iterate = 1;
    }
    __syncthreads();
    for (int i = tid; i < ns; i += nthr) {
      const float3 r = apply4_rn(sh.T0, src[3 * i], src[3 * i + 1], src[3 * i + 2]);
      reading[3 * i] = r.x, reading[3 * i + 1] = r.y, reading[3 * i + 2] = r.z;
    }
    __syncthreads();

    // ---- 3. iterations
    while (true) {
      float Ti[12];
#pragma unroll
      for (int i = 0; i < 12; ++i) Ti[i] = sh.Ti[i];
      auto step_of = [&](int i) { return apply4_rn(Ti, reading[3 * i], reading[3 * i + 1], reading[3 * i + 2]); };
      // 3a. exact nearest neighbour of every point
      int n_fin = 0;
      for (int i = tid; i < ns; i += nthr) {
        const float3 q = step_of(i);
        float bd;
        Pos bi;
        const int found = grid_knn_query3(g, q.x, q.y, q.z, [&](int j) { return zp[j]; }, max_d2, 1, &bd, &bi, 1);
        dist[i] = found ? bd : INFINITY;
        match[i] = found ? bi : (Pos)NONE;
        n_fin += found;
      }
      const int total_fin = block_total(n_fin, &sh.s.tot[0][0], tot_phase);  // (its barrier publishes dist[], match[])

      // 3b. trimmed-distance limit = element floor(float(n) * ratio) of the ascending finite distances
      float limit = INFINITY;
      if (prm.trim_ratio >= 0.f) {
        if (total_fin == 0) {
          if (tid == 0) sh.s.status = ICP_NO_OUTLIER;
          break;
        }
        if (prm.trim_ratio == 1.0f) {
          float m = 0.f;
          for (int i = tid; i < ns; i += nthr)
            if (dist[i] < INFINITY) m = fmaxf(m, dist[i]);
#pragma unroll
          for (int d = 16; d > 0; d >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, d));
          if ((tid & 31) == 0) sh.s.wred[tid >> 5] = m;
          __syncthreads();
          m = 0.f;
          for (int w = 0; w < (nthr >> 5); ++w) m = fmaxf(m, sh.s.wred[w]);
          limit = m;
          __syncthreads();
        } else {
          int kk = (int)(size_t)__fmul_rn((float)total_fin, prm.trim_ratio);
          if (kk >= total_fin) kk = total_fin - 1;
          limit = block_select_kth(dist, ns, kk, sh.s, sel_pass);
        }
      }

      // 3c. 0/1 weights: match[] keeps the kept pairs only
      int cnt = 0;
      for (int i = tid; i < ns; i += nthr) {
        bool keep = match[i] != (Pos)NONE;
        if (prm.outlier_max_dist > 0.f) keep = keep && (dist[i] <= out_d2);
        if (prm.trim_ratio >= 0.f) keep = keep && (dist[i] <= limit);
        if (!keep) match[i] = (Pos)NONE;
        cnt += keep;
      }
      const int n_keep = block_total(cnt, &sh.s.tot[0][0], tot_phase);  // (its barrier publishes match[])
      if (n_keep == 0) {
        if (tid == 0) sh.s.status = ICP_NO_POINT;
        break;
      }

      // 3d. means and cross-covariance: sequential sums in point order by warp 0; dropped pairs add +0
      if (tid < 32) {
        float sum = seq_sum9_warp<NONE>(ns, scratch, match, sorted, [&](int i, int m, float2 t, float (&v)[9]) {
          const float3 q = step_of(i);
          v[0] = q.x, v[1] = q.y, v[2] = q.z, v[3] = t.x, v[4] = t.y, v[5] = zp[m];
        });
        const float winv = __fdiv_rn(1.0f, (float)n_keep);
        float mr[3], mf[3];
#pragma unroll
        for (int k = 0; k < 3; ++k)
          mr[k] = __fmul_rn(__shfl_sync(0xffffffffu, sum, k), winv), mf[k] = __fmul_rn(__shfl_sync(0xffffffffu, sum, 3 + k), winv);
        __syncwarp();  // (scratch is rewritten by the next pass)
        // M[a][b] = sum (ref_a - mf_a) (step_b - mr_b)
        sum = seq_sum9_warp<NONE>(ns, scratch, match, sorted, [&](int i, int m, float2 t, float (&v)[9]) {
          const float3 q = step_of(i);
          const float p[3] = {__fsub_rn(q.x, mr[0]), __fsub_rn(q.y, mr[1]), __fsub_rn(q.z, mr[2])};
          const float r[3] = {__fsub_rn(t.x, mf[0]), __fsub_rn(t.y, mf[1]), __fsub_rn(zp[m], mf[2])};
#pragma unroll
          for (int a = 0; a < 3; ++a)
#pragma unroll
            for (int c = 0; c < 3; ++c) v[a * 3 + c] = __fmul_rn(r[a], p[c]);
        });
        float M[9];
#pragma unroll
        for (int k = 0; k < 9; ++k) M[k] = __shfl_sync(0xffffffffu, sum, k);
        __syncwarp();
        // 3e. rigid fit, T_iter update, checkers (one thread)
        if (tid == 0) icp3_update(sh, prm, smooth, n_keep, mr, mf, M);
      }
      __syncthreads();
      if (sh.s.status != ICP_OK || !sh.s.iterate) break;
    }

    // ---- 4. back to the caller's frame
    if (tid == 0) {
      if (sh.s.status == ICP_OK) {
        const float Tm[16] = {1.f, 0.f, 0.f, mx, 0.f, 1.f, 0.f, my, 0.f, 0.f, 1.f, mz, 0.f, 0.f, 0.f, 1.f};
        float tmp[16], out[16], Ti[16], T0[16];
#pragma unroll
        for (int i = 0; i < 16; ++i) Ti[i] = sh.Ti[i], T0[i] = sh.T0[i];
        mat4_mul_rn(Tm, Ti, tmp);
        mat4_mul_rn(tmp, T0, out);
#pragma unroll
        for (int i = 0; i < 16; ++i) b.T_out[16 * (size_t)p + i] = out[i];
      } else {
#pragma unroll
        for (int i = 0; i < 16; ++i) b.T_out[16 * (size_t)p + i] = guess[i];
      }
      b.iters[p] = sh.s.count;
      b.inliers[p] = sh.s.inliers;
      b.status[p] = sh.s.status;
    }
  }
}

// (mp is not read: the three kernels take the same parameters, as icp_kernel's classes do)
__global__ void __launch_bounds__(ICP3_THREADS, 1) icp3_kernel(const Icp3Batch b, const MapArgs mp) {
  icp3_body<false>(b, mp);
}

__global__ void __launch_bounds__(ICP3_THREADS, 2) icp3_map_kernel(const Icp3Batch b, const MapArgs mp) {
  icp3_body<true>(b, mp);
}

__global__ void __launch_bounds__(ICP3_THREADS, 2) icp3_gsrc_kernel(const Icp3Batch b, const MapArgs mp) {
  icp3_body<true, true>(b, mp);
}

// Map class: the centred z of every map-grid position and every slot's z mean (icp3_body's sequential sum), one CTA
// per slot
__global__ void __launch_bounds__(ICP3_THREADS) icp3_map_z_kernel(const float *tgt_pts, const int *tgt_off, MapWs w,
                                                                  float *zs, float *zm) {
  __shared__ float mean;
  const int s = blockIdx.x;
  if (s >= *w.n_slots) return;
  const int ti = w.slot_tgt[s], nt = tgt_off[ti + 1] - tgt_off[ti];
  const float *tgt = tgt_pts + 3 * (size_t)tgt_off[ti];
  if (threadIdx.x < 32) {
    const float sum = seq_sum_warp_global(tgt + 2, nt, 3);
    if (threadIdx.x == 0) mean = __fdiv_rn(sum, (float)nt), zm[s] = mean;
  }
  __syncthreads();
  const MapGrid &m = w.grid[s];
  const int *cs = w.cstart + (size_t)s * w.cell_cap;
  for (int i = cs[0] + (int)threadIdx.x; i < cs[m.nx * m.ny]; i += blockDim.x)
    zs[i] = __fsub_rn(tgt[3 * (size_t)w.orig[i] + 2], mean);
}

// Shared memory of icp3_kernel's layout for ns_max x nt_max points after big targets traded cell-table entries for
// room; *max_cells receives the table's size
static size_t icp3_cta_smem(int ns_max, int nt_max, size_t budget, int *max_cells) {
  auto smem_for = [&](int mc) {
    return ((sizeof(Icp3Shared) + 15) & ~size_t(15)) + (sizeof(float2) + sizeof(float)) * (size_t)nt_max +
           sizeof(uint32_t) * (size_t)((mc + 2) / 2 + 1) + 16 + (3 * sizeof(float) + sizeof(float)) * (size_t)ns_max +
           sizeof(uint16_t) * (size_t)ns_max + 16 + ICP3_SCRATCH * sizeof(float);
  };
  int mc = pick_max_cells(nt_max);
  while (smem_for(mc) > budget && mc > nt_max / 4 + 256) mc -= mc / 8;
  *max_cells = mc;
  return smem_for(mc);
}

static size_t icp3_map_smem(int ns_max) {
  return ((sizeof(Icp3Shared) + 15) & ~size_t(15)) + 16 + (3 * sizeof(float) + sizeof(float) + sizeof(int)) * (size_t)ns_max +
         16 + ICP3_SCRATCH * sizeof(float);
}

// The global-source class: one CTA's slice for sources of up to ns_max points (reading 12 B, dist and match 4 B each
// per point, 256-byte aligned), and icp3_gsrc_kernel's shared memory
static size_t icp3_src_slice(int ns_max) { return (20 * (size_t)ns_max + 255) & ~size_t(255); }
static size_t icp3_gsrc_smem() { return ((sizeof(Icp3Shared) + 15) & ~size_t(15)) + ICP3_SCRATCH * sizeof(float); }

}  // namespace sfe
