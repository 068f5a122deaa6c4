// ICP scan matcher and nearest-neighbour matcher (sm_90a).
//
// Replaces bruce_slam.pcl.ICP.compute and bruce_slam.pcl.match
// (bruce_slam/src/bruce_slam/cpp/pcl.cpp:161-174,185-212), i.e. libpointmatcher's
// PM::ICP::operator() under bruce_slam/config/icp.yaml: KD-tree NN (knn 1, maxDist 10) ->
// MaxDist(3.0) x TrimmedDist(0.8) outlier weights -> point-to-point rigid fit ->
// Counter(40) + Differential(0.01 rad, 0.1 m, smooth 4) checkers, all float32.
// Algorithm statement and conventions: oracle/icp_ref.c (same steps, same float32 expressions).
//
// One CTA solves one (source, target, guess) problem end to end: the target is centred on its
// mean and counting-sorted into a uniform grid held in shared memory (grid.cuh), the source is
// moved into the centred frame once, and every iteration runs entirely on chip:
//   transform + grid NN search per source point (seeded with the previous iteration's match: only the
//   cells overlapping the seed's disc are scanned)  ->  exact k-th smallest distance (4-pass radix
//   select on the float bits)  ->  0/1 weights  ->  warp-shuffle / shared-memory reductions of the
//   weighted means and the 2x2 cross-covariance (float32 products, float64 accumulation, fixed
//   order: deterministic)  ->  closed-form 2-D rotation and translation, T_iter update and the
//   Counter / Differential checkers on one thread.
// CTAs are persistent over the problem list (batch of keyframe pairs / of initial guesses).
#include <algorithm>
#include <type_traits>

#include <climits>
#include <cmath>

#include <cub/cub.cuh>

#include "grid.cuh"
#include "stages.cuh"

namespace sfe {

#ifndef SFE_SEQ_PIPE_MIN
#define SFE_SEQ_PIPE_MIN 256  // CTA sizes from which the sequential sums are software-pipelined (register budget)
#endif
constexpr int ICP_THREADS = 512;
constexpr int ICP_HIST = 16;  // differential-checker history kept (>= smoothLength + 1)
constexpr int ICP_COARSE = 8;            // fine cells per coarse cell edge
constexpr int ICP_COARSE_WORDS = 96;     // bitmap words: cnx*cny <= 2048 + margin
constexpr int ICP_PLANE_SCRATCH = 2 * 320;  // floats (seq_sum9_warp: two buffers of 9 rows, 36 apart, 32 used)
constexpr float ICP_PRUNED = 3.0e38f;    // "finite, but farther than we needed to know"

enum { ICP_OK = 0, ICP_NO_OUTLIER = 1, ICP_NO_POINT = 2, ICP_NAN_ROT = 3, ICP_NAN_TRANS = 4, ICP_NOT_RIGID = 5,
       ICP_EMPTY_REF = 6, ICP_SKIPPED = 7, ICP_TOO_LARGE = 8 };

// The problems one launch takes: those with ns_lo < ns <= ns_hi source and nt_lo < nt <= nt_hi target points.  The
// launches of one call take disjoint boxes that together hold every problem (icp_split_run), so each problem is solved
// and its results written by exactly one launch.
struct IcpBox {
  int ns_lo, ns_hi, nt_lo, nt_hi;
};
constexpr IcpBox ICP_BOX_ALL = {INT_MIN, INT_MAX, INT_MIN, INT_MAX};

__device__ __forceinline__ bool icp_takes(const IcpBox &x, int ns, int nt) {
  return x.ns_lo < ns && ns <= x.ns_hi && x.nt_lo < nt && nt <= x.nt_hi;
}

// One-pass exact path (per-lane searches with certified matches, no pruning passes): problems of up to
// ICP_SMALL_MULT source points per thread (and nt <= 4096) take it, and its certificates are ICP_MARGIN_MULT of the
// point's last step.  Both chosen on the config-4 replay (sources of ~360 points in 128-thread CTAs: a lower limit
// sends more problems down the slower pruned path); not re-measured on H100.  icp_run hands them to the kernel as
// IcpBatch fields: folded in as compile-time constants they change icp_kernel's register allocation and spills.
constexpr int ICP_SMALL_MULT = 5;
constexpr float ICP_MARGIN_MULT = 6.f;

struct IcpBatch {
  const float *src_pts;
  const int *src_off;
  const float *tgt_pts;
  const int *tgt_off;
  const int *src_cnt;  // optional counts (else off[c+1]-off[c])
  const int *tgt_cnt;
  int min_points;      // problems whose source or target has fewer points are skipped (ICP_SKIPPED)
  const int *raw_cnt;  // optional: un-clamped size of the source's raw cloud; > raw_cap -> ICP_TOO_LARGE
  int raw_cap;
  IcpBox box;         // the problems this launch takes (the others are another launch's; ICP_BOX_ALL: every problem)
  const int *src_id;  // may be null (problem p uses source p)
  const int *tgt_id;  // may be null
  const float *guess; // [P][9] row-major 3x3
  float *T_out;       // [P][9]
  int *iters, *inliers, *status;
  int P, ns_max, nt_max, max_cells;
  float cell_scale;  // grid cell = cell_scale * sqrt(area / n)
  sfe_icp_params prm;
  uint16_t *orig_ws;  // [slots][nt_max]
  float2 *nrm_ws;     // [slots][nt_max] point-to-plane only: normal of the target point at every sorted position
  int use_order;      // search passes visit the source points in spatially sorted order (big problems only)
  float margin_mult;  // ICP_MARGIN_MULT: certificate size in units of the point's last step (one-pass path)
  int small_mult;     // ICP_SMALL_MULT: ns <= small_mult * blockDim.x (and nt <= 4096) takes the one-pass path
  int slot_by_smid;   // workspace slot = %smid (one CTA per SM, one CTA per problem) instead of blockIdx.x
  int *next;          // persistent CTAs: work counter (next_work_item), or null: CTA c takes problems c, c + gridDim.x, ...
  const int *list;    // icp_run's classes: this launch's problems, largest first (icp_classify_kernel), or null: 0 .. P-1
  const int *list_n;  // ... and their number
  // sfe_icp_filters (the FILT kernels only): outlier filters MinDist (keep d2 > min_d2; < 0 off) and MedianDist (keep
  // d2 <= median_factor * median; < 0 off); gate_src_cnt / gate_tgt_cnt (may be null): the clouds' sizes before the
  // data filters, which the min_points test reads
  float min_d2, median_factor;
  const int *gate_src_cnt, *gate_tgt_cnt;
  // global-source class (icp_kernel's GSRC instantiations): CTA c keeps its per-source-point arrays at src_ws + c *
  // src_ws_stride in global memory
  unsigned char *src_ws;
  size_t src_ws_stride;  sfe_icp_robust robust;  // the ROBUST kernels only: the RobustOutlierFilter (last, so the other fields keep their offsets)
  const float2 *given_nrm;  // the GNRM kernels only: the targets' normals, laid out as tgt_pts (after the fields above)
};


// Per-phase cycle counts (development build, -DSFE_ICP_PHASE_CLOCKS; tools/build_icp_variants.sh, tools/icp_phases.py):
// thread 0 of every CTA reads clock64() at the phase boundaries below and adds its totals to a global array when the
// CTA exits.  Phases: 0 set-up (mean, grid, coarse map) per problem; per iteration 1 search + re-search list, 2
// trimmed-quantile select, 3 keep count, 4 means sums, 5 covariance sums, 6 fit + end barrier.  Thread 0 belongs to
// warp 0, which runs the sums and the fit, so the counts follow the CTA's critical path.  Off: no code at all.
#ifdef SFE_ICP_PHASE_CLOCKS
constexpr int ICP_PHASES = 7;
__device__ unsigned long long icp_phase_cycles[ICP_PHASES], icp_phase_count[ICP_PHASES];
static int icp_phase_per_sm[3];  // CTAs per SM of the last 128 / 256 / 512-thread launch
#define ICP_PH_DECL long long ph_t = 0, ph_acc[ICP_PHASES] = {}, ph_cnt[ICP_PHASES] = {};
#define ICP_PH_START() (threadIdx.x == 0 ? (void)(ph_t = clock64()) : (void)0)
#define ICP_PH_MARK(k)                           \
  do {                                           \
    if (threadIdx.x == 0) {                      \
      const long long t_ = clock64();            \
      ph_acc[k] += t_ - ph_t, ph_cnt[k] += 1;    \
      ph_t = t_;                                 \
    }                                            \
  } while (0)
#define ICP_PH_FLUSH()                                                                              \
  do {                                                                                              \
    if (threadIdx.x == 0)                                                                           \
      _Pragma("unroll") for (int k_ = 0; k_ < ICP_PHASES; ++k_)                                     \
        atomicAdd(&icp_phase_cycles[k_], (unsigned long long)ph_acc[k_]),                          \
            atomicAdd(&icp_phase_count[k_], (unsigned long long)ph_cnt[k_]);                       \
  } while (0)
#else
#define ICP_PH_DECL
#define ICP_PH_START() ((void)0)
#define ICP_PH_MARK(k) ((void)0)
#define ICP_PH_FLUSH() ((void)0)
#endif

// Problem of work item k: entry k of the launch's class list (P past its end), or k itself without a list
__device__ __forceinline__ int icp_work_item(const IcpBatch &b, int k) {
  if (!b.list) return k;
  return k < *b.list_n ? b.list[k] : b.P;
}

constexpr int ICP_SM_SLOTS = 256;  // >= %nsmid on every sm_90 part
__device__ __forceinline__ unsigned icp_smid() {
  unsigned r;
  asm volatile("mov.u32 %0, %%smid;" : "=r"(r));
  return r;
}

__device__ __forceinline__ void mat3_mul_rn(const float *a, const float *b, float *c) {
  float r[9];
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) {
      float acc = __fmul_rn(a[i * 3 + 0], b[0 * 3 + j]);
      acc = __fadd_rn(acc, __fmul_rn(a[i * 3 + 1], b[1 * 3 + j]));
      acc = __fadd_rn(acc, __fmul_rn(a[i * 3 + 2], b[2 * 3 + j]));
      r[i * 3 + j] = acc;
    }
#pragma unroll
  for (int i = 0; i < 9; ++i) c[i] = r[i];
}

__device__ __forceinline__ float2 apply_T(const float *T, float x, float y) {
  float2 o;
  o.x = __fadd_rn(__fadd_rn(__fmul_rn(T[0], x), __fmul_rn(T[1], y)), T[2]);
  o.y = __fadd_rn(__fadd_rn(__fmul_rn(T[3], x), __fmul_rn(T[4], y)), T[5]);
  return o;
}

// Eigen's rotation-matrix -> quaternion conversion for a 2-D rotation embedded in 3x3 (w and z)
__device__ __forceinline__ void rot_to_quat(const float *T, float &qw, float &qz) {
  const float m00 = T[0], m01 = T[1], m10 = T[3], m11 = T[4];
  float t = __fadd_rn(__fadd_rn(m00, m11), 1.0f);
  if (t > 0.f) {
    t = sqrtf(__fadd_rn(t, 1.0f));
    qw = __fmul_rn(0.5f, t);
    t = __fdiv_rn(0.5f, t);
    qz = __fmul_rn(__fsub_rn(m10, m01), t);
  } else {
    t = sqrtf(__fadd_rn(__fsub_rn(__fsub_rn(1.0f, m00), m11), 1.0f));
    qz = __fmul_rn(0.5f, t);
    t = __fdiv_rn(0.5f, t);
    qw = __fmul_rn(__fsub_rn(m10, m01), t);
  }
}

// same for one int
__device__ __forceinline__ int block_total(int v, int *scratch /* [2][16] smem */, int &phase) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  int *half = scratch + (phase & 1) * 16;
  ++phase;
  v = __reduce_add_sync(0xffffffffu, v);
  if (lane == 0) half[warp] = v;
  __syncthreads();
  return __reduce_add_sync(0xffffffffu, lane < nwarps ? half[lane] : 0);
}

struct IcpShared {  // small fixed-size part of the shared state
  float Ti[9];
  float Tprev[9];  // T_iter of the previous iteration (how far did every point move since?)
  float T0[9];
  float mean[2];
  float bbox[4];
  int iterate, status, count, inliers;
  uint32_t sel_val;  // radix select: the element found alone in its bin
  int todo_n;        // one-pass path: length of the re-search list
  int hist[3][256];  // radix-select histograms, used in rotation (block_select_kth)
  int scan[36];
  int tot[2][16];
  float wred[4 * 16];  // per-warp partials of the bounding-box / maximum reductions
  float hq_w[ICP_HIST], hq_z[ICP_HIST], ht_x[ICP_HIST], ht_y[ICP_HIST];
  int hn;
  float seq[2];  // reference mean (sequential sums)
  union {        // a launch runs one accumulation mode (flags bit 1)
    double red[2 * 5 * 16];                   // float64 mode: block_sum, <= 16 warps per CTA
    __align__(16) float seq_buf[2 * 4 * 36];  // sequential mode: staging of seq_sum4_warp
  };
  int cnx, cny;               // coarse occupancy grid (ICP_COARSE x ICP_COARSE fine cells per coarse cell)
  uint32_t coarse[ICP_COARSE_WORDS];
};

// k-th smallest (0-based) of the finite entries of vals[0..n): 4-pass radix select on the float bits
// (non-negative floats order like their bit patterns).  All threads call it; kk < number of finite entries.
// One barrier per pass: pass number `pass` (counted over the CTA's lifetime) fills histogram pass % 3 and clears
// histogram (pass + 1) % 3 -- last read two passes ago -- before its barrier; after the barrier every warp scans
// the 256 bins itself (8 per lane), so no second barrier is needed to publish the selected bin.
__device__ __forceinline__ float block_select_kth(const float *vals, int n, int kk, IcpShared &sh, int &pass) {
  const int tid = threadIdx.x, nthr = blockDim.x, lane = tid & 31;
  uint32_t prefix = 0, mask = 0;
  for (int shift = 24; shift >= 0; shift -= 8) {
    int *hist = sh.hist[pass % 3], *next = sh.hist[(pass + 1) % 3];
    ++pass;
    for (int h = tid; h < 256; h += nthr) next[h] = 0;
    for (int i = tid; i < n; i += nthr) {
      const float v = vals[i];
      if (!(v < INFINITY)) continue;
      const uint32_t u = __float_as_uint(v);
      if ((u & mask) == prefix) atomicAdd(&hist[(u >> shift) & 255u], 1);
    }
    __syncthreads();
    int c[8], sum = 0;  // lane l owns bins 8l .. 8l+7
#pragma unroll
    for (int j = 0; j < 8; ++j) c[j] = hist[lane * 8 + j], sum += c[j];
    int incl = sum;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const int t = __shfl_up_sync(0xffffffffu, incl, d);
      if (lane >= d) incl += t;
    }
    // the lane whose 8 bins contain rank kk, then lanes 0..7 look at those 8 bins together
    const unsigned owner = __ballot_sync(0xffffffffu, kk >= incl - sum && kk < incl);
    const int src = owner ? __ffs(owner) - 1 : 31;
    const int base = __shfl_sync(0xffffffffu, incl - sum, src);  // number of entries in the bins before lane src's
    const int cj = hist[src * 8 + (lane & 7)];
    int ij = cj;
#pragma unroll
    for (int d = 1; d < 8; d <<= 1) {
      const int t = __shfl_up_sync(0xffffffffu, ij, d);
      if ((lane & 7) >= d) ij += t;
    }
    const unsigned hit = __ballot_sync(0xffffffffu, kk - base < ij) & 0xffu;
    const int j = hit ? __ffs(hit) - 1 : 7;
    const int bin = src * 8 + j;
    const int in_bin = __shfl_sync(0xffffffffu, cj, j);
    kk = kk - base - (__shfl_sync(0xffffffffu, ij, j) - in_bin);
    prefix |= (uint32_t)bin << shift;
    mask |= 255u << shift;
    if (in_bin == 1 && shift > 0) {
      // the wanted element is alone in its bin: no need to resolve its remaining bits digit by digit -- the one
      // thread that holds it publishes it (typically after two of the four passes for a few hundred values)
      for (int i = tid; i < n; i += nthr) {
        const float v = vals[i];
        if (v < INFINITY && (__float_as_uint(v) & mask) == prefix) sh.sel_val = __float_as_uint(v);
      }
      __syncthreads();
      return __uint_as_float(sh.sel_val);  // (next written after at least one more barrier)
    }
  }
  return __uint_as_float(prefix);
}

// Exact SEQUENTIAL float32 sums in index order (the accumulation order of oracle/icp_ref.c; default mode), computed
// by one warp.  The dependent chain is the float add alone (~4 cycles per term); terms beyond n (or of dropped
// pairs) are +0, which leaves a sum unchanged bit for bit.  All 32 lanes of the warp must call these.
// Four sequential sums at once (the components of one float4 term per point), by ONE warp with few instructions:
// lane j evaluates the four terms of point base + j and parks them, transposed, in shared memory ([component][32],
// rows padded to 36 floats so that the four reading lanes hit different banks); lanes 0..3 then add "their"
// component's 32 values in order (eight LDS.128 + 32 dependent adds).  ~55 warp instructions per 32 points for all
// four sums; result: lane c (c < 4) returns the sum of component c.
// `scratch` = [2][4][36] floats (double-buffered: a batch is written while the previous one may still be read).
template <bool PIPELINED, typename F>
__device__ __forceinline__ float seq_sum4_warp(int n, float *scratch, F term4) {
  const int lane = threadIdx.x & 31;
  float s = 0.f;
  if (!PIPELINED) {
    int it = 0;
    for (int base = 0; base < n; base += 32, ++it) {
      float *buf = scratch + (it & 1) * (4 * 36);
      const float4 t = base + lane < n ? term4(base + lane) : make_float4(0.f, 0.f, 0.f, 0.f);
      buf[0 * 36 + lane] = t.x, buf[1 * 36 + lane] = t.y, buf[2 * 36 + lane] = t.z, buf[3 * 36 + lane] = t.w;
      __syncwarp();
      if (lane < 4) {
        const float4 *v = reinterpret_cast<const float4 *>(buf + lane * 36);
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          const float4 a = v[k];
          s = __fadd_rn(__fadd_rn(__fadd_rn(__fadd_rn(s, a.x), a.y), a.z), a.w);
        }
      }
      // (the buffer written two batches from now is this one: every lane passes the next batch's __syncwarp first)
    }
    return s;
  }
  // Software-pipelined form (CTA sizes with registers to spare): while lanes 0..3 add batch k from registers, all
  // lanes evaluate and park batch k + 1, so the add chain never waits for shared memory.
  float4 cur[8];
  {
    const float4 t = lane < n ? term4(lane) : make_float4(0.f, 0.f, 0.f, 0.f);
    scratch[0 * 36 + lane] = t.x, scratch[1 * 36 + lane] = t.y, scratch[2 * 36 + lane] = t.z, scratch[3 * 36 + lane] = t.w;
    __syncwarp();
    const float4 *v = reinterpret_cast<const float4 *>(scratch + (lane & 3) * 36);
#pragma unroll
    for (int k = 0; k < 8; ++k) cur[k] = v[k];
  }
  int it = 1;
  for (int base = 0; base < n; base += 32, ++it) {
    const int nb = base + 32;
    float *buf = scratch + (it & 1) * (4 * 36);
    if (nb < n) {  // (warp-uniform) park the next batch
      const float4 t = nb + lane < n ? term4(nb + lane) : make_float4(0.f, 0.f, 0.f, 0.f);
      buf[0 * 36 + lane] = t.x, buf[1 * 36 + lane] = t.y, buf[2 * 36 + lane] = t.z, buf[3 * 36 + lane] = t.w;
    }
#pragma unroll
    for (int k = 0; k < 8; ++k)
      s = __fadd_rn(__fadd_rn(__fadd_rn(__fadd_rn(s, cur[k].x), cur[k].y), cur[k].z), cur[k].w);
    __syncwarp();
    if (nb < n) {
      const float4 *v = reinterpret_cast<const float4 *>(buf + (lane & 3) * 36);
#pragma unroll
      for (int k = 0; k < 8; ++k) cur[k] = v[k];
    }
  }
  return s;  // lanes c, c + 4, c + 8, ... all hold the sum of component c
}

// Point-to-plane: the nine sequential sums of the normal equations in one pass.  Same scheme as seq_sum4_warp with
// nine rows -- lanes 0..8 each add one component's 32 values per batch, in point order -- and the per-pair normal
// (a gather from global memory, ~700 cycles) requested for eight batches at once so that its latency is paid once
// per 256 points, not once per batch.  `scratch` = 2 x 320 floats (nine rows 36 floats apart, 32 used).  term9(i, m, n, v): the nine terms of kept
// pair i (match m, normal n).  Lane c (c < 9) returns the sum of component c.
template <int NONE, typename Pos, typename F>
__device__ __forceinline__ float seq_sum9_warp(int n, float *scratch, const Pos *match, const float2 *nrm, F term9) {
  const int lane = threadIdx.x & 31;
  float s = 0.f;
  int it = 0;
  for (int chunk = 0; chunk < n; chunk += 256) {
    int mm[8];
    float2 nn[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const int i = chunk + 32 * k + lane;
      mm[k] = i < n ? match[i] : NONE;
      nn[k] = mm[k] != NONE ? nrm[mm[k]] : make_float2(0.f, 0.f);
    }
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      if (chunk + 32 * k >= n) break;  // (warp-uniform)
      float *buf = scratch + (it & 1) * 320;
      ++it;
      float v[9] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
      if (mm[k] != NONE) term9(chunk + 32 * k + lane, mm[k], nn[k], v);
#pragma unroll
      for (int c = 0; c < 9; ++c) buf[c * 36 + lane] = v[c];
      __syncwarp();
      if (lane < 9) {  // (8-byte loads: the scratch may sit on dist[], which is only 8-byte aligned)
        const float2 *r = reinterpret_cast<const float2 *>(buf + lane * 36);
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          const float2 a = r[j];
          s = __fadd_rn(__fadd_rn(s, a.x), a.y);
        }
      }
      // (this buffer is rewritten two batches from now: every lane passes the next batch's __syncwarp first)
    }
  }
  return s;
}

// ROBUST point-to-point: R (<= 8) sequential float32 sums in index order at once, by one warp: lane j parks the R terms
// of point base + j (term(i, v)) in `scratch` ([R][36] floats, single-buffered), lanes 0..R-1 add their row's 32 values
// in order.  Lane c (c < R) returns the sum of component c.  All 32 lanes of the warp must call it.
template <int R, typename F>
__device__ __forceinline__ float seq_sum_rows_warp(int n, float *scratch, F term) {
  static_assert(R >= 1 && R <= 8, "seq_sum_rows_warp: one row per lane of the first eight");
  const int lane = threadIdx.x & 31;
  float s = 0.f;
  for (int base = 0; base < n; base += 32) {
    float v[R];
    if (base + lane < n) {
      term(base + lane, v);
    } else {
#pragma unroll
      for (int c = 0; c < R; ++c) v[c] = 0.f;
    }
#pragma unroll
    for (int c = 0; c < R; ++c) scratch[c * 36 + lane] = v[c];
    __syncwarp();
    if (lane < R) {
      const float4 *r = reinterpret_cast<const float4 *>(scratch + lane * 36);
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const float4 a = r[k];
        s = __fadd_rn(__fadd_rn(__fadd_rn(__fadd_rn(s, a.x), a.y), a.z), a.w);
      }
    }
    __syncwarp();  // (the next batch rewrites the rows)
  }
  return s;
}

// RobustOutlierFilter weight of a pair of squared distance e2 (oracle/robust_ref.c): k = tuning, k2 = k * k, division
// and sqrt IEEE-rounded, nothing contracted, welsch's exp in float64 rounded to float32; 0 where e2 >= approximation
__device__ __forceinline__ float icp_robust_weight(const sfe_icp_robust &r, float e2) {
  const float k = r.tuning, k2 = __fmul_rn(k, k);
  float w = 1.f;
  switch (r.fct) {
    case SFE_ICP_ROBUST_CAUCHY: w = __fdiv_rn(1.f, __fadd_rn(1.f, __fdiv_rn(e2, k2))); break;
    case SFE_ICP_ROBUST_WELSCH: w = (float)exp((double)(-__fdiv_rn(e2, k2))); break;
    case SFE_ICP_ROBUST_SC: {
      const float t = __fadd_rn(k, e2);
      w = e2 >= k ? __fdiv_rn(__fmul_rn(4.f, k2), __fmul_rn(t, t)) : 1.f;
      break;
    }
    case SFE_ICP_ROBUST_GM: {
      const float t = __fadd_rn(k, e2);
      w = __fdiv_rn(k2, __fmul_rn(t, t));
      break;
    }
    case SFE_ICP_ROBUST_TUKEY: {
      const float u = __fsub_rn(1.f, __fdiv_rn(e2, k2));
      w = e2 >= k2 ? 0.f : __fmul_rn(u, u);
      break;
    }
    case SFE_ICP_ROBUST_HUBER: w = e2 >= k2 ? __fdiv_rn(k, __fsqrt_rn(e2)) : 1.f; break;
    case SFE_ICP_ROBUST_L1: w = __fdiv_rn(1.f, __fsqrt_rn(e2)); break;
  }
  return e2 >= r.approximation ? 0.f : w;
}

#include "icp_kernel_body.cuh"

// Data filters of sfe_icp_filters (MaxDist / MinDistDataPointsFilter): cloud c of a batch (cloud id[c], or c with id
// null) -> its survivors, in input order, at out_pts + 2 * c * n_max; out_off[c] = c * n_max, out_cnt[c] = their number,
// out_raw[c] = the cloud's size before the filters.  A cloud of more than n_max points is passed on uncompacted with its
// size (the ICP launch then reports it, SFE_ICP_TOO_LARGE).  One CTA per cloud.
struct IcpDataFilters {
  int n;
  sfe_icp_data_filter f[SFE_ICP_MAX_DATA_FILTERS];
};
constexpr int ICP_DF_THREADS = 256;

// ShadowDataPointsFilter: |n^ . p^| > sin_eps, v^ = v / sqrtf(v.v) when v.v > 0 else v (Eigen's normalized()), every
// operation rounded on its own (oracle/shadow_ref.c)
__device__ __forceinline__ bool icp_shadow_keep(float x, float y, float2 n, float sin_eps) {
  const float nn = __fadd_rn(__fmul_rn(n.x, n.x), __fmul_rn(n.y, n.y));
  const float pp = __fadd_rn(__fmul_rn(x, x), __fmul_rn(y, y));
  if (nn > 0.f) {
    const float l = __fsqrt_rn(nn);
    n.x = __fdiv_rn(n.x, l), n.y = __fdiv_rn(n.y, l);
  }
  if (pp > 0.f) {
    const float l = __fsqrt_rn(pp);
    x = __fdiv_rn(x, l), y = __fdiv_rn(y, l);
  }
  return fabsf(__fadd_rn(__fmul_rn(n.x, x), __fmul_rn(n.y, y))) > sin_eps;
}

// NRM: the pass after a SurfaceNormalDataPointsFilter -- SFE_ICP_DATA_SHADOW entries (dist = sinf(eps), set on the host)
// read the point's normal n
template <bool NRM = false>
__device__ __forceinline__ bool icp_data_keep(const IcpDataFilters &df, float x, float y, float2 n = {}) {
  bool keep = true;
  for (int k = 0; k < df.n; ++k) {
    const sfe_icp_data_filter &f = df.f[k];
    bool kk;
    if constexpr (NRM)
      if (f.kind == SFE_ICP_DATA_SHADOW) {
        keep = keep && icp_shadow_keep(x, y, n, f.dist);
        continue;
      }
    if (f.dim < 0) {  // sqrtf of the unfused float32 x*x + y*y (oracle/icp_filters_ref.c)
      const float r = __fsqrt_rn(__fadd_rn(__fmul_rn(x, x), __fmul_rn(y, y)));
      kk = f.kind == SFE_ICP_DATA_MAX_DIST ? r < fabsf(f.dist) : r > fabsf(f.dist);
    } else {
      const float v = f.dim == 0 ? x : y;
      kk = f.kind == SFE_ICP_DATA_MAX_DIST ? v < f.dist : v > f.dist;
    }
    keep = keep && kk;
  }
  return keep;
}

// After an octree stage (downsample_run, which reads at most n_max points of a cloud): the clouds passed on
// uncompacted keep their size, so that the ICP launch still reports them SFE_ICP_TOO_LARGE
__global__ void icp_keep_too_large_kernel(const int *in_cnt, int n_clouds, int n_max, int *out_cnt) {
  for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < n_clouds; c += gridDim.x * blockDim.x)
    if (in_cnt[c] > n_max) out_cnt[c] = in_cnt[c];
}

// NRM: the pass after a SurfaceNormalDataPointsFilter, whose normals in_nrm are laid out as the points (in.off, no id)
template <bool NRM>
__global__ void __launch_bounds__(ICP_DF_THREADS) icp_data_filter_kernel(const PackedClouds in, const int *id,
                                                                         int n_clouds, const IcpDataFilters df,
                                                                         float *out_pts, int *out_off, int *out_cnt,
                                                                         int *out_raw, const float2 *in_nrm) {
  __shared__ int warp_n[ICP_DF_THREADS / 32];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (int c = blockIdx.x; c < n_clouds; c += gridDim.x) {
    const int ci = id ? id[c] : c;
    const int n = in.cnt ? in.cnt[ci] : in.off[ci + 1] - in.off[ci];
    const float *src = in.pts + 2 * (size_t)in.off[ci];
    float *dst = out_pts + 2 * (size_t)c * in.n_max;
    if (tid == 0) out_off[c] = c * in.n_max, out_raw[c] = n;
    if (c == n_clouds - 1 && tid == 0) out_off[n_clouds] = n_clouds * in.n_max;
    if (n > in.n_max) {
      if (tid == 0) out_cnt[c] = n;
      continue;
    }
    int base = 0;
    for (int i0 = 0; i0 < n; i0 += ICP_DF_THREADS) {
      const int i = i0 + tid;
      float x = 0.f, y = 0.f;
      bool keep;
      if constexpr (NRM)
        keep = i < n && (x = src[2 * i], y = src[2 * i + 1], icp_data_keep<true>(df, x, y, in_nrm[in.off[ci] + i]));
      else
        keep = i < n && (x = src[2 * i], y = src[2 * i + 1], icp_data_keep(df, x, y));
      const unsigned m = __ballot_sync(0xffffffffu, keep);
      if (lane == 0) warp_n[warp] = __popc(m);
      __syncthreads();
      int before = base, total = 0;
      for (int w = 0; w < ICP_DF_THREADS / 32; ++w) {
        if (w < warp) before += warp_n[w];
        total += warp_n[w];
      }
      if (keep) {
        const int at = before + __popc(m & ((1u << lane) - 1u));
        dst[2 * at] = x, dst[2 * at + 1] = y;
      }
      base += total;
      __syncthreads();  // warp_n is rewritten by the next chunk
    }
    if (tid == 0) out_cnt[c] = base;
  }
}

// pcl.match: nearest reference point (within max_dist) of every query point; one CTA per (ref, query) pair
struct MatchBatch {
  const float *ref_pts;
  const int *ref_off;
  const float *in_pts;
  const int *in_off;
  int P, nt_max, max_cells;
  float max_dist;
  int32_t *ids;  // [total queries]
  float *dists;
  uint16_t *orig_ws;
  MapArgs map;  // map class (match_map_kernel): pair p reads its reference from the grid in slot map.slot[p]
};

// One pair's reference of nt points (nt >= 1) in match_kernel's layout: the bounding box over the CTA, the grid
// geometry and the counting sort into sorted / cells (shared), original indices in orig.  All threads call it.
// DIM 3: rows of x, y, z; the grid holds x, y.
template <int DIM = 2>
__device__ __forceinline__ void match_ref_grid(const MatchBatch &b, const float *ref, int nt, float2 *sorted,
                                               uint32_t *cells, uint16_t *orig, int *scan, float *bbox_w, float *bbox,
                                               GridView &g) {
  const int tid = threadIdx.x, nthr = blockDim.x;
  float mn_x = INFINITY, mn_y = INFINITY, mxx = -INFINITY, mxy = -INFINITY;
  for (int i = tid; i < nt; i += nthr) {
    const float x = ref[DIM * i], y = ref[DIM * i + 1];
    mn_x = fminf(mn_x, x), mxx = fmaxf(mxx, x), mn_y = fminf(mn_y, y), mxy = fmaxf(mxy, y);
  }
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) {
    mn_x = fminf(mn_x, __shfl_xor_sync(0xffffffffu, mn_x, d));
    mn_y = fminf(mn_y, __shfl_xor_sync(0xffffffffu, mn_y, d));
    mxx = fmaxf(mxx, __shfl_xor_sync(0xffffffffu, mxx, d));
    mxy = fmaxf(mxy, __shfl_xor_sync(0xffffffffu, mxy, d));
  }
  if ((tid & 31) == 0) {
    bbox_w[(tid >> 5) * 4 + 0] = mn_x, bbox_w[(tid >> 5) * 4 + 1] = mn_y;
    bbox_w[(tid >> 5) * 4 + 2] = mxx, bbox_w[(tid >> 5) * 4 + 3] = mxy;
  }
  __syncthreads();
  if (tid == 0) {
    float a = INFINITY, bb = INFINITY, c = -INFINITY, d = -INFINITY;
    for (int w = 0; w < (nthr >> 5); ++w) {
      a = fminf(a, bbox_w[w * 4 + 0]), bb = fminf(bb, bbox_w[w * 4 + 1]);
      c = fmaxf(c, bbox_w[w * 4 + 2]), d = fmaxf(d, bbox_w[w * 4 + 3]);
    }
    bbox[0] = a, bbox[1] = bb, bbox[2] = c, bbox[3] = d;
  }
  __syncthreads();
  grid_geometry(nt, bbox[0], bbox[1], bbox[2], bbox[3], 0.05f, g, b.max_cells);
  grid_build(ref, DIM, nt, 0.f, 0.f, g, sorted, cells, orig, scan);
}

__global__ void __launch_bounds__(ICP_THREADS) match_kernel(const MatchBatch b) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  __shared__ int scan[36];
  __shared__ float bbox_w[4 * 32];
  __shared__ float bbox[4];
  float2 *sorted = reinterpret_cast<float2 *>(smem_raw);
  uint32_t *cells = reinterpret_cast<uint32_t *>(smem_raw + sizeof(float2) * (size_t)b.nt_max);
  const int tid = threadIdx.x, nthr = blockDim.x;
  uint16_t *orig = b.orig_ws + (size_t)blockIdx.x * b.nt_max;
  const float max_d2 = __fmul_rn(b.max_dist, b.max_dist);
  for (int p = blockIdx.x; p < b.P; p += gridDim.x) {
    const float *ref = b.ref_pts + 2 * (size_t)b.ref_off[p];
    const int nt = b.ref_off[p + 1] - b.ref_off[p];
    const float *in = b.in_pts + 2 * (size_t)b.in_off[p];
    const int ns = b.in_off[p + 1] - b.in_off[p];
    int32_t *ids = b.ids + b.in_off[p];
    float *dists = b.dists + b.in_off[p];
    if (nt > b.nt_max) continue;  // the map class's (match_map_kernel)
    __syncthreads();
    if (nt <= 0) {
      for (int i = tid; i < ns; i += nthr) ids[i] = -1, dists[i] = INFINITY;
      continue;
    }
    GridView g;
    match_ref_grid(b, ref, nt, sorted, cells, orig, scan, bbox_w, bbox, g);
    for (int i = tid; i < ns; i += nthr) {
      const NNResult r = nn_query(g, in[2 * i], in[2 * i + 1], max_d2);
      ids[i] = r.pos >= 0 ? (int32_t)orig[r.pos] : -1;
      dists[i] = r.d2;
    }
  }
}

// The map class of pcl.match: references held as map grids in global memory.  The whole grid works on one pair's
// queries at a time (a map match is one large reference and a few thousand queries, not many small pairs).
__global__ void __launch_bounds__(ICP_THREADS) match_map_kernel(const MatchBatch b) {
  const float max_d2 = __fmul_rn(b.max_dist, b.max_dist);
  for (int p = 0; p < b.P; ++p) {
    const int ms = b.map.slot[p];
    if (ms < 0) continue;
    const MapGridView g = map_grid_view(b.map, ms);
    const float *in = b.in_pts + 2 * (size_t)b.in_off[p];
    const int ns = b.in_off[p + 1] - b.in_off[p];
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < ns; i += gridDim.x * blockDim.x) {
      const NNResult r = nn_query(g, in[2 * i], in[2 * i + 1], max_d2);
      b.ids[b.in_off[p] + i] = r.pos >= 0 ? (int32_t)g.orig[r.pos] : -1;
      b.dists[b.in_off[p] + i] = r.d2;
    }
  }
}

// pcl.match with knn > 1 (grid_knn_query).  Output rows: neighbour j of query i of pair p goes to j * total + in_off[p]
// + i (total = in_off[P]); the first `found` slots hold the neighbours, the others -1 / +inf.
template <typename Idx, typename B>
__device__ __forceinline__ void match_knn_rows(const Idx *orig, int found, int knn, const float *bd, const B *bi,
                                               int stride, int32_t *ids, float *dists, size_t total) {
  for (int j = 0; j < knn; ++j) {
    const bool hit = j < found;
    ids[j * total] = hit ? (int32_t)orig[bi[j * stride]] : -1;
    dists[j * total] = hit ? bd[j * stride] : INFINITY;
  }
}

// The in-CTA class: match_kernel's layout, then from byte list_off the best-knn lists, one column per thread
// (distances [knn][blockDim.x], then uint16 sorted positions [knn][blockDim.x]).  DIM 3: [x, y, z] clouds, any knn
// (grid_knn_query3 on the grid of x, y; z read from the reference's rows through the original indices).
template <int DIM>
__global__ void __launch_bounds__(ICP_THREADS) match_knn_kernel(const MatchBatch b, int knn, int list_off) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  __shared__ int scan[36];
  __shared__ float bbox_w[4 * 32];
  __shared__ float bbox[4];
  float2 *sorted = reinterpret_cast<float2 *>(smem_raw);
  uint32_t *cells = reinterpret_cast<uint32_t *>(smem_raw + sizeof(float2) * (size_t)b.nt_max);
  const int tid = threadIdx.x, nthr = blockDim.x;
  float *bd = reinterpret_cast<float *>(smem_raw + list_off) + tid;
  uint16_t *bi = reinterpret_cast<uint16_t *>(smem_raw + list_off + sizeof(float) * (size_t)nthr * knn) + tid;
  uint16_t *orig = b.orig_ws + (size_t)blockIdx.x * b.nt_max;
  const float max_d2 = __fmul_rn(b.max_dist, b.max_dist);
  const size_t total = (size_t)b.in_off[b.P];
  for (int p = blockIdx.x; p < b.P; p += gridDim.x) {
    const float *ref = b.ref_pts + DIM * (size_t)b.ref_off[p];
    const int nt = b.ref_off[p + 1] - b.ref_off[p];
    const float *in = b.in_pts + DIM * (size_t)b.in_off[p];
    const int ns = b.in_off[p + 1] - b.in_off[p];
    int32_t *ids = b.ids + b.in_off[p];
    float *dists = b.dists + b.in_off[p];
    if (nt > b.nt_max) continue;  // the map class's (match_knn_map_kernel)
    __syncthreads();
    if (nt <= 0) {
      for (int i = tid; i < ns; i += nthr) match_knn_rows(orig, 0, knn, bd, bi, nthr, ids + i, dists + i, total);
      continue;
    }
    GridView g;
    match_ref_grid<DIM>(b, ref, nt, sorted, cells, orig, scan, bbox_w, bbox, g);
    for (int i = tid; i < ns; i += nthr) {
      int found;
      if constexpr (DIM == 3)
        found = grid_knn_query3(g, in[3 * i], in[3 * i + 1], in[3 * i + 2],
                                [&](int j) { return ref[3 * (size_t)orig[j] + 2]; }, max_d2, knn, bd, bi, nthr);
      else
        found = grid_knn_query(g, in[2 * i], in[2 * i + 1], max_d2, knn, bd, bi, nthr);
      match_knn_rows(orig, found, knn, bd, bi, nthr, ids + i, dists + i, total);
    }
  }
}

// The map class of knn > 1: match_map_kernel with the best-knn lists in dynamic shared memory (distances
// [knn][blockDim.x], then int sorted positions [knn][blockDim.x]).  DIM 3 as match_knn_kernel's.
template <int DIM>
__global__ void __launch_bounds__(ICP_THREADS) match_knn_map_kernel(const MatchBatch b, int knn) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int tid = threadIdx.x, nthr = blockDim.x;
  float *bd = reinterpret_cast<float *>(smem_raw) + tid;
  int *bi = reinterpret_cast<int *>(smem_raw + sizeof(float) * (size_t)nthr * knn) + tid;
  const float max_d2 = __fmul_rn(b.max_dist, b.max_dist);
  const size_t total = (size_t)b.in_off[b.P];
  for (int p = 0; p < b.P; ++p) {
    const int ms = b.map.slot[p];
    if (ms < 0) continue;
    const MapGridView g = map_grid_view(b.map, ms);
    const float *in = b.in_pts + DIM * (size_t)b.in_off[p];
    const int ns = b.in_off[p + 1] - b.in_off[p];
    const float *ref = b.ref_pts + DIM * (size_t)b.ref_off[p];
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < ns; i += gridDim.x * blockDim.x) {
      int found;
      if constexpr (DIM == 3)
        found = grid_knn_query3(g, in[3 * i], in[3 * i + 1], in[3 * i + 2],
                                [&](int j) { return ref[3 * (size_t)g.orig[j] + 2]; }, max_d2, knn, bd, bi, nthr);
      else
        found = grid_knn_query(g, in[2 * i], in[2 * i + 1], max_d2, knn, bd, bi, nthr);
      match_knn_rows(g.orig, found, knn, bd, bi, nthr, b.ids + b.in_off[p] + i, b.dists + b.in_off[p] + i, total);
    }
  }
}

// ---------------------------------------------------------------------------- host side
constexpr int ICP_SN_KNN_MAX = 64;  // the largest box of a SamplingSurfaceNormalDataPointsFilter

// Whether the reference chain of f (may be null) ends with a SamplingSurfaceNormalDataPointsFilter
static bool icp_sampling_normals(const sfe_icp_filters *f) {
  return f && f->n_reference > 0 && f->n_reference <= SFE_ICP_MAX_DATA_FILTERS &&
         f->reference[f->n_reference - 1].kind == SFE_ICP_DATA_SAMPLING_NORMALS;
}

int icp_params_check(const sfe_icp_params *prm, int dim, const sfe_icp_filters *filt, const char *what,
                     const sfe_icp_robust *robust) {
  if (dim == 3 && (prm->minimizer != 0 || (prm->flags & 2) || filt || robust)) {
    set_error("%s: %s is not supported on [x, y, z] clouds by the 3-D scan matcher", what,
              prm->minimizer != 0 ? "the point-to-plane error minimizer"
              : (prm->flags & 2)  ? "float64 accumulation (flags bit 1)"
              : filt              ? "ICP filters (sfe_icp_set_filters)"
                                  : "the RobustOutlierFilter (sfe_icp_set_robust)");
    return SFE_ERR_UNSUPPORTED;
  }
  if (robust && (prm->flags & 2)) {
    set_error("%s: the RobustOutlierFilter (sfe_icp_set_robust) runs with float32 sums only, not with float64 "
              "accumulation (flags bit 1)", what);
    return SFE_ERR_UNSUPPORTED;
  }
  if (robust) {
    const int rc = icp_robust_check(robust, what);
    if (rc != SFE_OK) return rc;
  }
  SFE_REQUIRE(prm->max_iterations >= 1, "%s: maxIterationCount must be >= 1", what);
  SFE_REQUIRE(prm->minimizer == 0 || prm->minimizer == 1, "%s: unknown error minimizer %d", what, prm->minimizer);
  if (icp_sampling_normals(filt)) {
    SFE_REQUIRE(prm->normals_knn >= 3 && prm->normals_knn <= ICP_SN_KNN_MAX,
                "%s: SamplingSurfaceNormalDataPointsFilter knn %d is not supported (3..%d)", what, prm->normals_knn,
                ICP_SN_KNN_MAX);
  } else {
    SFE_REQUIRE(prm->minimizer == 0 || (prm->normals_knn >= 3 && prm->normals_knn <= GRID_KNN_MAX),
                "%s: SurfaceNormalDataPointsFilter knn %d is not supported (3..%d)", what, prm->normals_knn,
                GRID_KNN_MAX);
  }
  SFE_REQUIRE(prm->smooth_length < ICP_HIST, "%s: smoothLength %d is not supported (at most %d)", what,
              prm->smooth_length, ICP_HIST - 1);
  SFE_REQUIRE(!std::isnan(prm->matcher_max_dist) && !std::isnan(prm->outlier_max_dist) &&
                  !std::isnan(prm->trim_ratio) && !std::isnan(prm->min_diff_rot) && !std::isnan(prm->min_diff_trans),
              "%s: a NaN parameter (maxDist, ratio or minDiff*) is not supported", what);
  // (the quantile element floor(n * ratio) lies past the sorted distances for a ratio above 1)
  SFE_REQUIRE(prm->trim_ratio <= 1.0f, "%s: TrimmedDistOutlierFilter ratio %g is above 1", what,
              (double)prm->trim_ratio);
  return filt ? icp_filters_check(filt, what) : SFE_OK;
}

int icp_robust_check(const sfe_icp_robust *r, const char *what) {
  SFE_REQUIRE(r->fct >= SFE_ICP_ROBUST_CAUCHY && r->fct <= SFE_ICP_ROBUST_L1, "%s: unknown RobustOutlierFilter robustFct %d",
              what, r->fct);
  SFE_REQUIRE(std::isfinite(r->tuning) && r->tuning > 0.f, "%s: RobustOutlierFilter tuning %g (finite and positive)",
              what, (double)r->tuning);
  SFE_REQUIRE(!std::isnan(r->approximation), "%s: a NaN RobustOutlierFilter approximation is not supported", what);
  return SFE_OK;
}

int icp_filters_check(const sfe_icp_filters *f, const char *what) {
  SFE_REQUIRE(!std::isnan(f->min_dist) && !std::isnan(f->median_factor),
              "%s: a NaN MinDist / MedianDist outlier filter setting is not supported", what);
  SFE_REQUIRE(f->median_factor < 0.f || std::isfinite(f->median_factor), "%s: MedianDistOutlierFilter factor %g",
              what, (double)f->median_factor);
  SFE_REQUIRE(f->n_reading >= 0 && f->n_reading <= SFE_ICP_MAX_DATA_FILTERS && f->n_reference >= 0 &&
                  f->n_reference <= SFE_ICP_MAX_DATA_FILTERS,
              "%s: %d reading / %d reference data filters (0..%d each)", what, f->n_reading, f->n_reference,
              SFE_ICP_MAX_DATA_FILTERS);
  for (int side = 0; side < 2; ++side)
    for (int k = 0, normals = 0; k < (side ? f->n_reference : f->n_reading); ++k) {
      const sfe_icp_data_filter &d = side ? f->reference[k] : f->reading[k];
      SFE_REQUIRE(d.kind == SFE_ICP_DATA_MAX_DIST || d.kind == SFE_ICP_DATA_MIN_DIST || d.kind == SFE_ICP_DATA_OCTREE ||
                      d.kind == SFE_ICP_DATA_VOXEL || d.kind == SFE_ICP_DATA_SAMPLING_NORMALS ||
                      d.kind == SFE_ICP_DATA_NORMALS || d.kind == SFE_ICP_DATA_SHADOW,
                  "%s: unknown data filter kind %d", what, d.kind);
      // a reading SurfaceNormalDataPointsFilter: only per-point filters after it (their normals travel with the points)
      SFE_REQUIRE(!normals || d.kind == SFE_ICP_DATA_MAX_DIST || d.kind == SFE_ICP_DATA_MIN_DIST ||
                      d.kind == SFE_ICP_DATA_SHADOW,
                  "%s: data filter kind %d after the reading SurfaceNormalDataPointsFilter (only the distance filters "
                  "and ShadowDataPointsFilter may follow it)", what, d.kind);
      if (d.kind == SFE_ICP_DATA_NORMALS || d.kind == SFE_ICP_DATA_SHADOW) {
        const char *name = d.kind == SFE_ICP_DATA_NORMALS ? "SurfaceNormalDataPointsFilter (SFE_ICP_DATA_NORMALS)"
                                                          : "ShadowDataPointsFilter";
        SFE_REQUIRE(side == 0, "%s: %s is supported on the reading cloud only", what, name);
        if (d.kind == SFE_ICP_DATA_NORMALS) {
          SFE_REQUIRE(d.dim >= 3 && d.dim <= GRID_KNN_MAX, "%s: reading SurfaceNormalDataPointsFilter knn %d (3..%d)",
                      what, d.dim, GRID_KNN_MAX);
          normals = 1;
        } else {
          SFE_REQUIRE(normals, "%s: ShadowDataPointsFilter needs the reading's normals: put a "
                      "SurfaceNormalDataPointsFilter before it", what);
          SFE_REQUIRE(std::isfinite(d.dist), "%s: ShadowDataPointsFilter eps %g (finite)", what, (double)d.dist);
        }
        continue;
      }
      if (d.kind == SFE_ICP_DATA_SAMPLING_NORMALS) {
        SFE_REQUIRE(side == 1 && k == f->n_reference - 1,
                    "%s: SamplingSurfaceNormalDataPointsFilter is supported as the last reference filter only", what);
        SFE_REQUIRE(d.dim == 0 || d.dim == 1,
                    "%s: SamplingSurfaceNormalDataPointsFilter samplingMethod %d (0 with ratio 1, or 1)", what, d.dim);
        SFE_REQUIRE(!std::isnan(d.dist) && d.dist >= 0.f,
                    "%s: SamplingSurfaceNormalDataPointsFilter maxBoxDim %g (non-negative)", what, (double)d.dist);
        continue;
      }
      if (d.kind == SFE_ICP_DATA_VOXEL) {
        SFE_REQUIRE(d.dim == 1, "%s: VoxelGridDataPointsFilter useCentroid %d (only 1, the centroid, is supported)",
                    what, d.dim);
        SFE_REQUIRE(std::isfinite(d.dist) && d.dist > 0.f,
                    "%s: VoxelGridDataPointsFilter vSize %g (finite and positive)", what, (double)d.dist);
        continue;
      }
      if (d.kind == SFE_ICP_DATA_OCTREE) {
        SFE_REQUIRE(d.dim == DS_FIRST || d.dim == DS_CENTROID || d.dim == DS_MEDOID,
                    "%s: OctreeGridDataPointsFilter samplingMethod %d (0 first point, 2 centroid or 3 medoid)", what,
                    d.dim);
        SFE_REQUIRE(std::isfinite(d.dist) && d.dist > 0.f,
                    "%s: OctreeGridDataPointsFilter maxSizeByNode %g (finite and positive)", what, (double)d.dist);
        continue;
      }
      SFE_REQUIRE(d.dim >= -1 && d.dim <= 1, "%s: data filter dim %d (2-D clouds: -1, 0 or 1)", what, d.dim);
      SFE_REQUIRE(!std::isnan(d.dist), "%s: a NaN data filter distance is not supported", what);
    }
  return SFE_OK;
}

static int pick_max_cells(int nt_max) {
  int c = nt_max + nt_max / 2;  // the grid aims at one point per cell; the slack absorbs elongated bounding boxes
  if (c < 256) c = 256;
  if (c > GRID_MAX_CELLS) c = GRID_MAX_CELLS;
  return c;
}

// Shared memory of icp_kernel's layout for sources of up to ns_max points (>= 1).  In-CTA class: targets of up to
// nt_max points (>= 1), 16-bit target positions, after big problems traded cell-table entries (coarser cells) for room;
// *max_cells receives the table's size.  Map class: 32-bit target positions and no target arrays (*max_cells 0).
static size_t icp_cta_smem(int ns_max, int nt_max, bool plane, bool map, bool robust, size_t budget, int *max_cells) {
  const bool use_order = ns_max > 1024;
  const size_t pos = map ? sizeof(int) : sizeof(uint16_t);  // match[] and prev[]
  auto smem_for = [&](int mc) {
    return ((sizeof(IcpShared) + 15) & ~size_t(15)) +
           (map ? 0 : sizeof(float2) * (size_t)nt_max + sizeof(uint32_t) * (size_t)((mc + 2) / 2 + 1)) + 8 +
           sizeof(float2) * (size_t)ns_max + sizeof(float) * (size_t)ns_max + 2 * pos * (size_t)ns_max +
           (size_t)ns_max + 4 + sizeof(float) * (size_t)ns_max + (use_order ? sizeof(uint16_t) * (size_t)ns_max : 0) +
           16 + (plane && (robust || ns_max < ICP_PLANE_SCRATCH) ? 16 + ICP_PLANE_SCRATCH * sizeof(float) : 0);
  };
  int mc = 0;
  if (!map) {
    mc = pick_max_cells(nt_max);
    while (smem_for(mc) > budget && mc > nt_max / 4 + 256) mc -= mc / 8;
  }
  *max_cells = mc;
  return smem_for(mc);
}

static size_t match_cta_smem(int nt_max) {
  return sizeof(float2) * (size_t)nt_max + sizeof(uint32_t) * (size_t)((pick_max_cells(nt_max) + 2) / 2 + 1) + 16;
}

// CTA size follows the source size (one NN query per thread and iteration is the sweet spot)
// (chosen on the config-4 replay for ~360-point sources; not re-measured on H100)
static int icp_threads(int ns_max) { return ns_max <= 640 ? 128 : (ns_max <= 1536 ? 256 : ICP_THREADS); }

// icp_kernel's instantiation for `threads`-thread CTAs with `smem` bytes of layout: (threads, register budget), then
// the flags.  In-CTA class: 512-thread CTAs whose shared memory allows only one per SM get the full 128 registers;
// dense (icp_run's classes): 128-thread CTAs held to 64 registers, so that layouts small enough for 8 CTAs per SM get
// them (IcpClass::dense).  Map class: one instantiation per CTA size.  filt: sfe_icp_filters; robust: the
// RobustOutlierFilter (FILT instantiations with ROBUST); gnrm: given normals (in-CTA GNRM instantiations).
template <int THREADS, int MINB, bool MAP, bool GSRC = false>
static const void *icp_kernel_of(bool plane, bool filt, bool robust, bool gnrm = false) {
  if constexpr (!MAP)
    if (plane && gnrm)
      return robust ? (const void *)icp_kernel<THREADS, MINB, true, false, true, false, true, true>
                    : (const void *)icp_kernel<THREADS, MINB, true, false, true, false, false, true>;
  if (robust)
    return plane ? (const void *)icp_kernel<THREADS, MINB, true, MAP, true, GSRC, true>
                 : (const void *)icp_kernel<THREADS, MINB, false, MAP, true, GSRC, true>;
  if (filt)
    return plane ? (const void *)icp_kernel<THREADS, MINB, true, MAP, true, GSRC>
                 : (const void *)icp_kernel<THREADS, MINB, false, MAP, true, GSRC>;
  return plane ? (const void *)icp_kernel<THREADS, MINB, true, MAP, false, GSRC>
               : (const void *)icp_kernel<THREADS, MINB, false, MAP, false, GSRC>;
}

static const void *icp_kernel_for(int threads, size_t smem, bool plane, bool dense, bool filt, bool robust, bool map,
                                  bool gnrm) {
  if (map) {
    if (threads == 128) return icp_kernel_of<128, 7, true>(plane, filt, robust);
    if (threads == 256) return icp_kernel_of<256, 4, true>(plane, filt, robust);
    return icp_kernel_of<512, 1, true>(plane, filt, robust);
  }
  if (threads == 128 && dense) return icp_kernel_of<128, 8, false>(plane, filt, robust, gnrm);
  if (threads == 128) return icp_kernel_of<128, 7, false>(plane, filt, robust, gnrm);
  if (threads == 256) return icp_kernel_of<256, 4, false>(plane, filt, robust, gnrm);
  if (smem <= 110 * 1024) return icp_kernel_of<512, 2, false>(plane, filt, robust, gnrm);
  return icp_kernel_of<512, 1, false>(plane, filt, robust, gnrm);
}

// The global-source class: sources above what the shared-memory layouts hold (icp_source_limit).  Each persistent CTA
// keeps its per-source-point arrays in a slice of global workspace; all slices together stay within ICP_SRC_WS_CAP.
constexpr size_t ICP_SRC_WS_CAP = size_t(512) << 20;

// Bytes of one CTA's slice for sources of up to ns_max points: icp_kernel's reading (8 B), dist, match, prev, slack and
// order (4 B each) and qstate (1 B) per point, 256-byte aligned
static size_t icp_src_slice(int ns_max) {
  const size_t n = (size_t)ns_max;
  return (28 * n + ((n + 3) & ~size_t(3)) + 255) & ~size_t(255);
}

}  // namespace sfe

#include "icp3.cuh"

namespace sfe {
// The launch classes of an ICP call: in-CTA (the target's grid in shared memory), map (targets read as map_build's
// grids) and global-source (map grids, and the per-source-point arrays in a slice of global workspace)
enum { ICP_CTA = 0, ICP_MAP = 1, ICP_GSRC = 2 };

// One dimension's kernels and layouts: icp_kernel's instantiations for the minimizer and the filters (dim 2), or the
// icp3_body kernels (dim 3).  filt: sfe_icp_filters (icp_filters_on), or a robust filter; robust: the
// RobustOutlierFilter; gnrm: point-to-plane reads the normals of a SamplingSurfaceNormalDataPointsFilter.
struct IcpDim {
  int dim;
  bool plane, filt, robust, gnrm;
  int threads(int cls, int ns) const { return dim == 3 ? ICP3_THREADS : cls == ICP_GSRC ? ICP_THREADS : icp_threads(ns); }
  // class cls's kernel for `threads`-thread CTAs with `smem` bytes of layout; dense: IcpClass::dense
  const void *kernel(int cls, int threads, size_t smem, bool dense = false) const {
    if (dim == 3)
      return cls == ICP_CTA ? (const void *)icp3_kernel
             : cls == ICP_MAP ? (const void *)icp3_map_kernel
                              : (const void *)icp3_gsrc_kernel;
    if (cls == ICP_GSRC) return icp_kernel_of<ICP_THREADS, 1, true, true>(plane, filt, robust);
    return icp_kernel_for(threads, smem, plane, dense, filt, robust, cls == ICP_MAP, gnrm);
  }
  // shared memory class cls may take next to sources of ns points: the budget of the instantiation that runs the
  // largest of its layouts
  int budget(const sfe_ctx *ctx, int cls, int ns, size_t *bytes, bool dense = false) const {
    return cta_smem_budget(ctx, kernel(cls, threads(cls, ns), ctx->max_smem_optin, dense), bytes);
  }
  // class cls's layout for sources of ns and targets of nt points (>= 1); *max_cells: the in-CTA cell table's size
  size_t smem(int cls, int ns, int nt, size_t budget, int *max_cells) const {
    *max_cells = 0;
    if (cls == ICP_GSRC)
      return dim == 3 ? icp3_gsrc_smem()
                      : ((sizeof(IcpShared) + 15) & ~size_t(15)) + (plane ? ICP_PLANE_SCRATCH * sizeof(float) : 0);
    if (dim == 3) return cls == ICP_MAP ? icp3_map_smem(ns) : icp3_cta_smem(ns, nt, budget, max_cells);
    return icp_cta_smem(ns, nt, plane, cls == ICP_MAP, robust, budget, max_cells);
  }
  size_t slice(int ns) const { return dim == 3 ? icp3_src_slice(ns) : icp_src_slice(ns); }
  const char *what() const { return dim == 3 ? "icp (3-D)" : "icp"; }
};

// One launch of icp_kernel (IcpBatch) or an icp3_body kernel (Icp3Batch): sized by icp_plan, its workspace placed and
// the kernel enqueued by icp_enqueue.  Its arguments are b, then the map grids m, which the caller sets after map_build
// (the in-CTA class ignores them).  Workspace: orig_ws (orig_bytes), then nrm_ws (2-D point-to-plane); or the
// global-source class's slices.
template <class Batch>
struct IcpLaunch {
  Batch b;
  MapArgs m;
  const void *fn;
  int threads, grid;
  size_t smem, orig_bytes, ws_bytes;
};

// A launch of class cls over b's problems, laid out for sources of up to ns_max and targets of up to nt_max points.
// CTAs are persistent, min(P, SMs x CTAs per SM) of them, and in the global-source class no more than the slices
// ICP_SRC_WS_CAP holds (at least one) -- except 2-D in-CTA layouts that allow one CTA per SM: one CTA per problem, its
// workspace indexed by SM (IcpBatch::slot_by_smid).
template <class Batch>
static int icp_plan(sfe_ctx *ctx, const IcpDim &d, int cls, Batch b, int ns_max, int nt_max, IcpLaunch<Batch> &L,
                    bool dense = false) {
  b.ns_max = ns_max > 0 ? ns_max : 1, b.nt_max = nt_max > 0 ? nt_max : 1;
  const int threads = d.threads(cls, b.ns_max);
  const size_t slice = cls == ICP_GSRC ? d.slice(b.ns_max) : 0;
  if (slice > ICP_SRC_WS_CAP) {
    set_error("%s: a source of %d points needs %zu B of global workspace per CTA (at most %zu)", d.what(), b.ns_max,
              slice, ICP_SRC_WS_CAP);
    return SFE_ERR_UNSUPPORTED;
  }
  size_t budget;
  int rc = d.budget(ctx, cls, b.ns_max, &budget, dense);
  if (rc != SFE_OK) return rc;
  const size_t smem = d.smem(cls, b.ns_max, b.nt_max, budget, &b.max_cells);
  if (smem > budget) {
    set_error("%s: sources of %d points next to targets of %d need %zu B of shared memory per CTA (limit %zu)",
              d.what(), ns_max, nt_max, smem, budget);
    return SFE_ERR_UNSUPPORTED;
  }
  const void *fn = d.kernel(cls, threads, smem, dense);
  int per_sm;  // (the front end calls this per copy chunk: the context caches the query)
  if ((rc = ctas_per_sm(ctx, fn, threads, smem, &per_sm)) != SFE_OK) return rc;
#ifdef SFE_ICP_PHASE_CLOCKS
  if (d.dim == 2) icp_phase_per_sm[threads == 128 ? 0 : threads == 256 ? 1 : 2] = per_sm;
#endif
  int grid = std::min(ctx->sm_count * per_sm, b.P), slots = cls == ICP_CTA ? grid : 0;
  if constexpr (std::is_same_v<Batch, IcpBatch>) {
    b.use_order = cls == ICP_GSRC || b.ns_max > 1024;
    if (cls == ICP_CTA && per_sm == 1 && b.P > grid) b.slot_by_smid = 1, slots = ICP_SM_SLOTS, grid = b.P;
  }
  if (slice) grid = std::max(1, std::min(grid, (int)(ICP_SRC_WS_CAP / slice))), b.src_ws_stride = slice;
  L.orig_bytes = ((size_t)slots * b.nt_max * sizeof(uint16_t) + 15) & ~size_t(15);
  L.ws_bytes = slice ? (size_t)grid * slice : L.orig_bytes + (d.plane ? (size_t)slots * b.nt_max * sizeof(float2) : 0);
  L.b = b, L.m = {}, L.fn = fn, L.threads = threads, L.grid = grid, L.smem = smem;
  return SFE_OK;
}

// Whether L's CTAs take their problems from a work counter: fewer persistent CTAs than problems, or a class list (walked
// from a counter unless the launch runs one CTA per problem)
template <class Batch>
static bool icp_counted(const IcpLaunch<Batch> &L) {
  if constexpr (std::is_same_v<Batch, IcpBatch>)
    if (L.b.list) return !L.b.slot_by_smid;
  return L.grid < L.b.P;
}

// ws: L.ws_bytes of device memory; next: the launch's work counter, zero when the kernel starts (icp_counted)
template <class Batch>
static int icp_enqueue(sfe_ctx *ctx, cudaStream_t st, IcpLaunch<Batch> &L, char *ws, int *next) {
  Batch &b = L.b;
  b.orig_ws = (uint16_t *)ws;
  if constexpr (std::is_same_v<Batch, IcpBatch>) b.nrm_ws = b.prm.minimizer == 1 ? (float2 *)(ws + L.orig_bytes) : nullptr;
  if (b.src_ws_stride) b.src_ws = (unsigned char *)ws;  // (the global-source class: its slices, nothing else)
  if (icp_counted(L)) b.next = next;
  void *args[] = {(void *)&b, (void *)&L.m};
  SFE_CUDA(cudaLaunchKernel(L.fn, dim3(L.grid), dim3(L.threads), args, L.smem, st));
  ctx->launches++;
  return SFE_OK;
}

// Work lists of icp_run's classes.  Problem p goes to the first class c whose bounds it fits (the last class takes
// every other problem); lists[c][0 .. n[c]) holds class c's problems by decreasing cost -- source size in steps of
// ICP_COST_STEP points, ties in index order -- so that a launch ends on its shortest problems.  One CTA: warp w counts,
// then places, a contiguous segment of the problem indices; segments are laid out in warp order inside every (class,
// size step) run.  Also zeroes the classes' work counters next[c].
constexpr int ICP_COST_STEP = 32, ICP_COST_STEPS = 32;  // (sources of 992 points and more share the last step)
struct IcpClassBounds {
  int n, ns[ICP_MAX_CLASSES + 1], nt[ICP_MAX_CLASSES + 1];
};

__global__ void __launch_bounds__(1024) icp_classify_kernel(const IcpBatch b, const IcpClassBounds cb, int *lists,
                                                            int *n, int *next) {
  constexpr int KEYS = (ICP_MAX_CLASSES + 1) * ICP_COST_STEPS;
  __shared__ int cnt[32][KEYS];  // per warp: its problems per (class, cost step), then where the next one goes
  __shared__ int run_len[KEYS];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, P = b.P;
  const int seg = (P + 31) / 32, lo = min(warp * seg, P), hi = min(lo + seg, P);
  auto key_of = [&](int p) {
    const int si = b.src_id ? b.src_id[p] : p, ti = b.tgt_id ? b.tgt_id[p] : p;
    const int ns = b.src_cnt ? b.src_cnt[si] : b.src_off[si + 1] - b.src_off[si];
    const int nt = b.tgt_cnt ? b.tgt_cnt[ti] : b.tgt_off[ti + 1] - b.tgt_off[ti];
    int c = 0;
    while (c + 1 < cb.n && (ns > cb.ns[c] || nt > cb.nt[c])) ++c;
    return c * ICP_COST_STEPS + (ICP_COST_STEPS - 1 - min(max(ns, 0) / ICP_COST_STEP, ICP_COST_STEPS - 1));
  };
  for (int k = lane; k < KEYS; k += 32) cnt[warp][k] = 0;
  __syncwarp();
  for (int p = lo + lane; p < hi; p += 32) atomicAdd(&cnt[warp][key_of(p)], 1);
  __syncthreads();
  const int key = threadIdx.x;
  if (key < KEYS) {
    int s = 0;
    for (int w = 0; w < 32; ++w) s += cnt[w][key];
    run_len[key] = s;
  }
  __syncthreads();
  if (key < KEYS) {  // exclusive scan in (cost step, warp) order within the key's class
    const int c = key / ICP_COST_STEPS;
    int at = 0;
    for (int k = c * ICP_COST_STEPS; k < key; ++k) at += run_len[k];
    if (key % ICP_COST_STEPS == ICP_COST_STEPS - 1) n[c] = at + run_len[key], next[c] = 0;
    for (int w = 0; w < 32; ++w) {
      const int v = cnt[w][key];
      cnt[w][key] = at, at += v;
    }
  }
  __syncthreads();
  for (int base = lo; base < hi; base += 32) {  // in index order: lanes with the same key take consecutive places
    const int p = base + lane;
    const int k = p < hi ? key_of(p) : -1;
    const unsigned peers = __match_any_sync(0xffffffffu, k);
    if (k >= 0) lists[(size_t)(k / ICP_COST_STEPS) * P + cnt[warp][k] + __popc(peers & ((1u << lane) - 1u))] = p;
    __syncwarp();
    if (k >= 0 && lane == __ffs(peers) - 1) cnt[warp][k] += __popc(peers);
    __syncwarp();
  }
}

// class_of[p] = the class whose list holds p, class_of[P + p] = its place there (icp_run's class_of)
__global__ void icp_class_of_kernel(const int *lists, const int *n, int n_classes, int P, int *class_of) {
  for (int c = 0; c < n_classes; ++c)
    for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < n[c]; k += gridDim.x * blockDim.x) {
      const int p = lists[(size_t)c * P + k];
      class_of[p] = c, class_of[P + p] = k;
    }
}

// icp_run's class path: the classify kernel, then one launch per class, the widest first
static int icp_run_classes(sfe_ctx *ctx, cudaStream_t st, const IcpDim &d, const IcpBatch &b, const IcpClass *classes,
                           int n_classes, int ns_max, int nt_max, int *class_of) {
  IcpLaunch<IcpBatch> L[ICP_MAX_CLASSES + 1];
  IcpClassBounds cb{};
  cb.n = n_classes + 1;
  size_t ws_bytes = 0;
  for (int c = 0; c < cb.n; ++c) {
    const bool cap = c == n_classes;
    cb.ns[c] = cap ? ns_max : std::min(classes[c].ns, ns_max);
    cb.nt[c] = cap ? nt_max : std::min(classes[c].nt, nt_max);
    const int threads = icp_threads(cb.ns[c] > 0 ? cb.ns[c] : 1);
    int rc = icp_plan(ctx, d, ICP_CTA, b, cb.ns[c], cb.nt[c], L[c], !cap && classes[c].dense && threads == 128);
    if (rc != SFE_OK) return rc;
    ws_bytes = std::max(ws_bytes, L[c].ws_bytes);  // (the launches run one after the other)
  }
  // SCR_ICP: [work counters n, next][lists [class][P]][the launches' workspace]
  const size_t head = 256, list_bytes = ((size_t)cb.n * b.P * sizeof(int) + 255) & ~size_t(255);
  int rc = ensure(ctx, ctx->scratch[SCR_ICP], head + list_bytes + ws_bytes, st);
  if (rc != SFE_OK) return rc;
  char *base = (char *)ctx->scratch[SCR_ICP].ptr;
  int *n = (int *)base, *next = n + ICP_MAX_CLASSES + 1, *lists = (int *)(base + head);
  icp_classify_kernel<<<1, 1024, 0, st>>>(b, cb, lists, n, next);
  SFE_CUDA(cudaGetLastError());
  ctx->launches++;
  for (int c = cb.n - 1; c >= 0; --c) {
    L[c].b.list = lists + (size_t)c * b.P, L[c].b.list_n = n + c;
    rc = icp_enqueue(ctx, st, L[c], base + head + list_bytes, next + c);
    if (rc != SFE_OK) return rc;
  }
  if (class_of) {
    icp_class_of_kernel<<<ctx->sm_count, 256, 0, st>>>(lists, n, cb.n, b.P, class_of);
    SFE_CUDA(cudaGetLastError());
    ctx->launches++;
  }
  return SFE_OK;
}

// A persistent launch of fn over P problems: ctas_per_sm CTAs per SM, at most one per problem
static int persistent_grid(sfe_ctx *ctx, const void *fn, int threads, size_t smem, int P, int *grid) {
  int per_sm;
  const int rc = ctas_per_sm(ctx, fn, threads, smem, &per_sm);
  if (rc != SFE_OK) return rc;
  *grid = std::min(ctx->sm_count * per_sm, P);
  return SFE_OK;
}

// The one-CTA kernel of split_run: fn in `threads`-thread CTAs with `smem` bytes of layout for targets of up to nt
// points (>= 1)
struct SplitCta {
  const void *fn;
  int threads;
  size_t smem;
  int nt;
};

// One call of P problems split at `limit` target points (match_run, match_knn_run): the one-CTA kernel takes the targets
// of up to `limit` points in a persistent launch (persistent_grid), each CTA with a row of c.nt original indices
// (orig_ws, in scratch[SCR_ICP]); when the largest target, tgt.n_max, is above `limit`, map_build builds map grids of
// the larger ones (`dim` columns, problem p's target is cloud p, not centred) and the map class reads them.
// cta(grid, orig_ws) enqueues the one-CTA kernel; map(MapWs) enqueues the map class and returns an SFE_* code.
template <typename Cta, typename Map>
static int split_run(sfe_ctx *ctx, cudaStream_t st, const SplitCta &c, int P, int limit, const PackedClouds &tgt,
                     int dim, Cta cta, Map map) {
  int grid, rc;
  if ((rc = persistent_grid(ctx, c.fn, c.threads, c.smem, P, &grid)) != SFE_OK) return rc;
  if ((rc = ensure(ctx, ctx->scratch[SCR_ICP], (size_t)grid * c.nt * sizeof(uint16_t), st)) != SFE_OK) return rc;
  cta(grid, (uint16_t *)ctx->scratch[SCR_ICP].ptr);
  SFE_CUDA(cudaGetLastError());
  ctx->launches++;
  if (tgt.n_max <= limit) return SFE_OK;
  MapWs w;
  if ((rc = map_build(ctx, st, tgt, dim, nullptr, P, limit, P, false, true, 0, w)) != SFE_OK) return rc;
  if ((rc = map(w)) != SFE_OK) return rc;
  SFE_CUDA(cudaGetLastError());
  ctx->launches++;
  return SFE_OK;
}

// How a call of sources of up to ns_max and targets of up to nt_max points splits into launches (icp_run without
// classes, icp3_run; icp_cta_limit and icp_source_limit report its limits).  S: the largest source the map class's
// layout holds (at most 65 535 points).  L: the largest target the in-CTA layout holds next to sources of ns_lay points,
// the size both shared-memory launches are laid out for.  Sources above S take the global-source launch -- unless every
// target fits the in-CTA layout next to them (it holds a few more source points than the map class's), and ns_lay is
// then S.  L = 0 (MAP_CLASS_ALL): no in-CTA launch, the map launch takes every target.
struct IcpSplit {
  int S, L, ns_lay;
  bool cta, map, gsrc;
};

static int icp_split(const sfe_ctx *ctx, const IcpDim &d, int ns_max, int nt_max, IcpSplit &s) {
  size_t budget;
  int mc, rc = d.budget(ctx, ICP_MAP, 65535, &budget);  // (sources that large run in the widest CTAs)
  if (rc != SFE_OK) return rc;
  s.S = largest_layout(65535, budget, [&](int ns) { return d.smem(ICP_MAP, ns, 1, budget, &mc); });
  auto cta_limit = [&](int ns, int *L) -> int {
    *L = 0;
    if (MAP_CLASS_ALL || ns > 65535) return SFE_OK;
    const int rc = d.budget(ctx, ICP_CTA, ns, &budget);
    if (rc == SFE_OK) *L = largest_layout(65535, budget, [&](int nt) { return d.smem(ICP_CTA, ns, nt, budget, &mc); });
    return rc;
  };
  s.ns_lay = ns_max > 0 ? ns_max : 1;
  if ((rc = cta_limit(s.ns_lay, &s.L)) != SFE_OK) return rc;
  s.gsrc = s.ns_lay > s.S && !(s.L > 0 && nt_max <= s.L);
  if (s.gsrc) {
    s.ns_lay = s.S;
    if ((rc = cta_limit(s.S, &s.L)) != SFE_OK) return rc;
  }
  s.cta = s.L > 0;
  s.map = !s.cta || nt_max > s.L;
  return SFE_OK;
}

// Enqueues the launches of icp_split's s on st, in this order: the in-CTA launch; map_build, when a launch reads map
// grids (the map launch: the targets above L; the global-source launch: every target); dim 3: the grids' z
// (icp3_map_z_kernel); the map launch; the global-source launch.  Their boxes partition the problems:
//   without a global-source launch: in-CTA {nt <= L}, map {nt > L} (every nt when there is no in-CTA launch);
//   with one: in-CTA {ns <= S, nt <= L}, map {ns <= S, nt > L}, global-source {ns > S}.
// (A launch with no neighbour on one side takes everything on that side.)  Admission reports the sources above
// src.n_max and the targets above tgt.n_max SFE_ICP_TOO_LARGE in whichever launch takes them.  Workspace,
// scratch[SCR_ICP]: [dim 3 with map grids: the centred z of every map-grid position, the z mean of every slot][the
// workspace of one launch at a time]; launch k takes its problems from the work counter ctx->work[WORK_ICP + k].
template <class Batch>
static int icp_split_run(sfe_ctx *ctx, cudaStream_t st, const IcpDim &d, const IcpSplit &s, Batch b,
                         const IcpProblems &pb) {
  const int nt_max = pb.tgt.n_max, ns_hi = s.gsrc ? s.S : INT_MAX;
  const bool run[3] = {s.cta, s.map, s.gsrc};
  const IcpBox box[3] = {{INT_MIN, ns_hi, INT_MIN, s.map ? s.L : INT_MAX},
                         {INT_MIN, ns_hi, s.cta ? s.L : INT_MIN, INT_MAX},
                         {s.S, INT_MAX, INT_MIN, INT_MAX}};
  const int ns[3] = {s.ns_lay, s.ns_lay, pb.src.n_max}, nt[3] = {std::min(nt_max, s.L), nt_max, nt_max};
  IcpLaunch<Batch> L[3];
  size_t ws = 0;
  bool counted = false;
  int rc;
  for (int k = 0; k < 3; ++k) {
    if (!run[k]) continue;
    b.box = box[k];
    if ((rc = icp_plan(ctx, d, k, b, ns[k], nt[k], L[k])) != SFE_OK) return rc;
    // (with no target points every problem fails admission before the global-source launch touches a slice)
    if (k == ICP_GSRC && nt_max == 0) L[k].ws_bytes = 0;
    ws = std::max(ws, L[k].ws_bytes), counted = counted || icp_counted(L[k]);
  }
  const int grid_limit = s.gsrc ? 0 : s.L;  // (the global-source launch reads every target as a map grid)
  const bool grids = nt_max > grid_limit;
  const int slot_cap = pb.n_tgt_clouds > 0 ? std::min(pb.n_tgt_clouds, pb.P) : pb.P;
  const size_t z_bytes = ((size_t)slot_cap * nt_max * sizeof(float) + 255) & ~size_t(255);
  const size_t side = grids && d.dim == 3 ? (z_bytes + sizeof(float) * slot_cap + 255) & ~size_t(255) : 0;
  if ((rc = ensure(ctx, ctx->scratch[SCR_ICP], side + ws, st)) != SFE_OK) return rc;
  char *base = (char *)ctx->scratch[SCR_ICP].ptr;
  int *next = ctx->work + WORK_ICP;
  if (counted) SFE_CUDA(cudaMemsetAsync(next, 0, 3 * sizeof(int), st));
  if (s.cta && (rc = icp_enqueue(ctx, st, L[ICP_CTA], base + side, next + ICP_CTA)) != SFE_OK) return rc;
  MapWs w{};
  if (grids) {
    const float2 *given = nullptr;
    if constexpr (std::is_same_v<Batch, IcpBatch>) given = d.gnrm ? b.given_nrm : nullptr;
    const int knn = d.plane && !given ? std::min(std::max(b.prm.normals_knn, 1), GRID_KNN_MAX) : 0;
    rc = map_build(ctx, st, pb.tgt, d.dim, pb.tgt_id, pb.P, grid_limit, slot_cap, true, (b.prm.flags & 2) == 0, knn, w,
                   given);
    if (rc != SFE_OK) return rc;
    if constexpr (std::is_same_v<Batch, Icp3Batch>) {
      float *zs = (float *)base, *zm = (float *)(base + z_bytes);
      icp3_map_z_kernel<<<slot_cap, ICP3_THREADS, 0, st>>>(pb.tgt.pts, pb.tgt.off, w, zs, zm);
      SFE_CUDA(cudaGetLastError());
      ctx->launches++;
      for (int k = ICP_MAP; k <= ICP_GSRC; ++k) L[k].b.map_z = zs, L[k].b.map_zm = zm;
    }
  }
  for (int k = ICP_MAP; k <= ICP_GSRC; ++k) {
    if (!run[k]) continue;
    L[k].m = w.args();
    if ((rc = icp_enqueue(ctx, st, L[k], base + side, next + k)) != SFE_OK) return rc;
  }
  return SFE_OK;
}

// Whether a call with the filters f (may be null) runs icp_kernel's FILT instantiations
static bool icp_filters_on(const sfe_icp_filters *f) {
  return f && (f->n_reading > 0 || f->n_reference > 0 || f->min_dist >= 0.f || f->median_factor >= 0.f);
}

// Data filters: the clouds of one side of the batch, filtered into scratch[SCR_ICP_FILTER] once per cloud when the
// cloud count is known (no ids: one per problem), else once per problem (the ids then name the filtered clouds no
// more).  The chain f[0 .. n) runs as stages in its order: every maximal run of distance filters is one
// icp_data_filter_kernel pass, every octree filter one downsample_run call on the clouds the stage before left.  The
// first stage is always a compaction pass (with no filter when the chain starts with an octree filter): it lays the
// clouds out n_max points apart and records their sizes before any filter, the `gate` counts.  Every voxel filter is
// one voxel_filter_run call likewise; a cloud whose voxel index would overflow sets *vox_overflow.  Two passes over
// the Carver: the first sizes the block, the second launches.
static int icp_filter_side(sfe_ctx *ctx, cudaStream_t st, const sfe_icp_data_filter *f, int n, PackedClouds &c,
                           const int *&id, int n_clouds, int P, Carver &cv, const int *&gate, int *vox_overflow,
                           int knn = 0, const float2 **nrm_out = nullptr) {
  const int jobs = id && n_clouds > 0 ? n_clouds : P;
  const int n_max = c.n_max > 0 ? c.n_max : 1;
  const size_t pts_bytes = sizeof(float) * 2 * (size_t)jobs * n_max;
  float *pts = (float *)cv.take(pts_bytes);
  int *off = (int *)cv.take(sizeof(int) * (size_t)(jobs + 1));
  int *cnt = (int *)cv.take(sizeof(int) * (size_t)jobs);
  int *raw = (int *)cv.take(sizeof(int) * (size_t)jobs);
  bool octree = false;
  for (int k = 0; k < n; ++k)
    octree = octree || f[k].kind == SFE_ICP_DATA_OCTREE || f[k].kind == SFE_ICP_DATA_VOXEL ||
             f[k].kind == SFE_ICP_DATA_SAMPLING_NORMALS || f[k].kind == SFE_ICP_DATA_NORMALS;
  // a reading SurfaceNormalDataPointsFilter whose normals a ShadowDataPointsFilter reads: the normals, laid out as the
  // points, and the stage's workspace (a filter with no shadow after it changes nothing and does not run)
  float2 *pnrm = nullptr;
  void *pn_ws = nullptr;
  int pn_at = -1;
  for (int k = 0; k < n; ++k)
    if (f[k].kind == SFE_ICP_DATA_NORMALS) pn_at = k;
  if (pn_at >= 0) {
    bool shadow = false;
    for (int k = pn_at + 1; k < n; ++k) shadow = shadow || f[k].kind == SFE_ICP_DATA_SHADOW;
    if (shadow) {
      size_t ws_bytes;
      const int rc = surface_normals_ws(jobs, n_max, &ws_bytes);
      if (rc != SFE_OK) return rc;
      pnrm = (float2 *)cv.take(sizeof(float2) * (size_t)jobs * n_max);
      pn_ws = cv.take(ws_bytes);
    }
  }
  // a sampling-normals stage (the chain's last): the normals it writes, laid out as the points, and its workspace
  float2 *nrm = nullptr;
  void *sn_ws = nullptr;
  if (n > 0 && f[n - 1].kind == SFE_ICP_DATA_SAMPLING_NORMALS) {
    size_t ws_bytes;
    const int rc = sampling_normals_ws(jobs, n_max, knn, &ws_bytes);
    if (rc != SFE_OK) return rc;
    nrm = (float2 *)cv.take(sizeof(float2) * (size_t)jobs * n_max);
    sn_ws = cv.take(ws_bytes);
  }
  // octree and voxel chains: a second set of points and counts the stages alternate with, the down-sample's indices,
  // and the offsets and sizes later compaction passes write (the same offsets; the sizes are not the gate's)
  float *pts2 = nullptr;
  int *cnt2 = nullptr, *idx = nullptr, *off2 = nullptr, *raw2 = nullptr;
  if (octree) {
    pts2 = (float *)cv.take(pts_bytes);
    cnt2 = (int *)cv.take(sizeof(int) * (size_t)jobs);
    idx = (int *)cv.take(sizeof(int) * (size_t)jobs * n_max);
    off2 = (int *)cv.take(sizeof(int) * (size_t)(jobs + 1));
    raw2 = (int *)cv.take(sizeof(int) * (size_t)jobs);
  }
  if (!cv.base) return SFE_OK;
  const bool per_problem = id && n_clouds <= 0;
  PackedClouds cur = c;
  const int *cur_id = per_problem ? id : nullptr;
  float *next_pts = pts;
  int *next_cnt = cnt;
  for (int k = 0, first = 1; k < n || first; first = 0) {
    if (!first && f[k].kind == SFE_ICP_DATA_NORMALS) {  // the points stay where they are
      if (pnrm) {
        const int rc = surface_normals_run(ctx, st, cur, jobs, f[k].dim, pn_ws, pnrm);
        if (rc != SFE_OK) return rc;
      }
      ++k;
      continue;
    }
    if (!first && f[k].kind == SFE_ICP_DATA_SAMPLING_NORMALS) {
      const int rc = sampling_normals_run(ctx, st, cur, jobs, knn, f[k].dim, f[k].dist, sn_ws, next_pts, off, next_cnt,
                                          nrm);
      if (rc != SFE_OK) return rc;
      icp_keep_too_large_kernel<<<std::min((jobs + 255) / 256, ctx->sm_count), 256, 0, st>>>(cur.cnt, jobs, n_max,
                                                                                             next_cnt);
      ++k;
    } else if (!first && f[k].kind == SFE_ICP_DATA_VOXEL) {
      const int rc = voxel_filter_run(ctx, st, cur, jobs, f[k].dist, next_pts, off, next_cnt, vox_overflow);
      if (rc != SFE_OK) return rc;
      icp_keep_too_large_kernel<<<std::min((jobs + 255) / 256, ctx->sm_count), 256, 0, st>>>(cur.cnt, jobs, n_max,
                                                                                             next_cnt);
      ++k;
    } else if (!first && f[k].kind == SFE_ICP_DATA_OCTREE) {
      const int rc = downsample_run(ctx, st, cur, jobs, 2, f[k].dist, next_pts, idx, next_cnt, DS_ANY_SIZE, SCR_CLOUD,
                                    WORK_DS, f[k].dim);
      if (rc != SFE_OK) return rc;
      icp_keep_too_large_kernel<<<std::min((jobs + 255) / 256, ctx->sm_count), 256, 0, st>>>(cur.cnt, jobs, n_max,
                                                                                             next_cnt);
      ++k;
    } else {
      IcpDataFilters df{0, {}};
      const bool nrm = !first && k > pn_at && pn_at >= 0;  // after the reading normals: the per-point filters
      for (; k < n && f[k].kind != SFE_ICP_DATA_OCTREE && f[k].kind != SFE_ICP_DATA_VOXEL &&
             f[k].kind != SFE_ICP_DATA_SAMPLING_NORMALS && f[k].kind != SFE_ICP_DATA_NORMALS;
           ++k) {
        df.f[df.n++] = f[k];
        // the threshold as upstream computes it, once on the host: the C library's sinf, not the device's
        if (f[k].kind == SFE_ICP_DATA_SHADOW) df.f[df.n - 1].dist = std::sin(f[k].dist);
      }
      if (nrm && pnrm)
        icp_data_filter_kernel<true><<<std::min(jobs, ctx->sm_count * 8), ICP_DF_THREADS, 0, st>>>(
            {cur.pts, cur.off, cur.cnt, n_max}, cur_id, jobs, df, next_pts, first ? off : off2, next_cnt,
            first ? raw : raw2, pnrm);
      else
        icp_data_filter_kernel<false><<<std::min(jobs, ctx->sm_count * 8), ICP_DF_THREADS, 0, st>>>(
            {cur.pts, cur.off, cur.cnt, n_max}, cur_id, jobs, df, next_pts, first ? off : off2, next_cnt,
            first ? raw : raw2, nullptr);
    }
    SFE_CUDA(cudaGetLastError());
    ctx->launches++;
    float *prev_pts = (float *)cur.pts;
    int *prev_cnt = (int *)cur.cnt;
    cur = {next_pts, off, next_cnt, c.n_max}, cur_id = nullptr;
    next_pts = first ? pts2 : prev_pts, next_cnt = first ? cnt2 : prev_cnt;
  }
  c = cur;
  if (per_problem) id = nullptr;
  gate = raw;
  if (nrm_out) *nrm_out = nrm;
  return SFE_OK;
}
}  // namespace sfe

// Size classes: every listed class gets a launch laid out for it, whose smaller shared-memory footprint fits more
// CTAs per SM, and a last launch, laid out for the capacities src.n_max x tgt.n_max, takes the problems that fit none
// (and reports oversize ones, SFE_ICP_TOO_LARGE).  Without classes the launches of icp_split_run partition the
// problems: in-CTA, map class (targets above the in-CTA layout's limit, read as map grids from global memory) and
// global-source class (sources above the shared-memory layouts).
int sfe::icp_run(sfe_ctx *ctx, cudaStream_t st, const sfe_icp_params *prm, const IcpProblems &pb_in,
                 const IcpClass *class_list, int n_classes, int *class_of, const sfe_icp_filters *filt,
                 const sfe_icp_robust *robust) {
  IcpProblems pb = pb_in;
  const int ns_max = pb.src.n_max, nt_max = pb.tgt.n_max;
  SFE_REQUIRE(ctx && prm, "icp: null context or parameters");
  SFE_REQUIRE(pb.P >= 0 && ns_max >= 0 && nt_max >= 0, "icp: negative sizes");
  if (pb.P == 0) return SFE_OK;
  SFE_REQUIRE(pb.src.pts && pb.src.off && pb.tgt.pts && pb.tgt.off && pb.guess && pb.T_out && pb.iters && pb.inliers &&
                  pb.status,
              "icp: null pointer");
  SFE_REQUIRE(n_classes >= 0 && n_classes <= ICP_MAX_CLASSES && (n_classes == 0 || class_list),
              "icp: %d size classes (at most %d)", n_classes, ICP_MAX_CLASSES);
  for (int c = 0; c < n_classes; ++c)
    SFE_REQUIRE(class_list[c].ns > 0 && class_list[c].nt > 0, "icp: size class %d of %d x %d points", c,
                class_list[c].ns, class_list[c].nt);
  const bool classes = n_classes > 0;
  SFE_REQUIRE((ns_max <= 65535 && nt_max <= 65535) || !classes,
              "icp: clouds of more than 65535 points are not supported (got %d, %d)", ns_max, nt_max);
  int rc = icp_params_check(prm, 2, filt, "icp", robust);
  if (rc != SFE_OK) return rc;
  const int *gate_src = nullptr, *gate_tgt = nullptr;
  const float2 *given_nrm = nullptr;
  if (filt && (filt->n_reading > 0 || filt->n_reference > 0)) {
    bool voxel = false;
    for (int k = 0; k < filt->n_reading; ++k) voxel = voxel || filt->reading[k].kind == SFE_ICP_DATA_VOXEL;
    for (int k = 0; k < filt->n_reference; ++k) voxel = voxel || filt->reference[k].kind == SFE_ICP_DATA_VOXEL;
    Carver cv;
    int *vox_overflow = nullptr;
    for (int pass = 0; pass < 2; ++pass) {
      IcpProblems q = pb;
      if (voxel) {
        vox_overflow = (int *)cv.take(sizeof(int));
        if (pass == 1) SFE_CUDA(cudaMemsetAsync(vox_overflow, 0, sizeof(int), st));
      }
      if (filt->n_reading > 0) {
        rc = icp_filter_side(ctx, st, filt->reading, filt->n_reading, q.src, q.src_id, q.n_src_clouds, q.P, cv,
                             gate_src, vox_overflow);
        if (rc != SFE_OK) return rc;
      }
      if (filt->n_reference > 0) {
        rc = icp_filter_side(ctx, st, filt->reference, filt->n_reference, q.tgt, q.tgt_id, q.n_tgt_clouds, q.P, cv,
                             gate_tgt, vox_overflow, prm->normals_knn, &given_nrm);
        if (rc != SFE_OK) return rc;
        if (q.tgt_id != pb.tgt_id) q.n_tgt_clouds = q.P;  // one compacted target per problem
      }
      if (pass == 0) {
        rc = ensure(ctx, ctx->scratch[SCR_ICP_FILTER], cv.off, st);
        if (rc != SFE_OK) return rc;
        cv.base = (char *)ctx->scratch[SCR_ICP_FILTER].ptr, cv.off = 0;
      } else {
        pb = q;
      }
    }
    // The voxel grid spans the cloud a voxel stage receives, known on the device only: wait for the stages, and refuse
    // the call before its ICP launch when a grid would need upstream's 32-bit voxel index to wrap (undefined there)
    if (voxel) {
      int overflow = 0;
      SFE_CUDA(cudaMemcpyAsync(&overflow, vox_overflow, sizeof(int), cudaMemcpyDeviceToHost, st));
      SFE_CUDA(cudaStreamSynchronize(st));
      if (overflow) {
        set_error("icp: VoxelGridDataPointsFilter: a cloud's voxel grid has more than 2^32 - 1 voxels (or its bounds "
                  "are not finite): its 32-bit voxel index would wrap; use a larger vSize");
        return SFE_ERR_UNSUPPORTED;
      }
    }
  }
  IcpBatch b{};
  b.min_d2 = b.median_factor = -1.f;
  if (filt) {
    b.min_d2 = filt->min_dist < 0.f ? -1.f : (prm->flags & 1) ? filt->min_dist : filt->min_dist * filt->min_dist;
    b.median_factor = filt->median_factor;
    b.gate_src_cnt = gate_src, b.gate_tgt_cnt = gate_tgt;
  }
  if (robust) b.robust = *robust;
  b.given_nrm = prm->minimizer == 1 ? given_nrm : nullptr;
  b.src_pts = pb.src.pts, b.src_off = pb.src.off, b.tgt_pts = pb.tgt.pts, b.tgt_off = pb.tgt.off;
  b.src_cnt = pb.src.cnt, b.tgt_cnt = pb.tgt.cnt, b.min_points = pb.min_points;
  b.raw_cnt = pb.raw_cnt, b.raw_cap = pb.raw_cap;
  b.src_id = pb.src_id, b.tgt_id = pb.tgt_id, b.guess = pb.guess;
  b.T_out = pb.T_out, b.iters = pb.iters, b.inliers = pb.inliers, b.status = pb.status;
  b.P = pb.P;
  b.box = ICP_BOX_ALL;
  b.cell_scale = 1.0f, b.prm = *prm;
  b.small_mult = ICP_SMALL_MULT, b.margin_mult = ICP_MARGIN_MULT;
  const IcpDim d{2, prm->minimizer == 1, icp_filters_on(filt) || robust, robust != nullptr, b.given_nrm != nullptr};
  if (classes) return icp_run_classes(ctx, st, d, b, class_list, n_classes, ns_max, nt_max, class_of);
  IcpSplit s;
  if ((rc = icp_split(ctx, d, ns_max, nt_max, s)) != SFE_OK) return rc;
  return icp_split_run(ctx, st, d, s, b, pb);
}

int sfe::icp_cta_limit(const sfe_ctx *ctx, int dim, int ns, int *limit) {
  SFE_REQUIRE(dim == 2 || dim == 3, "icp: points must have 2 or 3 columns (got %d)", dim);
  SFE_REQUIRE(ns >= 0 && ns <= 65535, "icp: sources of %d points are not supported (0..65535)", ns);
  IcpSplit s;
  const int rc = icp_split(ctx, {dim, false, false, false}, ns, 0, s);
  if (rc == SFE_OK) *limit = s.gsrc ? 0 : s.L;  // (a global-source launch: no in-CTA layout holds these sources)
  return rc;
}

int sfe::icp_source_limit(const sfe_ctx *ctx, const sfe_icp_params *prm, int dim, const sfe_icp_filters *filt,
                          int *limit, const sfe_icp_robust *robust) {
  SFE_REQUIRE(ctx && prm && limit, "icp_source_limit: null pointer");
  SFE_REQUIRE(dim == 2 || dim == 3, "icp: points must have 2 or 3 columns (got %d)", dim);
  int rc = icp_params_check(prm, dim, filt, "icp_source_limit", robust);
  if (rc != SFE_OK) return rc;
  IcpSplit s;
  const IcpDim d{dim, prm->minimizer == 1, icp_filters_on(filt) || robust, robust != nullptr,
                 prm->minimizer == 1 && icp_sampling_normals(filt)};
  if ((rc = icp_split(ctx, d, 1, 0, s)) == SFE_OK) *limit = s.S;
  return rc;
}

// [x, y, z] clouds: the launches of icp_split_run -- icp3_kernel (one CTA, the target's grid in shared memory),
// icp3_map_kernel (targets as map grids from map_build with dim 3, plus their z by grid position) and icp3_gsrc_kernel
// (sources above the shared-memory layouts) -- as in icp_run.
int sfe::icp3_run(sfe_ctx *ctx, cudaStream_t st, const sfe_icp_params *prm, const IcpProblems &pb,
                  const sfe_icp_filters *filt, const sfe_icp_robust *robust) {
  SFE_REQUIRE(ctx && prm, "icp (3-D): null context or parameters");
  SFE_REQUIRE(pb.P >= 0 && pb.src.n_max >= 0 && pb.tgt.n_max >= 0, "icp (3-D): negative sizes");
  int rc = icp_params_check(prm, 3, filt, "icp (3-D)", robust);
  if (rc != SFE_OK) return rc;
  if (pb.P == 0) return SFE_OK;
  SFE_REQUIRE(pb.src.pts && pb.src.off && pb.tgt.pts && pb.tgt.off && pb.guess && pb.T_out && pb.iters && pb.inliers &&
                  pb.status,
              "icp (3-D): null pointer");
  SFE_REQUIRE(!pb.src.cnt && !pb.tgt.cnt, "icp (3-D): per-cloud counts are not supported");
  Icp3Batch b{};
  b.src_pts = pb.src.pts, b.src_off = pb.src.off, b.tgt_pts = pb.tgt.pts, b.tgt_off = pb.tgt.off;
  b.src_id = pb.src_id, b.tgt_id = pb.tgt_id, b.guess = pb.guess;
  b.T_out = pb.T_out, b.iters = pb.iters, b.inliers = pb.inliers, b.status = pb.status;
  b.P = pb.P, b.prm = *prm;
  const IcpDim d{3, false, false, false};
  IcpSplit s;
  if ((rc = icp_split(ctx, d, pb.src.n_max, pb.tgt.n_max, s)) != SFE_OK) return rc;
  return icp_split_run(ctx, st, d, s, b, pb);
}

// References that fit one CTA's shared memory run in match_kernel, larger ones (whole maps) as map grids in
// match_map_kernel, in the same call.
int sfe::match_run(sfe_ctx *ctx, cudaStream_t st, const PackedClouds &ref, const PackedClouds &in, int P,
                   float max_dist, int32_t *ids, float *dists) {
  const int nt_max = ref.n_max;
  SFE_REQUIRE(ctx, "match: null context");
  SFE_REQUIRE(P >= 0 && nt_max >= 0, "match: negative sizes");
  if (P == 0) return SFE_OK;
  SFE_REQUIRE(ref.pts && ref.off && in.pts && in.off && ids && dists, "match: null pointer");
  SFE_REQUIRE(!ref.cnt && !in.cnt, "match: per-cloud counts are not supported");
  size_t budget;
  int rc = cta_smem_budget(ctx, (const void *)match_kernel, &budget);
  if (rc != SFE_OK) return rc;
  // (MAP_CLASS_ALL: references of one point are taken by both kernels, with the same result)
  const int limit = MAP_CLASS_ALL ? 0 : largest_layout(65535, budget, match_cta_smem);
  MatchBatch b{};
  b.ref_pts = ref.pts, b.ref_off = ref.off, b.in_pts = in.pts, b.in_off = in.off;
  b.P = P, b.max_dist = max_dist;
  b.ids = ids, b.dists = dists;
  const int nt_cta = std::min(nt_max, limit);
  b.nt_max = nt_cta > 0 ? nt_cta : 1, b.max_cells = pick_max_cells(b.nt_max);
  const size_t smem = match_cta_smem(b.nt_max);
  if (smem > (size_t)ctx->max_smem_optin) {
    set_error("match: a %d-point reference needs %zu B of shared memory per CTA (limit %d)", nt_max, smem,
              ctx->max_smem_optin);
    return SFE_ERR_UNSUPPORTED;
  }
  return split_run(
      ctx, st, {(const void *)match_kernel, ICP_THREADS, smem, b.nt_max}, P, limit, {ref.pts, ref.off, nullptr, nt_max},
      2,
      [&](int grid, uint16_t *orig_ws) {
        b.orig_ws = orig_ws;
        match_kernel<<<grid, ICP_THREADS, smem, st>>>(b);
      },
      [&](const MapWs &w) -> int {
        b.map = w.args();
        match_map_kernel<<<ctx->sm_count * 4, ICP_THREADS, 0, st>>>(b);
        return SFE_OK;
      });
}

// 2-D clouds, knn 1: match_run.  Otherwise (knn > 1, or [x, y, z] clouds at any knn): references whose layout fits one
// CTA next to the best-knn lists run in match_knn_kernel, larger ones as map grids in match_knn_map_kernel, in the same
// call; the split comes from the same limit search for both dims.
int sfe::match_knn_run(sfe_ctx *ctx, cudaStream_t st, const PackedClouds &ref, const PackedClouds &in, int P, int knn,
                       float max_dist, int32_t *ids, float *dists, int dim) {
  SFE_REQUIRE(knn >= 1 && knn <= GRID_KNN_MAX, "match: knn %d is not supported (1..%d)", knn, GRID_KNN_MAX);
  SFE_REQUIRE(dim == 2 || dim == 3, "match: points must have 2 or 3 columns (got %d)", dim);
  if (knn == 1 && dim == 2) return match_run(ctx, st, ref, in, P, max_dist, ids, dists);
  const int nt_max = ref.n_max;
  SFE_REQUIRE(ctx, "match: null context");
  SFE_REQUIRE(P >= 0 && nt_max >= 0, "match: negative sizes");
  if (P == 0) return SFE_OK;
  SFE_REQUIRE(ref.pts && ref.off && in.pts && in.off && ids && dists, "match: null pointer");
  SFE_REQUIRE(!ref.cnt && !in.cnt, "match: per-cloud counts are not supported");
  const size_t lists = (size_t)ICP_THREADS * knn * (sizeof(float) + sizeof(uint16_t));
  auto list_off = [](int nt) { return (match_cta_smem(nt) + 15) & ~size_t(15); };
  const void *cta_kernel = dim == 3 ? (const void *)match_knn_kernel<3> : (const void *)match_knn_kernel<2>;
  size_t budget;
  int rc = cta_smem_budget(ctx, cta_kernel, &budget);
  if (rc != SFE_OK) return rc;
  const int limit = MAP_CLASS_ALL ? 0 : largest_layout(65535, budget, [&](int nt) { return list_off(nt) + lists; });
  MatchBatch b{};
  b.ref_pts = ref.pts, b.ref_off = ref.off, b.in_pts = in.pts, b.in_off = in.off;
  b.P = P, b.max_dist = max_dist;
  b.ids = ids, b.dists = dists;
  const int nt_cta = std::min(nt_max, limit);
  b.nt_max = nt_cta > 0 ? nt_cta : 1, b.max_cells = pick_max_cells(b.nt_max);
  const size_t smem = list_off(b.nt_max) + lists;
  if (smem > budget) {
    set_error("match: knn %d needs %zu B of shared memory per CTA (limit %zu)", knn, smem, budget);
    return SFE_ERR_UNSUPPORTED;
  }
  return split_run(
      ctx, st, {cta_kernel, ICP_THREADS, smem, b.nt_max}, P, limit, {ref.pts, ref.off, nullptr, nt_max}, dim,
      [&](int grid, uint16_t *orig_ws) {
        b.orig_ws = orig_ws;
        if (dim == 3) match_knn_kernel<3><<<grid, ICP_THREADS, smem, st>>>(b, knn, (int)list_off(b.nt_max));
        else match_knn_kernel<2><<<grid, ICP_THREADS, smem, st>>>(b, knn, (int)list_off(b.nt_max));
      },
      [&](const MapWs &w) -> int {
        b.map = w.args();
        const size_t map_lists = (size_t)ICP_THREADS * knn * (sizeof(float) + sizeof(int));
        const void *map_kernel = dim == 3 ? (const void *)match_knn_map_kernel<3> : (const void *)match_knn_map_kernel<2>;
        int per_sm;
        const int rc = ctas_per_sm(ctx, map_kernel, ICP_THREADS, map_lists, &per_sm);
        if (rc != SFE_OK) return rc;
        if (dim == 3) match_knn_map_kernel<3><<<ctx->sm_count * per_sm, ICP_THREADS, map_lists, st>>>(b, knn);
        else match_knn_map_kernel<2><<<ctx->sm_count * per_sm, ICP_THREADS, map_lists, st>>>(b, knn);
        return SFE_OK;
      });
}

#ifdef SFE_ICP_PHASE_CLOCKS
// Development build only (not declared in include/sonarfe.h): out[0..6] cycles per phase, out[7..13] phase counts,
// out[14..16] CTAs per SM of the last 128 / 256 / 512-thread launch.  reset != 0 clears the totals afterwards.
extern "C" __attribute__((visibility("default"))) int sfe_icp_phase_clocks(unsigned long long *out, int reset) {
  using namespace sfe;
  if (cudaDeviceSynchronize() != cudaSuccess) return -1;
  if (cudaMemcpyFromSymbol(out, icp_phase_cycles, sizeof(icp_phase_cycles)) != cudaSuccess) return -1;
  if (cudaMemcpyFromSymbol(out + ICP_PHASES, icp_phase_count, sizeof(icp_phase_count)) != cudaSuccess) return -1;
  for (int k = 0; k < 3; ++k) out[2 * ICP_PHASES + k] = (unsigned long long)icp_phase_per_sm[k];
  if (reset) {
    const unsigned long long z[ICP_PHASES] = {};
    if (cudaMemcpyToSymbol(icp_phase_cycles, z, sizeof z) != cudaSuccess) return -1;
    if (cudaMemcpyToSymbol(icp_phase_count, z, sizeof z) != cudaSuccess) return -1;
  }
  return 0;
}
#endif
