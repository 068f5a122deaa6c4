// SamplingSurfaceNormalDataPointsFilter on the device: the last reference data filter of an ICP call (icp.cu's
// icp_filter_side).  Statement: oracle/sampling_normal_ref.c.
//
// Clouds of up to SN_CTA_MAX points take one CTA each (sn_cta_kernel): the keys stay in registers and every level is one
// block-wide radix sort of (segment, ordered coordinate, index).  Larger clouds (whole maps) take the grid-wide path:
// the partition is built level by level for every such cloud of the batch at once.  Its shape depends on the cloud's size
// alone (a range of count > knn points splits into count - count / 2 and count / 2), so segment s of level d is found
// by walking s's d bits down from the root; only the cut axis depends on the points, through the bounds each level
// hands its children.  Each level, every point gets the 64-bit key (ordered coordinate on its segment's cut axis,
// index) -- just its index inside a box -- and one CUB segmented sort orders every segment of every cloud; the next
// level's bounds take the cut value from the sorted keys.  After the last level every box lists its points in index
// order, and one thread per box forms its extent, normal and centroid; a compaction per cloud then writes the kept
// points and their normals in index order.
#include <algorithm>
#include <climits>
#include <cmath>

#include <cub/cub.cuh>

#include "stages.cuh"

namespace sfe {

constexpr int SN_THREADS = 256;

// Levels of the partition of clouds of up to n_max points: the first level at which every range holds <= knn points
__host__ __device__ inline int sn_levels(int n_max, int knn) {
  int d = 0;
  while (((long long)n_max + (1ll << d) - 1) >> d > knn) ++d;
  return d;
}

// Segment s of level d of a cloud of n points: [*first, *first + *count), or count 0 when the range stopped splitting
// at an earlier level and s is not its leftmost descendant (the leftmost one carries the box).
__device__ __forceinline__ void sn_segment(int n, int knn, int d, int s, int *first, int *count) {
  int f = 0, c = n;
  for (int l = d - 1; l >= 0; --l) {
    const int right = (s >> l) & 1;
    if (c <= knn) {
      if (right) c = 0;
      continue;
    }
    const int left = c - c / 2;
    if (right) f += left, c -= left;
    else c = left;
  }
  *first = f, *count = c;
}

// The segment of level d that holds position i (< n) of a cloud of n points
__device__ __forceinline__ int sn_segment_of(int n, int knn, int d, int i) {
  int f = 0, c = n, s = 0;
  for (int l = 0; l < d; ++l) {
    if (c <= knn) {
      s <<= 1;
      continue;
    }
    const int left = c - c / 2;
    const int right = i - f >= left;
    s = (s << 1) | right;
    if (right) f += left, c -= left;
    else c = left;
  }
  return s;
}

// float32 -> uint32 in the order of the float values, -0 as +0
__device__ __forceinline__ uint32_t sn_ord(float v) {
  const uint32_t u = __float_as_uint(v == 0.f ? 0.f : v);
  return u ^ ((u & 0x80000000u) ? 0xffffffffu : 0x80000000u);
}

__device__ __forceinline__ int sn_count(const PackedClouds &in, int c) {
  const int n = in.cnt ? in.cnt[c] : in.off[c + 1] - in.off[c];
  return n > in.n_max ? 0 : n;  // (a cloud above n_max is not read: the caller keeps its size)
}

// The one-CTA path's capacity: the keys of a cloud sit in registers, SN_CTA_ITEMS per thread
constexpr int SN_CTA_THREADS = 256, SN_CTA_ITEMS = 16, SN_CTA_MAX = SN_CTA_THREADS * SN_CTA_ITEMS;
constexpr int SN_IDX_BITS = 12;  // (an index below SN_CTA_MAX)
static_assert(SN_CTA_MAX <= (1 << SN_IDX_BITS), "sn_cta_kernel: indices in the low key bits");

// The grid-wide levels' view of cloud c: clouds the one-CTA path takes (n <= lo) are empty there
__device__ __forceinline__ int sn_grid_count(const PackedClouds &in, int c, int lo) {
  const int n = sn_count(in, c);
  return n <= lo ? 0 : n;
}

// the cut axis of bounds (minx, miny, maxx, maxy): the larger extent, x on a tie (Eigen's maxCoeff)
__device__ __forceinline__ int sn_cut_dim(float4 b) { return __fsub_rn(b.w, b.y) > __fsub_rn(b.z, b.x) ? 1 : 0; }

// Level 0: the identity order and every cloud's bounds.  One CTA per cloud.
__global__ void __launch_bounds__(SN_THREADS) sn_init_kernel(const PackedClouds in, int n_clouds,
                                                             unsigned long long *key, float4 *bounds, int seg_stride) {
  __shared__ float4 part[SN_THREADS / 32];
  for (int c = blockIdx.x; c < n_clouds; c += gridDim.x) {
    const int n = sn_count(in, c);
    const float *p = in.pts + 2 * (size_t)in.off[c];
    float4 b = make_float4(INFINITY, INFINITY, -INFINITY, -INFINITY);
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
      key[(size_t)c * in.n_max + i] = (unsigned)i;
      const float x = p[2 * i], y = p[2 * i + 1];
      b.x = fminf(b.x, x), b.y = fminf(b.y, y), b.z = fmaxf(b.z, x), b.w = fmaxf(b.w, y);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      b.x = fminf(b.x, __shfl_xor_sync(0xffffffffu, b.x, o)), b.y = fminf(b.y, __shfl_xor_sync(0xffffffffu, b.y, o));
      b.z = fmaxf(b.z, __shfl_xor_sync(0xffffffffu, b.z, o)), b.w = fmaxf(b.w, __shfl_xor_sync(0xffffffffu, b.w, o));
    }
    if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = b;
    __syncthreads();
    if (threadIdx.x == 0) {
      for (int w = 1; w < SN_THREADS / 32; ++w) {
        const float4 q = part[w];
        b.x = fminf(b.x, q.x), b.y = fminf(b.y, q.y), b.z = fmaxf(b.z, q.z), b.w = fmaxf(b.w, q.w);
      }
      bounds[(size_t)c * seg_stride] = b;
    }
    __syncthreads();
  }
}

// Level d: every segment's range (absolute positions, for the sort) -- one thread per (cloud, segment)
__global__ void sn_segments_kernel(const PackedClouds in, int n_clouds, int lo, int knn, int d, int *seg_begin,
                                   int *seg_end) {
  const long long total = (long long)n_clouds << d;
  for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(t >> d), s = (int)(t & ((1ll << d) - 1));
    int f, cnt;
    sn_segment(sn_grid_count(in, c, lo), knn, d, s, &f, &cnt);
    const int base = c * in.n_max + f;
    seg_begin[t] = base, seg_end[t] = base + cnt;
  }
}

// Level d: every point's key -- (ordered coordinate on the cut axis, index) in a segment that splits, the index alone in
// a box
__global__ void sn_keys_kernel(const PackedClouds in, int n_clouds, int lo, int knn, int d, unsigned long long *key,
                               const float4 *bounds, int seg_stride) {
  const long long total = (long long)n_clouds * in.n_max;
  for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(t / in.n_max), i = (int)(t - (long long)c * in.n_max), n = sn_grid_count(in, c, lo);
    if (i >= n) continue;
    const unsigned idx = (unsigned)key[t];
    const int s = sn_segment_of(n, knn, d, i);
    int f, cnt;
    sn_segment(n, knn, d, s, &f, &cnt);
    unsigned long long k = idx;
    if (cnt > knn) {
      const int cd = sn_cut_dim(bounds[(size_t)c * seg_stride + s]);
      k |= (unsigned long long)sn_ord(in.pts[2 * ((size_t)in.off[c] + idx) + cd]) << 32;
    }
    key[t] = k;
  }
}

// After level d's sort: the children's bounds of every segment that split
__global__ void sn_cut_kernel(const PackedClouds in, int n_clouds, int lo, int knn, int d, const unsigned long long *key,
                              const float4 *bounds, float4 *child, int seg_stride) {
  const long long total = (long long)n_clouds << d;
  for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(t >> d), s = (int)(t & ((1ll << d) - 1));
    int f, cnt;
    sn_segment(sn_grid_count(in, c, lo), knn, d, s, &f, &cnt);
    if (cnt <= knn) continue;
    const float4 b = bounds[(size_t)c * seg_stride + s];
    const int cd = sn_cut_dim(b);
    const unsigned idx = (unsigned)key[(size_t)c * in.n_max + f + (cnt - cnt / 2)];
    const float cut = in.pts[2 * ((size_t)in.off[c] + idx) + cd];
    float4 l = b, r = b;
    if (cd == 0) l.z = cut, r.x = cut;
    else l.w = cut, r.y = cut;
    child[(size_t)c * seg_stride + 2 * s] = l, child[(size_t)c * seg_stride + 2 * s + 1] = r;
  }
}

// The one-CTA path: the whole partition of every cloud of up to SN_CTA_MAX points, one CTA per cloud (persistent over
// the clouds).  Position i of the cloud is thread i / SN_CTA_ITEMS's item i % SN_CTA_ITEMS (CUB's blocked arrangement);
// level d's keys are (segment << 44 | ordered coordinate << 12 | index), the coordinate 0 in a box, so one sort orders
// every segment at once and leaves each box in index order.  bounds / child: the cloud's two slices of level bounds.
// Writes the final order's indices to key_out, the layout the grid-wide path leaves.
__global__ void __launch_bounds__(SN_CTA_THREADS) sn_cta_kernel(const PackedClouds in, int n_clouds, int knn,
                                                                unsigned long long *key_out, float4 *bounds0,
                                                                float4 *bounds1, int seg_stride) {
  using Sort = cub::BlockRadixSort<unsigned long long, SN_CTA_THREADS, SN_CTA_ITEMS>;
  __shared__ typename Sort::TempStorage tmp;
  __shared__ float4 part[SN_CTA_THREADS / 32];
  const int tid = threadIdx.x;
  for (int c = blockIdx.x; c < n_clouds; c += gridDim.x) {
    const int n = sn_count(in, c);
    if (n > SN_CTA_MAX) continue;  // (CTA-uniform) the grid-wide path's
    const float *p = in.pts + 2 * (size_t)in.off[c];
    float4 *bc = bounds0 + (size_t)c * seg_stride, *bn = bounds1 + (size_t)c * seg_stride;
    float4 b = make_float4(INFINITY, INFINITY, -INFINITY, -INFINITY);
    for (int i = tid; i < n; i += SN_CTA_THREADS) {
      const float x = p[2 * i], y = p[2 * i + 1];
      b.x = fminf(b.x, x), b.y = fminf(b.y, y), b.z = fmaxf(b.z, x), b.w = fmaxf(b.w, y);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      b.x = fminf(b.x, __shfl_xor_sync(0xffffffffu, b.x, o)), b.y = fminf(b.y, __shfl_xor_sync(0xffffffffu, b.y, o));
      b.z = fmaxf(b.z, __shfl_xor_sync(0xffffffffu, b.z, o)), b.w = fmaxf(b.w, __shfl_xor_sync(0xffffffffu, b.w, o));
    }
    if ((tid & 31) == 0) part[tid >> 5] = b;
    __syncthreads();
    if (tid == 0) {
      for (int w = 1; w < SN_CTA_THREADS / 32; ++w) {
        const float4 q = part[w];
        b.x = fminf(b.x, q.x), b.y = fminf(b.y, q.y), b.z = fmaxf(b.z, q.z), b.w = fmaxf(b.w, q.w);
      }
      bc[0] = b;
    }
    __syncthreads();
    const int D = sn_levels(n > 0 ? n : 1, knn);
    unsigned long long k[SN_CTA_ITEMS];
#pragma unroll
    for (int j = 0; j < SN_CTA_ITEMS; ++j) {
      const int i = tid * SN_CTA_ITEMS + j;
      k[j] = i < n ? (unsigned long long)i : ~0ull;  // (padding sorts last)
    }
    for (int d = 0; d <= D; ++d) {
#pragma unroll
      for (int j = 0; j < SN_CTA_ITEMS; ++j) {
        const int i = tid * SN_CTA_ITEMS + j;
        if (i >= n) continue;
        const unsigned idx = (unsigned)(k[j] & ((1u << SN_IDX_BITS) - 1));
        const int s = sn_segment_of(n, knn, d, i);
        int f, cnt;
        sn_segment(n, knn, d, s, &f, &cnt);
        const unsigned ord = cnt > knn ? sn_ord(p[2 * idx + sn_cut_dim(bc[s])]) : 0u;
        k[j] = ((unsigned long long)s << (32 + SN_IDX_BITS)) | ((unsigned long long)ord << SN_IDX_BITS) | idx;
      }
      Sort(tmp).Sort(k, 0, 32 + SN_IDX_BITS + d);
      __syncthreads();  // (tmp is reused by the next sort)
      if (d == D) break;
#pragma unroll
      for (int j = 0; j < SN_CTA_ITEMS; ++j) {  // the point at a splitting segment's cut hands its children the bounds
        const int i = tid * SN_CTA_ITEMS + j;
        if (i >= n) continue;
        const int s = sn_segment_of(n, knn, d, i);
        int f, cnt;
        sn_segment(n, knn, d, s, &f, &cnt);
        if (cnt <= knn || i != f + (cnt - cnt / 2)) continue;
        const float4 bb = bc[s];
        const int cd = sn_cut_dim(bb);
        const float cut = p[2 * (k[j] & ((1u << SN_IDX_BITS) - 1)) + cd];
        float4 l = bb, r = bb;
        if (cd == 0) l.z = cut, r.x = cut;
        else l.w = cut, r.y = cut;
        bn[2 * s] = l, bn[2 * s + 1] = r;
      }
      __syncthreads();
      float4 *t = bc;
      bc = bn, bn = t;
    }
#pragma unroll
    for (int j = 0; j < SN_CTA_ITEMS; ++j) {
      const int i = tid * SN_CTA_ITEMS + j;
      if (i < n) key_out[(size_t)c * in.n_max + i] = k[j] & ((1u << SN_IDX_BITS) - 1);
    }
    __syncthreads();
  }
}

// The boxes (level D, members in index order): extent test, normal (orc_surface_normals' closed form over the k members,
// every operation IEEE float32 in the oracle's order, as grid_surface_normal), centroid; results by original index
__global__ void sn_box_kernel(const PackedClouds in, int n_clouds, int knn, int D, int method, float max_box,
                              const unsigned long long *key, float2 *val, float2 *nrm, unsigned char *keep) {
  const long long total = (long long)n_clouds << D;
  for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(t >> D), s = (int)(t & ((1ll << D) - 1));
    int f, k;
    sn_segment(sn_count(in, c), knn, D, s, &f, &k);
    if (k == 0) continue;
    const unsigned long long *m = key + (size_t)c * in.n_max + f;
    const float2 *p = reinterpret_cast<const float2 *>(in.pts) + in.off[c];
    float2 q = p[(unsigned)m[0]];
    float mnx = q.x, mxx = q.x, mny = q.y, mxy = q.y, sx = 0.f, sy = 0.f;
    for (int j = 0; j < k; ++j) {
      q = p[(unsigned)m[j]];
      mnx = fminf(mnx, q.x), mxx = fmaxf(mxx, q.x), mny = fminf(mny, q.y), mxy = fmaxf(mxy, q.y);
      sx = __fadd_rn(sx, q.x), sy = __fadd_rn(sy, q.y);
    }
    const float ex = __fsub_rn(mxx, mnx), ey = __fsub_rn(mxy, mny);
    if ((ex > ey ? ex : ey) > max_box) continue;
    const float kf = (float)k, mx = __fdiv_rn(sx, kf), my = __fdiv_rn(sy, kf);
    float a = 0.f, b = 0.f, cc = 0.f;
    for (int j = 0; j < k; ++j) {
      q = p[(unsigned)m[j]];
      const float ux = __fsub_rn(q.x, mx), uy = __fsub_rn(q.y, my);
      a = __fadd_rn(a, __fmul_rn(ux, ux)), b = __fadd_rn(b, __fmul_rn(ux, uy)), cc = __fadd_rn(cc, __fmul_rn(uy, uy));
    }
    a = __fdiv_rn(a, kf), b = __fdiv_rn(b, kf), cc = __fdiv_rn(cc, kf);
    float2 n = make_float2(0.f, 0.f);
    if (a != 0.f || b != 0.f || cc != 0.f) {
      const float dd = __fmul_rn(0.5f, __fsub_rn(a, cc));
      const float r = __fsqrt_rn(__fadd_rn(__fmul_rn(dd, dd), __fmul_rn(b, b)));
      if (r == 0.f) {
        n = make_float2(1.f, 0.f);
      } else {
        const float ux = dd >= 0.f ? __fadd_rn(r, dd) : b, uy = dd >= 0.f ? b : __fsub_rn(r, dd);
        const float len = __fsqrt_rn(__fadd_rn(__fmul_rn(ux, ux), __fmul_rn(uy, uy)));
        n = make_float2(-__fdiv_rn(uy, len), __fdiv_rn(ux, len));
      }
    }
    for (int j = 0; j < (method == 1 ? 1 : k); ++j) {
      const size_t at = (size_t)c * in.n_max + (unsigned)m[j];
      keep[at] = 1, nrm[at] = n, val[at] = method == 1 ? make_float2(mx, my) : p[(unsigned)m[j]];
    }
  }
}

// The kept points and their normals, in index order, at c * n_max; out_cnt[c] their number.  One CTA per cloud.
__global__ void __launch_bounds__(SN_THREADS) sn_compact_kernel(const PackedClouds in, int n_clouds, const float2 *val,
                                                                const float2 *nrm, const unsigned char *keep,
                                                                float2 *out_pts, float2 *out_nrm, int *out_off,
                                                                int *out_cnt) {
  __shared__ int warp_n[SN_THREADS / 32];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (int c = blockIdx.x; c < n_clouds; c += gridDim.x) {
    const int n = sn_count(in, c);
    const size_t base_at = (size_t)c * in.n_max;
    if (tid == 0) out_off[c] = c * in.n_max;
    if (c == n_clouds - 1 && tid == 0) out_off[n_clouds] = n_clouds * in.n_max;
    int base = 0;
    for (int i0 = 0; i0 < n; i0 += SN_THREADS) {
      const int i = i0 + tid;
      const bool kp = i < n && keep[base_at + i];
      const unsigned m = __ballot_sync(0xffffffffu, kp);
      if (lane == 0) warp_n[warp] = __popc(m);
      __syncthreads();
      int before = base, tot = 0;
      for (int w = 0; w < SN_THREADS / 32; ++w) {
        if (w < warp) before += warp_n[w];
        tot += warp_n[w];
      }
      if (kp) {
        const int at = before + __popc(m & ((1u << lane) - 1u));
        out_pts[base_at + at] = val[base_at + i], out_nrm[base_at + at] = nrm[base_at + i];
      }
      base += tot;
      __syncthreads();
    }
    if (tid == 0) out_cnt[c] = base;
  }
}

// Workspace layout of sampling_normals_run for n_clouds clouds of up to n_max points
struct SnLayout {
  int D;
  size_t segs, pts, temp_bytes;
};

static int sn_layout(int n_clouds, int n_max, int knn, SnLayout &L) {
  L.D = sn_levels(n_max, knn);
  L.segs = (size_t)n_clouds << L.D;
  L.pts = (size_t)n_clouds * n_max;
  SFE_REQUIRE(L.segs < (size_t)INT_MAX && L.pts < (size_t)INT_MAX,
              "icp: SamplingSurfaceNormalDataPointsFilter: %d clouds of up to %d points at knn %d exceed the segment "
              "table", n_clouds, n_max, knn);
  cub::DoubleBuffer<unsigned long long> k;
  L.temp_bytes = 0;
  SFE_CUDA(cub::DeviceSegmentedSort::SortKeys(nullptr, L.temp_bytes, k, (int)L.pts, (int)L.segs, (const int *)nullptr,
                                              (const int *)nullptr));
  return SFE_OK;
}

static void sn_carve(Carver &cv, const SnLayout &L, unsigned long long **k0, unsigned long long **k1, float4 **b0,
                     float4 **b1, int **sb, int **se, float2 **val, float2 **nrm, unsigned char **keep, void **temp) {
  *k0 = (unsigned long long *)cv.take(sizeof(unsigned long long) * L.pts);
  *k1 = (unsigned long long *)cv.take(sizeof(unsigned long long) * L.pts);
  *b0 = (float4 *)cv.take(sizeof(float4) * L.segs);
  *b1 = (float4 *)cv.take(sizeof(float4) * L.segs);
  *sb = (int *)cv.take(sizeof(int) * L.segs);
  *se = (int *)cv.take(sizeof(int) * L.segs);
  *val = (float2 *)cv.take(sizeof(float2) * L.pts);
  *nrm = (float2 *)cv.take(sizeof(float2) * L.pts);
  *keep = (unsigned char *)cv.take(L.pts);
  *temp = cv.take(L.temp_bytes);
}

int sampling_normals_ws(int n_clouds, int n_max, int knn, size_t *bytes) {
  SnLayout L;
  const int rc = sn_layout(n_clouds, n_max > 0 ? n_max : 1, knn, L);
  if (rc != SFE_OK) return rc;
  Carver cv;
  unsigned long long *k0, *k1;
  float4 *b0, *b1;
  int *sb, *se;
  float2 *val, *nrm;
  unsigned char *keep;
  void *temp;
  sn_carve(cv, L, &k0, &k1, &b0, &b1, &sb, &se, &val, &nrm, &keep, &temp);
  *bytes = cv.off;
  return SFE_OK;
}

int sampling_normals_run(sfe_ctx *ctx, cudaStream_t st, const PackedClouds &in_c, int n_clouds, int knn, int method,
                         float max_box, void *ws, float *out_pts, int *out_off, int *out_cnt, float2 *out_nrm) {
  PackedClouds in = in_c;
  in.n_max = in.n_max > 0 ? in.n_max : 1;
  SnLayout L;
  int rc = sn_layout(n_clouds, in.n_max, knn, L);
  if (rc != SFE_OK) return rc;
  Carver cv;
  cv.base = (char *)ws;
  unsigned long long *k0, *k1;
  float4 *b0, *b1;
  int *sb, *se;
  float2 *val, *nrm;
  unsigned char *keep;
  void *temp;
  sn_carve(cv, L, &k0, &k1, &b0, &b1, &sb, &se, &val, &nrm, &keep, &temp);
  const int seg_stride = 1 << L.D;
  const int grid = ctx->sm_count * 8;
  SFE_CUDA(cudaMemsetAsync(keep, 0, L.pts, st));
  cub::DoubleBuffer<unsigned long long> keys(k0, k1);
  // the grid-wide levels, for the clouds above the one-CTA path's capacity (only when the capacity n_max allows one)
  if (in.n_max > SN_CTA_MAX) {
    sn_init_kernel<<<std::min(n_clouds, grid), SN_THREADS, 0, st>>>(in, n_clouds, k0, b0, seg_stride);
    SFE_CUDA(cudaGetLastError());
    ctx->launches++;
  }
  for (int d = 0; in.n_max > SN_CTA_MAX && d <= L.D; ++d) {
    const long long segs = (long long)n_clouds << d;
    const int sgrid = (int)std::min<long long>((segs + SN_THREADS - 1) / SN_THREADS, grid);
    const int pgrid = (int)std::min<long long>(((long long)L.pts + SN_THREADS - 1) / SN_THREADS, grid);
    sn_segments_kernel<<<sgrid, SN_THREADS, 0, st>>>(in, n_clouds, SN_CTA_MAX, knn, d, sb, se);
    sn_keys_kernel<<<pgrid, SN_THREADS, 0, st>>>(in, n_clouds, SN_CTA_MAX, knn, d, keys.Current(), b0, seg_stride);
    SFE_CUDA(cudaGetLastError());
    size_t tb = L.temp_bytes;
    SFE_CUDA(cub::DeviceSegmentedSort::SortKeys(temp, tb, keys, (int)L.pts, (int)segs, sb, se, st));
    ctx->launches += 3;
    if (d < L.D) {
      sn_cut_kernel<<<sgrid, SN_THREADS, 0, st>>>(in, n_clouds, SN_CTA_MAX, knn, d, keys.Current(), b0, b1,
                                                  seg_stride);
      SFE_CUDA(cudaGetLastError());
      ctx->launches++;
      std::swap(b0, b1);
    }
  }
  // the one-CTA path, after the grid-wide levels (it reuses their bounds slices), into the key buffer they left
  int per_sm;
  if ((rc = ctas_per_sm(ctx, (const void *)sn_cta_kernel, SN_CTA_THREADS, 0, &per_sm)) != SFE_OK) return rc;
  sn_cta_kernel<<<std::min(n_clouds, ctx->sm_count * per_sm), SN_CTA_THREADS, 0, st>>>(in, n_clouds, knn,
                                                                                      keys.Current(), b0, b1,
                                                                                      seg_stride);
  SFE_CUDA(cudaGetLastError());
  ctx->launches++;
  const int bgrid = (int)std::min<long long>(((long long)L.segs + SN_THREADS - 1) / SN_THREADS, grid);
  sn_box_kernel<<<bgrid, SN_THREADS, 0, st>>>(in, n_clouds, knn, L.D, method, max_box, keys.Current(), val, nrm, keep);
  sn_compact_kernel<<<std::min(n_clouds, grid), SN_THREADS, 0, st>>>(in, n_clouds, val, nrm, keep,
                                                                     reinterpret_cast<float2 *>(out_pts), out_nrm,
                                                                     out_off, out_cnt);
  SFE_CUDA(cudaGetLastError());
  ctx->launches += 2;
  return SFE_OK;
}

}  // namespace sfe
