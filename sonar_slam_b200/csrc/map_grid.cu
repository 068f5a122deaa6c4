// Map grids (sm_90a): clouds too large for a one-CTA layout, sorted into a uniform grid in global memory once per call.
//
// Shared by the scan matcher and the nearest-neighbour matcher (icp.cu: icp_kernel's map class, match_map_kernel) and the
// radius outlier filter (cloud.cu: ro_map_count_kernel).  The grid is the one grid.cuh describes -- row-major cells,
// every cell's points contiguous -- with 32-bit absolute cell starts and original indices (MapGridView).
#include <climits>

#include <cub/cub.cuh>

#include "grid.cuh"
#include "stages.cuh"

namespace sfe {

// Clouds too large for the in-CTA layout get one grid each per call, in global memory, shared by every problem that
// names the same cloud.  Slots: the distinct map-class clouds, numbered in cloud order on the device (a sort of the
// problems by cloud id), so nothing depends on how many problems share a cloud or in which order they come.
// Per slot: the mean (icp_kernel's own sequential float32 sum in point order; 0 without centring), the bounding box of the
// centred points, the geometry (grid_geometry, up to 1.5 cells per point), a stable radix sort of (slot, cell, index),
// the centred points in that order with their original indices, the cell starts, and for point-to-plane the normals
// (grid_surface_normal, one thread per point).  No coarse occupancy map: pass B of the pruned path searches instead.
constexpr int MAP_THREADS = 256;
constexpr int MAP_SETUP_THREADS = 512;
constexpr unsigned MAP_NONE = 0xffffffffu;

__device__ __forceinline__ int map_count(const PackedClouds &t, int c) {
  return t.cnt ? t.cnt[c] : t.off[c + 1] - t.off[c];
}

__global__ void map_flag_kernel(const PackedClouds t, const int *tgt_id, int P, int limit, unsigned *key, int *val,
                                int *slot) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= P) return;
  const int ti = tgt_id ? tgt_id[p] : p;
  key[p] = map_count(t, ti) > limit ? (unsigned)ti : MAP_NONE;
  val[p] = p;
  slot[p] = -1;
}

__global__ void map_head_kernel(const unsigned *key, int P, int *head) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < P) head[i] = key[i] != MAP_NONE && (i == 0 || key[i] != key[i - 1]);
}

__global__ void map_slot_kernel(const unsigned *key, const int *val, const int *head, const int *sid, int P, int *slot,
                                int *slot_tgt, int *n_slots) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= P) return;
  if (key[i] != MAP_NONE) {
    slot[val[i]] = sid[i] - 1;
    if (head[i]) slot_tgt[sid[i] - 1] = (int)key[i];
  }
  if (i == P - 1) *n_slots = sid[i];
}

// one CTA per slot: mean, bounding box, geometry
__global__ void __launch_bounds__(MAP_SETUP_THREADS) map_setup_kernel(const PackedClouds t, int dim, const int *slot_tgt,
                                                                       const int *n_slots, int center, int seq,
                                                                       MapGrid *grid) {
  __shared__ float mean[2];
  __shared__ float4 bred[MAP_SETUP_THREADS / 32];
  __shared__ double red[2 * 5 * 16];
  const int s = blockIdx.x, tid = threadIdx.x, nthr = blockDim.x;
  if (s >= *n_slots) return;
  const int ti = slot_tgt[s], nt = map_count(t, ti);
  const float *tgt = t.pts + dim * (size_t)t.off[ti];
  float mx = 0.f, my = 0.f;
  if (center) {  // as icp_body's set-up
    if (seq) {
      if (tid < 64) {
        const float sum = seq_sum_warp_global(tgt + (tid >> 5), nt, dim);
        if ((tid & 31) == 0) mean[tid >> 5] = __fdiv_rn(sum, (float)nt);
      }
      __syncthreads();
      mx = mean[0], my = mean[1];
    } else {  // (float64 mode: the reduction tree of a 512-thread CTA, not the in-CTA launch's -- that mode is not
              //  bit-reproducible across CTA sizes anyway)
      double sm[2] = {0.0, 0.0}, tot[2];
      int phase = 0;
      for (int i = tid; i < nt; i += nthr) sm[0] += (double)tgt[dim * i], sm[1] += (double)tgt[dim * i + 1];
      block_sum<2>(sm, red, phase, tot);
      mx = (float)(tot[0] / (double)nt), my = (float)(tot[1] / (double)nt);
    }
  }
  float4 bnd = make_float4(INFINITY, INFINITY, -INFINITY, -INFINITY);
  for (int i = tid; i < nt; i += nthr) {
    const float x = tgt[dim * i] - mx, y = tgt[dim * i + 1] - my;
    bnd.x = fminf(bnd.x, x), bnd.y = fminf(bnd.y, y), bnd.z = fmaxf(bnd.z, x), bnd.w = fmaxf(bnd.w, y);
  }
  bnd = block_bounds(bnd, bred);
  if (tid == 0) {
    MapGridView g;
    grid_geometry(nt, bnd.x, bnd.y, bnd.z, bnd.w, 0.05f, g, nt + nt / 2 > 256 ? nt + nt / 2 : 256);
    MapGrid m;
    m.mean[0] = mx, m.mean[1] = my;
    m.bbox[0] = bnd.x, m.bbox[1] = bnd.y, m.bbox[2] = bnd.z, m.bbox[3] = bnd.w;
    m.ox = g.ox, m.oy = g.oy, m.cell = g.cell, m.inv_cell = g.inv_cell;
    m.nx = g.nx, m.ny = g.ny, m.n = nt, m.pad = 0;
    grid[s] = m;
  }
}

// sort key of every (slot, point): slot above, cell below; unused positions get the padding key (all ones)
__global__ void map_keys_kernel(const PackedClouds t, int dim, const int *slot_tgt, const int *n_slots,
                                const MapGrid *grid, int nt_max, unsigned long long *key, int *val) {
  const int s = blockIdx.y;
  const bool live = s < *n_slots;
  const int ti = live ? slot_tgt[s] : 0, nt = live ? map_count(t, ti) : 0;
  const float *tgt = t.pts + dim * (size_t)(live ? t.off[ti] : 0);
  MapGrid m;
  if (live) m = grid[s];
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < nt_max; j += gridDim.x * blockDim.x) {
    const size_t i = (size_t)s * nt_max + j;
    if (j < nt) {
      const float x = tgt[dim * j] - m.mean[0], y = tgt[dim * j + 1] - m.mean[1];
      const int c = grid_cell_coord(y, m.oy, m.inv_cell, m.ny) * m.nx + grid_cell_coord(x, m.ox, m.inv_cell, m.nx);
      key[i] = ((unsigned long long)s << 32) | (unsigned)c;
      val[i] = j;
    } else {
      key[i] = ~0ull;
      val[i] = 0;
    }
  }
}

// after the sort: centred points in sorted order and every cell's first position (absolute in pts)
__global__ void map_scatter_kernel(const PackedClouds t, int dim, const int *slot_tgt, const MapGrid *grid,
                                   const unsigned long long *key, const int *val, int N, int cell_cap, float2 *pts,
                                   int *cstart) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  const unsigned long long k = key[i];
  if (k == ~0ull) return;
  const int s = (int)(k >> 32), c = (int)(k & 0xffffffffu), j = val[i];
  const MapGrid &m = grid[s];
  const float *src = t.pts + dim * ((size_t)t.off[slot_tgt[s]] + j);
  pts[i] = make_float2(src[0] - m.mean[0], src[1] - m.mean[1]);
  int *cs = cstart + (size_t)s * cell_cap;
  const int pc = (i > 0 && (int)(key[i - 1] >> 32) == s) ? (int)(key[i - 1] & 0xffffffffu) : -1;
  for (int cc = pc + 1; cc <= c; ++cc) cs[cc] = i;
  if (i + 1 == N || (key[i + 1] >> 32) != (unsigned long long)s)
    for (int cc = c + 1; cc <= m.nx * m.ny; ++cc) cs[cc] = i + 1;  // through the sentinel entry ncells
}

// point-to-plane: the normal at every sorted position, once per target
__global__ void map_normals_kernel(const unsigned long long *key, const MapArgs m, int N, int knn, float2 *nrm) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  const unsigned long long k = key[i];
  if (k == ~0ull) return;
  const MapGridView g = map_grid_view(m, (int)(k >> 32));
  float bd[GRID_KNN_MAX];
  int bi[GRID_KNN_MAX];
  nrm[i] = grid_surface_normal(g, i, knn, bd, bi, 1);
}

// point-to-plane with given normals (SamplingSurfaceNormalDataPointsFilter): the normal of every sorted position
__global__ void map_given_normals_kernel(const unsigned long long *key, const PackedClouds t, const int *slot_tgt,
                                         const int *orig, int N, const float2 *given, float2 *nrm) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  const unsigned long long k = key[i];
  if (k == ~0ull) return;
  nrm[i] = given[t.off[slot_tgt[(int)(k >> 32)]] + orig[i]];
}

// Builds the map grids of the problems whose target has more than `limit` points.  slot_cap bounds the number of
// distinct such targets.  Workspace (scratch[SCR_MAP]): 40 bytes per slot point (48 with normals) for slot_cap *
// nt_max slot points, 4 * (1.5 nt_max + 257) bytes of cell table per slot, 28 bytes per problem, CUB's temporary
// storage.  knn > 0: normals too.
int map_build(sfe_ctx *ctx, cudaStream_t st, const PackedClouds &t, int dim, const int *tgt_id, int P, int limit,
              int slot_cap, bool center, bool seq, int knn, MapWs &w, const float2 *given_nrm) {
  const int nt_max = t.n_max;
  const long long slots = (long long)slot_cap * nt_max;
  SFE_REQUIRE(slots < INT_MAX, "map grids: %d targets of up to %d points exceed %d slot points", slot_cap, nt_max,
              INT_MAX - 1);
  SFE_REQUIRE(slot_cap <= 65535, "map grids: at most 65535 distinct map-sized targets per call (got up to %d)",
              slot_cap);
  const int N = (int)slots;
  w.cell_cap = (nt_max + nt_max / 2 > 256 ? nt_max + nt_max / 2 : 256) + 1;
  int slot_bits = 1;
  while ((1ll << slot_bits) < slot_cap) ++slot_bits;
  const int end_bit = 32 + slot_bits;

  cub::DoubleBuffer<unsigned> pkeys;
  cub::DoubleBuffer<int> pvals;
  cub::DoubleBuffer<unsigned long long> keys;
  cub::DoubleBuffer<int> vals;
  size_t psort_bytes = 0, scan_bytes = 0, sort_bytes = 0;
  SFE_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, psort_bytes, pkeys, pvals, P, 0, 32, st));
  SFE_CUDA(cub::DeviceScan::InclusiveSum(nullptr, scan_bytes, (const int *)nullptr, (int *)nullptr, P, st));
  SFE_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, keys, vals, N, 0, end_bit, st));
  size_t temp_bytes = psort_bytes > scan_bytes ? psort_bytes : scan_bytes;
  if (sort_bytes > temp_bytes) temp_bytes = sort_bytes;
  Carver cv;
  unsigned *pk0, *pk1;
  int *pv0, *pv1, *head, *sid;
  unsigned long long *k0, *k1;
  int *v0, *v1;
  void *temp;
  for (int pass = 0; pass < 2; ++pass) {
    cv.off = 0;
    pk0 = (unsigned *)cv.take(sizeof(unsigned) * (size_t)P);
    pk1 = (unsigned *)cv.take(sizeof(unsigned) * (size_t)P);
    pv0 = (int *)cv.take(sizeof(int) * (size_t)P);
    pv1 = (int *)cv.take(sizeof(int) * (size_t)P);
    head = (int *)cv.take(sizeof(int) * (size_t)P);
    sid = (int *)cv.take(sizeof(int) * (size_t)P);
    w.slot = (int *)cv.take(sizeof(int) * (size_t)P);
    w.n_slots = (int *)cv.take(sizeof(int));
    w.slot_tgt = (int *)cv.take(sizeof(int) * (size_t)slot_cap);
    w.grid = (MapGrid *)cv.take(sizeof(MapGrid) * (size_t)slot_cap);
    k0 = (unsigned long long *)cv.take(sizeof(unsigned long long) * (size_t)N);
    k1 = (unsigned long long *)cv.take(sizeof(unsigned long long) * (size_t)N);
    v0 = (int *)cv.take(sizeof(int) * (size_t)N);
    v1 = (int *)cv.take(sizeof(int) * (size_t)N);
    w.pts = (float2 *)cv.take(sizeof(float2) * (size_t)N);
    w.nrm = knn > 0 || given_nrm ? (float2 *)cv.take(sizeof(float2) * (size_t)N) : nullptr;
    w.cstart = (int *)cv.take(sizeof(int) * (size_t)slot_cap * w.cell_cap);
    temp = cv.take(temp_bytes);
    if (pass == 0) {
      int rc = ensure(ctx, ctx->scratch[SCR_MAP], cv.off, st);
      if (rc != SFE_OK) return rc;
      cv.base = (char *)ctx->scratch[SCR_MAP].ptr;
    }
  }
  const int pb = (P + MAP_THREADS - 1) / MAP_THREADS;
  map_flag_kernel<<<pb, MAP_THREADS, 0, st>>>(t, tgt_id, P, limit, pk0, pv0, w.slot);
  SFE_CUDA(cudaGetLastError());
  pkeys = cub::DoubleBuffer<unsigned>(pk0, pk1);
  pvals = cub::DoubleBuffer<int>(pv0, pv1);
  SFE_CUDA(cub::DeviceRadixSort::SortPairs(temp, psort_bytes, pkeys, pvals, P, 0, 32, st));
  map_head_kernel<<<pb, MAP_THREADS, 0, st>>>(pkeys.Current(), P, head);
  SFE_CUDA(cudaGetLastError());
  SFE_CUDA(cub::DeviceScan::InclusiveSum(temp, scan_bytes, (const int *)head, sid, P, st));
  map_slot_kernel<<<pb, MAP_THREADS, 0, st>>>(pkeys.Current(), pvals.Current(), head, sid, P, w.slot, w.slot_tgt,
                                              w.n_slots);
  SFE_CUDA(cudaGetLastError());
  map_setup_kernel<<<slot_cap, MAP_SETUP_THREADS, 0, st>>>(t, dim, w.slot_tgt, w.n_slots, center ? 1 : 0, seq ? 1 : 0, w.grid);
  SFE_CUDA(cudaGetLastError());
  int bps = (nt_max + 4 * MAP_THREADS - 1) / (4 * MAP_THREADS);
  bps = bps < 1 ? 1 : (bps > 256 ? 256 : bps);
  map_keys_kernel<<<dim3(bps, slot_cap), MAP_THREADS, 0, st>>>(t, dim, w.slot_tgt, w.n_slots, w.grid, nt_max, k0, v0);
  SFE_CUDA(cudaGetLastError());
  keys = cub::DoubleBuffer<unsigned long long>(k0, k1);
  vals = cub::DoubleBuffer<int>(v0, v1);
  SFE_CUDA(cub::DeviceRadixSort::SortPairs(temp, sort_bytes, keys, vals, N, 0, end_bit, st));
  w.orig = vals.Current();
  const int nb = (N + MAP_THREADS - 1) / MAP_THREADS;
  map_scatter_kernel<<<nb, MAP_THREADS, 0, st>>>(t, dim, w.slot_tgt, w.grid, keys.Current(), w.orig, N, w.cell_cap, w.pts,
                                                 w.cstart);
  SFE_CUDA(cudaGetLastError());
  ctx->launches += 9;  // six kernels, the two sorts and the scan counted once each
  if (given_nrm) {
    map_given_normals_kernel<<<nb, MAP_THREADS, 0, st>>>(keys.Current(), t, w.slot_tgt, w.orig, N, given_nrm, w.nrm);
    SFE_CUDA(cudaGetLastError());
    ctx->launches++;
  } else if (knn > 0) {
    map_normals_kernel<<<nb, MAP_THREADS, 0, st>>>(keys.Current(), w.args(), N, knn, w.nrm);
    SFE_CUDA(cudaGetLastError());
    ctx->launches++;
  }
  return SFE_OK;
}

}  // namespace sfe
