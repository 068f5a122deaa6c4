// Uniform-grid nearest-neighbour machinery shared by the ICP, match and outlier kernels.
//
// This is the GPU counterpart of the KD-tree the reference reaches through libpointmatcher /
// libnabo (KDTreeMatcher, pcl.cpp:161-174 and icp.yaml:5-9) and PCL (RadiusOutlierRemoval,
// pcl.cpp:54-74): an exact search structure, rebuilt per call like the reference does, but laid
// out for a CTA: the reference cloud is counting-sorted by cell (row-major cells, so a row span of
// cells is one contiguous point range) and lives in shared memory together with 16-bit cell
// offsets; a query walks square rings of cells around its own cell until the ring boundary is
// farther than the best match.
//
// Conventions (same as oracle/cloud_ref.c): float32 squared distance dx*dx + dy*dy with each
// product and the sum rounded separately; ties go to the lowest ORIGINAL index.
#pragma once
#include "common.cuh"
#include "stages.cuh"

namespace sfe {

constexpr int GRID_MAX_CELLS = 16384;  // 16-bit offsets, two per 32-bit word

// Idx: type of the cell offsets and original indices.  uint16_t for the grids a CTA builds in shared memory
// (GridView); int for the map grids built once per cloud in global memory (map_grid.cu, MapGridView), whose
// offsets are absolute positions in the workspace's sorted-point array.
template <typename Idx>
struct GridViewT {
  const float2 *pts;   // points sorted by cell
  const Idx *cstart;   // [ncells + 1] first sorted position of every cell
  const Idx *orig;     // sorted position -> index in the caller's cloud
  int n, nx, ny;
  float ox, oy, cell, inv_cell;
};
using GridView = GridViewT<uint16_t>;
using MapGridView = GridViewT<int>;

// the grid of map slot `slot` (map_build)
__device__ __forceinline__ MapGridView map_grid_view(const MapArgs &m, int slot) {
  const MapGrid &mg = m.grid[slot];
  MapGridView g;
  g.pts = m.pts, g.cstart = m.cstart + (size_t)slot * m.cell_cap, g.orig = m.orig;
  g.n = mg.n, g.nx = mg.nx, g.ny = mg.ny, g.ox = mg.ox, g.oy = mg.oy, g.cell = mg.cell, g.inv_cell = mg.inv_cell;
  return g;
}

__device__ __forceinline__ float dist2_rn(float dx, float dy) {
  return __fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy));
}

__device__ __forceinline__ int grid_cell_coord(float v, float o, float inv_cell, int n) {
  const int c = (int)floorf((v - o) * inv_cell);
  return c < 0 ? 0 : (c >= n ? n - 1 : c);
}

// block-wide exclusive scan helper: returns the exclusive prefix of `v` over the CTA and the total
__device__ __forceinline__ int block_exclusive_scan(int v, int *warp_sums /* [33] smem */, int &total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = (blockDim.x + 31) >> 5;
  int incl = v;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const int t = __shfl_up_sync(0xffffffffu, incl, d);
    if (lane >= d) incl += t;
  }
  if (lane == 31) warp_sums[warp] = incl;
  __syncthreads();
  if (warp == 0) {
    int w = lane < nwarps ? warp_sums[lane] : 0;
    int wi = w;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const int t = __shfl_up_sync(0xffffffffu, wi, d);
      if (lane >= d) wi += t;
    }
    warp_sums[lane] = wi - w;
    if (lane == 31) warp_sums[32] = wi;
  }
  __syncthreads();
  const int excl = warp_sums[warp] + incl - v;
  total = warp_sums[32];
  __syncthreads();
  return excl;
}

// Sum K doubles over the CTA with ONE barrier: every warp publishes its partial sums, and after the barrier
// every warp reduces the (<= 16) partials itself with a butterfly, so all threads hold the bit-identical total.
// `scratch` has two halves used alternately (`phase` counts the calls): the half written by call n is last read
// before call n+1's barrier and not rewritten before call n+2.
template <int K>
__device__ __forceinline__ void block_sum(double (&v)[K], double *scratch /* [2][5][16] smem */, int &phase,
                                          double (&out)[K]) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  static_assert(K <= 5, "scratch holds five partial sums per warp");
  double *half = scratch + (phase & 1) * (5 * 16);
  ++phase;
#pragma unroll
  for (int k = 0; k < K; ++k) {
    double x = v[k];
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) x += __shfl_xor_sync(0xffffffffu, x, d);
    if (lane == 0) half[k * 16 + warp] = x;
  }
  __syncthreads();
#pragma unroll
  for (int k = 0; k < K; ++k) {
    double x = lane < nwarps ? half[k * 16 + lane] : 0.0;
#pragma unroll
    for (int d = 8; d > 0; d >>= 1) x += __shfl_xor_sync(0xffffffffu, x, d);  // nwarps <= 16
    out[k] = __shfl_sync(0xffffffffu, x, 0);
  }
}

// (min x, min y, max x, max y) over the CTA from every thread's partial bounds: warp shuffles, then thread 0 over the
// warps' results in `red` (shared, one entry per warp).  The result is valid in thread 0 only; min and max are exact,
// so the order does not matter.
__device__ __forceinline__ float4 block_bounds(float4 m, float4 *red) {
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) {
    m.x = fminf(m.x, __shfl_xor_sync(0xffffffffu, m.x, d));
    m.y = fminf(m.y, __shfl_xor_sync(0xffffffffu, m.y, d));
    m.z = fmaxf(m.z, __shfl_xor_sync(0xffffffffu, m.z, d));
    m.w = fmaxf(m.w, __shfl_xor_sync(0xffffffffu, m.w, d));
  }
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
  __syncthreads();
  if (threadIdx.x == 0)
    for (int w = 1; w < (int)(blockDim.x >> 5); ++w)
      m.x = fminf(m.x, red[w].x), m.y = fminf(m.y, red[w].y), m.z = fmaxf(m.z, red[w].z), m.w = fmaxf(m.w, red[w].w);
  return m;
}

// One sequential sum over values in global memory, p[0], p[stride], ... (the reference cloud's mean, once per
// problem): lane j holds term base + j and a shuffle hands term j to every lane, so all lanes carry the same
// running sum; eight batches (256 terms) are requested at once and the next eight are in flight while these are
// added, so the L2 latency hides behind the ~1000-cycle add chain.  s0: the value the chain starts from.  Lanes past n
// hold -0.f, the identity of IEEE addition, so that a chain from -0.f over -0.f terms stays -0.f.
__device__ __forceinline__ float seq_sum_warp_global(const float *p, int n, int stride, float s0 = 0.f) {
  const int lane = threadIdx.x & 31;
  float s = s0, cur[8], nxt[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const int i = k * 32 + lane;
    cur[k] = i < n ? p[(size_t)i * stride] : -0.f;
  }
  for (int base = 0; base < n; base += 256) {
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const int i = base + 256 + k * 32 + lane;
      nxt[k] = i < n ? p[(size_t)i * stride] : -0.f;
    }
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      if (base + k * 32 < n) {  // (warp-uniform)
#pragma unroll
        for (int j = 0; j < 32; ++j) s = __fadd_rn(s, __shfl_sync(0xffffffffu, cur[k], j));
      }
    }
#pragma unroll
    for (int k = 0; k < 8; ++k) cur[k] = nxt[k];
  }
  return s;
}

// Choose grid geometry for n points with bounding box [minx,maxx] x [miny,maxy].
template <typename Idx>
__device__ __forceinline__ void grid_geometry(int n, float minx, float miny, float maxx, float maxy, float min_cell,
                                              GridViewT<Idx> &g, int max_cells, float cell_scale = 1.0f) {
  const float w = maxx - minx, h = maxy - miny;
  float cell = cell_scale * sqrtf((w * h) / (float)(n > 0 ? n : 1));
  if (!(cell > min_cell)) cell = min_cell;
  if (!(cell > 1e-6f)) cell = 1.f;
  // keep the cell table within max_cells (<= GRID_MAX_CELLS for the 16-bit grids)
  for (int it = 0; it < 32; ++it) {
    const float inv = 1.f / cell;
    const long long nx = (long long)(w * inv) + 1, ny = (long long)(h * inv) + 1;
    if (nx * ny <= max_cells && nx < 32768 && ny < 32768) break;
    cell *= 1.5f;
  }
  g.cell = cell;
  g.inv_cell = 1.f / cell;
  g.ox = minx;
  g.oy = miny;
  g.nx = (int)(w * g.inv_cell) + 1;
  g.ny = (int)(h * g.inv_cell) + 1;
  g.n = n;
}

// Counting sort of `n` points (src[i] - (mx,my)) into cells.  All threads of the CTA call this.
//   sorted  [n]            float2, shared or global
//   cells   [ncells/2+1]   uint32 words holding two uint16 offsets each (shared), zeroed here
//   orig    [n]            uint16 original indices (global or shared), may be null
// g.nx/ny/ox/oy/cell must be set (grid_geometry).  n <= 65535.
__device__ __forceinline__ void grid_build(const float *__restrict__ src, int stride, int n, float mx, float my,
                                           GridView &g, float2 *sorted, uint32_t *cells, uint16_t *orig,
                                           int *scan_scratch /* [33] smem */) {
  const int tid = threadIdx.x, nt = blockDim.x;
  const int ncells = g.nx * g.ny;
  const int nwords = (ncells + 2) / 2;  // covers entries 0 .. ncells
  for (int w = tid; w < nwords; w += nt) cells[w] = 0;
  __syncthreads();
  // histogram
  for (int i = tid; i < n; i += nt) {
    const float x = src[(size_t)i * stride] - mx, y = src[(size_t)i * stride + 1] - my;
    const int c = grid_cell_coord(y, g.oy, g.inv_cell, g.ny) * g.nx + grid_cell_coord(x, g.ox, g.inv_cell, g.nx);
    atomicAdd(&cells[c >> 1], (c & 1) ? 0x10000u : 1u);
  }
  __syncthreads();
  // inclusive scan over cells: each thread owns a contiguous run of words
  const int per = (nwords + nt - 1) / nt;
  const int w0 = min(tid * per, nwords), w1 = min(w0 + per, nwords);
  int local = 0;
  for (int w = w0; w < w1; ++w) local += (int)(cells[w] & 0xffffu) + (int)(cells[w] >> 16);
  int total;
  int run = block_exclusive_scan(local, scan_scratch, total);
  for (int w = w0; w < w1; ++w) {
    const uint32_t v = cells[w];
    const int lo = run + (int)(v & 0xffffu), hi = lo + (int)(v >> 16);
    cells[w] = (uint32_t)lo | ((uint32_t)hi << 16);  // inclusive ends
    run = hi;
  }
  __syncthreads();
  // scatter from the back of every cell: the inclusive end counts down to the cell start
  for (int i = tid; i < n; i += nt) {
    const float x = src[(size_t)i * stride] - mx, y = src[(size_t)i * stride + 1] - my;
    const int c = grid_cell_coord(y, g.oy, g.inv_cell, g.ny) * g.nx + grid_cell_coord(x, g.ox, g.inv_cell, g.nx);
    const uint32_t old = atomicSub(&cells[c >> 1], (c & 1) ? 0x10000u : 1u);
    const int pos = (int)((c & 1) ? (old >> 16) : (old & 0xffffu)) - 1;
    sorted[pos] = make_float2(x, y);
    if (orig) orig[pos] = (uint16_t)i;
  }
  __syncthreads();
  if (tid == 0) {  // sentinel entry ncells = n
    uint16_t *cs = reinterpret_cast<uint16_t *>(cells);
    cs[ncells] = (uint16_t)n;
  }
  __syncthreads();
  g.pts = sorted;
  g.cstart = reinterpret_cast<const uint16_t *>(cells);
  g.orig = orig;
}

struct NNResult {
  float d2;
  int pos;   // sorted position, -1 if none
  int tie;   // another point at exactly the same distance was seen (resolved after the search)
};

// scan a contiguous range of sorted points (hot loop: no global memory, ties only flagged)
__device__ __forceinline__ void nn_update(float d2, int p, NNResult &r) {
  r.tie |= (d2 == r.d2) & (p != r.pos);
  if (d2 < r.d2) {
    r.d2 = d2;
    r.pos = p;
    r.tie = 0;
  }
}

// Four candidates per trip: the four shared-memory loads are issued together (a warp issues in order, so a
// load followed by its use costs the full latency per candidate), and the best / tie bookkeeping only runs
// when one of the four is at least as close as the current best -- O(log n) times per query.  Positions past
// the end are clamped to e - 1: re-evaluating a candidate never changes the result (same position, no tie).
template <typename Idx>
__device__ __forceinline__ void nn_scan(const GridViewT<Idx> &g, int s, int e, float qx, float qy, NNResult &r) {
  const int last = e - 1;
  for (int p = s; p < e; p += 4) {
    const int p1 = min(p + 1, last), p2 = min(p + 2, last), p3 = min(p + 3, last);
    const float2 t0 = g.pts[p], t1 = g.pts[p1], t2 = g.pts[p2], t3 = g.pts[p3];
    const float d0 = dist2_rn(qx - t0.x, qy - t0.y), d1 = dist2_rn(qx - t1.x, qy - t1.y);
    const float d2 = dist2_rn(qx - t2.x, qy - t2.y), d3 = dist2_rn(qx - t3.x, qy - t3.y);
    if (fminf(fminf(d0, d1), fminf(d2, d3)) <= r.d2) {
      nn_update(d0, p, r);
      nn_update(d1, p1, r);
      nn_update(d2, p2, r);
      nn_update(d3, p3, r);
    }
  }
}

// rare: among the points of the cell rectangle [xa, xb] x [ya, yb] at exactly distance r.d2, keep the lowest
// original index
template <typename Idx>
static __device__ __noinline__ void nn_resolve_tie_rect(const GridViewT<Idx> &g, int xa, int xb, int ya, int yb, float qx,
                                                        float qy, NNResult &r) {
  if (g.orig == nullptr || r.pos < 0) return;
  int best = r.pos;
  for (int y = ya; y <= yb; ++y)
    for (int p = g.cstart[y * g.nx + xa]; p < g.cstart[y * g.nx + xb + 1]; ++p) {
      const float2 t = g.pts[p];
      if (dist2_rn(qx - t.x, qy - t.y) == r.d2 && g.orig[p] < g.orig[best]) best = p;
    }
  r.pos = best;
  r.tie = 0;
}

template <typename Idx>
__device__ __forceinline__ void nn_resolve_tie(const GridViewT<Idx> &g, int cx, int cy, int k, float qx, float qy, NNResult &r) {
  nn_resolve_tie_rect(g, max(cx - k, 0), min(cx + k, g.nx - 1), max(cy - k, 0), min(cy + k, g.ny - 1), qx, qy, r);
}

// conservative lower bound (squared) on the distance from the query to anything outside the
// (2k+1)^2 block of cells around cell (cx, cy); +inf when the block covers the whole grid
template <typename Idx>
__device__ __forceinline__ float nn_block_bound2(const GridViewT<Idx> &g, float qx, float qy, int cx, int cy, int k) {
  const int x0 = cx - k, x1 = cx + k, y0 = cy - k, y1 = cy + k;
  float bound = INFINITY;
  if (x0 > 0) bound = fminf(bound, qx - (g.ox + (float)x0 * g.cell));
  if (x1 < g.nx - 1) bound = fminf(bound, (g.ox + (float)(x1 + 1) * g.cell) - qx);
  if (y0 > 0) bound = fminf(bound, qy - (g.oy + (float)y0 * g.cell));
  if (y1 < g.ny - 1) bound = fminf(bound, (g.oy + (float)(y1 + 1) * g.cell) - qy);
  if (bound == INFINITY) return INFINITY;
  const float b = bound * (1.0f - 1e-5f) - 1e-6f;  // conservative against float rounding
  return b > 0.f ? b * b * (1.0f - 1e-6f) : 0.f;
}

// scan the whole (2k+1)^2 block as one contiguous point range per cell row
template <typename Idx>
__device__ __forceinline__ void nn_scan_block(const GridViewT<Idx> &g, int cx, int cy, int k, float qx, float qy, NNResult &r) {
  const int xa = max(cx - k, 0), xb = min(cx + k, g.nx - 1);
  for (int y = max(cy - k, 0); y <= min(cy + k, g.ny - 1); ++y)
    nn_scan(g, g.cstart[y * g.nx + xa], g.cstart[y * g.nx + xb + 1], qx, qy, r);
}

// Continue a search that has already scanned the block of radius k_done (k_done = -1: nothing yet), until
//   (a) the nearest neighbour is certain                      -> returns 1, r = exact NN (if any within max_d2)
//   (b) every unscanned point is farther than sqrt(stop_d2)   -> returns 0, r = best so far (NOT exact); the
//       caller only learns "the NN distance exceeds stop_d2"
// The block of cells around the query doubles (k = 1, 2, 4, ...) while nothing has been found, each block
// scanned as row spans (two offset loads per row), so a query far from every point costs O(k) cell
// look-ups; once a candidate at distance d exists, one last block of radius ceil(d / cell) + 1 settles it.
// Re-scanning inner cells is harmless (same candidates, same tie rule).
template <typename Idx>
__device__ __forceinline__ int nn_search(const GridViewT<Idx> &g, float qx, float qy, float max_d2, float stop_d2,
                                         int k_done, NNResult &r) {
  if (g.n <= 0) return 1;
  const int cx = grid_cell_coord(qx, g.ox, g.inv_cell, g.nx), cy = grid_cell_coord(qy, g.oy, g.inv_cell, g.ny);
  const int kmax = max(g.nx, g.ny);
  const float lim = fminf(max_d2, stop_d2);
  int k = k_done;  // block radius scanned so far; -1 = nothing yet (start with the query's own cell, k = 0)
  int exact = -1;
  while (exact < 0) {
    if (k >= 0) {
      const float b2 = nn_block_bound2(g, qx, qy, cx, cy, k);
      if (b2 == INFINITY || b2 > r.d2 || b2 > max_d2) {
        exact = 1;  // nothing outside the block can beat the candidate / be accepted at all
      } else if (b2 > stop_d2) {
        exact = 0;  // NN is farther than the caller cares about
      } else if (r.pos >= 0 && r.d2 <= lim) {
        // a candidate the caller cares about: jump to the smallest block that contains every point at
        // distance <= sqrt(d2) (its bound is re-checked at the top of the loop)
        const float d = sqrtf(r.d2);
        int kk = (int)(d * g.inv_cell * 1.0001f) + 1;
        kk = min(max(kk, k + 1), kmax);
        nn_scan_block(g, cx, cy, kk, qx, qy, r);
        k = kk;
        continue;
      } else if (k >= kmax) {
        exact = 1;
      }
      if (exact >= 0) break;
    }
    k = k < 0 ? 0 : (k == 0 ? 1 : min(2 * k, kmax));
    nn_scan_block(g, cx, cy, k, qx, qy, r);
  }
  if (exact == 1 && r.tie) nn_resolve_tie(g, cx, cy, k, qx, qy, r);
  return exact;
}

// ---------------------------------------------------------------- search that certifies its answer for later
// nn_query plus a lower bound on the distance from the query to every OTHER point: the block of cells it scans is
// at least 3x3, the second-smallest distance met inside it is tracked, and everything outside the last block
// scanned is farther than the block's boundary.  *lb2 receives the square of that bound (min of the two).  The
// ICP keeps it per source point: while the point has moved less than (bound - distance to its match) since this
// search, the match is provably still the unique nearest neighbour and no search is needed (icp.cu).
struct NNResult2 {
  float d2, d2nd;  // smallest and second-smallest distance (over different positions)
  int pos, tie;
};

__device__ __forceinline__ void nn_update2(float d2, int p, NNResult2 &r) {
  if (p == r.pos) return;  // a re-scan of the current best
  if (d2 < r.d2) {
    r.d2nd = r.d2;  // the old best is now the runner-up (it was <= the old runner-up)
    r.d2 = d2, r.pos = p, r.tie = 0;
  } else {
    r.tie |= d2 == r.d2;
    r.d2nd = fminf(r.d2nd, d2);
  }
}

template <typename Idx>
__device__ __forceinline__ void nn_scan_block2(const GridViewT<Idx> &g, int cx, int cy, int k, float qx, float qy, NNResult2 &r) {
  const int xa = max(cx - k, 0), xb = min(cx + k, g.nx - 1);
  for (int y = max(cy - k, 0); y <= min(cy + k, g.ny - 1); ++y) {
    const int s = g.cstart[y * g.nx + xa], e = g.cstart[y * g.nx + xb + 1], last = e - 1;
    for (int p = s; p < e; p += 4) {
      const int p1 = min(p + 1, last), p2 = min(p + 2, last), p3 = min(p + 3, last);
      const float2 t0 = g.pts[p], t1 = g.pts[p1], t2 = g.pts[p2], t3 = g.pts[p3];
      const float d0 = dist2_rn(qx - t0.x, qy - t0.y), d1 = dist2_rn(qx - t1.x, qy - t1.y);
      const float d2 = dist2_rn(qx - t2.x, qy - t2.y), d3 = dist2_rn(qx - t3.x, qy - t3.y);
      if (fminf(fminf(d0, d1), fminf(d2, d3)) <= r.d2nd) {  // (clamped duplicates: same position, idempotent)
        nn_update2(d0, p, r);
        if (p1 != p) nn_update2(d1, p1, r);
        if (p2 != p1) nn_update2(d2, p2, r);
        if (p3 != p2) nn_update2(d3, p3, r);
      }
    }
  }
}

// exact nearest neighbour (accepted only when d2 <= max_d2, like nn_query) + *lb2
template <typename Idx>
__device__ __forceinline__ NNResult nn_query_certified(const GridViewT<Idx> &g, float qx, float qy, float max_d2, float *lb2) {
  NNResult out;
  out.d2 = INFINITY, out.pos = -1, out.tie = 0;
  *lb2 = 0.f;
  if (g.n <= 0) return out;
  const int cx = grid_cell_coord(qx, g.ox, g.inv_cell, g.nx), cy = grid_cell_coord(qy, g.oy, g.inv_cell, g.ny);
  const int kmax = max(g.nx, g.ny);
  NNResult2 r;
  r.d2 = INFINITY, r.d2nd = INFINITY, r.pos = -1, r.tie = 0;
  int k = min(1, kmax);
  nn_scan_block2(g, cx, cy, k, qx, qy, r);
  float b2;
  while (true) {
    b2 = nn_block_bound2(g, qx, qy, cx, cy, k);
    if (b2 == INFINITY || b2 > r.d2 || b2 > max_d2 || k >= kmax) break;  // nothing outside can beat / be accepted
    int kk;
    if (r.pos >= 0 && r.d2 <= max_d2) {
      kk = (int)(sqrtf(r.d2) * g.inv_cell * 1.0001f) + 1;  // the smallest block holding every point that close
      kk = min(max(kk, k + 1), kmax);
    } else {
      kk = min(2 * k, kmax);
    }
    nn_scan_block2(g, cx, cy, kk, qx, qy, r);
    k = kk;
  }
  out.d2 = r.d2, out.pos = r.pos, out.tie = r.tie;
  if (out.tie) nn_resolve_tie(g, cx, cy, k, qx, qy, out);
  *lb2 = out.tie || r.tie ? 0.f : fminf(r.d2nd, b2);  // a tie certifies nothing
  if (out.pos >= 0 && !(out.d2 <= max_d2)) out.pos = -1, out.d2 = INFINITY, *lb2 = 0.f;
  return out;
}

// The seeded search with a certificate of a chosen size.  The seed (last iteration's match) is at distance d from
// the query, so the nearest neighbour lies in the disc of radius d; scanning the cells that overlap the disc of
// radius d + margin settles the nearest neighbour exactly (as nn_query_seeded does) AND shows that every other
// point is farther than min(runner-up met, d + margin).  A small margin keeps the scan as narrow as the plain seeded
// search; the caller sizes it to a few of the point's recent steps, so that one search serves several iterations.
template <typename Idx>
__device__ __forceinline__ NNResult nn_query_seeded_certified(const GridViewT<Idx> &g, float qx, float qy, float max_d2,
                                                              int seed, float margin, float *lb2) {
  const float2 t = g.pts[seed];
  const float d0 = dist2_rn(qx - t.x, qy - t.y);
  if (!(d0 <= max_d2)) return nn_query_certified(g, qx, qy, max_d2, lb2);  // the seed is not acceptable any more
  const float cover = sqrtf(d0) * 1.0001f + 1e-4f * g.cell + margin;  // every point within `cover` gets scanned
  const int xa = grid_cell_coord(qx - cover, g.ox, g.inv_cell, g.nx), xb = grid_cell_coord(qx + cover, g.ox, g.inv_cell, g.nx);
  const int ya = grid_cell_coord(qy - cover, g.oy, g.inv_cell, g.ny), yb = grid_cell_coord(qy + cover, g.oy, g.inv_cell, g.ny);
  NNResult2 r;
  r.d2 = INFINITY, r.d2nd = INFINITY, r.pos = -1, r.tie = 0;
  for (int y = ya; y <= yb; ++y) {
    const int s = g.cstart[y * g.nx + xa], e = g.cstart[y * g.nx + xb + 1], last = e - 1;
    for (int p = s; p < e; p += 4) {
      const int p1 = min(p + 1, last), p2 = min(p + 2, last), p3 = min(p + 3, last);
      const float2 t0 = g.pts[p], t1 = g.pts[p1], t2 = g.pts[p2], t3 = g.pts[p3];
      const float e0 = dist2_rn(qx - t0.x, qy - t0.y), e1 = dist2_rn(qx - t1.x, qy - t1.y);
      const float e2 = dist2_rn(qx - t2.x, qy - t2.y), e3 = dist2_rn(qx - t3.x, qy - t3.y);
      if (fminf(fminf(e0, e1), fminf(e2, e3)) <= r.d2nd) {
        nn_update2(e0, p, r);
        if (p1 != p) nn_update2(e1, p1, r);
        if (p2 != p1) nn_update2(e2, p2, r);
        if (p3 != p2) nn_update2(e3, p3, r);
      }
    }
  }
  NNResult out;
  out.d2 = r.d2, out.pos = r.pos, out.tie = r.tie;  // r.pos >= 0: the seed's own cell is inside the rectangle
  if (out.tie) nn_resolve_tie_rect(g, xa, xb, ya, yb, qx, qy, out);
  const float c = cover * 0.9999f - 2e-4f * g.cell;  // what the rectangle certainly covers (float-safe)
  *lb2 = r.tie ? 0.f : fminf(r.d2nd, c > 0.f ? c * c : 0.f);
  return out;
}

// ---------------------------------------------------------------- warp-cooperative search
// The same search as nn_search, run by ALL 32 lanes of a warp for ONE query (arguments are warp-uniform).  Long
// searches -- a scan point far from every wall has to look at hundreds of candidates -- are the ones a warp should
// share: with one query per lane such a lane keeps its warp busy for the whole scan while the other lanes idle
// (ncu on 2 000 x 20 000-point problems: 7 of 32 lanes active on average, 2-5 in the candidate loops).
// Block scan: the rows of the (2k+1)^2 block are dealt to four groups of eight lanes, each group strides its row's
// contiguous point range; a butterfly picks the closest candidate, and ties (equal float32 distance at different
// positions, within a lane or across lanes) fall back to the exact lowest-original-index rule.  Blocks are nested,
// so the best of the last block scanned is the best of everything scanned.  Result = nn_search's, on every lane.
template <typename Idx>
__device__ __forceinline__ void nn_scan_block_warp(const GridViewT<Idx> &g, int cx, int cy, int k, float qx, float qy,
                                                   NNResult &r) {
  const int lane = threadIdx.x & 31, grp = lane >> 3, sub = lane & 7;
  const int xa = max(cx - k, 0), xb = min(cx + k, g.nx - 1);
  const int ya = max(cy - k, 0), yb = min(cy + k, g.ny - 1);
  NNResult m;
  m.d2 = INFINITY, m.pos = -1, m.tie = 0;
  for (int y = ya + grp; y <= yb; y += 4) {
    const int s = g.cstart[y * g.nx + xa], e = g.cstart[y * g.nx + xb + 1];
    for (int p = s + sub; p < e; p += 8) {
      const float2 t = g.pts[p];
      nn_update(dist2_rn(qx - t.x, qy - t.y), p, m);
    }
  }
  // closest over the warp; a tie is two different positions at the winning distance
  float d = m.d2;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) d = fminf(d, __shfl_xor_sync(0xffffffffu, d, o));
  const unsigned win = __ballot_sync(0xffffffffu, m.d2 == d && m.pos >= 0);
  if (win == 0u) {  // nothing in the block
    r.d2 = INFINITY, r.pos = -1, r.tie = 0;
    return;
  }
  const int first = __ffs(win) - 1;
  const int pos = __shfl_sync(0xffffffffu, m.pos, first);
  const unsigned other = __ballot_sync(0xffffffffu, m.d2 == d && m.pos >= 0 && (m.pos != pos || m.tie));
  r.d2 = d, r.pos = pos, r.tie = other != 0u;
}

// returns 1: r = exact nearest neighbour (if any within max_d2); 0: every point is farther than sqrt(stop_d2)
// (r is then not the NN).  `r` may carry a candidate from an earlier partial scan of the block of radius k_done.
template <typename Idx>
__device__ __forceinline__ int nn_search_warp(const GridViewT<Idx> &g, float qx, float qy, float max_d2, float stop_d2,
                                              int k_done, NNResult &r) {
  if (g.n <= 0) return 1;
  const int cx = grid_cell_coord(qx, g.ox, g.inv_cell, g.nx), cy = grid_cell_coord(qy, g.oy, g.inv_cell, g.ny);
  const int kmax = max(g.nx, g.ny);
  const float lim = fminf(max_d2, stop_d2);
  int k = k_done;
  int exact = -1;
  while (exact < 0) {
    if (k >= 0) {
      const float b2 = nn_block_bound2(g, qx, qy, cx, cy, k);
      if (b2 == INFINITY || b2 > r.d2 || b2 > max_d2) {
        exact = 1;
      } else if (b2 > stop_d2) {
        exact = 0;
      } else if (r.pos >= 0 && r.d2 <= lim) {
        const float d = sqrtf(r.d2);
        int kk = (int)(d * g.inv_cell * 1.0001f) + 1;
        kk = min(max(kk, k + 1), kmax);
        nn_scan_block_warp(g, cx, cy, kk, qx, qy, r);
        k = kk;
        continue;
      } else if (k >= kmax) {
        exact = 1;
      }
      if (exact >= 0) break;
    }
    k = k < 0 ? 0 : (k == 0 ? 1 : min(2 * k, kmax));
    nn_scan_block_warp(g, cx, cy, k, qx, qy, r);
  }
  if (exact == 1 && r.tie) nn_resolve_tie(g, cx, cy, k, qx, qy, r);  // rare; every lane computes the same answer
  return exact;
}

// exact nearest neighbour of (qx,qy); accepted only when d2 <= max_d2
template <typename Idx>
__device__ __forceinline__ NNResult nn_query(const GridViewT<Idx> &g, float qx, float qy, float max_d2) {
  NNResult r;
  r.d2 = INFINITY;
  r.pos = -1;
  r.tie = 0;
  nn_search(g, qx, qy, max_d2, INFINITY, -1, r);
  if (r.pos >= 0 && !(r.d2 <= max_d2)) {
    r.pos = -1;
    r.d2 = INFINITY;
  }
  return r;
}

// Exact nearest neighbour when a good candidate is already known (ICP: the match of the previous iteration).
// The candidate's distance d bounds the answer, so only the cells that overlap the disc of radius d around the
// query can hold the nearest neighbour or a tie with it -- typically 1-4 cells instead of the 3x3 block and its
// successors.  The result (position, distance, tie rule) is the same as nn_query's.
template <typename Idx>
__device__ __forceinline__ NNResult nn_query_seeded(const GridViewT<Idx> &g, float qx, float qy, float max_d2, int seed) {
  const float2 t = g.pts[seed];
  const float d0 = dist2_rn(qx - t.x, qy - t.y);
  if (!(d0 <= max_d2)) return nn_query(g, qx, qy, max_d2);  // the seed itself is not acceptable any more (or NaN)
  const float rad = sqrtf(d0) * 1.0001f + 1e-4f * g.cell;   // conservative against the rounding of d0 and of q -+ rad
  const int xa = grid_cell_coord(qx - rad, g.ox, g.inv_cell, g.nx), xb = grid_cell_coord(qx + rad, g.ox, g.inv_cell, g.nx);
  const int ya = grid_cell_coord(qy - rad, g.oy, g.inv_cell, g.ny), yb = grid_cell_coord(qy + rad, g.oy, g.inv_cell, g.ny);
  NNResult r;
  r.d2 = INFINITY, r.pos = -1, r.tie = 0;
  for (int y = ya; y <= yb; ++y) nn_scan(g, g.cstart[y * g.nx + xa], g.cstart[y * g.nx + xb + 1], qx, qy, r);
  if (r.tie) nn_resolve_tie_rect(g, xa, xb, ya, yb, qx, qy, r);
  return r;  // r.pos >= 0: the seed's own cell is inside the rectangle
}

// ---- k nearest neighbours: a best-knn list per query in ascending (squared distance, original index) order, held
// by the caller as bd[j * stride] (distances), bi[j * stride] (sorted positions), j < knn, and filled ring by ring of
// cells around the query's cell until the knn-th distance is below the bound of everything outside the rings scanned.
// Shared by the surface normals below and the k-nearest-neighbour matcher (grid_knn_query).
constexpr int GRID_KNN_MAX = 16;

// Offer the grid point at sorted position j, at squared distance d2, to the list: k = entries so far (grows to knn),
// kth = the knn-th distance (+inf until knn points are listed).  While the list is not full, d2 must be below +inf.
template <typename Idx, typename B>
__device__ __forceinline__ void knn_offer(const GridViewT<Idx> &g, float d2, int j, int knn, float *bd, B *bi,
                                          int stride, int &k, float &kth) {
  if (d2 > kth) return;
  if (d2 == kth && g.orig[j] > g.orig[bi[(k - 1) * stride]]) return;
  int at = k < knn ? k++ : knn - 1;
  while (at > 0 && (d2 < bd[(at - 1) * stride] || (d2 == bd[(at - 1) * stride] && g.orig[j] < g.orig[bi[(at - 1) * stride]]))) {
    bd[at * stride] = bd[(at - 1) * stride], bi[at * stride] = bi[(at - 1) * stride];
    --at;
  }
  bd[at * stride] = d2, bi[at * stride] = (B)j;
  if (k == knn) kth = bd[(k - 1) * stride];
}

// The ring loop: offer(s, e) gets every ring's cells as contiguous ranges of sorted positions, ring 0 being the cell
// (cx, cy) itself.  Stops when `kth` (the caller's, updated by offer) is below the bound of every unscanned cell, when
// that bound exceeds lim2 (nothing outside can be accepted), or when the rings cover the grid.
template <typename Idx, typename F>
__device__ __forceinline__ void knn_rings(const GridViewT<Idx> &g, float qx, float qy, int cx, int cy, const float &kth,
                                          float lim2, F &&offer) {
  for (int kr = 0;; ++kr) {
    const int x0 = cx - kr, x1 = cx + kr, y0 = cy - kr, y1 = cy + kr;
    for (int y = max(y0, 0); y <= min(y1, g.ny - 1); ++y) {
      const int row = y * g.nx;
      if (y == y0 || y == y1) {
        offer(g.cstart[row + max(x0, 0)], g.cstart[row + min(x1, g.nx - 1) + 1]);
      } else {
        if (x0 >= 0) offer(g.cstart[row + x0], g.cstart[row + x0 + 1]);
        if (x1 <= g.nx - 1) offer(g.cstart[row + x1], g.cstart[row + x1 + 1]);
      }
    }
    const float b2 = nn_block_bound2(g, qx, qy, cx, cy, kr);
    if (b2 == INFINITY || kth < b2 || b2 > lim2) break;
  }
}

// The knn nearest grid points of (qx, qy) among those with squared distance <= max_d2 (nn_query's radius test and
// distance expression; +inf and NaN distances never count, as in nn_query).  Returns how many were listed (<= knn);
// list entry 0 is nn_query's answer.
template <typename Idx, typename B>
__device__ __forceinline__ int grid_knn_query(const GridViewT<Idx> &g, float qx, float qy, float max_d2, int knn,
                                              float *bd, B *bi, int stride) {
  if (g.n <= 0) return 0;
  const int cx = grid_cell_coord(qx, g.ox, g.inv_cell, g.nx), cy = grid_cell_coord(qy, g.oy, g.inv_cell, g.ny);
  int k = 0;
  float kth = INFINITY;
  knn_rings(g, qx, qy, cx, cy, kth, max_d2, [&](int s, int e) {
    for (int j = s; j < e; ++j) {
      const float2 t = g.pts[j];
      const float d2 = dist2_rn(qx - t.x, qy - t.y);
      if (d2 <= max_d2 && d2 < INFINITY) knn_offer(g, d2, j, knn, bd, bi, stride, k, kth);
    }
  });
  return k;
}

// grid_knn_query for a 3-D query (qx, qy, qz) on the grid of the points' x, y: zof(j) is the z of sorted position j, and
// the distance is (dx*dx + dy*dy) + dz*dz, each operation rounded separately.  Adding dz*dz >= 0 never lowers the
// rounded xy distance, so the rings' xy bound still ends the search exactly; a cloud tall in z over a small xy
// footprint puts many points in every cell, and the search then scans those columns whole.
template <typename Idx, typename B, typename Z>
__device__ __forceinline__ int grid_knn_query3(const GridViewT<Idx> &g, float qx, float qy, float qz, const Z &zof,
                                               float max_d2, int knn, float *bd, B *bi, int stride) {
  if (g.n <= 0) return 0;
  const int cx = grid_cell_coord(qx, g.ox, g.inv_cell, g.nx), cy = grid_cell_coord(qy, g.oy, g.inv_cell, g.ny);
  int k = 0;
  float kth = INFINITY;
  knn_rings(g, qx, qy, cx, cy, kth, max_d2, [&](int s, int e) {
    for (int j = s; j < e; ++j) {
      const float2 t = g.pts[j];
      const float d2xy = dist2_rn(qx - t.x, qy - t.y);
      if (!(d2xy <= max_d2) || d2xy > kth) continue;  // the 3-D distance is at least d2xy
      const float dz = qz - zof(j);
      const float d2 = __fadd_rn(d2xy, __fmul_rn(dz, dz));
      if (d2 <= max_d2 && d2 < INFINITY) knn_offer(g, d2, j, knn, bd, bi, stride, k, kth);
    }
  });
  return k;
}

// ---- surface normals (point-to-plane minimiser, icp.yaml:18-19 + a SurfaceNormalDataPointsFilter{knn} on the
// reference; statement: oracle/icp_ref.c orc_surface_normals).  For the grid point at sorted position p: its knn
// nearest grid points (itself included) in ascending (squared distance, original index) order (knn_rings); then mean,
// 2x2 covariance and the unit eigenvector of the smaller eigenvalue in closed form -- every operation a float32
// IEEE operation in the oracle's order, so the normals are bit-identical to the oracle's.
// The scan matcher hands out shared memory that is idle while the normals are computed for the list (stride = CTA
// size, one column per thread): a list in local memory spills past the little L1 that a CTA's shared-memory carve-out
// leaves, so local arrays (stride 1) are only the fallback for CTAs without that room.
template <typename Idx, typename B>
__device__ inline float2 grid_surface_normal(const GridViewT<Idx> &g, int p, int knn, float *bd, B *bi, int stride) {
  const float2 q = g.pts[p];
  const int cx = grid_cell_coord(q.x, g.ox, g.inv_cell, g.nx), cy = grid_cell_coord(q.y, g.oy, g.inv_cell, g.ny);
  int k = 0;
  float kth = INFINITY;
  knn_rings(g, q.x, q.y, cx, cy, kth, INFINITY, [&](int s, int e) {
    for (int j = s; j < e; ++j) {
      const float2 t = g.pts[j];
      knn_offer(g, dist2_rn(q.x - t.x, q.y - t.y), j, knn, bd, bi, stride, k, kth);
    }
  });
  float sx = 0.f, sy = 0.f;
  for (int j = 0; j < k; ++j) sx = __fadd_rn(sx, g.pts[bi[j * stride]].x), sy = __fadd_rn(sy, g.pts[bi[j * stride]].y);
  const float kf = (float)k, mx = __fdiv_rn(sx, kf), my = __fdiv_rn(sy, kf);
  float a = 0.f, b = 0.f, c = 0.f;
  for (int j = 0; j < k; ++j) {
    const float ux = __fsub_rn(g.pts[bi[j * stride]].x, mx), uy = __fsub_rn(g.pts[bi[j * stride]].y, my);
    a = __fadd_rn(a, __fmul_rn(ux, ux)), b = __fadd_rn(b, __fmul_rn(ux, uy)), c = __fadd_rn(c, __fmul_rn(uy, uy));
  }
  a = __fdiv_rn(a, kf), b = __fdiv_rn(b, kf), c = __fdiv_rn(c, kf);
  if (a == 0.f && b == 0.f && c == 0.f) return make_float2(0.f, 0.f);
  const float d = __fmul_rn(0.5f, __fsub_rn(a, c));
  const float r = __fsqrt_rn(__fadd_rn(__fmul_rn(d, d), __fmul_rn(b, b)));
  if (r == 0.f) return make_float2(1.f, 0.f);
  const float ux = d >= 0.f ? __fadd_rn(r, d) : b, uy = d >= 0.f ? b : __fsub_rn(r, d);
  const float len = __fsqrt_rn(__fadd_rn(__fmul_rn(ux, ux), __fmul_rn(uy, uy)));
  return make_float2(-__fdiv_rn(uy, len), __fdiv_rn(ux, len));
}

}  // namespace sfe
