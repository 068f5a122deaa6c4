// SurfaceNormalDataPointsFilter on the reading cloud of an ICP call (icp.cu's icp_filter_side, SFE_ICP_DATA_NORMALS)
// and alone (sfe_icp_surface_normals_dev).  Statement: oracle/shadow_ref.c.
//
// Every point gets the normal point-to-plane forms for reference points: the cloud is centred on its mean (the
// sequential float32 sum icp_kernel takes), and grid_surface_normal lists each point's knn nearest points in (squared
// distance, index) order and applies the closed form.  Neither step depends on the grid's geometry, so both paths below
// give the same normals.
//   - Clouds of up to SNRM_CTA_MAX points: one CTA per cloud at a time (snrm_cta_kernel), the grid built in shared
//     memory, the knn lists in shared memory too (one column per thread), one thread per sorted position.
//   - Larger clouds: map grids in global memory (map_build, which forms the normals per sorted position), scattered back
//     to point order by snrm_scatter_kernel.
#include <algorithm>

#include "grid.cuh"
#include "stages.cuh"

namespace sfe {

constexpr int SNRM_THREADS = 256;
constexpr int SNRM_CTA_MAX = 4096;  // the largest cloud of the one-CTA path

__device__ __forceinline__ int snrm_count(const PackedClouds &in, int c) {
  return in.cnt ? in.cnt[c] : in.off[c + 1] - in.off[c];
}

// Shared memory of snrm_cta_kernel for clouds of up to cap points: sorted points, original indices, the cell table of
// max_cells cells, the knn lists
static size_t snrm_cta_smem(int cap, int max_cells, int knn) {
  return sizeof(float2) * (size_t)cap + sizeof(uint32_t) * (size_t)((max_cells + 2) / 2 + 1) +
         ((sizeof(uint16_t) * (size_t)cap + 3) & ~size_t(3)) + (sizeof(float) + sizeof(uint16_t)) * SNRM_THREADS * knn;
}

// Clouds of 1 .. limit points (and at most in.n_max): every point's normal at out + in.off[c] + its index
__global__ void __launch_bounds__(SNRM_THREADS) snrm_cta_kernel(const PackedClouds in, int n_clouds, int knn, int limit,
                                                                int max_cells, float2 *out) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  __shared__ float mean[2];
  __shared__ float4 bred[SNRM_THREADS / 32];
  __shared__ int scan[33];
  __shared__ GridView gs;
  const int cap = min(in.n_max, limit);
  float2 *sorted = reinterpret_cast<float2 *>(smem_raw);
  uint32_t *cells = reinterpret_cast<uint32_t *>(sorted + cap);
  uint16_t *orig = reinterpret_cast<uint16_t *>(cells + (max_cells + 2) / 2 + 1);
  float *bd = reinterpret_cast<float *>(smem_raw + ((reinterpret_cast<unsigned char *>(orig + cap) - smem_raw + 3) & ~3));
  uint16_t *bi = reinterpret_cast<uint16_t *>(bd + SNRM_THREADS * knn);
  const int tid = threadIdx.x, nthr = blockDim.x;
  for (int c = blockIdx.x; c < n_clouds; c += gridDim.x) {
    const int n = snrm_count(in, c);
    if (n <= 0 || n > cap) continue;  // (empty, too large for the capacity, or the map path's)
    const float *src = in.pts + 2 * (size_t)in.off[c];
    __syncthreads();  // the previous cloud fully retired
    if (tid < 64) {   // warps 0 and 1: x and y
      const float sum = seq_sum_warp_global(src + (tid >> 5), n, 2);
      if ((tid & 31) == 0) mean[tid >> 5] = __fdiv_rn(sum, (float)n);
    }
    __syncthreads();
    const float mx = mean[0], my = mean[1];
    float4 bnd = make_float4(INFINITY, INFINITY, -INFINITY, -INFINITY);
    for (int i = tid; i < n; i += nthr) {
      const float x = src[2 * i] - mx, y = src[2 * i + 1] - my;
      bnd.x = fminf(bnd.x, x), bnd.y = fminf(bnd.y, y), bnd.z = fmaxf(bnd.z, x), bnd.w = fmaxf(bnd.w, y);
    }
    bnd = block_bounds(bnd, bred);
    if (tid == 0) grid_geometry(n, bnd.x, bnd.y, bnd.z, bnd.w, 0.05f, gs, max_cells);
    __syncthreads();
    GridView g = gs;
    grid_build(src, 2, n, mx, my, g, sorted, cells, orig, scan);
    float2 *o = out + in.off[c];
    for (int j = tid; j < n; j += nthr) o[orig[j]] = grid_surface_normal(g, j, knn, bd + tid, bi + tid, nthr);
  }
}

// The map path's normals, by sorted position, to point order: slot s's points lie at cstart[s][0] .. cstart[s][nx * ny]
__global__ void snrm_scatter_kernel(const PackedClouds in, const MapArgs m, const int *n_slots, const int *slot_tgt,
                                    float2 *out) {
  const int s = blockIdx.y;
  if (s >= *n_slots) return;
  const int *cs = m.cstart + (size_t)s * m.cell_cap;
  const MapGrid g = m.grid[s];
  const int e = cs[g.nx * g.ny];
  float2 *o = out + in.off[slot_tgt[s]];
  for (int i = cs[0] + blockIdx.x * blockDim.x + threadIdx.x; i < e; i += gridDim.x * blockDim.x) o[m.orig[i]] = m.nrm[i];
}

// The counts map_build sees: clouds above n_max are not read (0 points)
__global__ void snrm_counts_kernel(const PackedClouds in, int n_clouds, int *cnt) {
  for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < n_clouds; c += gridDim.x * blockDim.x) {
    const int n = snrm_count(in, c);
    cnt[c] = n <= in.n_max ? n : 0;
  }
}

int surface_normals_ws(int n_clouds, int n_max, size_t *bytes) {
  *bytes = n_max > (MAP_CLASS_ALL ? 0 : SNRM_CTA_MAX) ? sizeof(int) * (size_t)n_clouds : 0;
  return SFE_OK;
}

int surface_normals_run(sfe_ctx *ctx, cudaStream_t st, const PackedClouds &in, int n_clouds, int knn, void *ws,
                        float2 *out_nrm) {
  SFE_REQUIRE(knn >= 3 && knn <= GRID_KNN_MAX, "surface normals: knn %d (3..%d)", knn, GRID_KNN_MAX);
  if (n_clouds <= 0 || in.n_max <= 0) return SFE_OK;
  const int limit = MAP_CLASS_ALL ? 0 : SNRM_CTA_MAX;
  const int cap = std::min(in.n_max, limit);
  if (cap > 0) {
    const int max_cells = std::min(std::max(cap + cap / 2, 256), GRID_MAX_CELLS);
    const size_t smem = snrm_cta_smem(cap, max_cells, knn);
    int per_sm;
    int rc = ctas_per_sm(ctx, (const void *)snrm_cta_kernel, SNRM_THREADS, smem, &per_sm);
    if (rc != SFE_OK) return rc;
    snrm_cta_kernel<<<std::min(n_clouds, ctx->sm_count * per_sm), SNRM_THREADS, smem, st>>>(in, n_clouds, knn, limit,
                                                                                          max_cells, out_nrm);
    SFE_CUDA(cudaGetLastError());
    ctx->launches++;
  }
  if (in.n_max > limit) {
    int *cnt = (int *)ws;
    snrm_counts_kernel<<<std::min((n_clouds + 255) / 256, ctx->sm_count), 256, 0, st>>>(in, n_clouds, cnt);
    SFE_CUDA(cudaGetLastError());
    ctx->launches++;
    MapWs w{};
    const int rc = map_build(ctx, st, {in.pts, in.off, cnt, in.n_max}, 2, nullptr, n_clouds, limit, n_clouds, true, true,
                             knn, w);
    if (rc != SFE_OK) return rc;
    const int bpc = std::max(1, std::min((in.n_max + 4 * 256 - 1) / (4 * 256), 256));
    snrm_scatter_kernel<<<dim3(bpc, n_clouds), 256, 0, st>>>(in, w.args(), w.n_slots, w.slot_tgt, out_nrm);
    SFE_CUDA(cudaGetLastError());
    ctx->launches++;
  }
  return SFE_OK;
}

}  // namespace sfe
