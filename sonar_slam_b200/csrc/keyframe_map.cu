// Keyframe clouds resident on the device (include/sonarfe.h: sfe_keyframe_map_*): SLAM.get_points (slam.py:229-292)
// assembled from an arena of local-coordinate clouds and a per-call table of transforms, then down-sampled by the
// launcher pcl.downsample uses (downsample_run, cloud.cu).
#include <climits>
#include <vector>

#include "stages.cuh"

namespace sfe {

constexpr int KFM_THREADS = 256;
constexpr int64_t KFM_FIRST_CAPACITY = 1 << 16;  // points of a new arena when the caller names none (512 KB)

// Entry table of one gather, in device memory: base [K + 1] output row of every entry's first point (base[K] = N),
// src [K] row of its first point in `from`, key [K], tf [K][6] = {r00, r01, r10, r11, tx, ty}.
struct GatherEntries {
  const int *base, *src;
  const float *key, *tf;
  int K;
};

// One thread per output point: the entry is the last one whose base is <= the point's row (an empty entry shares its
// base with the next one, so the search passes over it).  MOVE: the point moves as numpy's float32
// `points.dot(R.T) + t` (slam_objects.py:196), fma(y, r01, x * r00) + tx -- the convention of assemble_targets_kernel
// (pipeline.cu) and the costmap kernels, pinned against numpy in tests/test_host_logic_cpu.py.  Otherwise the point is
// copied bit for bit.  key_out (optional) receives the entry's key for every point.
template <bool MOVE>
__global__ void __launch_bounds__(KFM_THREADS)
    kfm_gather_kernel(const float2 *__restrict__ from, GatherEntries e, int N, float2 *__restrict__ to,
                      float *__restrict__ key_out) {
  const int i = blockIdx.x * KFM_THREADS + threadIdx.x;
  if (i >= N) return;
  int lo = 0, hi = e.K - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (__ldg(e.base + mid) <= i) lo = mid;
    else hi = mid - 1;
  }
  float2 p = from[(size_t)__ldg(e.src + lo) + (i - __ldg(e.base + lo))];
  if (MOVE) {
    const float *t = e.tf + 6 * (size_t)lo;
    const float r00 = __ldg(t), r01 = __ldg(t + 1), r10 = __ldg(t + 2), r11 = __ldg(t + 3);
    const float tx = __ldg(t + 4), ty = __ldg(t + 5);
    p = make_float2(__fadd_rn(__fmaf_rn(p.y, r01, __fmul_rn(p.x, r00)), tx),
                    __fadd_rn(__fmaf_rn(p.y, r11, __fmul_rn(p.x, r10)), ty));
  }
  to[i] = p;
  if (key_out) key_out[i] = __ldg(e.key + lo);
}

// keys of the down-sampled cloud: the key of the assembled point every output point came from (out_idx)
__global__ void __launch_bounds__(KFM_THREADS)
    kfm_keys_kernel(const float *__restrict__ key_in, const int32_t *__restrict__ idx,
                    const int32_t *__restrict__ count, int N, float *__restrict__ key_out) {
  const int i = blockIdx.x * KFM_THREADS + threadIdx.x;
  if (i < N && i < __ldg(count)) key_out[i] = key_in[__ldg(idx + i)];
}

}  // namespace sfe

using namespace sfe;

// The arena holds every stored cloud once, contiguous, in append order: cloud s is points off[s] .. off[s] + cnt[s] - 1.
// The table (off, cnt) lives on the host: an assemble resolves its entries against it and uploads them resolved.
struct sfe_keyframe_map {
  sfe_ctx *ctx = nullptr;
  int device = 0;
  float2 *arena = nullptr;
  int64_t cap = 0, n_points = 0;
  std::vector<int32_t> off, cnt;
  Buffer ws;   // per-call workspace: entry table, assembled cloud and its keys, down-sample indices
  Buffer out;  // device outputs of the host flavour
};

namespace {

// Room for `more` further points in the arena: doubles it, keeping the stored points (copied device to device on the
// context's stream).
int kfm_reserve(sfe_keyframe_map *km, int64_t more) {
  const int64_t need = km->n_points + more;
  if (need <= km->cap) return SFE_OK;
  int64_t cap = km->cap > 0 ? km->cap : need;  // the first allocation takes what the creator asked for
  while (cap < need) cap *= 2;
  float2 *grown = nullptr;
  SFE_CUDA(cudaMallocAsync((void **)&grown, sizeof(float2) * (size_t)cap, km->ctx->stream));
  if (km->n_points > 0)
    SFE_CUDA(cudaMemcpyAsync(grown, km->arena, sizeof(float2) * (size_t)km->n_points, cudaMemcpyDeviceToDevice,
                             km->ctx->stream));
  if (km->arena) SFE_CUDA(cudaFreeAsync(km->arena, km->ctx->stream));
  km->arena = grown;
  km->cap = cap;
  return SFE_OK;
}

// Uploads a gather table packed on the host as int32 words: base [K + 1] | src [K] | key [K] | tf [6K], followed by
// `extra` words (the assemble's down-sample offsets).  Returns the device copy in *e and the extra words in *extra_dev.
int kfm_upload(sfe_keyframe_map *km, const std::vector<int32_t> &h, int K, size_t at, GatherEntries *e,
               int32_t **extra_dev) {
  const int32_t *d = (const int32_t *)((const char *)km->ws.ptr + at);
  SFE_CUDA(cudaMemcpyAsync((char *)km->ws.ptr + at, h.data(), sizeof(int32_t) * h.size(), cudaMemcpyHostToDevice,
                           km->ctx->stream));
  e->base = d, e->src = d + K + 1;
  e->key = (const float *)(d + 2 * K + 1), e->tf = (const float *)(d + 3 * K + 1);
  e->K = K;
  if (extra_dev) *extra_dev = (int32_t *)(d + 9 * K + 1);
  return SFE_OK;
}

std::vector<int32_t> kfm_table(int K, size_t extra) { return std::vector<int32_t>((size_t)9 * K + 1 + extra, 0); }

// Shared body of the two assemble flavours, after the arguments are checked: N assembled points (> 0), outputs in
// device memory.
int kfm_assemble(sfe_keyframe_map *km, const int32_t *slots, const float *keys, const float *tf, int K, int N,
                 float resolution, float *out_pts, float *out_keys, int32_t *n_out) {
  sfe_ctx *ctx = km->ctx;
  cudaStream_t st = ctx->stream;
  std::vector<int32_t> h = kfm_table(K, 2);
  int32_t *base = h.data(), *src = base + K + 1;
  float *hkey = (float *)(base + 2 * K + 1), *htf = (float *)(base + 3 * K + 1);
  for (int k = 0; k < K; ++k) {
    base[k + 1] = base[k] + km->cnt[slots[k]];
    src[k] = km->off[slots[k]];
    hkey[k] = keys ? keys[k] : 0.f;
    for (int j = 0; j < 6; ++j) htf[6 * k + j] = tf[6 * k + j];
  }
  int32_t *ds_off = base + 9 * K + 1;
  ds_off[0] = 0, ds_off[1] = N;
  // workspace: assembled cloud [N], its keys [N], down-sample indices [N], entry table
  const size_t a_pts = 0, a_key = a_pts + ((sizeof(float2) * (size_t)N + 255) & ~size_t(255));
  const size_t a_idx = a_key + (out_keys ? (sizeof(float) * (size_t)N + 255) & ~size_t(255) : 0);
  const size_t a_tab = a_idx + ((sizeof(int32_t) * (size_t)N + 255) & ~size_t(255));
  int rc = ensure(ctx, km->ws, a_tab + sizeof(int32_t) * h.size(), st);
  if (rc != SFE_OK) return rc;
  char *ws = (char *)km->ws.ptr;
  float2 *asm_pts = (float2 *)(ws + a_pts);
  float *asm_key = out_keys ? (float *)(ws + a_key) : nullptr;
  int32_t *idx = (int32_t *)(ws + a_idx);
  GatherEntries e;
  int32_t *d_off;
  if ((rc = kfm_upload(km, h, K, a_tab, &e, &d_off)) != SFE_OK) return rc;
  const int blocks = (N + KFM_THREADS - 1) / KFM_THREADS;
  kfm_gather_kernel<true><<<blocks, KFM_THREADS, 0, st>>>(km->arena, e, N, asm_pts, asm_key);
  SFE_CUDA(cudaGetLastError());
  ctx->launches++;
  rc = downsample_run(ctx, st, {(const float *)asm_pts, d_off, nullptr, N}, 1, 2, resolution, out_pts, idx, n_out,
                      DS_ANY_SIZE, SCR_CLOUD, WORK_DS);
  if (rc != SFE_OK) return rc;
  if (out_keys) {
    kfm_keys_kernel<<<blocks, KFM_THREADS, 0, st>>>(asm_key, idx, n_out, N, out_keys);
    SFE_CUDA(cudaGetLastError());
    ctx->launches++;
  }
  return SFE_OK;
}

// Argument checks of both assemble flavours, before any device work; *N receives the assembled point count.
int kfm_check_assemble(const sfe_keyframe_map *km, const int32_t *slots, const float *keys, const float *tf, int K,
                       float resolution, int capacity, const void *out_pts, const void *out_keys, const void *n_out,
                       const char *what, int *N) {
  SFE_REQUIRE(km != nullptr, "%s: null map", what);
  SFE_REQUIRE(K >= 0, "%s: negative entry count %d", what, K);
  SFE_REQUIRE(resolution > 0.f, "%s: resolution must be positive (got %g)", what, (double)resolution);
  SFE_REQUIRE(n_out != nullptr, "%s: null count pointer", what);
  SFE_REQUIRE(K == 0 || (slots && tf), "%s: null entry table", what);
  SFE_REQUIRE(!out_keys || K == 0 || keys, "%s: keys requested without entry keys", what);
  const int n_clouds = (int)km->cnt.size();
  int64_t total = 0;
  for (int k = 0; k < K; ++k) {
    SFE_REQUIRE(slots[k] >= 0 && slots[k] < n_clouds, "%s: entry %d names slot %d (the map holds %d clouds)", what, k,
                slots[k], n_clouds);
    total += km->cnt[slots[k]];
  }
  SFE_REQUIRE(total <= INT_MAX - 1, "%s: %lld assembled points exceed %d", what, (long long)total, INT_MAX - 1);
  if (total > capacity) {
    set_error("%s: %lld assembled points exceed the output capacity %d", what, (long long)total, capacity);
    return SFE_ERR_CAPACITY;
  }
  SFE_REQUIRE(total == 0 || out_pts, "%s: null output pointer", what);
  *N = (int)total;
  return SFE_OK;
}

// Appends n clouds whose counts the host knows (clamped rows of `from`, cloud c at row src[c]) by one gather.
int kfm_append(sfe_keyframe_map *km, const float2 *from, const int64_t *src, const int32_t *counts, int n,
               int32_t *slots_host, const char *what) {
  int64_t total = 0;
  for (int c = 0; c < n; ++c) {
    SFE_REQUIRE(counts[c] >= 0, "%s: cloud %d has a negative count %d", what, c, counts[c]);
    total += counts[c];
  }
  SFE_REQUIRE(km->n_points + total <= INT_MAX - 1, "%s: the map would hold %lld points (at most %d)", what,
              (long long)(km->n_points + total), INT_MAX - 1);
  SFE_REQUIRE((int64_t)km->cnt.size() + n <= INT_MAX - 1, "%s: too many clouds", what);
  int rc = kfm_reserve(km, total);
  if (rc != SFE_OK) return rc;
  const int first = (int)km->cnt.size();
  if (total > 0) {
    std::vector<int32_t> h = kfm_table(n, 0);
    int32_t *base = h.data(), *hs = base + n + 1;
    for (int c = 0; c < n; ++c) {
      base[c + 1] = base[c] + counts[c];
      hs[c] = (int32_t)src[c];
    }
    rc = ensure(km->ctx, km->ws, sizeof(int32_t) * h.size(), km->ctx->stream);
    if (rc != SFE_OK) return rc;
    GatherEntries e;
    if ((rc = kfm_upload(km, h, n, 0, &e, nullptr)) != SFE_OK) return rc;
    kfm_gather_kernel<false><<<(int)((total + KFM_THREADS - 1) / KFM_THREADS), KFM_THREADS, 0, km->ctx->stream>>>(
        from, e, (int)total, km->arena + km->n_points, nullptr);
    SFE_CUDA(cudaGetLastError());
    km->ctx->launches++;
  }
  for (int c = 0; c < n; ++c) {
    km->off.push_back((int32_t)km->n_points);
    km->cnt.push_back(counts[c]);
    km->n_points += counts[c];
    if (slots_host) slots_host[c] = first + c;
  }
  return SFE_OK;
}

}  // namespace

extern "C" {

int sfe_keyframe_map_create(sfe_ctx *ctx, int initial_points, sfe_keyframe_map **out) {
  SFE_REQUIRE(ctx && out, "sfe_keyframe_map_create: null argument");
  SFE_REQUIRE(initial_points >= 0, "sfe_keyframe_map_create: negative capacity %d", initial_points);
  *out = nullptr;
  SFE_CUDA(cudaSetDevice(ctx->device));
  sfe_keyframe_map *km = new sfe_keyframe_map();
  km->ctx = ctx, km->device = ctx->device;
  km->cap = 0;
  int rc = kfm_reserve(km, initial_points > 0 ? initial_points : KFM_FIRST_CAPACITY);
  if (rc != SFE_OK) {
    delete km;
    return rc;
  }
  *out = km;
  return SFE_OK;
}

void sfe_keyframe_map_destroy(sfe_keyframe_map *km) {
  if (!km) return;
  cudaSetDevice(km->device);
  // cudaFree waits for the device, so the context's enqueued work on these blocks has finished; the context itself is
  // not touched (it may already be gone)
  if (km->arena) cudaFree(km->arena);
  if (km->ws.ptr) cudaFree(km->ws.ptr);
  if (km->out.ptr) cudaFree(km->out.ptr);
  delete km;
}

int sfe_keyframe_map_size(const sfe_keyframe_map *km, int *n_clouds, int64_t *n_points) {
  SFE_REQUIRE(km != nullptr, "sfe_keyframe_map_size: null map");
  if (n_clouds) *n_clouds = (int)km->cnt.size();
  if (n_points) *n_points = km->n_points;
  return SFE_OK;
}

int sfe_keyframe_map_append_host(sfe_keyframe_map *km, const float *pts_host, const int32_t *counts_host, int n_clouds,
                                 int32_t *slots_host) {
  SFE_REQUIRE(km != nullptr, "sfe_keyframe_map_append_host: null map");
  SFE_REQUIRE(n_clouds >= 0, "sfe_keyframe_map_append_host: negative cloud count %d", n_clouds);
  if (n_clouds == 0) return SFE_OK;
  SFE_REQUIRE(counts_host != nullptr, "sfe_keyframe_map_append_host: null counts");
  int64_t total = 0;
  std::vector<int64_t> src((size_t)n_clouds);
  for (int c = 0; c < n_clouds; ++c) {
    SFE_REQUIRE(counts_host[c] >= 0, "sfe_keyframe_map_append_host: cloud %d has a negative count %d", c,
                counts_host[c]);
    src[c] = km->n_points + total;
    total += counts_host[c];
  }
  SFE_REQUIRE(total == 0 || pts_host, "sfe_keyframe_map_append_host: null points");
  SFE_REQUIRE(km->n_points + total <= INT_MAX - 1, "sfe_keyframe_map_append_host: the map would hold %lld points (at "
              "most %d)", (long long)(km->n_points + total), INT_MAX - 1);
  SFE_CUDA(cudaSetDevice(km->device));
  int rc = kfm_reserve(km, total);
  if (rc != SFE_OK) return rc;
  if (total > 0)
    SFE_CUDA(cudaMemcpyAsync(km->arena + km->n_points, pts_host, sizeof(float2) * (size_t)total,
                             cudaMemcpyHostToDevice, km->ctx->stream));
  const int first = (int)km->cnt.size();
  for (int c = 0; c < n_clouds; ++c) {
    km->off.push_back((int32_t)src[c]);
    km->cnt.push_back(counts_host[c]);
    if (slots_host) slots_host[c] = first + c;
  }
  km->n_points += total;
  // the copy reads pageable (or the caller's) host memory: done before returning, so the caller may reuse it
  SFE_CUDA(cudaStreamSynchronize(km->ctx->stream));
  return SFE_OK;
}

int sfe_keyframe_map_append_dev(sfe_keyframe_map *km, const float *cloud_xy_dev, const int32_t *cloud_count_dev,
                                int cloud_stride, int n_clouds, int32_t *slots_host, int32_t *counts_host) {
  SFE_REQUIRE(km != nullptr, "sfe_keyframe_map_append_dev: null map");
  SFE_REQUIRE(n_clouds >= 0 && cloud_stride > 0, "sfe_keyframe_map_append_dev: bad sizes (%d clouds, stride %d)",
              n_clouds, cloud_stride);
  SFE_REQUIRE((int64_t)n_clouds * cloud_stride <= INT_MAX, "sfe_keyframe_map_append_dev: %d clouds of stride %d",
              n_clouds, cloud_stride);
  if (n_clouds == 0) return SFE_OK;
  SFE_REQUIRE(cloud_xy_dev && cloud_count_dev, "sfe_keyframe_map_append_dev: null cloud pointer");
  SFE_CUDA(cudaSetDevice(km->device));
  std::vector<int32_t> cnt((size_t)n_clouds);
  SFE_CUDA(cudaMemcpyAsync(cnt.data(), cloud_count_dev, sizeof(int32_t) * cnt.size(), cudaMemcpyDeviceToHost,
                           km->ctx->stream));
  SFE_CUDA(cudaStreamSynchronize(km->ctx->stream));
  std::vector<int64_t> src((size_t)n_clouds);
  for (int c = 0; c < n_clouds; ++c) {
    // a frame whose cloud overflowed the front end's capacity holds its first cloud_stride points (as its window
    // assembly reads it, assemble_targets_kernel)
    cnt[c] = cnt[c] < cloud_stride ? cnt[c] : cloud_stride;
    src[c] = (int64_t)c * cloud_stride;
  }
  int rc = kfm_append(km, (const float2 *)cloud_xy_dev, src.data(), cnt.data(), n_clouds, slots_host,
                      "sfe_keyframe_map_append_dev");
  if (rc != SFE_OK) return rc;
  if (counts_host)
    for (int c = 0; c < n_clouds; ++c) counts_host[c] = cnt[c];
  return SFE_OK;
}

int sfe_keyframe_map_assemble_dev(sfe_keyframe_map *km, const int32_t *slots_host, const float *keys_host,
                                  const float *transforms_host, int n_entries, float resolution, int capacity,
                                  float *out_pts_dev, float *out_keys_dev, int32_t *n_out_dev) {
  int N = 0;
  int rc = kfm_check_assemble(km, slots_host, keys_host, transforms_host, n_entries, resolution, capacity, out_pts_dev,
                              out_keys_dev, n_out_dev, "sfe_keyframe_map_assemble_dev", &N);
  if (rc != SFE_OK) return rc;
  SFE_CUDA(cudaSetDevice(km->device));
  if (N == 0) {
    SFE_CUDA(cudaMemsetAsync(n_out_dev, 0, sizeof(int32_t), km->ctx->stream));
    return SFE_OK;
  }
  return kfm_assemble(km, slots_host, keys_host, transforms_host, n_entries, N, resolution, out_pts_dev, out_keys_dev,
                      n_out_dev);
}

int sfe_keyframe_map_assemble_host(sfe_keyframe_map *km, const int32_t *slots_host, const float *keys_host,
                                   const float *transforms_host, int n_entries, float resolution, int capacity,
                                   float *out_pts_host, float *out_keys_host, int32_t *n_out) {
  int N = 0;
  int rc = kfm_check_assemble(km, slots_host, keys_host, transforms_host, n_entries, resolution, capacity, out_pts_host,
                              out_keys_host, n_out, "sfe_keyframe_map_assemble_host", &N);
  if (rc != SFE_OK) return rc;
  *n_out = 0;
  if (N == 0) return SFE_OK;
  SFE_CUDA(cudaSetDevice(km->device));
  const size_t a_key = (sizeof(float2) * (size_t)N + 255) & ~size_t(255);
  const size_t a_cnt = a_key + (out_keys_host ? (sizeof(float) * (size_t)N + 255) & ~size_t(255) : 0);
  if ((rc = ensure(km->ctx, km->out, a_cnt + sizeof(int32_t), km->ctx->stream)) != SFE_OK) return rc;
  char *o = (char *)km->out.ptr;
  float *d_keys = out_keys_host ? (float *)(o + a_key) : nullptr;
  int32_t *d_n = (int32_t *)(o + a_cnt);
  rc = kfm_assemble(km, slots_host, keys_host, transforms_host, n_entries, N, resolution, (float *)o, d_keys, d_n);
  if (rc != SFE_OK) return rc;
  int32_t M = 0;
  SFE_CUDA(cudaMemcpyAsync(&M, d_n, sizeof(int32_t), cudaMemcpyDeviceToHost, km->ctx->stream));
  SFE_CUDA(cudaStreamSynchronize(km->ctx->stream));
  SFE_CUDA(cudaMemcpyAsync(out_pts_host, o, sizeof(float2) * (size_t)M, cudaMemcpyDeviceToHost, km->ctx->stream));
  if (out_keys_host)
    SFE_CUDA(cudaMemcpyAsync(out_keys_host, d_keys, sizeof(float) * (size_t)M, cudaMemcpyDeviceToHost,
                             km->ctx->stream));
  SFE_CUDA(cudaStreamSynchronize(km->ctx->stream));
  *n_out = M;
  return SFE_OK;
}

}  // extern "C"
