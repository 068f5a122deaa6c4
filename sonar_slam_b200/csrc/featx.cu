// Polar -> Cartesian feature cloud (sm_90a).
//
// Replaces the numeric body of FeatureExtraction.callback between the CFAR detector and the
// point-cloud filters, bruce_slam/src/bruce_slam/feature_extraction.py:231-238:
//
//     peaks = cv2.remap(peaks, self.map_x, self.map_y, cv2.INTER_LINEAR)   (:231)
//     locs  = np.c_[np.nonzero(peaks)]                                      (:232)
//     x, y  = pixel -> metres ; points = np.column_stack((y, x))            (:235-238)
//
// cv2.remap of an 8-bit image with float maps runs in fixed point (OpenCV imgwarp.cpp): the
// sampling coordinates are quantised to 1/32 px (cvRound = round-half-even), the integer part is
// saturated to int16, and the four bilinear taps are weighted by 15-bit integers that for 1/32
// fractions are exactly 32*(32-fx)(32-fy), 32*fx(32-fy), 32*(32-fx)fy, 32*fx*fy; the result is
// (sum + 2^14) >> 15 with taps outside the image contributing 0.  For a 0/1 mask a Cartesian pixel is
// therefore non-zero  <=>  sum over set taps of (weight/32) >= 512.  That integer rule is evaluated
// here per Cartesian pixel from a per-geometry table (8 B/pixel, built once on the host from the same
// float32 maps the reference builds in generate_map_xy :134-173), against the polar mask held as a
// bit plane in shared memory; detections are compacted in row-major order (what np.nonzero returns)
// and converted to metres with the reference's float64 expressions.
//
// One CTA handles FPB frames per pass over the table so the table is read once per FPB frames.
#include <algorithm>
#include <vector>

#include "stages.cuh"

namespace sfe {

__device__ __forceinline__ int block_exclusive_scan_fx(int v, int *warp_sums /* [33] */, int &total) {
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
    const int w = lane < nwarps ? warp_sums[lane] : 0;
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

struct __align__(8) MapEntry {
  int16_t ix, iy;   // top-left tap (saturated like cv::saturate_cast<short>)
  uint8_t fx, fy;   // 1/32-pixel fractions
  uint8_t flags;    // bit 0: the pixel can reach weight 512 with in-image taps
                    // bit 1: the map coordinate is NaN, infinite or |map * 32| >= 1e9: cv2.remap gives 0 there
  uint8_t pad;
};
constexpr uint8_t MAP_FIRES = 1, MAP_DEAD = 2;

constexpr int FX_THREADS = 1024;
constexpr int FXS_THREADS = 512;  // detection-driven variant

// cv2.remap's fixed-point bilinear rule for one Cartesian pixel against a 0/1 polar bit plane
__device__ __forceinline__ bool cart_pixel_fires(const MapEntry e, const uint32_t *__restrict__ sb, int R, int B, int wpr) {
  const int ix = e.ix, iy = e.iy, fx = e.fx, fy = e.fy;
  const bool x0 = (unsigned)ix < (unsigned)B, x1 = (unsigned)(ix + 1) < (unsigned)B;
  const bool y0 = (unsigned)iy < (unsigned)R, y1 = (unsigned)(iy + 1) < (unsigned)R;
  const int w00 = (x0 && y0) ? (32 - fx) * (32 - fy) : 0, w01 = (x1 && y0) ? fx * (32 - fy) : 0;
  const int w10 = (x0 && y1) ? (32 - fx) * fy : 0, w11 = (x1 && y1) ? fx * fy : 0;
  const int cx0 = x0 ? ix : 0, cx1 = x1 ? ix + 1 : 0, cy0 = y0 ? iy : 0, cy1 = y1 ? iy + 1 : 0;
  const int sum = w00 * (int)((sb[cy0 * wpr + (cx0 >> 5)] >> (cx0 & 31)) & 1u) +
                  w01 * (int)((sb[cy0 * wpr + (cx1 >> 5)] >> (cx1 & 31)) & 1u) +
                  w10 * (int)((sb[cy1 * wpr + (cx0 >> 5)] >> (cx0 & 31)) & 1u) +
                  w11 * (int)((sb[cy1 * wpr + (cx1 >> 5)] >> (cx1 & 31)) & 1u);
  return sum >= 512;
}

// (row, col) and metres of one fired pixel from the per-geometry tables: the pixel -> metres expressions depend on
// the column alone (lateral) and on the row alone (forward), so sfe_maps_create evaluates them once per column /
// row with the reference's float64 operations and the kernels only look them up.
__device__ __forceinline__ void cart_emit_lut(int pix, int cols, float inv_cols, const float *__restrict__ metres,
                                              int32_t *ij, float *xy, size_t o) {
  int row = __float2int_rz(__fmul_rn((float)pix, inv_cols));
  int col = pix - row * cols;
  if (col < 0) --row, col += cols;           // the float quotient is within one of the exact one (pix < 2^24)
  else if (col >= cols) ++row, col -= cols;
  *reinterpret_cast<int2 *>(ij + o) = make_int2(row, col);
  *reinterpret_cast<float2 *>(xy + o) = make_float2(metres[cols + row], metres[col]);
}

__device__ __forceinline__ void cart_emit(int pix, int cols, int rows, double width, double height, int32_t *ij,
                                          float *xy, size_t o) {
  const int row = pix / cols, col = pix - row * cols;
  ij[o] = row;
  ij[o + 1] = col;
  // feature_extraction.py:235-237, float64, operation by operation (no contraction)
  double x = __dsub_rn((double)col, __ddiv_rn((double)cols, 2.0));
  x = __dmul_rn(__ddiv_rn(x, __ddiv_rn((double)cols, 2.0)), __ddiv_rn(width, 2.0));
  x = __dmul_rn(-1.0, x);
  double y = __dmul_rn(-1.0, __ddiv_rn((double)row, (double)rows));
  y = __dadd_rn(__dmul_rn(y, height), height);
  xy[o] = (float)y;
  xy[o + 1] = (float)x;
}

// Detection-driven variant.  A Cartesian pixel can only be non-zero if one of its four taps is a
// detection, and detections are sparse (~0.5 % of the polar image), so instead of testing all rows*cols
// pixels the CTA walks the set bits of the polar plane and, for each, the precomputed list of Cartesian
// pixels that sample it; firing pixels are marked in a Cartesian bit plane in shared memory, which is then
// scanned once, in order, to emit the points (np.nonzero order).  One CTA per frame.
__global__ void __launch_bounds__(FXS_THREADS)
    cart_scatter_kernel(const MapEntry *__restrict__ tab, const int32_t *__restrict__ inv_off,
                        const int32_t *__restrict__ inv_idx, int npix, int cols, int rows, int R, int B, int wpr,
                        const uint8_t *__restrict__ mask, const uint32_t *__restrict__ bits, int F, int cap,
                        const float *__restrict__ metres, int32_t *__restrict__ ij, float *__restrict__ xy,
                        int32_t *__restrict__ count, int *__restrict__ next) {
  extern __shared__ uint32_t fxs_smem[];
  __shared__ int scan_s[36], next_s;
  const float inv_cols = 1.0f / (float)cols;
  const int words = R * wpr, cwords = (npix + 31) / 32;
  uint32_t *sb = fxs_smem;           // polar bit plane
  uint32_t *cm = fxs_smem + words;   // Cartesian bit plane
  uint32_t *doff = fxs_smem + words + cwords;  // [(words + 1) / 2]: rank of the first set bit of every pair of polar words
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarps = FXS_THREADS / 32;

  for (int f = blockIdx.x; f < F; f = next_work_item(next, &next_s)) {
    __syncthreads();
    if (bits != nullptr) {
      const uint32_t *src = bits + (size_t)f * words;
      for (int w = tid; w < words; w += FXS_THREADS) sb[w] = src[w];
    } else {
      const uint8_t *src = mask + (size_t)f * R * B;
      for (int w = tid; w < words; w += FXS_THREADS) {
        const int r = w / wpr, q = w - r * wpr;
        const uint8_t *row = src + (size_t)r * B + q * 32;
        const int nb = min(32, B - q * 32);
        uint32_t word = 0;
        for (int t = 0; t < nb; ++t) word |= (row[t] ? 1u : 0u) << t;
        sb[w] = word;
      }
    }
    for (int w = tid; w < cwords; w += FXS_THREADS) cm[w] = 0;
    __syncthreads();
    // ---- detections -> candidate pixels.  The set bits of the polar plane are enumerated DENSELY: a block scan
    //      gives every pair of words the rank of its first set bit (`doff`), and thread d then finds detection d by
    //      a binary search over those ranks plus a find-n-th-set-bit -- every lane of every warp has a detection
    //      (walking the bits of one's own words left 4-6 lanes of 32 busy: set bits cluster in a few words).
    //      Each detection walks its inverse list with its own chain of loads in flight.
    {
      const int npair = (words + 1) / 2;
      const int per = (npair + FXS_THREADS - 1) / FXS_THREADS;
      const int k0 = min(tid * per, npair), k1 = min(k0 + per, npair);
      auto pair_count = [&](int k) { return __popc(sb[2 * k]) + (2 * k + 1 < words ? __popc(sb[2 * k + 1]) : 0); };
      int mycount = 0;
      for (int k = k0; k < k1; ++k) mycount += pair_count(k);
      int total;
      int pos = block_exclusive_scan_fx(mycount, scan_s, total);
      for (int k = k0; k < k1; ++k) {
        doff[k] = (uint32_t)pos;
        pos += pair_count(k);
      }
      __syncthreads();
      for (int d = tid; d < total; d += FXS_THREADS) {
        int lo = 0, hi = npair;  // last pair whose first rank is <= d (pairs without bits share their successor's rank)
        while (hi - lo > 1) {
          const int mid = (lo + hi) >> 1;
          if (doff[mid] <= (uint32_t)d) lo = mid; else hi = mid;
        }
        int r = d - (int)doff[lo], w = 2 * lo;
        const int c0 = __popc(sb[w]);
        if (r >= c0) r -= c0, ++w;
        const int bit = __fns(sb[w], 0, r + 1);
        const int y = w / wpr, x = (w - y * wpr) * 32 + bit;
        if (x >= B) continue;  // padding bits of the last word of a row
        const int q = y * B + x;
        const int s0 = inv_off[q], e0 = inv_off[q + 1];
        for (int t = s0; t < e0; ++t) {
          const int pix = inv_idx[t];
          if (cart_pixel_fires(tab[pix], sb, R, B, wpr)) atomicOr(&cm[pix >> 5], 1u << (pix & 31));
        }
      }
    }
    __syncthreads();
    // ---- ordered emission (np.nonzero order), dense in the same way: ranks of the Cartesian word pairs by a block
    //      scan (they go into the polar plane's memory, dead by now), then thread j finds point j and writes
    //      (row, col) and metres straight to slot j.
    {
      const int npair = (cwords + 1) / 2;
      const int per = (npair + FXS_THREADS - 1) / FXS_THREADS;
      const int k0 = min(tid * per, npair), k1 = min(k0 + per, npair);
      auto pair_count = [&](int k) { return __popc(cm[2 * k]) + (2 * k + 1 < cwords ? __popc(cm[2 * k + 1]) : 0); };
      int mine_cnt = 0;
      for (int k = k0; k < k1; ++k) mine_cnt += pair_count(k);
      int total;
      int idx = block_exclusive_scan_fx(mine_cnt, scan_s, total);
      uint32_t *woff = sb;  // [npair] <= [words]: checked by the host (else the dense kernel is used)
      for (int k = k0; k < k1; ++k) {
        woff[k] = (uint32_t)idx;
        idx += pair_count(k);
      }
      __syncthreads();
      const int n_out = min(total, cap);
      for (int j = tid; j < n_out; j += FXS_THREADS) {
        int lo = 0, hi = npair;
        while (hi - lo > 1) {
          const int mid = (lo + hi) >> 1;
          if (woff[mid] <= (uint32_t)j) lo = mid; else hi = mid;
        }
        int r = j - (int)woff[lo], w = 2 * lo;
        const int c0 = __popc(cm[w]);
        if (r >= c0) r -= c0, ++w;
        const int bit = __fns(cm[w], 0, r + 1);
        cart_emit_lut(w * 32 + bit, cols, inv_cols, metres, ij, xy, ((size_t)f * cap + j) * 2);
      }
      if (tid == 0) count[f] = total;
    }
  }
}

template <int FPB>
__global__ void __launch_bounds__(FX_THREADS)
    cart_points_kernel(const MapEntry *__restrict__ tab, int npix, int cols, int rows, int R, int B, int wpr,
                       const uint8_t *__restrict__ mask, const uint32_t *__restrict__ bits, int F, int cap,
                       double width, double height, int32_t *__restrict__ ij, float *__restrict__ xy,
                       int32_t *__restrict__ count) {
  extern __shared__ uint32_t sbits[];  // [FPB][R * wpr]
  __shared__ int wcount[FPB][32];
  __shared__ int wprefix[FPB][32];
  __shared__ int wtotal[FPB];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int f0 = blockIdx.x * FPB;
  const int words = R * wpr;

  // ---- stage the polar masks of this CTA's frames as bit planes
#pragma unroll
  for (int j = 0; j < FPB; ++j) {
    const int f = f0 + j;
    uint32_t *sb = sbits + (size_t)j * words;
    if (f >= F) {
      for (int w = tid; w < words; w += FX_THREADS) sb[w] = 0;
    } else if (bits != nullptr) {
      const uint32_t *src = bits + (size_t)f * words;
      for (int w = tid; w < words; w += FX_THREADS) sb[w] = src[w];
    } else {
      const uint8_t *src = mask + (size_t)f * R * B;
      const bool vec = (B % 16 == 0) && ((uintptr_t)src % 16 == 0);
      for (int w = tid; w < words; w += FX_THREADS) {
        const int r = w / wpr, q = w - r * wpr;
        const uint8_t *row = src + (size_t)r * B + q * 32;
        uint32_t word = 0;
        const int nb = min(32, B - q * 32);
        if (vec && nb == 32) {
          const uint4 a = *reinterpret_cast<const uint4 *>(row);
          const uint4 b = *reinterpret_cast<const uint4 *>(row + 16);
          const uint32_t v[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
#pragma unroll
          for (int t = 0; t < 8; ++t) {
            const uint32_t nz = v[t];  // four mask bytes (0/1)
            const uint32_t nib = ((nz & 0xffu) ? 1u : 0u) | ((nz & 0xff00u) ? 2u : 0u) | ((nz & 0xff0000u) ? 4u : 0u) |
                                 ((nz & 0xff000000u) ? 8u : 0u);
            word |= nib << (4 * t);
          }
        } else {
          for (int t = 0; t < nb; ++t) word |= (row[t] ? 1u : 0u) << t;
        }
        sb[w] = word;
      }
    }
  }
  __syncthreads();

  int running[FPB];
#pragma unroll
  for (int j = 0; j < FPB; ++j) running[j] = 0;
  const unsigned lt_mask = (1u << lane) - 1u;

  for (int base = 0; base < npix; base += FX_THREADS) {
    const int pix = base + tid;
    bool pass[FPB];
#pragma unroll
    for (int j = 0; j < FPB; ++j) pass[j] = false;
    if (pix < npix) {
      const MapEntry e = tab[pix];
      if (e.flags & 1) {
        const int ix = e.ix, iy = e.iy, fx = e.fx, fy = e.fy;
        const bool x0 = (unsigned)ix < (unsigned)B, x1 = (unsigned)(ix + 1) < (unsigned)B;
        const bool y0 = (unsigned)iy < (unsigned)R, y1 = (unsigned)(iy + 1) < (unsigned)R;
        const int w00 = (x0 && y0) ? (32 - fx) * (32 - fy) : 0, w01 = (x1 && y0) ? fx * (32 - fy) : 0;
        const int w10 = (x0 && y1) ? (32 - fx) * fy : 0, w11 = (x1 && y1) ? fx * fy : 0;
        // clamp addresses of dead taps onto a valid word (their weight is 0)
        const int cx0 = x0 ? ix : 0, cx1 = x1 ? ix + 1 : 0, cy0 = y0 ? iy : 0, cy1 = y1 ? iy + 1 : 0;
        const int a00 = cy0 * wpr + (cx0 >> 5), a01 = cy0 * wpr + (cx1 >> 5);
        const int a10 = cy1 * wpr + (cx0 >> 5), a11 = cy1 * wpr + (cx1 >> 5);
        const int s0 = cx0 & 31, s1 = cx1 & 31;
#pragma unroll
        for (int j = 0; j < FPB; ++j) {
          const uint32_t *sb = sbits + (size_t)j * words;
          const int sum = w00 * (int)((sb[a00] >> s0) & 1u) + w01 * (int)((sb[a01] >> s1) & 1u) +
                          w10 * (int)((sb[a10] >> s0) & 1u) + w11 * (int)((sb[a11] >> s1) & 1u);
          pass[j] = sum >= 512;
        }
      }
    }
    unsigned bal[FPB];
    unsigned any = 0;
#pragma unroll
    for (int j = 0; j < FPB; ++j) {
      bal[j] = __ballot_sync(0xffffffffu, pass[j]);
      any |= bal[j];
      if (lane == 0) wcount[j][warp] = __popc(bal[j]);
    }
    if (__syncthreads_or(any != 0)) {
      if (warp < FPB) {  // warp j scans the 32 warp counts of frame j
        const int c = wcount[warp][lane];
        int incl = c;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
          const int t = __shfl_up_sync(0xffffffffu, incl, d);
          if (lane >= d) incl += t;
        }
        wprefix[warp][lane] = incl - c;
        if (lane == 31) wtotal[warp] = incl;
      }
      __syncthreads();
#pragma unroll
      for (int j = 0; j < FPB; ++j) {
        if (pass[j]) {
          const int idx = running[j] + wprefix[j][warp] + __popc(bal[j] & lt_mask);
          if (idx < cap) {
            const int row = pix / cols, col = pix - row * cols;
            const size_t o = ((size_t)(f0 + j) * cap + idx) * 2;
            ij[o] = row;
            ij[o + 1] = col;
            // feature_extraction.py:235-237, float64, operation by operation (no contraction)
            double x = __dsub_rn((double)col, __ddiv_rn((double)cols, 2.0));
            x = __dmul_rn(__ddiv_rn(x, __ddiv_rn((double)cols, 2.0)), __ddiv_rn(width, 2.0));
            x = __dmul_rn(-1.0, x);
            double y = __dmul_rn(-1.0, __ddiv_rn((double)row, (double)rows));
            y = __dadd_rn(__dmul_rn(y, height), height);
            xy[o] = (float)y;
            xy[o + 1] = (float)x;
          }
        }
        running[j] += wtotal[j];
      }
    }
  }
  if (tid == 0) {
#pragma unroll
    for (int j = 0; j < FPB; ++j)
      if (f0 + j < F) count[f0 + j] = running[j];
  }
}

// ---------------------------------------------------------------------------- feature image
// feature_extraction.py:226-227: cv2.remap(img, map_x, map_y, INTER_LINEAR) of the uint8 polar frame, then
// cv2.applyColorMap(., COLORMAP_JET) -- here the caller's 256-entry BGR table.  The remap is cart_pixel_fires' fixed-point
// rule on the full 8-bit frame: v = (32 * sum w_k img[tap_k] + 2^14) >> 15, taps outside the frame contribute 0, and a
// MAP_DEAD entry gives 0, as cv2 does for such coordinates.
//
// A CTA owns FI_TILE consecutive Cartesian pixels of FI_FPB frames: it loads their table entries once, into registers,
// and uses them for every frame.  Lanes take consecutive pixels, so a warp's tap gathers fall in a few polar rows (read
// through the read-only path).  Each frame's tile is assembled in shared memory and written with coalesced 16-B
// evict-first stores, three per thread: the images are written once and should not push the table and the frames out
// of L2.
constexpr int FI_THREADS = 256, FI_PPT = 16, FI_TILE = FI_THREADS * FI_PPT, FI_FPB = 8;
struct FeatureLut {
  uint8_t bgr[256 * 3];
};

__device__ __forceinline__ uint32_t remap_u8(uint2 e, const uint8_t *__restrict__ img, int R, int B) {
  if ((e.y >> 16) & MAP_DEAD) return 0;
  const int ix = (int16_t)(e.x & 0xffffu), iy = (int16_t)(e.x >> 16);
  const int fx = e.y & 0xff, fy = (e.y >> 8) & 0xff;
  const bool x0 = (unsigned)ix < (unsigned)B, x1 = (unsigned)(ix + 1) < (unsigned)B;
  const bool y0 = (unsigned)iy < (unsigned)R, y1 = (unsigned)(iy + 1) < (unsigned)R;
  const int v00 = (x0 && y0) ? __ldg(img + iy * B + ix) : 0, v01 = (x1 && y0) ? __ldg(img + iy * B + ix + 1) : 0;
  const int v10 = (x0 && y1) ? __ldg(img + (iy + 1) * B + ix) : 0, v11 = (x1 && y1) ? __ldg(img + (iy + 1) * B + ix + 1) : 0;
  const int sum = (32 - fx) * (32 - fy) * v00 + fx * (32 - fy) * v01 + (32 - fx) * fy * v10 + fx * fy * v11;
  return (uint32_t)((32 * sum + (1 << 14)) >> 15);
}

__global__ void __launch_bounds__(FI_THREADS)
    feature_image_kernel(const uint2 *__restrict__ tab, int npix, int R, int B, const uint8_t *__restrict__ frames,
                         int F, int n_tiles, const FeatureLut lut, uint8_t *__restrict__ out) {
  __shared__ uint32_t slut[256];  // B | G << 8 | R << 16
  __shared__ __align__(16) uint8_t simg[FI_TILE * 3];
  const int tid = threadIdx.x;
  const int p0 = (blockIdx.x % n_tiles) * FI_TILE, f0 = (blockIdx.x / n_tiles) * FI_FPB;
  const int np = min(FI_TILE, npix - p0), nf = min(FI_FPB, F - f0);
  for (int i = tid; i < 256; i += FI_THREADS)
    slut[i] = lut.bgr[3 * i] | (uint32_t)lut.bgr[3 * i + 1] << 8 | (uint32_t)lut.bgr[3 * i + 2] << 16;
  uint2 e[FI_PPT];
#pragma unroll
  for (int k = 0; k < FI_PPT; ++k) {
    const int p = k * FI_THREADS + tid;
    e[k] = p < np ? __ldg(tab + p0 + p) : make_uint2(0u, (uint32_t)MAP_DEAD << 16);
  }
  __syncthreads();
  const size_t img_bytes = (size_t)npix * 3;
  for (int j = 0; j < nf; ++j) {
    const uint8_t *img = frames + (size_t)(f0 + j) * R * B;
#pragma unroll
    for (int k = 0; k < FI_PPT; ++k) {
      const int p = k * FI_THREADS + tid;
      const uint32_t c = slut[remap_u8(e[k], img, R, B)];
      simg[3 * p] = (uint8_t)c, simg[3 * p + 1] = (uint8_t)(c >> 8), simg[3 * p + 2] = (uint8_t)(c >> 16);
    }
    __syncthreads();
    uint8_t *dst = out + (size_t)(f0 + j) * img_bytes + (size_t)p0 * 3;
    if (np == FI_TILE && ((uintptr_t)dst & 15) == 0) {
      const uint4 *s = reinterpret_cast<const uint4 *>(simg);
      uint4 *d = reinterpret_cast<uint4 *>(dst);
#pragma unroll
      for (int q = 0; q < 3; ++q) __stcs(d + q * FI_THREADS + tid, s[q * FI_THREADS + tid]);
    } else {  // the last tile of a frame, or a frame base that is not 16-B aligned (rows * cols * 3 % 16 != 0)
      for (int b = tid; b < np * 3; b += FI_THREADS) dst[b] = simg[b];
    }
    __syncthreads();
  }
}

template <int FPB>
static int launch_cart(sfe_ctx *ctx, cudaStream_t st, const sfe_maps *m, const uint8_t *mask, const uint32_t *bits, int F, int cap,
                       int32_t *ij, float *xy, int32_t *count) {
  const int wpr = (m->B + 31) / 32;
  const size_t smem = (size_t)FPB * m->R * wpr * sizeof(uint32_t);
  if (smem > (size_t)ctx->max_smem_optin - 1024) return SFE_ERR_UNSUPPORTED;
  if (smem > 40 * 1024) {
    const int rc = raise_smem_limit(ctx, (const void *)cart_points_kernel<FPB>, smem);
    if (rc != SFE_OK) return rc;
  }
  const int grid = (F + FPB - 1) / FPB;
  cart_points_kernel<FPB><<<grid, FX_THREADS, smem, st>>>(
      (const MapEntry *)m->table, m->rows * m->cols, m->cols, m->rows, m->R, m->B, wpr, mask, bits, F, cap, m->width,
      m->height, ij, xy, count);
  SFE_CUDA(cudaGetLastError());
  ctx->launches++;
  return SFE_OK;
}

}  // namespace sfe

int sfe::feature_image_run(sfe_ctx *ctx, cudaStream_t st, const sfe_maps *m, const uint8_t *frames, int F,
                           const uint8_t *lut_bgr, uint8_t *out, const char *what) {
  SFE_REQUIRE(ctx && m, "%s: null context or maps", what);
  SFE_REQUIRE(ctx->device == m->device, "%s: maps were created on device %d, context is on %d", what, m->device,
              ctx->device);
  SFE_REQUIRE(F >= 0, "%s: negative frame count", what);
  if (F == 0) return SFE_OK;
  SFE_REQUIRE(frames && lut_bgr && out, "%s: null frames, table or output pointer", what);
  SFE_REQUIRE((long long)m->R * m->B < (1ll << 31), "%s: a %d x %d polar frame is too large", what, m->R, m->B);
  const int npix = m->rows * m->cols, n_tiles = (npix + FI_TILE - 1) / FI_TILE;
  const long long grid = (long long)n_tiles * (((long long)F + FI_FPB - 1) / FI_FPB);
  SFE_REQUIRE(grid <= 0x7fffffffll, "%s: %d frames of %d x %d are too many for one call", what, F, m->rows, m->cols);
  FeatureLut lut;
  memcpy(lut.bgr, lut_bgr, sizeof(lut.bgr));
  feature_image_kernel<<<(unsigned)grid, FI_THREADS, 0, st>>>((const uint2 *)m->table, npix, m->R, m->B, frames, F,
                                                               n_tiles, lut, out);
  SFE_CUDA(cudaGetLastError());
  ctx->launches++;
  return SFE_OK;
}

int sfe::cart_points_run(sfe_ctx *ctx, cudaStream_t st, const sfe_maps *m, const uint8_t *mask, const uint32_t *bits,
                         int F, int cap, int32_t *ij, float *xy, int32_t *count) {
  SFE_REQUIRE(ctx && m, "cart_points: null context or maps");
  SFE_REQUIRE(ctx->device == m->device, "cart_points: maps were created on device %d, context is on %d", m->device,
              ctx->device);
  SFE_REQUIRE((mask != nullptr) != (bits != nullptr), "cart_points: pass exactly one of mask / bits");
  SFE_REQUIRE(F >= 0 && cap >= 0, "cart_points: negative frame count or capacity");
  SFE_REQUIRE(F == 0 || (ij && xy && count), "cart_points: null output pointer");
  if (F == 0) return SFE_OK;
  // detection-driven kernel whenever both bit planes fit in shared memory
  {
    const int wpr = (m->B + 31) / 32, npix = m->rows * m->cols;
    const size_t pw = (size_t)m->R * wpr, cw = (size_t)(npix + 31) / 32;
    const size_t smem = sizeof(uint32_t) * (pw + cw + (pw + 1) / 2 + 1);
    // (the emission's rank table of Cartesian word pairs reuses the polar plane: it must fit there)
    if (m->inv_off != nullptr && smem <= (size_t)ctx->max_smem_optin - 2048 && (cw + 1) / 2 <= pw) {
      int per_sm;
      const int rc = ctas_per_sm(ctx, (const void *)cart_scatter_kernel, FXS_THREADS, smem, &per_sm);
      if (rc != SFE_OK) return rc;
      int grid = ctx->sm_count * per_sm;
      if (grid > F) grid = F;
      SFE_CUDA(cudaMemsetAsync(ctx->work + WORK_CART, 0, sizeof(int), st));
      cart_scatter_kernel<<<grid, FXS_THREADS, smem, st>>>(
          (const MapEntry *)m->table, m->inv_off, m->inv_idx, npix, m->cols, m->rows, m->R, m->B, wpr, mask, bits, F,
          cap, m->metres, ij, xy, count, ctx->work + WORK_CART);
      SFE_CUDA(cudaGetLastError());
      ctx->launches++;
      return SFE_OK;
    }
  }
  // dense variant: several frames per CTA amortise the table read once there are enough frames
  int rc = SFE_ERR_UNSUPPORTED;
  if (F >= 4 * ctx->sm_count) rc = launch_cart<4>(ctx, st, m, mask, bits, F, cap, ij, xy, count);
  if (rc == SFE_ERR_UNSUPPORTED && F >= 2 * ctx->sm_count) rc = launch_cart<2>(ctx, st, m, mask, bits, F, cap, ij, xy, count);
  if (rc == SFE_ERR_UNSUPPORTED) rc = launch_cart<1>(ctx, st, m, mask, bits, F, cap, ij, xy, count);
  if (rc == SFE_ERR_UNSUPPORTED)
    set_error("cart_points: a %d x %d polar bit plane does not fit in shared memory", m->R, m->B);
  return rc;
}

namespace sfe {

// ---------------------------------------------------------------------------- host side: per-geometry tables
// cv2.remap's fixed-point sampling position of every Cartesian pixel (see cart_pixel_fires)
static void build_map_table(const float *map_x_host, const float *map_y_host, int rows, int cols, int R, int B,
                            std::vector<MapEntry> &tab) {
  const size_t n = (size_t)rows * cols;
  tab.assign(n, MapEntry{});
  for (size_t p = 0; p < n; ++p) {
    MapEntry e{};
    const float mx = map_x_host[p] * 32.0f, my = map_y_host[p] * 32.0f;
    if (fabsf(mx) < 1.0e9f && fabsf(my) < 1.0e9f) {  // finite and convertible (NaN fails the compare)
      const int sx = (int)lrintf(mx), sy = (int)lrintf(my);  // cvRound: nearest, ties to even
      int ix = sx >> 5, iy = sy >> 5;
      ix = ix < -32768 ? -32768 : (ix > 32767 ? 32767 : ix);
      iy = iy < -32768 ? -32768 : (iy > 32767 ? 32767 : iy);
      const int fx = sx & 31, fy = sy & 31;
      const bool x0 = ix >= 0 && ix < B, x1 = ix + 1 >= 0 && ix + 1 < B;
      const bool y0 = iy >= 0 && iy < R, y1 = iy + 1 >= 0 && iy + 1 < R;
      const int reach = (x0 && y0 ? (32 - fx) * (32 - fy) : 0) + (x1 && y0 ? fx * (32 - fy) : 0) +
                        (x0 && y1 ? (32 - fx) * fy : 0) + (x1 && y1 ? fx * fy : 0);
      e.ix = (int16_t)ix, e.iy = (int16_t)iy, e.fx = (uint8_t)fx, e.fy = (uint8_t)fy;
      e.flags = reach >= 512 ? MAP_FIRES : 0;
    } else {
      e.flags = MAP_DEAD;
    }
    tab[p] = e;
  }
}

// Inverse lists: polar cell -> Cartesian pixels the detection-driven kernel must test when that cell is a
// detection.  A pixel fires iff the weights of its lit taps add up to >= 512 (of 1024), so it need not be listed
// under every tap: taking its in-image taps by decreasing weight until the REMAINING ones together weigh less than
// 512 gives a set S such that every firing configuration lights a tap of S (if none is lit, the lit taps are among
// the remaining ones and cannot reach 512).  The kernel tests each listed candidate with the full rule, so the
// result is unchanged while the lists shrink from ~3.9 to ~1.4 entries per pixel (625 of the 1024 (fx, fy)
// fractions have one dominant tap).  Checked by enumeration and against cv2.remap in tests/test_oracle_featx.py.
static void build_inverse_lists(const std::vector<MapEntry> &tab, int R, int B, std::vector<int32_t> &inv_off,
                                std::vector<int32_t> &inv_idx) {
  const size_t n = tab.size();
  inv_off.assign((size_t)R * B + 1, 0);
  auto each_tap = [&](size_t p, auto &&fn) {
    const MapEntry &e = tab[p];
    if (!(e.flags & 1)) return;
    int w[4] = {(32 - e.fx) * (32 - e.fy), e.fx * (32 - e.fy), (32 - e.fx) * e.fy, e.fx * e.fy};
    int rest = 0;
    for (int t = 0; t < 4; ++t) {
      const int x = e.ix + (t & 1), y = e.iy + (t >> 1);
      if (!(x >= 0 && x < B && y >= 0 && y < R)) w[t] = 0;  // out-of-image taps never contribute
      rest += w[t];
    }
    while (rest >= 512) {
      int best = 0;
      for (int t = 1; t < 4; ++t)
        if (w[t] > w[best]) best = t;  // largest remaining weight, lowest tap on ties
      if (w[best] == 0) break;
      fn((size_t)(e.iy + (best >> 1)) * B + (size_t)(e.ix + (best & 1)));
      rest -= w[best];
      w[best] = 0;
    }
  };
  for (size_t p = 0; p < n; ++p) each_tap(p, [&](size_t q) { inv_off[q + 1]++; });
  for (size_t q = 0; q < (size_t)R * B; ++q) inv_off[q + 1] += inv_off[q];
  inv_idx.assign((size_t)inv_off.back() + 1, 0);
  std::vector<int32_t> cur(inv_off.begin(), inv_off.end() - 1);
  for (size_t p = 0; p < n; ++p) each_tap(p, [&](size_t q) { inv_idx[cur[q]++] = (int32_t)p; });
}

// feature_extraction.py:235-237 per column / per row, float64, operation by operation (volatile: no contraction,
// no re-association), then the float32 cast of the cloud (pybind / the ROS message)
static void build_metre_tables(int rows, int cols, double width, double height, std::vector<float> &t) {
  t.resize((size_t)cols + rows);
  for (int col = 0; col < cols; ++col) {
    volatile double half = (double)cols / 2.0;
    volatile double x = (double)col - half;
    x = x / half;
    volatile double hw = width / 2.0;
    x = x * hw;
    x = -1.0 * x;
    t[col] = (float)x;
  }
  for (int row = 0; row < rows; ++row) {
    volatile double y = (double)row / (double)rows;
    y = -1.0 * y;
    y = y * height;
    y = y + height;
    t[(size_t)cols + row] = (float)y;
  }
}

}  // namespace sfe

using namespace sfe;

extern "C" {

int sfe_maps_create(sfe_ctx *ctx, const float *map_x_host, const float *map_y_host, int rows, int cols, int R, int B,
                    double width, double height, sfe_maps **out) {
  SFE_REQUIRE(ctx && out, "sfe_maps_create: null context or out pointer");
  *out = nullptr;
  SFE_REQUIRE(map_x_host && map_y_host, "sfe_maps_create: null map pointer");
  SFE_REQUIRE(rows > 0 && cols > 0 && R > 0 && B > 0, "sfe_maps_create: non-positive shape");
  SFE_REQUIRE((long long)rows * cols < (1ll << 31), "sfe_maps_create: Cartesian image too large");
  SFE_CUDA(cudaSetDevice(ctx->device));
  std::vector<MapEntry> tab;
  std::vector<int32_t> inv_off, inv_idx;
  build_map_table(map_x_host, map_y_host, rows, cols, R, B, tab);
  build_inverse_lists(tab, R, B, inv_off, inv_idx);
  const size_t n = tab.size();
  sfe_maps *m = new sfe_maps();
  m->rows = rows, m->cols = cols, m->R = R, m->B = B, m->width = width, m->height = height, m->device = ctx->device;
  m->table = nullptr, m->inv_off = nullptr, m->inv_idx = nullptr, m->metres = nullptr;
  std::vector<float> metres;
  build_metre_tables(rows, cols, width, height, metres);
  cudaError_t e = cudaMalloc(&m->table, n * sizeof(MapEntry));
  if (e == cudaSuccess) e = cudaMalloc((void **)&m->metres, metres.size() * sizeof(float));
  if (e == cudaSuccess) e = cudaMemcpy(m->metres, metres.data(), metres.size() * sizeof(float), cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaMemcpy(m->table, tab.data(), n * sizeof(MapEntry), cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaMalloc((void **)&m->inv_off, inv_off.size() * sizeof(int32_t));
  if (e == cudaSuccess)
    e = cudaMemcpy(m->inv_off, inv_off.data(), inv_off.size() * sizeof(int32_t), cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaMalloc((void **)&m->inv_idx, inv_idx.size() * sizeof(int32_t));
  if (e == cudaSuccess)
    e = cudaMemcpy(m->inv_idx, inv_idx.data(), inv_idx.size() * sizeof(int32_t), cudaMemcpyHostToDevice);
  if (e != cudaSuccess) {
    set_error("sfe_maps_create: %s", cudaGetErrorString(e));
    if (m->table) cudaFree(m->table);
    if (m->inv_off) cudaFree(m->inv_off);
    if (m->inv_idx) cudaFree(m->inv_idx);
    if (m->metres) cudaFree(m->metres);
    delete m;
    return SFE_ERR_CUDA;
  }
  *out = m;
  return SFE_OK;
}

void sfe_maps_destroy(sfe_maps *m) {
  if (!m) return;
  cudaSetDevice(m->device);
  if (m->table) cudaFree(m->table);
  if (m->inv_off) cudaFree(m->inv_off);
  if (m->inv_idx) cudaFree(m->inv_idx);
  if (m->metres) cudaFree(m->metres);
  delete m;
}

int sfe_maps_inverse_lists_host(const float *map_x_host, const float *map_y_host, int rows, int cols, int R, int B,
                                int32_t *off_out, int32_t *idx_out, int64_t idx_capacity, int64_t *n_entries) {
  SFE_REQUIRE(map_x_host && map_y_host && off_out && n_entries, "sfe_maps_inverse_lists_host: null pointer");
  SFE_REQUIRE(rows > 0 && cols > 0 && R > 0 && B > 0 && (long long)rows * cols < (1ll << 31),
              "sfe_maps_inverse_lists_host: bad shape");
  std::vector<MapEntry> tab;
  std::vector<int32_t> inv_off, inv_idx;
  build_map_table(map_x_host, map_y_host, rows, cols, R, B, tab);
  build_inverse_lists(tab, R, B, inv_off, inv_idx);
  *n_entries = inv_off.back();
  memcpy(off_out, inv_off.data(), inv_off.size() * sizeof(int32_t));
  if (*n_entries > idx_capacity || (idx_out == nullptr && *n_entries > 0)) {
    set_error("sfe_maps_inverse_lists_host: %lld entries do not fit the index buffer", (long long)*n_entries);
    return SFE_ERR_CAPACITY;
  }
  memcpy(idx_out, inv_idx.data(), (size_t)*n_entries * sizeof(int32_t));
  return SFE_OK;
}

int sfe_cart_points_dev(sfe_ctx *ctx, const sfe_maps *maps, const uint8_t *mask_dev, const uint32_t *bits_dev,
                        int n_frames, int capacity, int32_t *ij_dev, float *xy_dev, int32_t *count_dev) {
  SFE_REQUIRE(ctx != nullptr, "sfe_cart_points_dev: null context");
  SFE_CUDA(cudaSetDevice(ctx->device));
  return cart_points_run(ctx, ctx->stream, maps, mask_dev, bits_dev, n_frames, capacity, ij_dev, xy_dev, count_dev);
}

int sfe_cart_points_host(sfe_ctx *ctx, const sfe_maps *maps, const uint8_t *mask_host, int n_frames, int capacity,
                         int32_t *ij_host, float *xy_host, int32_t *count_host) {
  SFE_REQUIRE(ctx && maps, "sfe_cart_points_host: null context or maps");
  SFE_REQUIRE(n_frames >= 0 && capacity >= 0, "sfe_cart_points_host: negative frame count or capacity");
  if (n_frames == 0) return SFE_OK;
  SFE_REQUIRE(mask_host && ij_host && xy_host && count_host, "sfe_cart_points_host: null pointer");
  SFE_CUDA(cudaSetDevice(ctx->device));
  const size_t cells = (size_t)n_frames * maps->R * maps->B, slots = (size_t)n_frames * capacity * 2;
  int rc;
  if ((rc = ensure(ctx, ctx->stage_in[0], cells)) != SFE_OK) return rc;
  if ((rc = ensure(ctx, ctx->stage_out[0], slots * sizeof(int32_t) + 16)) != SFE_OK) return rc;
  if ((rc = ensure(ctx, ctx->stage_out[1], slots * sizeof(float) + 16)) != SFE_OK) return rc;
  if ((rc = ensure(ctx, ctx->stage_out[2], (size_t)n_frames * sizeof(int32_t))) != SFE_OK) return rc;
  SFE_CUDA(cudaMemcpyAsync(ctx->stage_in[0].ptr, mask_host, cells, cudaMemcpyHostToDevice, ctx->stream));
  rc = cart_points_run(ctx, ctx->stream, maps, (const uint8_t *)ctx->stage_in[0].ptr, nullptr, n_frames, capacity,
                       (int32_t *)ctx->stage_out[0].ptr, (float *)ctx->stage_out[1].ptr,
                       (int32_t *)ctx->stage_out[2].ptr);
  if (rc != SFE_OK) return rc;
  SFE_CUDA(cudaMemcpyAsync(count_host, ctx->stage_out[2].ptr, (size_t)n_frames * sizeof(int32_t),
                           cudaMemcpyDeviceToHost, ctx->stream));
  SFE_CUDA(cudaMemcpyAsync(ij_host, ctx->stage_out[0].ptr, slots * sizeof(int32_t), cudaMemcpyDeviceToHost,
                           ctx->stream));
  SFE_CUDA(cudaMemcpyAsync(xy_host, ctx->stage_out[1].ptr, slots * sizeof(float), cudaMemcpyDeviceToHost,
                           ctx->stream));
  SFE_CUDA(cudaStreamSynchronize(ctx->stream));
  for (int f = 0; f < n_frames; ++f)
    if (count_host[f] > capacity) {
      set_error("sfe_cart_points_host: frame %d has %d points, capacity is %d", f, count_host[f], capacity);
      return SFE_ERR_CAPACITY;
    }
  return SFE_OK;
}

int sfe_feature_image_dev(sfe_ctx *ctx, const sfe_maps *maps, const uint8_t *frames_dev, int n_frames,
                          const uint8_t *lut_bgr_host, uint8_t *out_dev) {
  SFE_REQUIRE(ctx != nullptr, "sfe_feature_image_dev: null context");
  SFE_CUDA(cudaSetDevice(ctx->device));
  return feature_image_run(ctx, ctx->stream, maps, frames_dev, n_frames, lut_bgr_host, out_dev,
                           "sfe_feature_image_dev");
}

// Chunks of FI_HOST_CHUNK frames: the copies in and out run on the context's copy stream, in the order
// in(0) in(1) out(0) in(2) out(1) ..., so the kernel of chunk k overlaps the copy-out of chunk k-1 and the copy-in of
// chunk k+1.  Staging is double-buffered both ways.
constexpr int FI_HOST_CHUNK = 16;

static int feature_image_host(sfe_ctx *ctx, const sfe_maps *m, const uint8_t *frames_host, int n,
                              const uint8_t *lut_bgr, uint8_t *out_host) {
  const char *what = "sfe_feature_image_host";
  const size_t fbytes = (size_t)m->R * m->B, ibytes = (size_t)m->rows * m->cols * 3;
  const int chunk = n < FI_HOST_CHUNK ? n : FI_HOST_CHUNK;
  int rc;
  for (int b = 0; b < 2; ++b) {
    if ((rc = ensure(ctx, ctx->stage_in[b], chunk * fbytes)) != SFE_OK) return rc;
    if ((rc = ensure(ctx, ctx->stage_out[b], chunk * ibytes)) != SFE_OK) return rc;
  }
  if (!ctx->copy_stream) SFE_CUDA(cudaStreamCreateWithFlags(&ctx->copy_stream, cudaStreamNonBlocking));
  for (auto &ev : ctx->copy_ev)
    if (!ev) SFE_CUDA(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
  cudaEvent_t *in_done = ctx->copy_ev, *kernel_done = ctx->copy_ev + 2;
  // the staging buffers are allocated (and may be still in use) in the launch stream's order
  SFE_CUDA(cudaEventRecord(kernel_done[1], ctx->stream));
  SFE_CUDA(cudaStreamWaitEvent(ctx->copy_stream, kernel_done[1], 0));
  const int n_chunks = (n + chunk - 1) / chunk;
  auto copy_in = [&](int k) -> int {
    const int f0 = k * chunk, nf = std::min(chunk, n - f0);
    if (k >= 2) SFE_CUDA(cudaStreamWaitEvent(ctx->copy_stream, kernel_done[k & 1], 0));  // kernel k-2 read the buffer
    SFE_CUDA(cudaMemcpyAsync(ctx->stage_in[k & 1].ptr, frames_host + f0 * fbytes, nf * fbytes, cudaMemcpyHostToDevice,
                             ctx->copy_stream));
    SFE_CUDA(cudaEventRecord(in_done[k & 1], ctx->copy_stream));
    return SFE_OK;
  };
  if ((rc = copy_in(0)) != SFE_OK) return rc;
  for (int k = 0; k < n_chunks; ++k) {
    const int f0 = k * chunk, nf = std::min(chunk, n - f0);
    if (k + 1 < n_chunks && (rc = copy_in(k + 1)) != SFE_OK) return rc;
    // the copy-out of chunk k-2 (enqueued on the copy stream before in_done[k]) has drained this output buffer
    SFE_CUDA(cudaStreamWaitEvent(ctx->stream, in_done[k & 1], 0));
    rc = feature_image_run(ctx, ctx->stream, m, (const uint8_t *)ctx->stage_in[k & 1].ptr, nf, lut_bgr,
                           (uint8_t *)ctx->stage_out[k & 1].ptr, what);
    if (rc != SFE_OK) return rc;
    SFE_CUDA(cudaEventRecord(kernel_done[k & 1], ctx->stream));
    SFE_CUDA(cudaStreamWaitEvent(ctx->copy_stream, kernel_done[k & 1], 0));
    SFE_CUDA(cudaMemcpyAsync(out_host + f0 * ibytes, ctx->stage_out[k & 1].ptr, nf * ibytes, cudaMemcpyDeviceToHost,
                             ctx->copy_stream));
  }
  return SFE_OK;
}

int sfe_feature_image_host(sfe_ctx *ctx, const sfe_maps *maps, const uint8_t *frames_host, int n_frames,
                           const uint8_t *lut_bgr_host, uint8_t *out_host) {
  SFE_REQUIRE(ctx && maps, "sfe_feature_image_host: null context or maps");
  SFE_REQUIRE(ctx->device == maps->device, "sfe_feature_image_host: maps were created on device %d, context is on %d",
              maps->device, ctx->device);
  SFE_REQUIRE(n_frames >= 0, "sfe_feature_image_host: negative frame count");
  if (n_frames == 0) return SFE_OK;
  SFE_REQUIRE(frames_host && lut_bgr_host && out_host, "sfe_feature_image_host: null frames, table or output pointer");
  SFE_CUDA(cudaSetDevice(ctx->device));
  const int rc = feature_image_host(ctx, maps, frames_host, n_frames, lut_bgr_host, out_host);
  // copies already enqueued finish before the call returns, also on an error
  if (ctx->copy_stream) SFE_CUDA(cudaStreamSynchronize(ctx->copy_stream));
  SFE_CUDA(cudaStreamSynchronize(ctx->stream));
  return rc;
}

}  // extern "C"
