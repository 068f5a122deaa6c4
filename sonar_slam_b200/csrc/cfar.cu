// CFAR detector kernels (sm_90a).
//
// Replaces bruce_slam/src/bruce_slam/cpp/cfar.cpp:10-192 (ca/soca/goca/os and the
// "2" variants) for batches of polar sonar frames laid out [frame][range][beam].
//
// Two kernels:
//
//  cfar_ring_tma_kernel   the streaming path for the shipped configuration
//      (train_hs = 20, guard_hs = 5; CA / SOCA / GOCA).  One CTA owns a strip of
//      128 beams of one frame and marches down the range axis once.  [16 range
//      bins x 128 beams] boxes of the frame stream through a 4-stage
//      shared-memory ring with TMA (cp.async.bulk.tensor + mbarrier), refilled by
//      one thread after every block's barrier (no producer warp: cfar_refill);
//      each of the 128 threads owns ONE beam, reads every cell of its
//      beam exactly once from shared memory and keeps the last 32 cells and the
//      last 32 window sums in two register rings.  With W[i] = sum of the 20
//      cells ending at range bin i, the lagging window of the cell under test r
//      is W[r+25] and the leading window is W[r-6] = W[(r+25)-31], so one add and
//      one subtract per cell maintain both.  Nothing is re-read from shared or
//      global memory.  The 0/1 mask (and/or a bit plane) leaves through a
//      double-buffered shared tile and TMA stores.  HBM traffic = the image once
//      + the mask once (no halo: a strip spans the whole range axis).
//
//      Exactness: for integer-valued cells with |x| <= 2^18 every float32 sum is
//      exact whatever the order, so sliding sums equal the reference's sequential
//      sums.  The double-precision compare of cfar.cpp (`img > tau * sum /
//      train_hs`) is decided from a two-term float32 evaluation of
//      xc - S*(c_hi + c_lo) (c_hi + c_lo = tau/div to ~2^-48), whose error is
//      < 2e-9; cells with |xc - S*c| <= 1e-7 (about one in a million) are re-done
//      with the reference's own double expression.  A strip that sees any other
//      value (fraction, |x| > 2^18, inf, nan) raises a flag and is re-done by ...
//
//  cfar_exact_kernel      ... the general path: any train_hs/guard_hs, OS-CFAR, any
//      float input.  It accumulates each window in the reference's order
//      (ascending range, one float32 accumulator per sum) and evaluates the
//      threshold in double exactly as written in cfar.cpp, so it is bit-exact for
//      arbitrary float32 images.  It is a device path, not a CPU fallback.
#include <vector>

#include "stages.cuh"

namespace sfe {

constexpr int CF_W = 128;     // beams per strip / consumer threads per CTA
constexpr int CF_CH = 16;     // range bins per TMA box
constexpr int CF_NSTAGE = 4;     // input ring depth (stages of CF_CH rows)
constexpr int CF_NSTAGE_U8 = 4;  // same for the uint8 kernel
constexpr int CF_RING = 32;   // two 32-deep register rings per thread (cells, window sums)
constexpr int CF_T = 20;      // train_hs of the streaming path
constexpr int CF_G = 5;       // guard_hs of the streaming path
constexpr int CF_HALF = CF_T + CF_G;
constexpr int CF_SPLIT = CF_CH - (CF_HALF % CF_CH);  // step of an output block at which the input box changes (7)
constexpr float CF_AMBIG = 1e-7f;                    // |xc - S*c| below this is decided in double

struct CfarParams {
  int F, R, B, strips;
  int alg, T, G, k;
  double tau;   // threshold factor (exact compare)
  double div;   // 2*T (CA), T (SOCA/GOCA), 1 (OS)
  float c_hi;   // float(tau / div)
  float c_lo;   // float(tau / div - c_hi)
  int gate_on;
  float gate_f;   // float g with (x > g) <=> ((double)x > gate) for every float x
  double gate_d;
  const void *img;
  uint8_t *mask;  // may be null
  float *thr;     // may be null
  uint32_t *bits; // may be null
  int words_per_row;
  uint8_t *flags; // per (frame, strip): streaming path saw a non-integer cell
  const CUtensorMap *out_map;  // device-side: address of the kernel's __grid_constant__ copy
};

__device__ __forceinline__ float cell_to_float(float v) { return v; }
__device__ __forceinline__ float cell_to_float(uint8_t v) {
  // exact u8 -> f32 on the FMA/ALU pipes (no I2F): 2^23 + v, minus 2^23
  return __uint_as_float(0x4B000000u | (uint32_t)v) - 8388608.0f;
}

// The reference's arithmetic for one cell (cfar.cpp:16-25, 36-48, 59-71, 82-93), reading the
// column straight from global memory.  `train` is OS scratch: element i at train[i * tstride].
template <typename InT>
__device__ bool cfar_cell_exact(const InT *__restrict__ colp, size_t B, int r, const CfarParams &p, float *train,
                                int tstride, double *thr_out) {
  const int T = p.T, G = p.G, half = T + G;
  double d;
  if (p.alg == SFE_CFAR_CA) {
    float acc = 0.f;
    for (int i = r - half; i <= r + half; ++i)
      if (abs(i - r) > G) acc = __fadd_rn(acc, cell_to_float(colp[(size_t)i * B]));
    d = p.tau * (double)acc / p.div;
  } else if (p.alg == SFE_CFAR_OS) {
    int n = 0;
    for (int i = r - half; i <= r + half; ++i)
      if (abs(i - r) > G) train[(n++) * tstride] = cell_to_float(colp[(size_t)i * B]);
    float v = __int_as_float(0x7fc00000);
    for (int a = 0; a < n; ++a) {  // k-th smallest by rank counting
      const float va = train[a * tstride];
      int less = 0, leq = 0;
      for (int b = 0; b < n; ++b) {
        const float vb = train[b * tstride];
        less += vb < va;
        leq += vb <= va;
      }
      if (less <= p.k && p.k < leq) {
        v = va;
        break;
      }
    }
    d = p.tau * (double)v;
  } else {
    float ld = 0.f, lg = 0.f;
    for (int i = r - half; i < r - G; ++i) ld = __fadd_rn(ld, cell_to_float(colp[(size_t)i * B]));
    for (int i = r + G + 1; i <= r + half; ++i) lg = __fadd_rn(lg, cell_to_float(colp[(size_t)i * B]));
    // std::min(lead, lag) / std::max(lead, lag) as written in cfar.cpp:46,69
    const float S = (p.alg == SFE_CFAR_SOCA) ? (lg < ld ? lg : ld) : (ld < lg ? lg : ld);
    d = p.tau * (double)S / p.div;
  }
  const float xc = cell_to_float(colp[(size_t)r * B]);
  bool pass = (double)xc > d;
  if (p.gate_on) pass = pass && ((double)xc > p.gate_d);
  if (thr_out) *thr_out = d;
  return pass;
}

// Rare path of the streaming kernel: this thread met a cell too close to its threshold for the
// float32 evaluation; redo its 16 output rows with the reference's expressions.
template <typename InT>
__device__ __noinline__ void cfar_resolve_block(const CfarParams &p, uint8_t (*obuf_ob)[CF_W], uint32_t *pass_bits,
                                                int f, int col, int r0, int tid) {
  if (col >= p.B) return;
  const InT *colp = (const InT *)p.img + (size_t)f * p.R * p.B + col;
  uint32_t pb = 0;
  for (int i = 0; i < CF_CH; ++i) {
    const int r = r0 + i;
    bool pass = false;
    if (r >= CF_HALF && r < p.R - CF_HALF) pass = cfar_cell_exact<InT>(colp, p.B, r, p, nullptr, 0, nullptr);
    if (obuf_ob) obuf_ob[i][tid] = pass ? 1 : 0;
    pb |= (pass ? 1u : 0u) << i;
  }
  *pass_bits = pb;
}

// Input ring without a producer warp.  Every 16-row block reads its two TMA boxes into registers up
// front and ends with a CTA-wide barrier, so after the barrier of block `blk` box blk-1 is dead and its
// stage can take box blk + NS - 1 (NS = ring depth): one thread re-arms the stage's mbarrier and issues the load.
template <typename InT, int NS>
__device__ __forceinline__ void cfar_refill(InT (*tile)[CF_CH][CF_W], uint64_t *full_bar, const CUtensorMap *in_map,
                                            const int blk, const int nchunks, const int tid, const int f,
                                            const int col0) {
  const int c = blk + NS - 1;
  if (tid == 0 && c < nchunks) {
    const int st = c & (NS - 1);
    mbar_arrive_expect_tx(&full_bar[st], CF_CH * CF_W * (int)sizeof(InT));
    tma_load_3d(&tile[st][0][0], in_map, &full_bar[st], col0, c * CF_CH, f);
  }
}

struct CfarStep {  // per-thread streaming state (all in registers; indices are static after unrolling)
  float xr[CF_RING];  // x[rn - a]      at slot (J - a) & 31
  float wr[CF_RING];  // W[rn - a] = sum of the 20 cells ending at rn - a
  float w;            // W[rn - 1]
  bool bad;           // set once a cell was seen that is not an integer of magnitude < 2^22 (fraction, NaN, +-inf)
  float mx;           // max |cell|
};

// One range bin.  J = position in the 32-step unrolled body (I = J % 16 = output row in its block);
// EDGE = this block touches the image border / the ends of the input (row validity is checked).
template <typename InT, int ALG, bool WITH_THR, bool MASK, bool BITS, bool EDGE, int J>
__device__ __forceinline__ void cfar_step(CfarStep &s, const float xn, uint8_t (*obuf_ob)[CF_W],
                                          const CfarParams &p, const int r, const int tid,
                                          const int f, const int col, const float c_hi, const float c_lo,
                                          const float gate, bool &amb, uint32_t &pass_bits) {
  constexpr int I = J % CF_CH;
  if (sizeof(InT) == 4) {
    // integer-valued?  (x + 1.5*2^23) - 1.5*2^23 == x  <=>  x integer and |x| < 2^22
    // (`!=` is true for unordered operands: a NaN cell, or inf - inf, flags the strip; fmaxf would drop the NaN)
    const float rt = (xn + 12582912.0f) - 12582912.0f;
    s.bad = s.bad || (rt - xn != 0.f);
    s.mx = fmaxf(s.mx, fabsf(xn));
  }
  // cell under test r, newest cell rn = r + 25:
  //   lagging window r+6 .. r+25  = the 20 cells ending at rn       -> W[rn]
  //   leading window r-25 .. r-6  = the 20 cells ending at rn - 31  -> W[rn-31]
  const float x20 = s.xr[(J + CF_RING - CF_T) % CF_RING];
  const float xc = s.xr[(J + CF_RING - CF_HALF) % CF_RING];
  const float lead = s.wr[(J + CF_RING - (CF_HALF + CF_G + 1)) % CF_RING];
  const float lag = (s.w + xn) - x20;
  s.w = lag;
  s.wr[J % CF_RING] = lag;
  s.xr[J % CF_RING] = xn;

  bool pass = false;
  if (!EDGE || (r >= CF_HALF && r < p.R - CF_HALF)) {
    float S;
    if (ALG == SFE_CFAR_CA)
      S = lead + lag;
    else if (ALG == SFE_CFAR_SOCA)
      S = fminf(lead, lag);
    else
      S = fmaxf(lead, lag);
    if (WITH_THR) {
      const double d = p.tau * (double)S / p.div;
      pass = (double)xc > d;
      if (col < p.B) p.thr[((size_t)f * p.R + r) * p.B + col] = (float)d;
    } else {
      const float u = fmaf(-S, c_lo, fmaf(-S, c_hi, xc));  // xc - S*(tau/div), |error| < 2e-9
      pass = u > 0.f;
      amb = amb || (fabsf(u) <= CF_AMBIG);
    }
    pass = pass && (xc > gate);  // gate = -inf when the amplitude gate is off
  }
  if (MASK) obuf_ob[I][tid] = pass ? 1 : 0;
  if (BITS) pass_bits |= (pass ? 1u : 0u) << I;
}

// 16 consecutive output rows r0 .. r0+15 (r0 % 16 == 0).  Needs cells r0+25 .. r0+40: rows 9..15 of
// TMA box `blk-1` (steps 0..6) and rows 0..8 of box `blk` (steps 7..15), where blk = r0/16 + 2.
template <typename InT, int ALG, bool WITH_THR, bool MASK, bool BITS, bool EDGE, int Q>
__device__ __forceinline__ void cfar_block16(CfarStep &s, InT (*tile)[CF_CH][CF_W], uint8_t (*obuf)[CF_CH][CF_W],
                                             uint32_t (*obits)[CF_CH][CF_W / 32], uint64_t *full_bar,
                                             const CUtensorMap *in_map, const CfarParams &p, const int blk,
                                             const int nchunks, const int tid, const int f, const int col0,
                                             const float c_hi, const float c_lo, const float gate) {
  const int r0 = (blk - 2) * CF_CH;
  const int col = col0 + tid;
  const int cA = blk - 1, cB = blk;
  const bool hasA = EDGE ? (cA >= 0 && cA < nchunks) : true;
  const bool hasB = EDGE ? (cB < nchunks) : true;
  const InT(*tileA)[CF_W] = tile[cA & (CF_NSTAGE - 1)];
  const InT(*tileB)[CF_W] = tile[cB & (CF_NSTAGE - 1)];
  constexpr int ob = Q & 1;  // blocks alternate output buffers; Q = blk & 1
  bool amb = false;
  uint32_t pass_bits = 0;
  // All 16 shared-memory reads of the block are issued before any arithmetic so that their latency
  // is paid once per block, not once per row (a warp issues in order).
  float xin[CF_CH];
#pragma unroll
  for (int i = 0; i < CF_SPLIT; ++i)  // x[r0 + 25 + i] = row 9 + i of box blk-1
    xin[i] = (!EDGE || hasA) ? cell_to_float(tileA[i + CF_CH - CF_SPLIT][tid]) : 0.f;
  if (hasB) mbar_wait(&full_bar[cB & (CF_NSTAGE - 1)], (cB / CF_NSTAGE) & 1);
#pragma unroll
  for (int i = CF_SPLIT; i < CF_CH; ++i)  // row i - 7 of box blk
    xin[i] = (!EDGE || hasB) ? cell_to_float(tileB[i - CF_SPLIT][tid]) : 0.f;
#define SFE_STEP(I)                                                                                          \
  cfar_step<InT, ALG, WITH_THR, MASK, BITS, EDGE, Q * CF_CH + I>(s, xin[I], obuf[ob], p, r0 + I, tid, f, col, \
                                                                 c_hi, c_lo, gate, amb, pass_bits);
  SFE_STEP(0) SFE_STEP(1) SFE_STEP(2) SFE_STEP(3) SFE_STEP(4) SFE_STEP(5) SFE_STEP(6) SFE_STEP(7)
  SFE_STEP(8) SFE_STEP(9) SFE_STEP(10) SFE_STEP(11) SFE_STEP(12) SFE_STEP(13) SFE_STEP(14) SFE_STEP(15)
#undef SFE_STEP
  if (EDGE && r0 < 0) {  // priming blocks: no output rows
    named_bar_sync(1, CF_W);
    cfar_refill<InT, CF_NSTAGE>(tile, full_bar, in_map, blk, nchunks, tid, f, col0);
    return;
  }
  if (!WITH_THR && amb) {
    uint32_t fixed = 0;
    cfar_resolve_block<InT>(p, MASK ? obuf[ob] : nullptr, &fixed, f, col, r0, tid);
    if (BITS) pass_bits = fixed;
  }
  if (BITS) {
    // transpose this thread's 16 row-bits into per-row ballots
#pragma unroll
    for (int i = 0; i < CF_CH; ++i) {
      const unsigned b = __ballot_sync(0xffffffffu, ((pass_bits >> i) & 1u) && col < p.B);
      if ((tid & 31) == i) obits[ob][i][tid >> 5] = b;
    }
  }
  // hand the 16 finished rows to global memory
  if (MASK) fence_proxy_async_smem();
  if (MASK && tid == 0) tma_wait_read<0>();  // the other buffer's TMA store has finished reading it
  named_bar_sync(1, CF_W);
  cfar_refill<InT, CF_NSTAGE>(tile, full_bar, in_map, blk, nchunks, tid, f, col0);
  if (MASK && tid == 0) {
    tma_store_3d(p.out_map, &obuf[ob][0][0], col0, r0, f);
    tma_commit();
  }
  if (BITS && tid < CF_CH * (CF_W / 32)) {
    const int i = tid / (CF_W / 32), wq = tid % (CF_W / 32);
    const int w = (col0 >> 5) + wq;
    if (r0 + i < p.R && w < p.words_per_row)
      p.bits[((size_t)f * p.R + r0 + i) * p.words_per_row + w] = obits[ob][i][wq];
  }
}

template <typename InT, int ALG, bool WITH_THR, bool MASK, bool BITS>
__global__ void __launch_bounds__(CF_W, 4)
    cfar_ring_tma_kernel(const __grid_constant__ CUtensorMap in_map, const __grid_constant__ CUtensorMap out_map,
                         CfarParams p) {
  __shared__ __align__(128) InT tile[CF_NSTAGE][CF_CH][CF_W];
  __shared__ __align__(128) uint8_t obuf[2][CF_CH][CF_W];
  __shared__ uint32_t obits[2][CF_CH][CF_W / 32];
  __shared__ __align__(8) uint64_t full_bar[CF_NSTAGE];

  const int tid = threadIdx.x;
  const int f = blockIdx.x / p.strips;
  const int col0 = (blockIdx.x % p.strips) * CF_W;
  const int R = p.R;
  p.out_map = &out_map;
  const int nchunks = (R + CF_CH - 1) / CF_CH;

  if (tid == 0) {
    prefetch_tmap(&in_map);
    for (int s = 0; s < CF_NSTAGE; ++s) mbar_init(&full_bar[s], 1);
    fence_mbar_init();
    for (int c = 0; c < CF_NSTAGE - 1 && c < nchunks; ++c) {  // the ring is refilled block by block (cfar_refill)
      mbar_arrive_expect_tx(&full_bar[c], CF_CH * CF_W * (int)sizeof(InT));
      tma_load_3d(&tile[c][0][0], &in_map, &full_bar[c], col0, c * CF_CH, f);
    }
  }
  __syncthreads();

  // one beam per thread
  CfarStep s;
#pragma unroll
  for (int i = 0; i < CF_RING; ++i) s.xr[i] = 0.f, s.wr[i] = 0.f;
  s.w = 0.f, s.bad = false, s.mx = 0.f;
  const float c_hi = p.c_hi, c_lo = p.c_lo;
  const float gate = p.gate_on ? p.gate_f : -INFINITY;

  // block `blk` emits output rows 16*(blk-2) .. +15; blocks 0 and 1 only prime the rings.
  const int nblk = nchunks + 2;
  for (int b2 = 0; b2 * 2 < nblk; ++b2) {
#pragma unroll
    for (int q = 0; q < 2; ++q) {
      const int blk = b2 * 2 + q;
      if (blk < nblk) {
        const int r0 = (blk - 2) * CF_CH;
        const bool interior = (r0 >= CF_HALF) && (r0 + CF_CH - 1 < R - CF_HALF);  // implies both boxes exist
#define SFE_BLOCK(EDGE_, Q_)                                                                                       \
  cfar_block16<InT, ALG, WITH_THR, MASK, BITS, EDGE_, Q_>(s, tile, obuf, obits, full_bar, &in_map, p, blk, nchunks, \
                                                          tid, f, col0, c_hi, c_lo, gate)
        if (interior) {
          if (q == 0) SFE_BLOCK(false, 0); else SFE_BLOCK(false, 1);
        } else {
          if (q == 0) SFE_BLOCK(true, 0); else SFE_BLOCK(true, 1);
        }
#undef SFE_BLOCK
      }
    }
  }
  if (sizeof(InT) == 4 && (s.bad || !(s.mx <= 262144.0f))) p.flags[blockIdx.x] = 1;
  if (MASK && tid == 0) tma_wait_all<0>();
}

// ------------------------------------------------------------------------------------------------
// uint8 streaming kernel: the node's native image type (feature_extraction.py:217).  Same TMA ring and
// per-beam register rings as above, but everything is integer: window sums are exact int32, and the
// reference's double-precision compare `(double)x > tau * S / div` (and the amplitude gate) is folded
// into a table M[S] = smallest cell value that passes for window statistic S, built on the host with
// the reference's own double expression for every possible S (S <= 2*T*255).  Per cell: one add/sub,
// one min/max, one table look-up in shared memory, one compare -- no floating point, no ambiguity path.
constexpr int CF_LUT_MAX = 2 * CF_T * 255 + 1;  // CA: sum of 40 uint8 cells

struct CfarStepI {
  int xr[CF_RING];
  int wr[CF_RING];
  int w;
};

template <int ALG, bool MASK, bool BITS, bool EDGE, int J>
__device__ __forceinline__ void cfar_step_u8(CfarStepI &s, const int xn, uint8_t (*obuf_ob)[CF_W],
                                             const uint16_t *__restrict__ lut, const int R, const int r,
                                             const int tid, const bool col_ok, unsigned &keep_bits) {
  constexpr int I = J % CF_CH;
  const int x20 = s.xr[(J + CF_RING - CF_T) % CF_RING];
  const int xc = s.xr[(J + CF_RING - CF_HALF) % CF_RING];
  const int lead = s.wr[(J + CF_RING - (CF_HALF + CF_G + 1)) % CF_RING];
  const int lag = s.w + xn - x20;
  s.w = lag;
  s.wr[J % CF_RING] = lag;
  s.xr[J % CF_RING] = xn;
  bool pass = false;
  if (!EDGE || (r >= CF_HALF && r < R - CF_HALF)) {
    const int S = ALG == SFE_CFAR_CA ? lead + lag : (ALG == SFE_CFAR_SOCA ? min(lead, lag) : max(lead, lag));
    pass = xc >= (int)lut[S];
  }
  if (MASK) obuf_ob[I][tid] = pass ? 1 : 0;
  if (BITS) {
    const unsigned b = __ballot_sync(0xffffffffu, pass && col_ok);
    if ((tid & 31) == I) keep_bits = b;  // lane i keeps the ballot of output row i
  }
}

template <int ALG, bool MASK, bool BITS, bool EDGE, int Q>
__device__ __forceinline__ void cfar_block16_u8(CfarStepI &s, uint8_t (*tile)[CF_CH][CF_W],
                                                uint8_t (*obuf)[CF_CH][CF_W], uint32_t (*obits)[CF_CH][CF_W / 32],
                                                uint64_t *full_bar, const CUtensorMap *in_map, const uint16_t *lut,
                                                const CfarParams &p, const int blk, const int nchunks,
                                                const int tid, const int f, const int col0) {
  const int r0 = (blk - 2) * CF_CH;
  const int cA = blk - 1, cB = blk;
  const bool hasA = EDGE ? (cA >= 0 && cA < nchunks) : true;
  const bool hasB = EDGE ? (cB < nchunks) : true;
  const uint8_t(*tileA)[CF_W] = tile[cA & (CF_NSTAGE_U8 - 1)];
  const uint8_t(*tileB)[CF_W] = tile[cB & (CF_NSTAGE_U8 - 1)];
  constexpr int ob = Q & 1;
  const bool col_ok = col0 + tid < p.B;
  unsigned keep_bits = 0;
  int xin[CF_CH];
#pragma unroll
  for (int i = 0; i < CF_SPLIT; ++i) xin[i] = (!EDGE || hasA) ? (int)tileA[i + CF_CH - CF_SPLIT][tid] : 0;
  if (hasB) mbar_wait(&full_bar[cB & (CF_NSTAGE_U8 - 1)], (cB / CF_NSTAGE_U8) & 1);
#pragma unroll
  for (int i = CF_SPLIT; i < CF_CH; ++i) xin[i] = (!EDGE || hasB) ? (int)tileB[i - CF_SPLIT][tid] : 0;
#define SFE_STEP(I) \
  cfar_step_u8<ALG, MASK, BITS, EDGE, Q * CF_CH + I>(s, xin[I], obuf[ob], lut, p.R, r0 + I, tid, col_ok, keep_bits);
  SFE_STEP(0) SFE_STEP(1) SFE_STEP(2) SFE_STEP(3) SFE_STEP(4) SFE_STEP(5) SFE_STEP(6) SFE_STEP(7)
  SFE_STEP(8) SFE_STEP(9) SFE_STEP(10) SFE_STEP(11) SFE_STEP(12) SFE_STEP(13) SFE_STEP(14) SFE_STEP(15)
#undef SFE_STEP
  if (EDGE && r0 < 0) {
    named_bar_sync(1, CF_W);
    cfar_refill<uint8_t, CF_NSTAGE_U8>(tile, full_bar, in_map, blk, nchunks, tid, f, col0);
    return;
  }
  if (BITS && (tid & 31) < CF_CH) obits[ob][tid & 31][tid >> 5] = keep_bits;
  if (MASK) fence_proxy_async_smem();
  if (MASK && tid == 0) tma_wait_read<0>();
  named_bar_sync(1, CF_W);
  cfar_refill<uint8_t, CF_NSTAGE_U8>(tile, full_bar, in_map, blk, nchunks, tid, f, col0);
  if (MASK && tid == 0) {
    tma_store_3d(p.out_map, &obuf[ob][0][0], col0, r0, f);
    tma_commit();
  }
  if (BITS && tid < CF_CH * (CF_W / 32)) {
    const int i = tid / (CF_W / 32), wq = tid % (CF_W / 32);
    const int w = (col0 >> 5) + wq;
    if (r0 + i < p.R && w < p.words_per_row)
      p.bits[((size_t)f * p.R + r0 + i) * p.words_per_row + w] = obits[ob][i][wq];
  }
}

template <int ALG, bool MASK, bool BITS>
__global__ void __launch_bounds__(CF_W, 5)
    cfar_u8_lut_kernel(const __grid_constant__ CUtensorMap in_map, const __grid_constant__ CUtensorMap out_map,
                       CfarParams p, const uint16_t *__restrict__ lut_g, const int lut_n) {
  __shared__ __align__(128) uint8_t tile[CF_NSTAGE_U8][CF_CH][CF_W];
  __shared__ __align__(128) uint8_t obuf[2][CF_CH][CF_W];
  __shared__ uint32_t obits[2][CF_CH][CF_W / 32];
  __shared__ __align__(8) uint64_t full_bar[CF_NSTAGE_U8];
  __shared__ __align__(16) uint16_t lut[(ALG == SFE_CFAR_CA ? CF_LUT_MAX : CF_T * 255 + 1) + 7];

  const int tid = threadIdx.x;
  const int f = blockIdx.x / p.strips;
  const int col0 = (blockIdx.x % p.strips) * CF_W;
  const int R = p.R;
  p.out_map = &out_map;
  const int nchunks = (R + CF_CH - 1) / CF_CH;

  if (tid == 0) {
    prefetch_tmap(&in_map);
    for (int st = 0; st < CF_NSTAGE_U8; ++st) mbar_init(&full_bar[st], 1);
    fence_mbar_init();
    for (int c = 0; c < CF_NSTAGE_U8 - 1 && c < nchunks; ++c) {
      mbar_arrive_expect_tx(&full_bar[c], CF_CH * CF_W);
      tma_load_3d(&tile[c][0][0], &in_map, &full_bar[c], col0, c * CF_CH, f);
    }
  }
  // 16-byte copies (the device table is padded to a multiple of 8 entries)
  for (int i = tid; i * 8 < lut_n; i += CF_W)
    reinterpret_cast<uint4 *>(lut)[i] = reinterpret_cast<const uint4 *>(lut_g)[i];
  __syncthreads();

  CfarStepI s;
#pragma unroll
  for (int i = 0; i < CF_RING; ++i) s.xr[i] = 0, s.wr[i] = 0;
  s.w = 0;
  const int nblk = nchunks + 2;
  for (int b2 = 0; b2 * 2 < nblk; ++b2) {
#pragma unroll
    for (int q = 0; q < 2; ++q) {
      const int blk = b2 * 2 + q;
      if (blk < nblk) {
        const int r0 = (blk - 2) * CF_CH;
        const bool interior = (r0 >= CF_HALF) && (r0 + CF_CH - 1 < R - CF_HALF);
#define SFE_BLOCK(EDGE_, Q_) \
  cfar_block16_u8<ALG, MASK, BITS, EDGE_, Q_>(s, tile, obuf, obits, full_bar, &in_map, lut, p, blk, nchunks, tid, f, col0)
        if (interior) {
          if (q == 0) SFE_BLOCK(false, 0); else SFE_BLOCK(false, 1);
        } else {
          if (q == 0) SFE_BLOCK(true, 0); else SFE_BLOCK(true, 1);
        }
#undef SFE_BLOCK
      }
    }
  }
  if (MASK && tid == 0) tma_wait_all<0>();
}

// ------------------------------------------------------------------------------------------------
// uint8 streaming kernel for the node's configuration (CFAR + amplitude gate fused, feature_extraction.py:223-224):
// FOUR beams per thread, SIMD inside 32-bit registers.  With the gate on, a cell can only be a detection when
// x >= g_min = min_S M[S] (M = the pass table of cfar_u8_lut_kernel; g_min is the gate for the shipped parameters),
// which holds for a few per cent of the cells of a sonar image (speckle tail + echoes).  The per-cell work is only
// what keeps the window statistic current; the table look-up / compare / bit set is done per CANDIDATE:
//   * one LDS.32 brings the new cells of 4 adjacent beams (bytes); the raw words also form the cell ring;
//   * window sums (<= 20*255 < 2^16) live as 16-bit lanes, two beams per register: PRMT spreads the bytes of the
//     entering and the leaving cell to 16-bit lanes, one IADD3 per beam pair updates the sums (lanes cannot carry
//     into each other: every lane stays in [0, 5100]); a 32-deep register delay line yields the leading sum and
//     VIMNMX.U16x2 the SOCA / GOCA statistic;
//   * "does any of the 4 cells under test reach g_min" is two integer instructions on the packed bytes
//     (((x + k) | x) & 0x80808080, k = (128 - g_min) * 0x01010101); a thread whose word qualifies parks
//     (cells, statistic) in its own shared-memory slot of that row with predicated stores and sets a bit in a
//     16-bit row mask -- the 16-row block is branch-free;
//   * after the block each warp compacts its parked (lane, row) pairs into a queue and decides them 32 at a time
//     against the table M[S] (atomicOr into a zero-initialised bit tile / byte stores into a mask tile): the
//     cost follows the NUMBER of candidates, not how they are spread over rows and lanes.
// 15 instructions per row of 4 cells, about half the warp instructions of the table kernel per frame.  All-integer,
// exact: identical to the table
// kernel by construction (the gate test is a necessary condition; the decision is the same table compare).
// A strip is 512 beams (128 threads x 4); 16-row chunks arrive by TMA as two [16 x 256] boxes per stage.  Block b
// consumes chunk b (newest cell rn = 16 b + i) and decides cell r = rn - 25, so every block touches ONE tile.
// The four warps of a CTA only share the tiles: no CTA barrier in the loop (see cfar_block16_g).
constexpr int CG_BEAMS = 4;
constexpr int CG_W = CF_W * CG_BEAMS;  // beams per strip
// Ring depth / occupancy: 2 stages with 4 CTAs per SM (128 registers, 55 KB of shared memory each) -- the kernel is
// latency-bound, so a fourth CTA per SM buys more than a deeper ring (chosen on replay frames; not re-measured on
// H100).
#ifndef SFE_CG_NS
#define SFE_CG_NS 2    // input ring depth (stages of 16 rows x 512 beams)
#endif
#ifndef SFE_CG_MINB
#define SFE_CG_MINB 4  // CTAs per SM the register budget is set for
#endif
constexpr int CG_NS = SFE_CG_NS;
constexpr int CG_GMIN_LO = 16;         // below this nearly every word qualifies: use the table kernel

struct CfarStepG {
  uint32_t xr[CF_RING];                // cells, 4 beams per word
  uint32_t wl[CF_RING], wh[CF_RING];   // window sums W[rn - a]: beams 0,1 / beams 2,3 as 16-bit lanes
  uint32_t w_lo, w_hi;                 // W[rn - 1]
  uint32_t hit;                        // rows of the current block with a parked candidate word
};

// shared-memory layout of cfar_u8_gate4_kernel (dynamic): tile [CG_NS][2][16][256] | obits [16][16] |
// full_bar [CG_NS] + stage counters [CG_NS] | parked statistic [16][128] uint2 | parked cells [16][128] u32 | candidate queues [4][512] u16 |
// lut [lut_n padded to 8] | omask [16][512] (MASK only)
constexpr size_t CG_OFF_OBITS = (size_t)CG_NS * CF_CH * CG_W;
constexpr size_t CG_OFF_BAR = CG_OFF_OBITS + sizeof(uint32_t) * CF_CH * (CG_W / 32);
constexpr size_t CG_OFF_RECS = CG_OFF_BAR + 64;
constexpr size_t CG_OFF_RECX = CG_OFF_RECS + sizeof(uint2) * CF_CH * CF_W;
constexpr size_t CG_OFF_WQ = CG_OFF_RECX + sizeof(uint32_t) * CF_CH * CF_W;  // per-warp candidate queues [4][512] u16
constexpr size_t CG_OFF_LUT = CG_OFF_WQ + sizeof(uint16_t) * (CF_W / 32) * 32 * CF_CH;
__host__ __device__ __forceinline__ size_t cg_off_omask(int lut_n) {
  return CG_OFF_LUT + ((sizeof(uint16_t) * (size_t)((lut_n + 7) / 8 * 8) + 15) & ~size_t(15));
}
extern __shared__ __align__(128) unsigned char cg_smem[];

template <int ALG, int J>
__device__ __forceinline__ void cfar_step_g(CfarStepG &s, const uint32_t xn4, const uint32_t gate_add,
                                            uint2 (*rec_s)[CF_W], uint32_t (*rec_x)[CF_W], const int tid) {
  constexpr int I = J % CF_CH;
  const uint32_t x20 = s.xr[(J + CF_RING - CF_T) % CF_RING];
  const uint32_t xc4 = s.xr[(J + CF_RING - CF_HALF) % CF_RING];
  const uint32_t lead_lo = s.wl[(J + CF_RING - (CF_HALF + CF_G + 1)) % CF_RING];
  const uint32_t lead_hi = s.wh[(J + CF_RING - (CF_HALF + CF_G + 1)) % CF_RING];
  const uint32_t lag_lo = s.w_lo + __byte_perm(xn4, 0u, 0x4140u) - __byte_perm(x20, 0u, 0x4140u);
  const uint32_t lag_hi = s.w_hi + __byte_perm(xn4, 0u, 0x4342u) - __byte_perm(x20, 0u, 0x4342u);
  s.w_lo = lag_lo, s.w_hi = lag_hi;
  s.wl[J % CF_RING] = lag_lo, s.wh[J % CF_RING] = lag_hi;
  s.xr[J % CF_RING] = xn4;
  uint32_t s_lo, s_hi;
  if (ALG == SFE_CFAR_CA) s_lo = lead_lo + lag_lo, s_hi = lead_hi + lag_hi;  // <= 10200 per lane
  else if (ALG == SFE_CFAR_SOCA) s_lo = __vminu2(lead_lo, lag_lo), s_hi = __vminu2(lead_hi, lag_hi);
  else s_lo = __vmaxu2(lead_lo, lag_lo), s_hi = __vmaxu2(lead_hi, lag_hi);
  // any of the four cells under test >= g_min?  (a carry out of a byte only happens when that byte already
  // qualifies, so the any-test is exact; which bytes pass is settled against the table after the block)
  if (((xc4 + gate_add) | xc4) & 0x80808080u) {  // (predicated stores, no branch)
    rec_s[I][tid] = make_uint2(s_lo, s_hi);
    rec_x[I][tid] = xc4;
    s.hit |= 1u << I;
  }
}

// One 16-row block of one WARP (128 beams).  The four warps of a CTA share the TMA tiles and nothing else: each has
// its own slice of the output tiles, its own parked records and queue, so there is no CTA barrier in the loop --
// an echo-rich warp does not hold the others up.  A stage of the input ring is refilled by whichever warp is the
// last to have read it (a shared-memory counter per stage; the reads are ordered before the TMA write by the
// fences around the counter update).
template <int ALG, bool MASK, bool BITS, bool EDGE, int Q>
__device__ __forceinline__ void cfar_block16_g(CfarStepG &s, uint8_t (*tile)[2][CF_CH][CG_W / 2],
                                               uint32_t (*obits)[CG_W / 32], uint8_t (*omask)[CG_W],
                                               uint64_t *full_bar, int *stage_cnt, const CUtensorMap *in_map,
                                               const uint16_t *__restrict__ lut, const CfarParams &p, const int blk,
                                               const int nchunks, const int tid, const int f, const int col0,
                                               const uint32_t gate_add) {
  const int r0 = blk * CF_CH - CF_HALF;  // first output row of this block
  const int st = blk & (CG_NS - 1);
  const bool has = EDGE ? (blk < nchunks) : true;
  const int lane = tid & 31, warp = tid >> 5, wbase = tid & ~31;
  uint2(*rec_s)[CF_W] = reinterpret_cast<uint2(*)[CF_W]>(cg_smem + CG_OFF_RECS);
  uint32_t(*rec_x)[CF_W] = reinterpret_cast<uint32_t(*)[CF_W]>(cg_smem + CG_OFF_RECX);
  uint32_t xin[CF_CH];
  if (has) {
    mbar_wait(&full_bar[st], (blk / CG_NS) & 1);
    const uint32_t *trow = reinterpret_cast<const uint32_t *>(&tile[st][tid >> 6][0][(tid & 63) * CG_BEAMS]);
#pragma unroll
    for (int i = 0; i < CF_CH; ++i) xin[i] = trow[i * (CG_W / 2 / 4)];
  } else {
#pragma unroll
    for (int i = 0; i < CF_CH; ++i) xin[i] = 0u;  // below the image: zero cells (never decide anything)
  }
  s.hit = 0u;
#define SFE_STEP(I) cfar_step_g<ALG, Q * CF_CH + I>(s, xin[I], gate_add, rec_s, rec_x, tid);
  SFE_STEP(0) SFE_STEP(1) SFE_STEP(2) SFE_STEP(3) SFE_STEP(4) SFE_STEP(5) SFE_STEP(6) SFE_STEP(7)
  SFE_STEP(8) SFE_STEP(9) SFE_STEP(10) SFE_STEP(11) SFE_STEP(12) SFE_STEP(13) SFE_STEP(14) SFE_STEP(15)
#undef SFE_STEP
  // ---- this warp is done with tile[st]: the last of the four warps to say so refills the stage
  if (has) {
    __syncwarp();
    if (lane == 0) {
      __threadfence_block();  // our reads of the tile come before the counter update ...
      if (atomicAdd(&stage_cnt[st], 1) == CF_W / 32 - 1) {
        stage_cnt[st] = 0;
        __threadfence_block();  // ... and everybody's counter update before the refill
        if (blk + CG_NS < nchunks) {
          mbar_arrive_expect_tx(&full_bar[st], CF_CH * CG_W);
          tma_load_3d(&tile[st][0][0][0], in_map, &full_bar[st], col0, (blk + CG_NS) * CF_CH, f);
          tma_load_3d(&tile[st][1][0][0], in_map, &full_bar[st], col0 + CG_W / 2, (blk + CG_NS) * CF_CH, f);
        }
      }
    }
  }
  // ---- the parked candidates: the reference's compare, via the table.  Echoes make candidates a few per cent of
  //      the cells and put them in runs (a wall crosses a lane on two or three consecutive rows), so a lane
  //      walking its own list would keep its warp for as many trips as the unluckiest lane has rows.  Instead the
  //      warp compacts its (lane, row) pairs into a small queue (prefix sum of the per-lane counts, each lane
  //      appends its own rows) and then decides them 32 at a time.
  {
    uint16_t *wq = reinterpret_cast<uint16_t *>(cg_smem + CG_OFF_WQ) + warp * (32 * CF_CH);
    uint32_t hit = s.hit;
    if (EDGE) {  // border rows stay 0: keep only rows r0 + i in [HALF, R - HALF)
      const int lo = max(CF_HALF - r0, 0), hi = min(p.R - CF_HALF - r0, CF_CH);
      hit &= hi > lo ? ((1u << hi) - (1u << lo)) : 0u;
    }
    const int cnt = __popc(hit);
    int incl = cnt;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const int t = __shfl_up_sync(0xffffffffu, incl, d);
      if (lane >= d) incl += t;
    }
    const int tot = __shfl_sync(0xffffffffu, incl, 31);
    if (tot) {  // (warp-uniform)
      int pos = incl - cnt;
      while (hit) {
        const int i = __ffs(hit) - 1;
        hit &= hit - 1;
        wq[pos++] = (uint16_t)((lane << 4) | i);
      }
      __syncwarp();  // queue and parked records (written by other lanes of this warp) are visible
      for (int e = lane; e < tot; e += 32) {
        const int code = wq[e], i = code & 15, t = wbase + (code >> 4);
        const uint2 sv = rec_s[i][t];
        const uint32_t xc4 = rec_x[i][t];
        const int nv = min(max(p.B - (col0 + CG_BEAMS * t), 0), CG_BEAMS);
        uint32_t set = 0;
#pragma unroll
        for (int k = 0; k < CG_BEAMS; ++k) {
          const int x = (int)((xc4 >> (8 * k)) & 255u);
          const int S = (int)(((k < 2 ? sv.x : sv.y) >> (16 * (k & 1))) & 0xffffu);
          if (k < nv && x >= (int)lut[S]) set |= 1u << k;
        }
        if (set) {
          if (BITS) atomicOr(&obits[i][t >> 3], set << ((t & 7) * CG_BEAMS));
          if (MASK)  // bytes 0/1 of the four beams: spread the 4 bits to 4 bytes
            *reinterpret_cast<uint32_t *>(&omask[i][CG_BEAMS * t]) =
                (set & 1u) | ((set & 2u) << 7) | ((set & 4u) << 14) | ((set & 8u) << 21);
        }
      }
    }
    __syncwarp();  // the warp's slice of the output tiles is complete
  }
  if (EDGE && r0 + CF_CH <= 0) return;  // nothing to write yet (and nothing was set)
  // ---- hand the warp's 16 rows x 128 beams to global memory and clear them for the next block
  if (BITS) {
    const int i = lane >> 1, wq2 = warp * (CF_W / 32) + (lane & 1) * 2;  // 16 rows x 4 words = 32 x uint2
    uint2 *src = reinterpret_cast<uint2 *>(&obits[i][wq2]);
    const uint2 v = *src;
    *src = make_uint2(0u, 0u);
    const int r = r0 + i, w = (col0 >> 5) + wq2;
    if (r >= 0 && r < p.R) {
      uint32_t *dst = p.bits + ((size_t)f * p.R + r) * p.words_per_row + w;
      if (w + 1 < p.words_per_row && (reinterpret_cast<uintptr_t>(dst) & 7u) == 0) {
        *reinterpret_cast<uint2 *>(dst) = v;
      } else {
        if (w < p.words_per_row) dst[0] = v.x;
        if (w + 1 < p.words_per_row) dst[1] = v.y;
      }
    }
  }
  if (MASK) {
#pragma unroll
    for (int j = 0; j < CF_CH * (CG_W / 4 / 16) / 32; ++j) {  // 16 rows x 8 uint4 (this warp's 128 beams) over 32 lanes
      const int idx = lane + j * 32, i = idx >> 3, sg = idx & 7;
      uint4 *src = reinterpret_cast<uint4 *>(&omask[i][warp * (CG_W / 4) + sg * 16]);
      const uint4 v = *src;
      *src = make_uint4(0u, 0u, 0u, 0u);
      const int r = r0 + i, c = col0 + warp * (CG_W / 4) + sg * 16;
      if (r >= 0 && r < p.R && c < p.B)  // B % 16 == 0 and mask 16-byte aligned (checked by the host)
        *reinterpret_cast<uint4 *>(p.mask + ((size_t)f * p.R + r) * p.B + c) = v;
    }
  }
  __syncwarp();
}

template <int ALG, bool MASK, bool BITS>
__global__ void __launch_bounds__(CF_W, MASK ? SFE_CG_MINB - 1 : SFE_CG_MINB)
    cfar_u8_gate4_kernel(const __grid_constant__ CUtensorMap in_map, CfarParams p, const uint16_t *__restrict__ lut_g,
                         const int lut_n, const uint32_t gate_add) {
  uint8_t(*tile)[2][CF_CH][CG_W / 2] = reinterpret_cast<uint8_t(*)[2][CF_CH][CG_W / 2]>(cg_smem);
  uint32_t(*obits)[CG_W / 32] = reinterpret_cast<uint32_t(*)[CG_W / 32]>(cg_smem + CG_OFF_OBITS);
  uint64_t *full_bar = reinterpret_cast<uint64_t *>(cg_smem + CG_OFF_BAR);
  int *stage_cnt = reinterpret_cast<int *>(cg_smem + CG_OFF_BAR + 8 * CG_NS);
  uint16_t *lut = reinterpret_cast<uint16_t *>(cg_smem + CG_OFF_LUT);
  uint8_t(*omask)[CG_W] = reinterpret_cast<uint8_t(*)[CG_W]>(cg_smem + cg_off_omask(lut_n));

  const int tid = threadIdx.x;
  const int f = blockIdx.x / p.strips;
  const int col0 = (blockIdx.x % p.strips) * CG_W;
  const int R = p.R;
  const int nchunks = (R + CF_CH - 1) / CF_CH;
  if (tid == 0) {
    prefetch_tmap(&in_map);
    for (int st = 0; st < CG_NS; ++st) mbar_init(&full_bar[st], 1), stage_cnt[st] = 0;
    fence_mbar_init();
    for (int c = 0; c < CG_NS && c < nchunks; ++c) {
      mbar_arrive_expect_tx(&full_bar[c], CF_CH * CG_W);
      tma_load_3d(&tile[c][0][0][0], &in_map, &full_bar[c], col0, c * CF_CH, f);
      tma_load_3d(&tile[c][1][0][0], &in_map, &full_bar[c], col0 + CG_W / 2, c * CF_CH, f);
    }
  }
  for (int i = tid; i * 8 < lut_n; i += CF_W) reinterpret_cast<uint4 *>(lut)[i] = reinterpret_cast<const uint4 *>(lut_g)[i];
  if (BITS)
    for (int i = tid; i < CF_CH * (CG_W / 32); i += CF_W) (&obits[0][0])[i] = 0u;
  if (MASK)
    for (int i = tid; i < CF_CH * CG_W / 16; i += CF_W) reinterpret_cast<uint4 *>(&omask[0][0])[i] = make_uint4(0u, 0u, 0u, 0u);
  __syncthreads();

  CfarStepG s;
#pragma unroll
  for (int i = 0; i < CF_RING; ++i) s.xr[i] = 0u, s.wl[i] = 0u, s.wh[i] = 0u;
  s.w_lo = 0u, s.w_hi = 0u, s.hit = 0u;
  // block b: newest cells rn = 16 b .. 16 b + 15, decides rows rn - 25; the last decided row is R - 1
  const int nblk = (R + CF_HALF + CF_CH - 1) / CF_CH;
  for (int b2 = 0; b2 * 2 < nblk; ++b2) {
#pragma unroll
    for (int q = 0; q < 2; ++q) {
      const int blk = b2 * 2 + q;
      if (blk < nblk) {
        const int r0 = blk * CF_CH - CF_HALF;
        const bool interior = (r0 >= CF_HALF) && (r0 + CF_CH - 1 < R - CF_HALF) && blk < nchunks;
#define SFE_BLOCK(EDGE_, Q_) \
  cfar_block16_g<ALG, MASK, BITS, EDGE_, Q_>(s, tile, obits, omask, full_bar, stage_cnt, &in_map, lut, p, blk, nchunks, tid, f, col0, gate_add)
        if (interior) {
          if (q == 0) SFE_BLOCK(false, 0); else SFE_BLOCK(false, 1);
        } else {
          if (q == 0) SFE_BLOCK(true, 0); else SFE_BLOCK(true, 1);
        }
#undef SFE_BLOCK
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// OS-CFAR on uint8 images (cfar.cpp:76-96): the k-th smallest of the 2T training cells.  One thread per
// beam marches down the range axis keeping a 256-bin histogram of its current training window (byte
// counters, four per 32-bit word, word-interleaved over the 128 threads of the CTA so every access is
// conflict free) and the running order statistic (value v, number of cells below it): moving one range bin
// removes two cells and adds two, after which v moves by at most a few bins (Huang's sliding median,
// generalised to rank k).  The double compare `x > tau * v` and the amplitude gate come from a 256-entry
// table built on the host with the reference's expression.  Any train_hs <= 127 / guard_hs.
__global__ void __launch_bounds__(CF_W) cfar_os_hist_kernel(const uint8_t *__restrict__ img, const CfarParams p,
                                                            const uint16_t *__restrict__ lut_g) {
  __shared__ uint32_t hs[64 * CF_W];
  __shared__ uint16_t lut[256];
  const int tid = threadIdx.x;
  const int f = blockIdx.x / p.strips;
  const int col0 = (blockIdx.x % p.strips) * CF_W;
  const int col = col0 + tid;
  const bool live = col < p.B;
  const int R = p.R, B = p.B, T = p.T, G = p.G, half = T + G, k = p.k;
  const uint8_t *colp = img + (size_t)f * R * B + (live ? col : 0);
  for (int i = tid; i < 256; i += CF_W) lut[i] = lut_g[i];
  for (int w = 0; w < 64; ++w) hs[w * CF_W + tid] = 0;
  __syncthreads();
  auto cnt = [&](int v) -> int { return (int)((hs[(v >> 2) * CF_W + tid] >> ((v & 3) * 8)) & 0xffu); };
  auto bump = [&](int v, int up) {
    const uint32_t d = 1u << ((v & 3) * 8);
    if (up) hs[(v >> 2) * CF_W + tid] += d; else hs[(v >> 2) * CF_W + tid] -= d;
  };
  const int r_first = half, r_last = R - half - 1;  // rows with a full window
  int v = 0, below = 0;
  if (r_first <= r_last) {
    for (int i = r_first - half; i <= r_first + half; ++i)
      if (abs(i - r_first) > G) bump(colp[(size_t)i * B], 1);
    while (below + cnt(v) <= k) below += cnt(v), ++v;
  }
  for (int r = 0; r < R; ++r) {
    bool pass = false;
    if (r >= r_first && r <= r_last) {
      const int xc = colp[(size_t)r * B];
      pass = live && xc >= (int)lut[v];
      if (p.thr != nullptr && live) p.thr[((size_t)f * R + r) * B + col] = (float)(p.tau * (double)(float)v);
      if (r < r_last) {  // slide the window to r + 1
        const int a_out = colp[(size_t)(r - half) * B], a_in = colp[(size_t)(r - G) * B];
        const int b_out = colp[(size_t)(r + G + 1) * B], b_in = colp[(size_t)(r + half + 1) * B];
        bump(a_out, 0), bump(a_in, 1), bump(b_out, 0), bump(b_in, 1);
        below += (a_in < v) + (b_in < v) - (a_out < v) - (b_out < v);
        while (below > k) --v, below -= cnt(v);
        while (below + cnt(v) <= k) below += cnt(v), ++v;
      }
    }
    if (p.mask != nullptr && live) p.mask[((size_t)f * R + r) * B + col] = pass ? 1 : 0;
    if (p.bits != nullptr) {
      const unsigned bal = __ballot_sync(0xffffffffu, pass);
      const int w = (col0 >> 5) + (tid >> 5);
      if ((tid & 31) == 0 && w < p.words_per_row) p.bits[((size_t)f * R + r) * p.words_per_row + w] = bal;
    }
  }
}

// General / exact path.  One CTA per (frame, strip of CF_W beams); thread = beam.
template <typename InT>
__global__ void __launch_bounds__(CF_W) cfar_exact_kernel(const InT *__restrict__ img, const CfarParams p,
                                                          const uint8_t *__restrict__ only_flagged) {
  extern __shared__ float train_smem[];  // OS only: [2*T][CF_W]
  if (only_flagged != nullptr && only_flagged[blockIdx.x] == 0) return;
  const int tid = threadIdx.x;
  const int f = blockIdx.x / p.strips;
  const int col0 = (blockIdx.x % p.strips) * CF_W;
  const int col = col0 + tid;
  const bool live = col < p.B;
  const int R = p.R, B = p.B;
  const int half = p.T + p.G;
  const InT *colp = img + (size_t)f * R * B + (live ? col : 0);

  for (int r = 0; r < R; ++r) {
    bool pass = false;
    if (r >= half && r < R - half) {
      double d;
      pass = cfar_cell_exact<InT>(colp, (size_t)B, r, p, train_smem + tid, CF_W, &d);
      if (p.thr != nullptr && live) p.thr[((size_t)f * R + r) * B + col] = (float)d;
    }
    pass = pass && live;
    if (p.mask != nullptr && live) p.mask[((size_t)f * R + r) * B + col] = pass ? 1 : 0;
    if (p.bits != nullptr) {
      const unsigned b = __ballot_sync(0xffffffffu, pass);
      const int w = (col0 >> 5) + (tid >> 5);
      if ((tid & 31) == 0 && w < p.words_per_row) p.bits[((size_t)f * R + r) * p.words_per_row + w] = b;
    }
  }
}

// ---------------------------------------------------------------------------- host side
// float g such that (x > g) <=> ((double)x > t) for every float x
static float gate_as_float(double t) {
  if (t != t) return __builtin_nanf("");  // x > nan is false, like numpy
  if (t >= 3.4028234663852886e38) return 3.4028234663852886e38f;  // only +inf can pass
  if (t < -3.4028234663852886e38) return -INFINITY;
  float g = (float)t;
  if ((double)g > t) g = nextafterf(g, -INFINITY);  // largest float <= t
  return g;
}

template <typename InT, int ALG, bool WITH_THR, bool MASK, bool BITS>
static int launch_ring(sfe_ctx *ctx, cudaStream_t st, const CUtensorMap &in_map, const CUtensorMap &out_map, const CfarParams &p) {
  cfar_ring_tma_kernel<InT, ALG, WITH_THR, MASK, BITS>
      <<<p.F * p.strips, CF_W, 0, st>>>(in_map, out_map, p);
  SFE_CUDA(cudaGetLastError());
  ctx->launches++;
  return SFE_OK;
}

template <typename InT, int ALG, bool WITH_THR>
static int launch_ring_out(sfe_ctx *ctx, cudaStream_t st, const CUtensorMap &in_map, const CUtensorMap &out_map, const CfarParams &p) {
  const bool m = p.mask != nullptr, b = p.bits != nullptr;
  if (m && b) return launch_ring<InT, ALG, WITH_THR, true, true>(ctx, st, in_map, out_map, p);
  if (m) return launch_ring<InT, ALG, WITH_THR, true, false>(ctx, st, in_map, out_map, p);
  if (b) return launch_ring<InT, ALG, WITH_THR, false, true>(ctx, st, in_map, out_map, p);
  if constexpr (WITH_THR) return launch_ring<InT, ALG, true, false, false>(ctx, st, in_map, out_map, p);
  return SFE_OK;  // nothing to write
}

template <typename InT, bool WITH_THR>
static int launch_ring_alg(sfe_ctx *ctx, cudaStream_t st, const CUtensorMap &in_map, const CUtensorMap &out_map, const CfarParams &p) {
  switch (p.alg) {
    case SFE_CFAR_CA:
      return launch_ring_out<InT, SFE_CFAR_CA, WITH_THR>(ctx, st, in_map, out_map, p);
    case SFE_CFAR_SOCA:
      return launch_ring_out<InT, SFE_CFAR_SOCA, WITH_THR>(ctx, st, in_map, out_map, p);
    default:
      return launch_ring_out<InT, SFE_CFAR_GOCA, WITH_THR>(ctx, st, in_map, out_map, p);
  }
}

// smallest uint8 value x with (double)x > d; 256 when there is none (d >= 255 or NaN)
static int u8_above(double d) {
  if (d != d || d >= 255.0) return 256;
  return d < 0 ? 0 : (int)floor(d) + 1;
}

// M[S] = smallest uint8 cell value x with (double)x > tau*S/div (the reference's compare) and
// (double)x > gate (the node's amplitude gate); 256 = no value passes.
static void build_u8_lut(const CfarParams &p, std::vector<uint16_t> &lut) {
  const int n = (p.alg == SFE_CFAR_CA ? 2 : 1) * CF_T * 255 + 1;
  lut.resize(n);
  const int g = p.gate_on ? u8_above(p.gate_d) : 0;
  for (int S = 0; S < n; ++S) {
    const int m = u8_above(p.tau * (double)(float)S / p.div);
    lut[S] = (uint16_t)(m > g ? m : g);
  }
}

template <int ALG>
static int launch_u8_lut(sfe_ctx *ctx, cudaStream_t st, const CUtensorMap &in_map, const CUtensorMap &out_map, const CfarParams &p,
                         const uint16_t *lut, int lut_n) {
  const bool m = p.mask != nullptr, b = p.bits != nullptr;
  const int grid = p.F * p.strips, thr = CF_W;
  if (m && b) cfar_u8_lut_kernel<ALG, true, true><<<grid, thr, 0, st>>>(in_map, out_map, p, lut, lut_n);
  else if (m) cfar_u8_lut_kernel<ALG, true, false><<<grid, thr, 0, st>>>(in_map, out_map, p, lut, lut_n);
  else if (b) cfar_u8_lut_kernel<ALG, false, true><<<grid, thr, 0, st>>>(in_map, out_map, p, lut, lut_n);
  else return SFE_OK;
  SFE_CUDA(cudaGetLastError());
  ctx->launches++;
  return SFE_OK;
}

template <int ALG>
static int launch_u8_gate4(sfe_ctx *ctx, cudaStream_t st, const CUtensorMap &in_map, const CfarParams &p, const uint16_t *lut, int lut_n,
                           uint32_t gate_add) {
  const bool m = p.mask != nullptr, b = p.bits != nullptr;
  const int grid = p.F * p.strips;
  const size_t smem = cg_off_omask(lut_n) + (m ? CF_CH * CG_W : 0);
#define SFE_GO(M_, B_)                                                                                              \
  do {                                                                                                              \
    const int rc = raise_smem_limit(ctx, (const void *)cfar_u8_gate4_kernel<ALG, M_, B_>, smem);                    \
    if (rc != SFE_OK) return rc;                                                                                    \
    cfar_u8_gate4_kernel<ALG, M_, B_><<<grid, CF_W, smem, st>>>(in_map, p, lut, lut_n, gate_add);          \
  } while (0)
  if (m && b) SFE_GO(true, true);
  else if (m) SFE_GO(true, false);
  else SFE_GO(false, true);
#undef SFE_GO
  SFE_CUDA(cudaGetLastError());
  ctx->launches++;
  return SFE_OK;
}

template <typename InT>
static int launch_exact(sfe_ctx *ctx, cudaStream_t st, const InT *img, const CfarParams &p, const uint8_t *only_flagged) {
  size_t smem = 0;
  if (p.alg == SFE_CFAR_OS) {
    smem = (size_t)2 * p.T * CF_W * sizeof(float);
    if (smem > 48 * 1024) {
      if (smem > (size_t)ctx->max_smem_optin) {
        set_error("OS-CFAR: train_hs=%d needs %zu B of shared memory (max %d)", p.T, smem, ctx->max_smem_optin);
        return SFE_ERR_UNSUPPORTED;
      }
      const int rc = raise_smem_limit(ctx, (const void *)cfar_exact_kernel<InT>, smem);
      if (rc != SFE_OK) return rc;
    }
  }
  cfar_exact_kernel<InT><<<p.F * p.strips, CF_W, smem, st>>>(img, p, only_flagged);
  SFE_CUDA(cudaGetLastError());
  ctx->launches++;
  return SFE_OK;
}

}  // namespace sfe

int sfe::cfar_run(sfe_ctx *ctx, cudaStream_t st, const void *img, int dtype, int F, int R, int B, int alg, int T, int G,
                  int k, double tau, int gate_on, double gate, uint8_t *mask, float *thr, uint32_t *bits) {
  SFE_REQUIRE(ctx != nullptr, "cfar: null context");
  SFE_REQUIRE(img != nullptr || F == 0, "cfar: null image pointer");
  SFE_REQUIRE(dtype == SFE_U8 || dtype == SFE_F32, "cfar: dtype must be SFE_U8 or SFE_F32 (got %d)", dtype);
  SFE_REQUIRE(F >= 0 && R >= 0 && B >= 0, "cfar: negative shape (%d, %d, %d)", F, R, B);
  SFE_REQUIRE(alg >= SFE_CFAR_CA && alg <= SFE_CFAR_OS, "cfar: unknown variant %d", alg);
  SFE_REQUIRE(T >= 0 && G >= 0, "cfar: train_hs/guard_hs must be >= 0 (got %d, %d)", T, G);
  SFE_REQUIRE(alg != SFE_CFAR_OS || (k >= 0 && k < 2 * T), "cfar: OS rank k=%d outside [0, %d)", k, 2 * T);
  if (F == 0 || R == 0 || B == 0) return SFE_OK;

  CfarParams p{};
  p.F = F, p.R = R, p.B = B;
  p.strips = (B + CF_W - 1) / CF_W;
  p.alg = alg, p.T = T, p.G = G, p.k = k;
  p.tau = tau;
  p.div = alg == SFE_CFAR_CA ? 2.0 * T : (alg == SFE_CFAR_OS ? 1.0 : (double)T);
  const double c = tau / p.div;
  p.c_hi = (float)c;
  p.c_lo = (float)(c - (double)p.c_hi);
  p.gate_on = gate_on != 0;
  p.gate_d = gate;
  p.gate_f = gate_as_float(gate);
  p.img = img;
  p.mask = mask, p.thr = thr, p.bits = bits;
  p.words_per_row = (B + 31) / 32;
  const size_t es = dtype == SFE_U8 ? 1 : 4;

  // the streaming path's preconditions (shape of the register rings; TMA alignment rules; a slope
  // whose two-float split is accurate)
  bool fast = T == CF_T && G == CF_G && alg != SFE_CFAR_OS && R > 2 * CF_HALF;
  fast = fast && ((uintptr_t)img % 16 == 0) && ((size_t)B * es % 16 == 0);
  if (mask != nullptr) fast = fast && ((uintptr_t)mask % 16 == 0) && (B % 16 == 0);
  fast = fast && isfinite(c) && fabs(c) > 1e-20 && fabs(c) < 1e20;

  if (thr != nullptr) SFE_CUDA(cudaMemsetAsync(thr, 0, (size_t)F * R * B * sizeof(float), st));

  if (fast) {
    CUtensorMap in_map, out_map;
    int rc = encode_tensor_map_3d(&in_map, dtype == SFE_U8 ? CU_TENSOR_MAP_DATA_TYPE_UINT8 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32,
                                  es, img, B, R, F, CF_W, CF_CH, 1);
    if (rc != SFE_OK) return rc;
    if (mask != nullptr) {
      rc = encode_tensor_map_3d(&out_map, CU_TENSOR_MAP_DATA_TYPE_UINT8, 1, mask, B, R, F, CF_W, CF_CH, 1);
      if (rc != SFE_OK) return rc;
    } else {
      out_map = in_map;  // unused
    }
    if (dtype == SFE_F32) {
      rc = ensure(ctx, ctx->scratch[SCR_CFAR_FLAGS], (size_t)F * p.strips, st);
      if (rc != SFE_OK) return rc;
      p.flags = (uint8_t *)ctx->scratch[SCR_CFAR_FLAGS].ptr;
      SFE_CUDA(cudaMemsetAsync(p.flags, 0, (size_t)F * p.strips, st));
      rc = thr != nullptr ? launch_ring_alg<float, true>(ctx, st, in_map, out_map, p)
                          : launch_ring_alg<float, false>(ctx, st, in_map, out_map, p);
      if (rc != SFE_OK) return rc;
      return launch_exact<float>(ctx, st, (const float *)img, p, p.flags);  // re-does flagged strips only
    }
    if (thr == nullptr) {  // (tau is finite: `fast` requires a finite tau / div)
      // integer kernels with the threshold table (re-uploaded only when the parameters change; the cache key lives
      // in the context next to the buffer it describes)
      std::vector<uint16_t> lut_host;
      build_u8_lut(p, lut_host);
      const int lut_n = (int)lut_host.size();
      int g_min = 256;
      for (uint16_t v : lut_host) g_min = v < g_min ? v : g_min;
      lut_host.resize((lut_host.size() + 7) / 8 * 8, 256);  // pad for the kernels' 16-byte copies
      rc = ensure(ctx, ctx->scratch[SCR_CFAR_LUT], 65536, st);  // [0, 32 KiB): this table, [32 KiB, 64 KiB): the OS table
      if (rc != SFE_OK) return rc;
      const double k6[6] = {(double)alg, tau, (double)p.gate_on, p.gate_d, (double)lut_host.size(), 1.0};
      if (memcmp(k6, ctx->cfar_lut_key, sizeof(k6)) != 0 || ctx->cfar_lut_buf != ctx->scratch[SCR_CFAR_LUT].ptr) {
        SFE_CUDA(cudaMemcpyAsync(ctx->scratch[SCR_CFAR_LUT].ptr, lut_host.data(), lut_host.size() * sizeof(uint16_t),
                                 cudaMemcpyHostToDevice, st));
        SFE_CUDA(cudaStreamSynchronize(st));  // lut_host is a local
        memcpy(ctx->cfar_lut_key, k6, sizeof(k6));
        ctx->cfar_lut_buf = ctx->scratch[SCR_CFAR_LUT].ptr;
      }
      const uint16_t *lut = (const uint16_t *)ctx->scratch[SCR_CFAR_LUT].ptr;
      const int n = lut_n;
      if (g_min >= CG_GMIN_LO && g_min <= 128 && (mask != nullptr || bits != nullptr)) {
        // gated 4-beams-per-thread kernel: its own tensor map (two [16 x 256] boxes per chunk)
        CUtensorMap in4;
        rc = encode_tensor_map_3d(&in4, CU_TENSOR_MAP_DATA_TYPE_UINT8, 1, img, B, R, F, CG_W / 2, CF_CH, 1);
        if (rc != SFE_OK) return rc;
        CfarParams q = p;
        q.strips = (B + CG_W - 1) / CG_W;
        const uint32_t gate_add = 0x01010101u * (uint32_t)(128 - g_min);
        switch (alg) {
          case SFE_CFAR_CA: return launch_u8_gate4<SFE_CFAR_CA>(ctx, st, in4, q, lut, n, gate_add);
          case SFE_CFAR_SOCA: return launch_u8_gate4<SFE_CFAR_SOCA>(ctx, st, in4, q, lut, n, gate_add);
          default: return launch_u8_gate4<SFE_CFAR_GOCA>(ctx, st, in4, q, lut, n, gate_add);
        }
      }
      switch (alg) {
        case SFE_CFAR_CA: return launch_u8_lut<SFE_CFAR_CA>(ctx, st, in_map, out_map, p, lut, n);
        case SFE_CFAR_SOCA: return launch_u8_lut<SFE_CFAR_SOCA>(ctx, st, in_map, out_map, p, lut, n);
        default: return launch_u8_lut<SFE_CFAR_GOCA>(ctx, st, in_map, out_map, p, lut, n);
      }
    }
    return launch_ring_alg<uint8_t, true>(ctx, st, in_map, out_map, p);  // uint8 with a threshold image
  }
  if (dtype == SFE_U8 && alg == SFE_CFAR_OS && T >= 1 && T <= 127 && R > 2 * (T + G) && isfinite(tau)) {
    // sliding-histogram OS-CFAR; 256-entry pass table M[v] = smallest cell value with x > tau*v (and the gate)
    std::vector<uint16_t> lut(256);
    const int g = p.gate_on ? u8_above(p.gate_d) : 0;
    for (int v = 0; v < 256; ++v) {
      const int m = u8_above(tau * (double)(float)v);
      lut[v] = (uint16_t)(m > g ? m : g);
    }
    int rc = ensure(ctx, ctx->scratch[SCR_CFAR_LUT], 65536, st);
    if (rc != SFE_OK) return rc;
    uint16_t *lut_dev = (uint16_t *)((char *)ctx->scratch[SCR_CFAR_LUT].ptr + 32768);  // second half: OS table
    SFE_CUDA(cudaMemcpyAsync(lut_dev, lut.data(), 512, cudaMemcpyHostToDevice, st));
    SFE_CUDA(cudaStreamSynchronize(st));  // `lut` is a local
    cfar_os_hist_kernel<<<F * p.strips, CF_W, 0, st>>>((const uint8_t *)img, p, lut_dev);
    SFE_CUDA(cudaGetLastError());
    ctx->launches++;
    return SFE_OK;
  }
  if (dtype == SFE_F32) return launch_exact<float>(ctx, st, (const float *)img, p, nullptr);
  return launch_exact<uint8_t>(ctx, st, (const uint8_t *)img, p, nullptr);
}
