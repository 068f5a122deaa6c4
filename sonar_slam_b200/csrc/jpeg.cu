// Baseline / extended-sequential Huffman JPEG decoder for compressed sonar pings (SURVEY 8(f) N4).
//
// The reference decodes every compressed ping on the host with
//     cv2.cvtColor(cv2.imdecode(buf, cv2.IMREAD_COLOR), cv2.COLOR_BGR2GRAY)      (feature_extraction.py:210-213)
// i.e. libjpeg-turbo's default decompression (JDCT_ISLOW, fancy upsampling) to BGR, then OpenCV's fixed-point
// BGR -> gray.  This file computes the same uint8 frames on the device, bit for bit, for the streams it accepts
// (include/sonarfe.h: sfe_jpeg_*).
//
// Host: the headers (a few hundred bytes per frame) are parsed here; every frame gets a descriptor (geometry,
// component layout, quantisation and Huffman tables -- pooled per chunk of frames, so frames sharing tables ship
// them once) and only the entropy-coded bytes travel to the device.
//
// Device, per chunk of frames:
//   jpeg_unstuff_kernel  one CTA per frame:
//     1. unstuff: a block-wide scan drops the 0x00 after every 0xFF and the RSTn markers, records the restart
//        segments and stops at the first other marker;
//   jpeg_entropy_kernel  one CTA per frame:
//     2. the bits of every segment are cut into CHUNK_BITS chunks, one thread each (the last chunk of a segment
//        takes the remainder).  Self-synchronising decoding (Weissenberger & Schmidt): a chunk is first decoded from
//        a guessed state (the segment's first chunk from the true one); then, round after round, every chunk whose
//        entry changed re-decodes its right neighbour from its exit state until no exit state (bit position,
//        block-in-MCU, zig-zag index) changes -- a fixed point, so every chunk's entry is the true one;
//     3. per-chunk block counts -> exclusive scan -> every chunk's first block; a last pass decodes every chunk
//        again and writes its coefficients (and the zero runs it covers) into their final places.  Data after a
//        segment's last MCU is skipped, as libjpeg-turbo skips it; a segment whose data ends before its last MCU is
//        corrupt (libjpeg-turbo would pad it with zero bits);
//     4. DC prediction: a block-wide scan of the DC differences per component, restarted at every segment.
//   jpeg_idct_kernel     dequantisation + jidctint.c's JDCT_ISLOW (CONST_BITS 13, PASS1_BITS 2, its 10-bit wrap
//                        range limit), 8 threads per 8x8 block; gray frames are written straight into the output;
//   jpeg_color_kernel    YCbCr frames: jdsample.c's upsampling (fancy h2v1 / h2v2, or replication for components
//                        at most 2 samples wide), jdcolor.c's YCbCr -> RGB tables, OpenCV's BGR2GRAY; also writes
//                        zeros over every frame that was rejected or failed to decode.
// Every device read of entropy-coded data is bounded by the frame's own byte range.
#include <algorithm>
#include <string>
#include <unordered_map>
#include <vector>

#include "stream_decode.cuh"

namespace sfe {

enum { JT = 512, CHUNK_BITS = 512, MAXTAB = 6 };  // MAXTAB: a DC and an AC table for each of 3 components

// ------------------------------------------------------------------ host-side header parsing
struct JHuffSpec {
  uint8_t bits[17];
  uint8_t vals[256];
  bool defined;
};

struct JHeader {
  int status = SFE_JPEG_OK;
  int H = 0, W = 0, nc = 0, sampling = -1, Ri = 0;
  int64_t ecs = 0, len = 0;  // first entropy-coded byte, stream length
  int cid[4] = {}, hs[4] = {}, vs[4] = {}, tq[4] = {}, td[4] = {}, ta[4] = {};
  uint16_t q[4][64];
  bool qdef[4] = {};
  JHuffSpec dc[4], ac[4];
  bool jfif = false, adobe = false;
  int adobe_tf = -1, orient = 1;
};

static const uint8_t kNatural[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,
                                     12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6,  7,  14, 21, 28,
                                     35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51,
                                     58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};
__constant__ uint8_t c_natural[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,
                                      12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6,  7,  14, 21, 28,
                                      35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51,
                                      58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

// EXIF orientation (tag 0x0112 of IFD0) of an APP1 "Exif" segment; 1 when absent or unreadable
static int exif_orientation(const uint8_t *s, int64_t sl) {
  if (sl < 14 || memcmp(s, "Exif\0\0", 6) != 0) return 1;
  return tiff_orientation(s + 6, sl - 6);
}

// Headers up to the start of the (single) scan.  Mirrors libjpeg-turbo's marker reader where it decides what is
// accepted (jdmarker.c) and how three components are interpreted (jdapimin.c: default_decompress_parms).
static void parse_header(const uint8_t *p, int64_t n, JHeader &h) {
  h = JHeader();
  h.len = n;
  for (int k = 0; k < 4; ++k) h.dc[k].defined = h.ac[k].defined = false;
  auto fail = [&](int st) { h.status = st; };
  if (n < 2 || p[0] != 0xFF || p[1] != 0xD8) return fail(SFE_JPEG_NOT_JPEG);
  int64_t i = 2;
  bool sof = false;
  for (;;) {
    while (i < n && p[i] != 0xFF) ++i;  // libjpeg skips (and warns about) garbage before a marker
    while (i < n && p[i] == 0xFF) ++i;
    if (i >= n) return fail(SFE_JPEG_TRUNCATED);
    const int m = p[i++];
    if (m == 0x00 || m == 0x01 || (m >= 0xD0 && m <= 0xD7)) continue;  // no length field
    if (m == 0xD8) return fail(SFE_JPEG_BAD_HEADER);
    if (m == 0xD9) return fail(SFE_JPEG_TRUNCATED);  // EOI before any scan
    if (i + 2 > n) return fail(SFE_JPEG_TRUNCATED);
    const int L = p[i] << 8 | p[i + 1];
    if (L < 2) return fail(SFE_JPEG_BAD_HEADER);
    if (i + L > n) return fail(SFE_JPEG_TRUNCATED);
    const uint8_t *s = p + i + 2;
    const int sl = L - 2;
    i += L;
    if (m == 0xC0 || m == 0xC1) {
      if (sof) return fail(SFE_JPEG_BAD_HEADER);
      sof = true;
      if (sl < 6) return fail(SFE_JPEG_BAD_HEADER);
      if (s[0] != 8) return fail(SFE_JPEG_PRECISION);
      h.H = s[1] << 8 | s[2], h.W = s[3] << 8 | s[4], h.nc = s[5];
      if (h.nc != 1 && h.nc != 3) return fail(SFE_JPEG_COLORSPACE);
      if (sl < 6 + 3 * h.nc || h.H == 0 || h.W == 0) return fail(SFE_JPEG_BAD_HEADER);
      for (int c = 0; c < h.nc; ++c) {
        h.cid[c] = s[6 + 3 * c], h.hs[c] = s[7 + 3 * c] >> 4, h.vs[c] = s[7 + 3 * c] & 15, h.tq[c] = s[8 + 3 * c];
        if (h.hs[c] < 1 || h.hs[c] > 4 || h.vs[c] < 1 || h.vs[c] > 4 || h.tq[c] > 3) return fail(SFE_JPEG_BAD_HEADER);
      }
    } else if (m == 0xC2 || m == 0xC6) {
      return fail(SFE_JPEG_PROGRESSIVE);
    } else if (m == 0xC3 || m == 0xC7) {
      return fail(SFE_JPEG_LOSSLESS);
    } else if (m >= 0xC9 && m <= 0xCF && m != 0xCC) {
      return fail(SFE_JPEG_ARITHMETIC);
    } else if (m == 0xC5 || m == 0xC8) {
      return fail(SFE_JPEG_BAD_HEADER);  // hierarchical / reserved
    } else if (m == 0xC4) {
      int o = 0;
      while (o < sl) {
        if (o + 17 > sl) return fail(SFE_JPEG_BAD_HEADER);
        const int tc = s[o] >> 4, th = s[o] & 15;
        int cnt = 0;
        for (int l = 1; l <= 16; ++l) cnt += s[o + l];
        if (tc > 1 || th > 3 || cnt > 256 || o + 17 + cnt > sl) return fail(SFE_JPEG_BAD_HEADER);
        JHuffSpec &t = tc ? h.ac[th] : h.dc[th];
        t.bits[0] = 0;
        memcpy(t.bits + 1, s + o + 1, 16);
        memset(t.vals, 0, sizeof(t.vals));
        memcpy(t.vals, s + o + 17, cnt);
        // jpeg_make_d_derived_tbl: codes must fit their lengths, DC categories must be <= 15
        int code = 0, k = 0;
        for (int l = 1; l <= 16; ++l) {
          code += t.bits[l];
          if (code > (1 << l)) return fail(SFE_JPEG_BAD_HEADER);
          code <<= 1;
          k += t.bits[l];
        }
        if (!tc)
          for (int j = 0; j < cnt; ++j)
            if (t.vals[j] > 15) return fail(SFE_JPEG_BAD_HEADER);
        t.defined = true;
        o += 17 + cnt;
      }
    } else if (m == 0xDB) {
      int o = 0;
      while (o < sl) {
        const int pq = s[o] >> 4, tq = s[o] & 15;
        const int need = 1 + 64 * (pq ? 2 : 1);
        if (pq > 1 || tq > 3 || o + need > sl) return fail(SFE_JPEG_BAD_HEADER);
        for (int k = 0; k < 64; ++k)
          h.q[tq][kNatural[k]] = pq ? (uint16_t)(s[o + 1 + 2 * k] << 8 | s[o + 2 + 2 * k]) : s[o + 1 + k];
        h.qdef[tq] = true;
        o += need;
      }
    } else if (m == 0xDD) {
      if (sl < 2) return fail(SFE_JPEG_BAD_HEADER);
      h.Ri = s[0] << 8 | s[1];
    } else if (m == 0xE0) {
      if (sl >= 14 && memcmp(s, "JFIF\0", 5) == 0) h.jfif = true;
    } else if (m == 0xEE) {
      if (sl >= 12 && memcmp(s, "Adobe", 5) == 0) h.adobe = true, h.adobe_tf = s[11];
    } else if (m == 0xE1) {
      if (h.orient == 1) h.orient = exif_orientation(s, sl);
    } else if (m == 0xDA) {
      if (!sof) return fail(SFE_JPEG_BAD_HEADER);
      if (sl < 1) return fail(SFE_JPEG_BAD_HEADER);
      const int ns = s[0];
      // one interleaved scan over every component, in frame order (what a sequential encoder writes by default)
      if (ns != h.nc || sl < 1 + 2 * ns + 3) return fail(SFE_JPEG_BAD_HEADER);
      for (int c = 0; c < ns; ++c) {
        if (s[1 + 2 * c] != h.cid[c]) return fail(SFE_JPEG_BAD_HEADER);
        h.td[c] = s[2 + 2 * c] >> 4, h.ta[c] = s[2 + 2 * c] & 15;
        if (h.td[c] > 3 || h.ta[c] > 3) return fail(SFE_JPEG_BAD_HEADER);
      }
      if (s[1 + 2 * ns] != 0 || s[2 + 2 * ns] != 63 || s[3 + 2 * ns] != 0) return fail(SFE_JPEG_BAD_HEADER);
      h.ecs = i;
      break;
    }
    // APPn, COM and anything else with a length: skipped
  }
  for (int c = 0; c < h.nc; ++c)
    if (!h.qdef[h.tq[c]] || !h.dc[h.td[c]].defined || !h.ac[h.ta[c]].defined) return fail(SFE_JPEG_BAD_HEADER);
  if (h.nc == 3) {
    // jdapimin.c default_decompress_parms: YCbCr unless an Adobe transform 0 or R/G/B component ids say RGB
    bool rgb = false;
    if (!h.jfif) {
      if (h.adobe)
        rgb = h.adobe_tf == 0;
      else
        rgb = h.cid[0] == 82 && h.cid[1] == 71 && h.cid[2] == 66;
    }
    if (rgb) return fail(SFE_JPEG_COLORSPACE);
  }
  if (h.orient >= 2 && h.orient <= 8) return fail(SFE_JPEG_ORIENTATION);
  if (h.nc == 1) {
    h.sampling = SFE_JPEG_GRAY;  // a single-component scan is non-interleaved: one block per MCU whatever the factors
  } else {
    if (h.hs[1] != 1 || h.vs[1] != 1 || h.hs[2] != 1 || h.vs[2] != 1) return fail(SFE_JPEG_SAMPLING);
    if (h.hs[0] == 1 && h.vs[0] == 1)
      h.sampling = SFE_JPEG_444;
    else if (h.hs[0] == 2 && h.vs[0] == 1)
      h.sampling = SFE_JPEG_422;
    else if (h.hs[0] == 2 && h.vs[0] == 2)
      h.sampling = SFE_JPEG_420;
    else
      return fail(SFE_JPEG_SAMPLING);
  }
}

// ------------------------------------------------------------------ device descriptors
struct HT {                // derived Huffman table
  uint16_t lut[512];       // 9-bit lookahead: (length << 8) | symbol, 0 = longer code or invalid
  int32_t maxcode[18];     // largest code of each length (-1: none), lengths 1..16
  int32_t valoff[18];      // index of the first symbol of a length minus its first code
  uint8_t vals[256];
};

struct JDesc {
  int32_t status;          // 0: decode; otherwise the host's SFE_JPEG_* verdict
  int32_t H, W, mode, bpm, mcux, mcuy, nmcu, Ri, nseg, nblocks, chunk_cap;
  int32_t tab[MAXTAB];     // pool index of Huffman table slot k
  int32_t qtab[3];         // pool index of every component's quantisation table
  int8_t bcomp[8], bdc[8], bac[8];  // per block of an MCU: component, DC slot, AC slot
  int32_t cw[3], ch[3];    // component size in samples (downsampled_width / _height)
  int32_t pw[3], ph[3];    // component plane size (whole MCUs)
  int64_t src, src_len;    // entropy-coded bytes in the chunk's byte buffer
  int64_t scr;             // this frame's scratch (byte offset)
  int64_t coef;            // this frame's first block in the coefficient buffer
};

struct JLayout {
  int64_t comp, segstart, segbase, segchunk, exit, pend, cnt, pcnt, cseg, flags, dcs, plane[3], total;
};

__host__ __device__ inline int64_t al16(int64_t x) { return (x + 15) & ~(int64_t)15; }

__host__ __device__ inline JLayout jlayout(const JDesc &d) {
  JLayout L;
  int64_t o = d.scr;
  L.comp = o, o += al16(d.src_len + 8);
  L.segstart = o, o += al16(4 * (int64_t)(d.nseg + 1));
  L.segbase = o, o += al16(12 * (int64_t)d.nseg);
  L.segchunk = o, o += al16(4 * (int64_t)(d.nseg + 1));
  L.exit = o, o += al16(8 * (int64_t)d.chunk_cap);
  L.pend = o, o += al16(8 * (int64_t)d.chunk_cap);
  L.cnt = o, o += al16(4 * (int64_t)d.chunk_cap);
  L.pcnt = o, o += al16(4 * (int64_t)d.chunk_cap);
  L.cseg = o, o += al16(4 * (int64_t)d.chunk_cap);
  L.flags = o, o += al16((int64_t)d.chunk_cap);
  L.dcs = o, o += al16(4 * (int64_t)d.nblocks);
  for (int c = 0; c < 3; ++c) {
    L.plane[c] = o;
    if (d.mode != SFE_JPEG_GRAY) o += al16((int64_t)d.pw[c] * d.ph[c]);
  }
  L.total = o - d.scr;
  return L;
}

// ------------------------------------------------------------------ device: entropy decoding
struct JSt {  // decoder state at a symbol boundary; bz = (block-in-MCU << 8) | zig-zag index, -1 = error
  int pos, bz;
};

__device__ __forceinline__ uint32_t peek32(const uint8_t *__restrict__ p, int pos) {
  const uint8_t *q = p + (pos >> 3);
  const uint64_t w = ((uint64_t)q[0] << 32) | ((uint64_t)q[1] << 24) | ((uint64_t)q[2] << 16) |
                     ((uint64_t)q[3] << 8) | (uint64_t)q[4];
  return (uint32_t)(w >> (8 - (pos & 7)));
}

__device__ __forceinline__ int huff(const HT &t, uint32_t w, int &len) {
  const int e = t.lut[w >> 23];
  if (e) {
    len = e >> 8;
    return e & 255;
  }
  int l = 10;
  int code = (int)(w >> 22);
  while (code > t.maxcode[l]) {
    if (++l > 16) return -1;
    code = (int)(w >> (32 - l));
  }
  len = l;
  return t.vals[t.valoff[l] + code];
}

__device__ __forceinline__ int extend(uint32_t r, int s) {
  return (int)r < (1 << (s - 1)) ? (int)r - (1 << s) + 1 : (int)r;
}

// Decode from state `s`.  WRITE = false: stop at the first symbol boundary at or after `end`, count completed blocks.
// WRITE = true: blocks are numbered from blk0 (< blk_end) and written; a chunk stops at `end` (the segment's last chunk:
// at the segment's end) or when block blk_end is reached, so no write reaches a block at or past blk_end.  `se` = end of the segment's data (bits): a symbol reaching past it is an error.
// Without WRITE the decoder is lenient: an invalid code skips one bit, a run past coefficient 63 ends the block.  A
// decode from a guessed state meets such codes all the time and must keep going to fall into step with the true one;
// from a true state on valid data the rules never fire, and the writing pass, which is strict, flags every chunk
// whose data is corrupt.
template <bool WRITE>
__device__ JSt run_chunk(const HT *__restrict__ T, const JDesc &d, const uint8_t *__restrict__ comp, JSt s, int end,
                         int se, bool last, int &blocks, int blk0, int blk_end, int16_t *__restrict__ coef,
                         int32_t *__restrict__ dcs) {
  const JSt ERR = {-1, -1};
  blocks = 0;
  if (s.bz < 0) return ERR;
  int pos = s.pos, b = s.bz >> 8, z = s.bz & 255;
  int blk = blk0;
  for (;;) {
    if (!(WRITE && last) && pos >= end) break;
    if (z == 0) {
      if (WRITE && blk >= blk_end) break;  // the segment's last MCU is complete; what follows is not decoded
      int len;
      const int sym = huff(T[d.bdc[b]], peek32(comp, pos), len);
      if (sym < 0) {
        if (WRITE) return ERR;
        ++pos;
        continue;
      }
      pos += len;
      int v = 0;
      if (sym) {
        v = extend(peek32(comp, pos) >> (32 - sym), sym);
        pos += sym;
      }
      if (pos > se) return ERR;
      if (WRITE) dcs[blk] = v;
      z = 1;
    } else {
      int len;
      const int rs = huff(T[d.bac[b]], peek32(comp, pos), len);
      if (rs < 0) {
        if (WRITE) return ERR;
        ++pos;
        continue;
      }
      pos += len;
      const int r = rs >> 4, sz = rs & 15;
      int zn;
      if (sz) {
        zn = z + r;
        const int v = extend(peek32(comp, pos) >> (32 - sz), sz);
        pos += sz;
        if (pos > se) return ERR;
        if (zn > 63) {  // a run past coefficient 63
          if (WRITE) return ERR;
          zn = 63;
        }
        if (WRITE) {
          int16_t *cb = coef + (int64_t)blk * 64;
          for (int k = z; k < zn; ++k) cb[c_natural[k]] = 0;
          cb[c_natural[zn]] = (int16_t)v;
        }
        ++zn;
      } else {
        if (pos > se) return ERR;
        zn = r == 15 ? z + 16 : 64;  // ZRL / EOB
        if (zn > 64) {
          if (WRITE) return ERR;
          zn = 64;
        }
        if (WRITE) {
          int16_t *cb = coef + (int64_t)blk * 64;
          for (int k = z; k < zn; ++k) cb[c_natural[k]] = 0;
        }
      }
      z = zn;
      if (z == 64) {
        z = 0;
        if (++b == d.bpm) b = 0;
        ++blocks, ++blk;
      }
    }
  }
  return JSt{pos, (b << 8) | z};
}

__device__ __forceinline__ int warp_incl(int v) {
  const int lane = threadIdx.x & 31;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int t = __shfl_up_sync(0xffffffffu, v, o);
    if (lane >= o) v += t;
  }
  return v;
}

// exclusive block-wide scan over JT threads; *total = sum.  Every thread must call it.
__device__ int block_exscan(int v, int *sh, int *total) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int inc = warp_incl(v);
  if (lane == 31) sh[w] = inc;
  __syncthreads();
  if (w == 0) {
    int s = lane < JT / 32 ? sh[lane] : 0;
    s = warp_incl(s);
    if (lane < JT / 32) sh[lane] = s;
  }
  __syncthreads();
  const int base = w ? sh[w - 1] : 0;
  *total = sh[JT / 32 - 1];
  __syncthreads();
  return base + inc - v;
}

// 1. unstuff: a block-wide scan drops the 0x00 after every 0xFF and the RSTn markers, records where every restart
// segment starts in the compacted stream and stops at the first other marker.  Writes the frame's status: the host's
// verdict, SFE_JPEG_CORRUPT (missing, surplus or out-of-sequence RSTn) or SFE_JPEG_OK.
__global__ void __launch_bounds__(JT) jpeg_unstuff_kernel(const JDesc *__restrict__ desc, const uint8_t *__restrict__ bytes,
                                                          uint8_t *__restrict__ scr, int32_t *__restrict__ status) {
  const int f = blockIdx.x, tid = threadIdx.x;
  const JDesc &d = desc[f];
  if (d.status != SFE_JPEG_OK) {
    if (tid == 0) status[f] = d.status;
    return;
  }
  __shared__ int sh[32];
  __shared__ int s_err, s_end;
  if (tid == 0) s_err = 0, s_end = INT_MAX;
  const JLayout L = jlayout(d);
  uint8_t *comp = scr + L.comp;
  int32_t *segstart = reinterpret_cast<int32_t *>(scr + L.segstart);
  const uint8_t *src = bytes + d.src;
  const int64_t n = d.src_len;
  __syncthreads();
  int kept = 0, rsts = 0;
  if (tid == 0) segstart[0] = 0;
  for (int64_t t0 = 0; t0 < n; t0 += JT) {
    const int64_t i = t0 + tid;
    int keep = 0, rst = 0, endh = 0;
    uint8_t c = 0;
    if (i < n) {
      c = src[i];
      const int next = i + 1 < n ? src[i + 1] : -1;
      const int prev = i > 0 ? src[i - 1] : -1;
      if (c == 0xFF) {
        if (next == 0x00)
          keep = 1;
        else if (next >= 0xD0 && next <= 0xD7)
          rst = 1;
        else if (next != 0xFF)
          endh = 1;  // any other marker (normally EOI), or the stream's end
      } else {
        keep = !(prev == 0xFF);  // the stuffed 0x00 or the RSTn byte after an 0xFF
      }
    }
    if (endh) atomicMin(&s_end, (int)i);
    __syncthreads();
    const int e = s_end;
    if (i >= e) keep = rst = 0;
    int tot;
    const int pre = block_exscan(keep | (rst << 16), sh, &tot);
    if (keep) comp[kept + (pre & 0xFFFF)] = c;
    int over = 0;
    if (rst) {
      const int k = rsts + (pre >> 16) + 1;  // segment that starts here
      if (k < d.nseg) {
        if (src[i + 1] != 0xD0 + ((k - 1) & 7))
          s_err = 1;
        else
          segstart[k] = kept + (pre & 0xFFFF);
      } else if (k == d.nseg) {  // past the last MCU: libjpeg-turbo never reads this far, neither does the decoder
        segstart[d.nseg] = kept + (pre & 0xFFFF);
        over = 1;
      }
    }
    kept += tot & 0xFFFF, rsts += tot >> 16;
    if (__syncthreads_or(over)) {
      if (tid == 0) s_end = -1;  // the last segment's end is set
      break;
    }
    if (e != INT_MAX) break;
  }
  if (tid < 8) comp[kept + tid] = 0;
  if (tid == 0 && s_end != -1) {
    if (rsts != d.nseg - 1) s_err = 1;
    segstart[d.nseg] = kept;
  }
  __syncthreads();
  if (tid == 0) status[f] = s_err ? SFE_JPEG_CORRUPT : SFE_JPEG_OK;
}

// 2.-4. chunked self-synchronising entropy decoding, coefficient writes, DC prediction (see the top of the file)
__global__ void __launch_bounds__(JT) jpeg_entropy_kernel(const JDesc *__restrict__ desc, const HT *__restrict__ pool,
                                                          uint8_t *__restrict__ scr, int16_t *__restrict__ coef_all,
                                                          int32_t *__restrict__ status) {
  const int f = blockIdx.x, tid = threadIdx.x;
  const JDesc &d = desc[f];
  if (status[f] != SFE_JPEG_OK) return;  // rejected on the host or by the unstuff kernel
  __shared__ HT T[MAXTAB];
  __shared__ int sh[32];
  __shared__ int s_err;
  {
    const int4 *src = reinterpret_cast<const int4 *>(pool);
    int4 *dst = reinterpret_cast<int4 *>(T);
    constexpr int W = sizeof(HT) / 16;
    for (int k = tid; k < MAXTAB * W; k += JT) {
      const int slot = k / W;
      if (d.tab[slot] >= 0) dst[k] = src[(int64_t)d.tab[slot] * W + (k % W)];
    }
  }
  if (tid == 0) s_err = 0;
  const JLayout L = jlayout(d);
  const uint8_t *comp = scr + L.comp;
  const int32_t *segstart = reinterpret_cast<const int32_t *>(scr + L.segstart);
  int32_t *segbase = reinterpret_cast<int32_t *>(scr + L.segbase);
  int32_t *segchunk = reinterpret_cast<int32_t *>(scr + L.segchunk);
  JSt *ex = reinterpret_cast<JSt *>(scr + L.exit);
  JSt *pend = reinterpret_cast<JSt *>(scr + L.pend);
  int32_t *cnt = reinterpret_cast<int32_t *>(scr + L.cnt);
  int32_t *pcnt = reinterpret_cast<int32_t *>(scr + L.pcnt);
  int32_t *cseg = reinterpret_cast<int32_t *>(scr + L.cseg);
  uint8_t *flags = scr + L.flags;
  int32_t *dcs = reinterpret_cast<int32_t *>(scr + L.dcs);
  int16_t *coef = coef_all + d.coef * 64;
  __syncthreads();

  // ---- 2. chunks: every segment's bits in CHUNK_BITS pieces, the last one taking the remainder
  int nch = 0;
  for (int s0 = 0; s0 < d.nseg; s0 += JT) {
    const int s = s0 + tid;
    int k = 0;
    if (s < d.nseg) k = max(1, (segstart[s + 1] - segstart[s]) * 8 / CHUNK_BITS);
    int tot;
    const int pre = block_exscan(k, sh, &tot);
    if (s < d.nseg) {
      segchunk[s] = nch + pre;
      for (int j = 0; j < k && nch + pre + j < d.chunk_cap; ++j) cseg[nch + pre + j] = s;
    }
    nch += tot;
  }
  if (tid == 0) segchunk[d.nseg] = nch;
  if (nch > d.chunk_cap) {  // cannot happen: the host sized chunk_cap for the byte count
    if (tid == 0) status[f] = SFE_JPEG_CORRUPT;
    return;
  }
  __syncthreads();
  auto chunk_geom = [&](int k, int &s, int &b0, int &b1, int &se, bool &first, bool &last) {
    s = cseg[k];
    const int j = k - segchunk[s], nk = segchunk[s + 1] - segchunk[s];
    const int sb = segstart[s] * 8;
    se = segstart[s + 1] * 8;
    b0 = sb + j * CHUNK_BITS;
    first = j == 0, last = j == nk - 1;
    b1 = last ? se : b0 + CHUNK_BITS;
  };

  // phase 1: every chunk from a guessed state (segment starts from the true one)
  for (int k = tid; k < nch; k += JT) {
    int s, b0, b1, se, blocks;
    bool first, last;
    chunk_geom(k, s, b0, b1, se, first, last);
    if (last) continue;
    ex[k] = run_chunk<false>(T, d, comp, JSt{b0, 0}, b1, se, false, blocks, 0, 0, nullptr, nullptr);
    cnt[k] = blocks;
    flags[k] = 1;  // dirty: its right neighbour must be re-decoded from this exit
  }
  __syncthreads();
  // rounds until no exit state changes
  for (;;) {
    for (int k = tid; k < nch; k += JT) {
      int s, b0, b1, se, blocks;
      bool first, last;
      chunk_geom(k, s, b0, b1, se, first, last);
      if (last || !(flags[k] & 1)) continue;
      const int k1 = k + 1;
      int s1, c0, c1, se1;
      bool f1, l1;
      chunk_geom(k1, s1, c0, c1, se1, f1, l1);
      if (l1) continue;
      pend[k1] = run_chunk<false>(T, d, comp, ex[k], c1, se1, false, blocks, 0, 0, nullptr, nullptr);
      pcnt[k1] = blocks;
      flags[k1] |= 2;
    }
    __syncthreads();
    int any = 0;
    for (int k = tid; k < nch; k += JT) {
      const int fl = flags[k];
      int nf = 0;
      if (fl & 2) {
        cnt[k] = pcnt[k];
        const JSt p = pend[k], o = ex[k];
        if (p.pos != o.pos || p.bz != o.bz) ex[k] = p, nf = 1, any = 1;
      }
      flags[k] = nf;
    }
    if (!__syncthreads_or(any)) break;
  }

  // ---- 3. first block of every chunk, then the writing pass
  const int seg_blocks = d.Ri ? d.Ri * d.bpm : d.nmcu * d.bpm;
  int run = 0;
  for (int k0 = 0; k0 < nch; k0 += JT) {
    const int k = k0 + tid;
    int v = 0;
    if (k < nch) {
      const int s = cseg[k];
      v = (k == segchunk[s + 1] - 1) ? 0 : cnt[k];
    }
    int tot;
    const int pre = block_exscan(v, sh, &tot);
    if (k < nch) pcnt[k] = run + pre;  // running count, made segment-relative below
    run += tot;
  }
  __syncthreads();
  for (int k = tid; k < nch; k += JT) {
    int s, b0, b1, se, blocks;
    bool first, last;
    chunk_geom(k, s, b0, b1, se, first, last);
    const int sblk = s * seg_blocks;
    const int send = min(sblk + seg_blocks, d.nblocks);
    const int blk0 = sblk + pcnt[k] - pcnt[segchunk[s]];
    // A chunk that starts after the segment's last MCU holds extraneous data: libjpeg-turbo skips it (with a
    // warning), and so does this decoder.  It writes nothing: every write below is to a block in [blk0, send).
    if (blk0 >= send) continue;
    const JSt in = first ? JSt{b0, 0} : ex[k - 1];
    if (in.bz < 0 || ((in.bz >> 8) != blk0 % d.bpm)) {
      s_err = 1;
      continue;
    }
    const JSt o = run_chunk<true>(T, d, comp, in, b1, se, last, blocks, blk0, send, coef, dcs);
    if (o.bz < 0 || (last && blk0 + blocks != send)) s_err = 1;
  }
  __syncthreads();
  if (s_err) {
    if (tid == 0) status[f] = SFE_JPEG_CORRUPT;
    return;
  }

  // ---- 4. DC prediction: per component, restarted at every segment
  int carry0 = 0, carry1 = 0, carry2 = 0;
  const bool color = d.mode != SFE_JPEG_GRAY;
  for (int i0 = 0; i0 < d.nblocks; i0 += JT) {
    const int i = i0 + tid;
    const int c = i < d.nblocks ? d.bcomp[i % d.bpm] : -1;
    const int v = i < d.nblocks ? dcs[i] : 0;
    int tot, i1 = 0, i2 = 0;
    const int i0c = carry0 + block_exscan(c == 0 ? v : 0, sh, &tot) + (c == 0 ? v : 0);
    carry0 += tot;
    if (color) {
      i1 = carry1 + block_exscan(c == 1 ? v : 0, sh, &tot) + (c == 1 ? v : 0);
      carry1 += tot;
      i2 = carry2 + block_exscan(c == 2 ? v : 0, sh, &tot) + (c == 2 ? v : 0);
      carry2 += tot;
    }
    if (i < d.nblocks) {
      dcs[i] = c == 0 ? i0c : c == 1 ? i1 : i2;
      if (d.Ri && (i + 1) % seg_blocks == 0 && (i + 1) / seg_blocks < d.nseg) {
        int32_t *sb = segbase + 3 * ((i + 1) / seg_blocks);
        sb[0] = i0c, sb[1] = i1, sb[2] = i2;
      }
    }
  }
  if (tid < 3) segbase[tid] = 0;
  __syncthreads();
  for (int i = tid; i < d.nblocks; i += JT) dcs[i] -= segbase[3 * (i / seg_blocks) + d.bcomp[i % d.bpm]];
  if (tid == 0) status[f] = SFE_JPEG_OK;
}

// ------------------------------------------------------------------ device: dequantisation + ISLOW IDCT
// jidctint.c, JDCT_ISLOW: CONST_BITS 13, PASS1_BITS 2, JLONG arithmetic, int workspace; the output index is taken
// modulo 1024 (RANGE_MASK) into the post-IDCT range-limit table, i.e. a 10-bit signed wrap and then a clamp.
#define FIX_0_298631336 ((int64_t)2446)
#define FIX_0_390180644 ((int64_t)3196)
#define FIX_0_541196100 ((int64_t)4433)
#define FIX_0_765366865 ((int64_t)6270)
#define FIX_0_899976223 ((int64_t)7373)
#define FIX_1_175875602 ((int64_t)9633)
#define FIX_1_501321110 ((int64_t)12299)
#define FIX_1_847759065 ((int64_t)15137)
#define FIX_1_961570560 ((int64_t)16069)
#define FIX_2_053119869 ((int64_t)16819)
#define FIX_2_562915447 ((int64_t)20995)
#define FIX_3_072711026 ((int64_t)25172)

__device__ __forceinline__ void idct_1d(const int64_t *in, int64_t *out) {
  // in[0..7] = coefficient u = 0..7; out[0..7] un-descaled sums (tmp10 + tmp3, ...)
  int64_t z2 = in[2], z3 = in[6];
  int64_t z1 = (z2 + z3) * FIX_0_541196100;
  const int64_t tmp2e = z1 + z3 * -FIX_1_847759065;
  const int64_t tmp3e = z1 + z2 * FIX_0_765366865;
  z2 = in[0], z3 = in[4];
  const int64_t tmp0e = (z2 + z3) * 8192, tmp1e = (z2 - z3) * 8192;
  const int64_t tmp10 = tmp0e + tmp3e, tmp13 = tmp0e - tmp3e, tmp11 = tmp1e + tmp2e, tmp12 = tmp1e - tmp2e;
  int64_t tmp0 = in[7], tmp1 = in[5], tmp2 = in[3], tmp3 = in[1];
  z1 = tmp0 + tmp3;
  z2 = tmp1 + tmp2;
  z3 = tmp0 + tmp2;
  int64_t z4 = tmp1 + tmp3;
  const int64_t z5 = (z3 + z4) * FIX_1_175875602;
  tmp0 *= FIX_0_298631336;
  tmp1 *= FIX_2_053119869;
  tmp2 *= FIX_3_072711026;
  tmp3 *= FIX_1_501321110;
  z1 *= -FIX_0_899976223;
  z2 *= -FIX_2_562915447;
  z3 *= -FIX_1_961570560;
  z4 *= -FIX_0_390180644;
  z3 += z5;
  z4 += z5;
  tmp0 += z1 + z3;
  tmp1 += z2 + z4;
  tmp2 += z2 + z3;
  tmp3 += z1 + z4;
  out[0] = tmp10 + tmp3, out[7] = tmp10 - tmp3;
  out[1] = tmp11 + tmp2, out[6] = tmp11 - tmp2;
  out[2] = tmp12 + tmp1, out[5] = tmp12 - tmp1;
  out[3] = tmp13 + tmp0, out[4] = tmp13 - tmp0;
}

__device__ __forceinline__ int64_t descale(int64_t x, int n) { return (x + ((int64_t)1 << (n - 1))) >> n; }

__device__ __forceinline__ uint8_t range_limit_idct(int x) {
  const int v = x & 1023;  // RANGE_MASK
  return (uint8_t)(v < 128 ? v + 128 : v < 512 ? 255 : v < 896 ? 0 : v - 896);
}

// dequantised coefficients of block `blk` of frame d, natural order (the int16 coefficient as libjpeg stores it,
// times its quantisation value)
__device__ __forceinline__ int dequant(const JDesc &d, const uint16_t *__restrict__ qpool, const int16_t *cb,
                                       const int32_t *dcs, int blk, int k) {
  const int c = d.bcomp[blk % d.bpm];
  const int co = k == 0 ? (int)(int16_t)dcs[blk] : (int)cb[k];
  return co * (int)qpool[(int64_t)d.qtab[c] * 64 + k];
}

__global__ void __launch_bounds__(128) jpeg_idct_kernel(const JDesc *__restrict__ desc, const uint16_t *__restrict__ qpool,
                                                        uint8_t *__restrict__ scr, const int16_t *__restrict__ coef_all,
                                                        const int32_t *__restrict__ status, uint8_t *__restrict__ out,
                                                        int64_t fstride) {
  const int f = blockIdx.y;
  const JDesc &d = desc[f];
  if (status[f] != SFE_JPEG_OK) return;
  const int g = threadIdx.x >> 3, t = threadIdx.x & 7;
  const int blk = blockIdx.x * 16 + g;
  __shared__ int ws[16][64];
  if (blk >= d.nblocks) return;  // whole 8-thread groups leave together
  const JLayout L = jlayout(d);
  const int32_t *dcs = reinterpret_cast<const int32_t *>(scr + L.dcs);
  const int16_t *cb = coef_all + (d.coef + blk) * 64;
  const unsigned gm = 0xFFu << (threadIdx.x & 24);
#pragma unroll
  for (int j = 0; j < 8; ++j) ws[g][t * 8 + j] = dequant(d, qpool, cb, dcs, blk, t * 8 + j);
  __syncwarp(gm);
  // pass 1: column t
  int64_t in[8], o[8];
#pragma unroll
  for (int r = 0; r < 8; ++r) in[r] = ws[g][r * 8 + t];
  idct_1d(in, o);
  __syncwarp(gm);
#pragma unroll
  for (int r = 0; r < 8; ++r) ws[g][r * 8 + t] = (int)descale(o[r], 13 - 2);
  __syncwarp(gm);
  // pass 2: row t
#pragma unroll
  for (int j = 0; j < 8; ++j) in[j] = ws[g][t * 8 + j];
  idct_1d(in, o);
  uint8_t px[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) px[j] = range_limit_idct((int)descale(o[j], 13 + 2 + 3));
  // where the block lies
  const int m = blk / d.bpm, b = blk % d.bpm;
  const int c = d.bcomp[b];
  int bx, by;
  if (d.mode == SFE_JPEG_GRAY) {
    bx = m % d.mcux, by = m / d.mcux;
  } else {
    // luma: hc x vc blocks per MCU in raster order, then one Cb and one Cr block
    const int hc = c == 0 ? (d.mode == SFE_JPEG_444 ? 1 : 2) : 1;
    const int vc = c == 0 ? (d.mode == SFE_JPEG_420 ? 2 : 1) : 1;
    const int idx = c == 0 ? b : 0;
    bx = (m % d.mcux) * hc + idx % hc, by = (m / d.mcux) * vc + idx / hc;
  }
  const int y = by * 8 + t;
  if (d.mode == SFE_JPEG_GRAY) {
    if (y >= d.H) return;
    uint8_t *row = out + (int64_t)f * fstride + (int64_t)y * d.W;
#pragma unroll
    for (int j = 0; j < 8; ++j)
      if (bx * 8 + j < d.W) row[bx * 8 + j] = px[j];
  } else {
    uint8_t *row = scr + L.plane[c] + (int64_t)y * d.pw[c] + bx * 8;
    uint2 v;
    v.x = px[0] | px[1] << 8 | px[2] << 16 | (uint32_t)px[3] << 24;
    v.y = px[4] | px[5] << 8 | px[6] << 16 | (uint32_t)px[7] << 24;
    *reinterpret_cast<uint2 *>(row) = v;
  }
}

// diagnostic: dequantised coefficient blocks, natural order, int32 [n][cap_blocks][64]
__global__ void jpeg_dequant_kernel(const JDesc *__restrict__ desc, const uint16_t *__restrict__ qpool,
                                    const uint8_t *__restrict__ scr, const int16_t *__restrict__ coef_all,
                                    const int32_t *__restrict__ status, int cap_blocks, int32_t *__restrict__ out) {
  const int f = blockIdx.y;
  const JDesc &d = desc[f];
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)cap_blocks * 64) return;
  const int blk = (int)(i >> 6), k = (int)(i & 63);
  int v = 0;
  if (status[f] == SFE_JPEG_OK && blk < d.nblocks) {
    const JLayout L = jlayout(d);
    v = dequant(d, qpool, coef_all + (d.coef + blk) * 64, reinterpret_cast<const int32_t *>(scr + L.dcs), blk, k);
  }
  out[(int64_t)f * cap_blocks * 64 + i] = v;
}

// ------------------------------------------------------------------ device: upsampling + colour + gray
__device__ __forceinline__ int chroma(const JDesc &d, const uint8_t *P, int c, int y, int x) {
  const int pw = d.pw[c], wc = d.cw[c];
  if (d.mode == SFE_JPEG_444) return P[(int64_t)y * pw + x];
  const int cx = x >> 1;
  if (d.mode == SFE_JPEG_422) {  // jdsample.c h2v1_fancy_upsample (downsampled_width > 2), else h2v1_upsample
    const uint8_t *row = P + (int64_t)y * pw;
    if (wc <= 2) return row[cx];
    return (x & 1) ? (3 * row[cx] + row[min(cx + 1, wc - 1)] + 2) >> 2 : (3 * row[cx] + row[max(cx - 1, 0)] + 1) >> 2;
  }
  // 4:2:0: h2v2_fancy_upsample with context rows (the image's first / last row repeated), else h2v2_upsample
  const int cy = y >> 1;
  if (wc <= 2) return P[(int64_t)cy * pw + cx];
  const int ny = (y & 1) ? min(cy + 1, d.ch[c] - 1) : max(cy - 1, 0);
  const uint8_t *r0 = P + (int64_t)cy * pw, *r1 = P + (int64_t)ny * pw;
  const int cs = 3 * r0[cx] + r1[cx];
  if (x & 1) {
    const int nx = min(cx + 1, wc - 1);
    return (3 * cs + 3 * r0[nx] + r1[nx] + 7) >> 4;
  }
  const int px = max(cx - 1, 0);
  return (3 * cs + 3 * r0[px] + r1[px] + 8) >> 4;
}

__device__ __forceinline__ int clamp255(int v) { return v < 0 ? 0 : v > 255 ? 255 : v; }

__global__ void __launch_bounds__(256) jpeg_color_kernel(const JDesc *__restrict__ desc, const uint8_t *__restrict__ scr,
                                                         const int32_t *__restrict__ status, uint8_t *__restrict__ out,
                                                         int64_t fstride, int R, int B) {
  const int f = blockIdx.y;
  const JDesc &d = desc[f];
  const bool ok = status[f] == SFE_JPEG_OK;
  if (ok && d.mode == SFE_JPEG_GRAY) return;  // written by the IDCT
  const JLayout L = jlayout(d);
  uint8_t *o = out + (int64_t)f * fstride;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < (int64_t)R * B; i += (int64_t)gridDim.x * blockDim.x) {
    if (!ok) {
      o[i] = 0;
      continue;
    }
    const int y = (int)(i / B), x = (int)(i % B);
    const int Y = scr[L.plane[0] + (int64_t)y * d.pw[0] + x];
    const int cb = chroma(d, scr + L.plane[1], 1, y, x) - 128;
    const int cr = chroma(d, scr + L.plane[2], 2, y, x) - 128;
    // jdcolor.c build_ycc_rgb_table (SCALEBITS 16) and ycc_rgb_convert
    const int r = clamp255(Y + ((91881 * cr + 32768) >> 16));
    const int g = clamp255(Y + ((-22554 * cb + 32768 - 46802 * cr) >> 16));
    const int b = clamp255(Y + ((116130 * cb + 32768) >> 16));
    o[i] = bgr2gray(b, g, r);
  }
}

// ------------------------------------------------------------------ host: batches of streams
static void derive_table(const JHuffSpec &s, HT &t) {
  memset(&t, 0, sizeof(t));
  int code = 0, k = 0;
  for (int l = 1; l <= 16; ++l) {
    if (s.bits[l]) {
      t.valoff[l] = k - code;
      for (int j = 0; j < s.bits[l]; ++j, ++k, ++code) {
        t.vals[k] = s.vals[k];
        if (l <= 9)
          for (int p = 0; p < (1 << (9 - l)); ++p) t.lut[(code << (9 - l)) | p] = (uint16_t)(l << 8 | s.vals[k]);
      }
      t.maxcode[l] = code - 1;
    } else {
      t.maxcode[l] = -1;
    }
    code <<= 1;
  }
  t.maxcode[17] = -1;
}

// descriptor of frame h (everything but the buffer offsets)
static void describe(const JHeader &h, JDesc &d) {
  memset(&d, 0, sizeof(d));
  d.status = h.status;
  for (int k = 0; k < MAXTAB; ++k) d.tab[k] = -1;
  if (h.status != SFE_JPEG_OK) return;
  d.H = h.H, d.W = h.W, d.mode = h.sampling, d.Ri = h.Ri;
  const int hmax = h.nc == 1 ? 1 : h.hs[0], vmax = h.nc == 1 ? 1 : h.vs[0];
  d.mcux = (h.W + 8 * hmax - 1) / (8 * hmax), d.mcuy = (h.H + 8 * vmax - 1) / (8 * vmax);
  d.nmcu = d.mcux * d.mcuy;
  d.bpm = h.nc == 1 ? 1 : hmax * vmax + 2;
  d.nblocks = d.nmcu * d.bpm;
  d.nseg = h.Ri ? (d.nmcu + h.Ri - 1) / h.Ri : 1;
  for (int c = 0; c < h.nc; ++c) {
    const int hc = h.nc == 1 ? 1 : h.hs[c], vc = h.nc == 1 ? 1 : h.vs[c];
    d.cw[c] = (h.W * hc + hmax - 1) / hmax, d.ch[c] = (h.H * vc + vmax - 1) / vmax;
    d.pw[c] = d.mcux * hc * 8, d.ph[c] = d.mcuy * vc * 8;
  }
  d.src_len = h.len - h.ecs;
  d.chunk_cap = (int)(d.src_len * 8 / CHUNK_BITS) + d.nseg + 1;
}

// the device-side bytes of a chunk of frames [f0, f0 + nf): descriptors, table pools, entropy-coded data
struct ChunkPlan {
  std::vector<JDesc> desc;
  std::vector<HT> huff;
  std::vector<uint16_t> quant;
  int64_t ecs_bytes = 0, scr_bytes = 0, coef_blocks = 0;
  size_t off_huff = 0, off_quant = 0, off_bytes = 0, total = 0;
};

static void plan_chunk(const StreamBatch<JHeader> &bt, int f0, int nf, ChunkPlan &p) {
  p = ChunkPlan();
  p.desc.resize(nf);
  std::unordered_map<std::string, int> hmap, qmap;
  for (int i = 0; i < nf; ++i) {
    const JHeader &h = bt.hdr[f0 + i];
    JDesc &d = p.desc[i];
    describe(h, d);
    if (d.status != SFE_JPEG_OK) continue;
    int nslot = 0;
    int slot_of[2][4] = {{-1, -1, -1, -1}, {-1, -1, -1, -1}};
    auto use_table = [&](int cls, int id) {
      if (slot_of[cls][id] >= 0) return slot_of[cls][id];
      const JHuffSpec &s = cls ? h.ac[id] : h.dc[id];
      std::string key(reinterpret_cast<const char *>(s.bits), 17);
      key.append(reinterpret_cast<const char *>(s.vals), 256);
      auto it = hmap.find(key);
      int pi;
      if (it == hmap.end()) {
        pi = (int)p.huff.size();
        p.huff.emplace_back();
        derive_table(s, p.huff.back());
        hmap.emplace(key, pi);
      } else {
        pi = it->second;
      }
      d.tab[nslot] = pi;
      return slot_of[cls][id] = nslot++;
    };
    for (int c = 0; c < h.nc; ++c) {
      const std::string key(reinterpret_cast<const char *>(h.q[h.tq[c]]), 128);
      auto it = qmap.find(key);
      if (it == qmap.end()) {
        it = qmap.emplace(key, (int)(p.quant.size() / 64)).first;
        p.quant.insert(p.quant.end(), h.q[h.tq[c]], h.q[h.tq[c]] + 64);
      }
      d.qtab[c] = it->second;
    }
    int b = 0;
    for (int c = 0; c < h.nc; ++c) {
      const int nb = h.nc == 1 ? 1 : h.hs[c] * h.vs[c];
      const int sd = use_table(0, h.td[c]), sa = use_table(1, h.ta[c]);
      for (int j = 0; j < nb; ++j, ++b) d.bcomp[b] = (int8_t)c, d.bdc[b] = (int8_t)sd, d.bac[b] = (int8_t)sa;
    }
    if (h.H != bt.R_of(f0 + i) || h.W != bt.B_of(f0 + i)) {
      d.status = SFE_JPEG_SIZE;
      continue;
    }
    d.src = p.ecs_bytes;
    p.ecs_bytes += al16(d.src_len);
    d.scr = p.scr_bytes;
    p.scr_bytes += jlayout(d).total;
    d.coef = p.coef_blocks;
    p.coef_blocks += d.nblocks;
  }
  if (p.huff.empty()) p.huff.emplace_back();
  if (p.quant.empty()) p.quant.resize(64);
  p.off_huff = al16(sizeof(JDesc) * nf);
  p.off_quant = p.off_huff + al16(sizeof(HT) * p.huff.size());
  p.off_bytes = p.off_quant + al16(2 * p.quant.size());
  p.total = p.off_bytes + p.ecs_bytes + 16;
}

enum { JPEG_CHUNK = 256 };

struct JpegState final : StreamDecoder {
  StreamBatch<JHeader> bt;
  Buffer scr, coef;
  // sfe_jpeg_coefficients_host: with cap_blocks > 0 every chunk also writes its dequantised coefficients
  // (int32 [nf][cap_blocks][64], in ctx->stage_out[0]) and copies them to coef_host
  int cap_blocks = 0;
  int32_t *coef_host = nullptr;

  ~JpegState() override {
    for (Buffer *b : {&scr, &coef})
      if (b->ptr) cudaFree(b->ptr);
  }
  int chunk_frames(const sfe_ctx *) const override { return cap_blocks > 0 ? 16 : JPEG_CHUNK; }
  void parse(const uint8_t *bytes, const int64_t *offsets, int n, int R, int B, const int32_t *shape) override {
    bt.parse(bytes, offsets, n, R, B, shape, parse_header, SFE_JPEG_SIZE);
  }
  int frame_status(int i) const override { return bt.hdr[i].status; }
  const char *message(int status) const override { return sfe_jpeg_status_message(status); }
  int reserve(sfe_ctx *ctx, int chunk, size_t out_bytes) override;
  int decode_chunk(sfe_ctx *ctx, int f0, int nf, uint8_t *out_dev) override;
};

StreamDecoder *jpeg_decoder(sfe_ctx *ctx) {
  if (!ctx->jpeg) ctx->jpeg = new JpegState();
  return ctx->jpeg;
}
void destroy(JpegState *s) { delete s; }

int JpegState::reserve(sfe_ctx *ctx, int chunk, size_t out_bytes) {
  size_t in_max = 0, scr_max = 0, coef_max = 0;
  ChunkPlan p;
  for (int f0 = 0; f0 < bt.n; f0 += chunk) {
    plan_chunk(bt, f0, std::min(chunk, bt.n - f0), p);
    in_max = std::max(in_max, p.total);
    scr_max = std::max(scr_max, (size_t)p.scr_bytes);
    coef_max = std::max(coef_max, (size_t)p.coef_blocks * 128);
  }
  int rc = ensure(ctx, scr, scr_max + 16);
  if (rc == SFE_OK) rc = ensure(ctx, coef, coef_max + 16);
  if (rc == SFE_OK && cap_blocks > 0) rc = ensure(ctx, ctx->stage_out[0], (size_t)chunk * cap_blocks * 64 * 4);
  return rc == SFE_OK ? reserve_common(ctx, bt.n, in_max, out_bytes) : rc;
}

int JpegState::decode_chunk(sfe_ctx *ctx, int f0, int nf, uint8_t *out_dev) {
  ChunkPlan p;
  plan_chunk(bt, f0, nf, p);
  uint8_t *pin, *dev;
  int rc = stager.acquire(&pin);
  if (rc != SFE_OK) return rc;
  memcpy(pin, p.desc.data(), sizeof(JDesc) * nf);
  memcpy(pin + p.off_huff, p.huff.data(), sizeof(HT) * p.huff.size());
  memcpy(pin + p.off_quant, p.quant.data(), 2 * p.quant.size());
  for (int i = 0; i < nf; ++i) {
    const JDesc &d = p.desc[i];
    if (d.status != SFE_JPEG_OK) continue;
    const JHeader &h = bt.hdr[f0 + i];
    memcpy(pin + p.off_bytes + d.src, bt.bytes + bt.offsets[f0 + i] + h.ecs, d.src_len);
  }
  rc = stager.upload(ctx, p.off_bytes + p.ecs_bytes, &dev);
  if (rc != SFE_OK) return rc;
  const JDesc *desc = reinterpret_cast<const JDesc *>(dev);
  const HT *huff = reinterpret_cast<const HT *>(dev + p.off_huff);
  const uint16_t *quant = reinterpret_cast<const uint16_t *>(dev + p.off_quant);
  uint8_t *s = static_cast<uint8_t *>(scr.ptr);
  int16_t *c = static_cast<int16_t *>(coef.ptr);
  int32_t *st = static_cast<int32_t *>(status.ptr) + f0;
  const int R = bt.R_of(f0), B = bt.B_of(f0);
  const int64_t fstride = (int64_t)R * B;
  timer.tic(ctx->stream, SFE_JPEG_T_UNSTUFF);
  jpeg_unstuff_kernel<<<nf, JT, 0, ctx->stream>>>(desc, dev + p.off_bytes, s, st);
  timer.toc(ctx->stream);
  timer.tic(ctx->stream, SFE_JPEG_T_ENTROPY);
  jpeg_entropy_kernel<<<nf, JT, 0, ctx->stream>>>(desc, huff, s, c, st);
  timer.toc(ctx->stream);
  int maxblk = 1;
  for (const JDesc &d : p.desc) maxblk = std::max(maxblk, d.nblocks);
  timer.tic(ctx->stream, SFE_JPEG_T_PIXELS);
  jpeg_idct_kernel<<<dim3((maxblk + 15) / 16, nf), 128, 0, ctx->stream>>>(desc, quant, s, c, st, out_dev, fstride);
  const int per = (int)std::min<int64_t>((fstride + 1023) / 1024, 64);
  jpeg_color_kernel<<<dim3(per, nf), 256, 0, ctx->stream>>>(desc, s, st, out_dev, fstride, R, B);
  timer.toc(ctx->stream);
  ctx->launches += 4;
  int32_t *coef_dev = static_cast<int32_t *>(ctx->stage_out[0].ptr);
  if (cap_blocks > 0) {
    jpeg_dequant_kernel<<<dim3((int)(((int64_t)cap_blocks * 64 + 255) / 256), nf), 256, 0, ctx->stream>>>(
        desc, quant, s, c, st, cap_blocks, coef_dev);
    ctx->launches++;
  }
  SFE_CUDA(cudaGetLastError());
  rc = stager.done(ctx);
  if (rc != SFE_OK || !coef_host) return rc;
  SFE_CUDA(cudaMemcpyAsync(coef_host + (size_t)f0 * cap_blocks * 64, coef_dev, (size_t)nf * cap_blocks * 64 * 4,
                           cudaMemcpyDeviceToHost, ctx->stream));
  return SFE_OK;
}

}  // namespace sfe

using namespace sfe;

extern "C" {

const char *sfe_jpeg_status_message(int status) {
  switch (status) {
    case SFE_JPEG_OK: return "ok";
    case SFE_JPEG_NOT_JPEG: return "not a JPEG stream (no SOI marker; PNG and other formats stay on the host path)";
    case SFE_JPEG_TRUNCATED: return "headers truncated before the start of scan";
    case SFE_JPEG_PROGRESSIVE: return "progressive JPEG is not supported";
    case SFE_JPEG_LOSSLESS: return "lossless JPEG is not supported";
    case SFE_JPEG_ARITHMETIC: return "arithmetic-coded JPEG is not supported";
    case SFE_JPEG_PRECISION: return "sample precision other than 8 bits (e.g. 12-bit) is not supported";
    case SFE_JPEG_SAMPLING: return "chroma sampling other than 4:4:4, 4:2:2 (2x1) or 4:2:0 (2x2) is not supported";
    case SFE_JPEG_COLORSPACE: return "colour space other than gray or YCbCr (CMYK, RGB) is not supported";
    case SFE_JPEG_ORIENTATION: return "EXIF orientation other than 1 (imdecode would rotate the image)";
    case SFE_JPEG_SIZE: return "frame size differs from the call's R x B";
    case SFE_JPEG_CORRUPT: return "corrupt entropy-coded data";
    case SFE_JPEG_BAD_HEADER: return "malformed or unsupported header (tables, scan layout, hierarchical mode)";
    default: return "unknown status";
  }
}

int sfe_jpeg_inspect_host(const uint8_t *bytes, const int64_t *offsets, int n, int32_t *info) {
  SFE_REQUIRE(bytes && offsets && info, "sfe_jpeg_inspect_host: null argument");
  SFE_REQUIRE(n >= 0, "sfe_jpeg_inspect_host: negative count");
  SFE_REQUIRE(offsets_ok(offsets, n), "sfe_jpeg_inspect_host: offsets must be non-decreasing");
  for (int i = 0; i < n; ++i) {
    JHeader h;
    parse_header(bytes + offsets[i], offsets[i + 1] - offsets[i], h);
    int32_t *o = info + (size_t)SFE_JPEG_INFO * i;
    o[0] = h.status, o[1] = h.H, o[2] = h.W, o[3] = h.nc, o[4] = h.status == SFE_JPEG_OK ? h.sampling : -1, o[5] = h.Ri;
  }
  return SFE_OK;
}

int sfe_jpeg_decode_host(sfe_ctx *ctx, const uint8_t *bytes, const int64_t *offsets, int n, int R, int B,
                         uint8_t *out_host, int32_t *status_host) {
  SFE_REQUIRE(out_host, "sfe_jpeg_decode_host: null output");
  return decode_all(ctx, jpeg_decoder, bytes, offsets, n, R, B, nullptr, out_host, status_host, "sfe_jpeg_decode_host");
}

int sfe_jpeg_decode_to_dev(sfe_ctx *ctx, const uint8_t *bytes_host, const int64_t *offsets_host, int n, int R, int B,
                           uint8_t *out_dev, int32_t *status_host) {
  SFE_REQUIRE(out_dev, "sfe_jpeg_decode_to_dev: null output");
  return decode_all(ctx, jpeg_decoder, bytes_host, offsets_host, n, R, B, out_dev, nullptr, status_host,
                    "sfe_jpeg_decode_to_dev");
}

int sfe_jpeg_coefficients_host(sfe_ctx *ctx, const uint8_t *bytes, const int64_t *offsets, int n, int R, int B,
                               int cap_blocks, int32_t *coef_host, int32_t *status_host) {
  SFE_REQUIRE(coef_host && cap_blocks > 0, "sfe_jpeg_coefficients_host: null output or cap_blocks <= 0");
  SFE_REQUIRE(ctx && bytes && offsets && status_host && n >= 0, "sfe_jpeg_coefficients_host: null argument");
  SFE_REQUIRE(offsets_ok(offsets, n), "sfe_jpeg_coefficients_host: offsets must be non-decreasing");
  for (int i = 0; i < n; ++i) {
    JHeader h;
    parse_header(bytes + offsets[i], offsets[i + 1] - offsets[i], h);
    if (h.status != SFE_JPEG_OK) continue;
    JDesc d;
    describe(h, d);
    if (d.nblocks > cap_blocks) {
      set_error("sfe_jpeg_coefficients_host: frame %d has %d blocks, cap_blocks is %d", i, d.nblocks, cap_blocks);
      return SFE_ERR_CAPACITY;
    }
  }
  JpegState *js = static_cast<JpegState *>(jpeg_decoder(ctx));
  js->cap_blocks = cap_blocks, js->coef_host = coef_host;
  const int rc = decode_all(ctx, jpeg_decoder, bytes, offsets, n, R, B, nullptr, nullptr, status_host,
                            "sfe_jpeg_coefficients_host");
  js->cap_blocks = 0, js->coef_host = nullptr;
  return rc;
}

int sfe_jpeg_set_timing(sfe_ctx *ctx, int enable) {
  SFE_REQUIRE(ctx != nullptr, "sfe_jpeg_set_timing: null context");
  SFE_CUDA(cudaSetDevice(ctx->device));
  jpeg_decoder(ctx)->timer.reset(enable != 0);
  return SFE_OK;
}

int sfe_jpeg_get_timing(sfe_ctx *ctx, double *stage_ms, int64_t *stage_calls) {
  SFE_REQUIRE(ctx && stage_ms, "sfe_jpeg_get_timing: null argument");
  SFE_CUDA(cudaSetDevice(ctx->device));
  return jpeg_decoder(ctx)->timer.collect(ctx->stream, SFE_JPEG_STAGES, stage_ms, stage_calls);
}

}  // extern "C"
