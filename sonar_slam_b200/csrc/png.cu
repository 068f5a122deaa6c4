// PNG decoder for compressed sonar pings (SURVEY 8(f) N4).
//
// The reference decodes every compressed ping on the host with
//     cv2.cvtColor(cv2.imdecode(buf, cv2.IMREAD_COLOR), cv2.COLOR_BGR2GRAY)      (feature_extraction.py:210-213)
// For a PNG that is libpng + zlib, then OpenCV's fixed-point BGR -> gray.  This file computes the same uint8 frames on
// the device, bit for bit, for the streams it accepts (include/sonarfe.h: sfe_png_*): 8-bit gray or truecolour, not
// interlaced, any deflate content and any row filter.
//
// Host: the chunk list is walked (signature, IHDR and its CRC, every chunk header, IEND); nothing is inflated or
// checksummed there.  The span holding the IDAT chunks travels to the device.
//
// Device, per chunk of frames:
//   png_check_kernel     one CTA per frame: every IDAT's data is cut into 1 KB slices, one thread each; a thread
//                        computes the CRC-32 of its slice, shifts it to the chunk's end (multiplication by
//                        x^(8 n) mod P) and XORs it into the chunk's CRC, so no slice waits for another; it also
//                        gathers the slice into the frame's contiguous zlib stream.
//   png_inflate_kernel   one warp per frame, 4 frames per CTA: all 32 lanes decode the same Huffman symbols from a
//                        64-bit bit buffer (tables in the warp's shared memory: a 10-bit lookahead for literal /
//                        length codes, 8 bits for distances, canonical decoding for longer codes); literals are
//                        stored by one lane, back-references and stored blocks are copied by the whole warp
//                        (byte i of a copy is byte i mod distance of the source, so short distances replicate).
//                        The output is the filtered scanlines; bytes past the last row go to a 32 KB ring, so they
//                        still serve as a window, and their Adler-32 sums are taken on the fly.
//   png_unfilter_kernel  one warp per frame: rows in order, 32 pixels per step: None / Up are per pixel, Sub is a
//                        per-channel warp scan, Average / Paeth pass the left pixel lane to lane (32 dependent steps
//                        per 32 pixels).  Unfiltered rows replace the filtered ones in place (the next row's "up"),
//                        gray goes straight to the output frame (truecolour through BGR2GRAY in the same pass).  The
//                        Adler-32 of the whole inflated data is summed here in any order (s1 = 1 + sum b_i,
//                        s2 = L + sum (L - i) b_i) and checked; a frame that fails anything is written as zeros.
// Every device read and write is bounded by the frame's own bytes and scratch.
#include <algorithm>
#include <vector>

#include "stream_decode.cuh"

namespace sfe {

enum { PNG_CHECK_T = 256, PNG_SLICE = 1024, PNG_WARPS = 4, PNG_LBITS = 10, PNG_DBITS = 8, PNG_RING = 32768 };
static const uint32_t kAdlerMod = 65521;
static const int64_t kPngMaxDim = 1000000;  // libpng's default user limit on width and height

// ------------------------------------------------------------------ host-side chunk walk
struct PHeader {
  int status = SFE_PNG_OK;
  int H = 0, W = 0, ctype = 0;
  int64_t span0 = 0, span1 = 0;                   // bytes of the IDAT chunks (first length field .. last CRC)
  std::vector<std::pair<int64_t, int32_t>> idat;  // data offset in the stream, length
};

static uint32_t be32(const uint8_t *p) { return (uint32_t)p[0] << 24 | p[1] << 16 | p[2] << 8 | p[3]; }

static uint32_t crc32_host(const uint8_t *p, int64_t n) {
  uint32_t c = 0xFFFFFFFFu;
  for (int64_t i = 0; i < n; ++i) {
    c ^= p[i];
    for (int k = 0; k < 8; ++k) c = (c >> 1) ^ (0xEDB88320u & (0u - (c & 1)));
  }
  return c ^ 0xFFFFFFFFu;
}

// What libpng (as OpenCV 4.13 drives it) decides from the chunk list; decode-time checks are the device's.
static void parse_png(const uint8_t *p, int64_t n, PHeader &h) {
  h = PHeader();
  auto fail = [&](int st) { h.status = st; };
  static const uint8_t sig[8] = {0x89, 'P', 'N', 'G', 0x0D, 0x0A, 0x1A, 0x0A};
  if (n < 8 || memcmp(p, sig, 8) != 0) return fail(SFE_PNG_NOT_PNG);
  int64_t i = 8;
  bool after_idat = false;
  int orient = 1, depth = 0;
  for (int k = 0;; ++k) {
    if (i + 8 > n) return fail(SFE_PNG_TRUNCATED);
    const uint32_t len = be32(p + i);
    const uint8_t *t = p + i + 4;
    if (len > 0x7FFFFFFFu) return fail(SFE_PNG_BAD_HEADER);
    if (i + 12 + (int64_t)len > n) return fail(SFE_PNG_TRUNCATED);
    const uint8_t *d = p + i + 8;
    for (int c = 0; c < 4; ++c)
      if (!((t[c] >= 'A' && t[c] <= 'Z') || (t[c] >= 'a' && t[c] <= 'z'))) return fail(SFE_PNG_BAD_HEADER);
    const bool is_idat = !memcmp(t, "IDAT", 4);
    if (k == 0) {
      if (memcmp(t, "IHDR", 4) || len != 13 || crc32_host(t, 17) != be32(d + 13)) return fail(SFE_PNG_BAD_HEADER);
      const uint32_t w = be32(d), hh = be32(d + 4);
      depth = d[8], h.ctype = d[9];
      if (w == 0 || hh == 0 || w > kPngMaxDim || hh > kPngMaxDim) return fail(SFE_PNG_BAD_HEADER);
      h.W = (int)w, h.H = (int)hh;
      const int ct = h.ctype;
      const bool depth_ok = ct == 0   ? (depth == 1 || depth == 2 || depth == 4 || depth == 8 || depth == 16)
                            : ct == 3 ? (depth == 1 || depth == 2 || depth == 4 || depth == 8)
                            : (ct == 2 || ct == 4 || ct == 6) && (depth == 8 || depth == 16);
      if (!depth_ok || d[10] != 0 || d[11] != 0 || d[12] > 1) return fail(SFE_PNG_BAD_HEADER);
    } else if (is_idat) {
      if (after_idat && (h.idat.empty() || h.span1 != i)) return fail(SFE_PNG_BAD_HEADER);  // not consecutive
      if (h.idat.empty()) h.span0 = i;
      h.idat.emplace_back(i + 8, (int32_t)len);
      h.span1 = i + 12 + len;
      after_idat = true;
    } else if (!memcmp(t, "IEND", 4)) {  // its CRC is not read: libpng only warns
      break;
    } else if (!memcmp(t, "IHDR", 4)) {
      return fail(SFE_PNG_BAD_HEADER);
    } else if (!memcmp(t, "PLTE", 4)) {
      if (after_idat || h.ctype == 3) return fail(h.ctype == 3 ? SFE_PNG_COLORTYPE : SFE_PNG_BAD_HEADER);
      // types 0 / 2: libpng ignores it (a suggested palette); the image does not change
    } else if (!(t[0] & 0x20)) {
      return fail(SFE_PNG_BAD_HEADER);  // unknown critical chunk
    } else if (!memcmp(t, "acTL", 4)) {
      return fail(SFE_PNG_ANIMATED);
    } else if (!memcmp(t, "eXIf", 4)) {
      if (orient == 1) orient = tiff_orientation(d, len);
    }
    // other ancillary chunks (and their CRCs) are ignored, as libpng ignores them
    i += 12 + (int64_t)len;
  }
  if (h.idat.empty()) return fail(SFE_PNG_BAD_HEADER);
  if (depth != 8) return fail(SFE_PNG_DEPTH);
  if (h.ctype != 0 && h.ctype != 2) return fail(SFE_PNG_COLORTYPE);
  if (p[8 + 8 + 12] == 1) return fail(SFE_PNG_INTERLACED);
  if (orient >= 2 && orient <= 8) return fail(SFE_PNG_ORIENTATION);
}

// ------------------------------------------------------------------ device descriptors
struct PDesc {
  int32_t status;          // 0: decode; otherwise the host's SFE_PNG_* verdict
  int32_t H, W, C;         // geometry, channels (1 gray, 3 truecolour)
  int32_t idat0, nidat;    // the frame's IDAT entries in the chunk's table
  int64_t zlen;            // zlib stream bytes (sum of the IDAT lengths)
  int64_t nslice;          // CRC slices over all IDATs
  int64_t img;             // filtered scanline bytes, H * (1 + W * C)
  int64_t scr;             // this frame's scratch (byte offset)
};

struct PIdat {
  int64_t data;            // first data byte in the chunk's byte buffer (the CRC follows the data)
  int64_t zoff;            // where the data goes in the frame's zlib stream
  int64_t slice0;          // first CRC slice
  int32_t len, pad;
};

struct PRes {              // inflate -> unfilter hand-over
  int64_t olen;            // inflated bytes (may exceed img)
  uint32_t adler;          // the stream's stored Adler-32
  uint32_t ex_sum;         // sum of the inflated bytes past img, mod 65521
  uint32_t ex_isum;        // sum of i * b_i over those bytes, mod 65521
  uint32_t pad[3];
};

struct PLayout {
  int64_t res, acc, zbuf, img, total;
};

__host__ __device__ inline int64_t pal16(int64_t x) { return (x + 15) & ~(int64_t)15; }

__host__ __device__ inline PLayout playout(const PDesc &d) {
  PLayout L;
  int64_t o = d.scr;
  L.res = o, o += pal16(sizeof(PRes));
  L.acc = o, o += pal16(4 * (int64_t)d.nidat);
  L.zbuf = o, o += pal16(d.zlen + 16);
  L.img = o, o += pal16(d.img + PNG_RING);
  L.total = o - d.scr;
  return L;
}

struct X2N {               // x^(2^k) mod P (reflected CRC-32 polynomial), k = 0..31
  uint32_t t[32];
};

// ------------------------------------------------------------------ device: CRC-32 and gather
__device__ __forceinline__ uint32_t multmodp(uint32_t a, uint32_t b) {  // a * b mod P, reflected
  uint32_t m = 1u << 31, p = 0;
  for (;;) {
    if (a & m) {
      p ^= b;
      if ((a & (m - 1)) == 0) break;
    }
    m >>= 1;
    b = b & 1 ? (b >> 1) ^ 0xEDB88320u : b >> 1;
  }
  return p;
}

// the CRC register `crc` followed by n zero bytes (x^(8 n) mod P times crc)
__device__ uint32_t crc_shift(const X2N &x, uint32_t crc, int64_t n) {
  uint32_t p = 1u << 31;
  int k = 3;
  while (n) {
    if (n & 1) p = multmodp(x.t[k & 31], p);
    n >>= 1, ++k;
  }
  return multmodp(p, crc);
}

__global__ void __launch_bounds__(PNG_CHECK_T) png_check_kernel(const PDesc *__restrict__ desc,
                                                                const PIdat *__restrict__ idat,
                                                                const uint8_t *__restrict__ bytes,
                                                                uint8_t *__restrict__ scr, int32_t *__restrict__ status,
                                                                X2N x2n) {
  const int f = blockIdx.x, tid = threadIdx.x;
  const PDesc &d = desc[f];
  if (d.status != SFE_PNG_OK) {
    if (tid == 0) status[f] = d.status;
    return;
  }
  __shared__ uint32_t tab[256];
  __shared__ int s_bad;
  {
    uint32_t c = tid;
    for (int k = 0; k < 8; ++k) c = (c >> 1) ^ (0xEDB88320u & (0u - (c & 1)));
    tab[tid] = c;
  }
  if (tid == 0) s_bad = 0;
  const PLayout L = playout(d);
  uint32_t *acc = reinterpret_cast<uint32_t *>(scr + L.acc);
  uint8_t *z = scr + L.zbuf;
  const PIdat *id = idat + d.idat0;
  __syncthreads();
  // the register after 0xFFFFFFFF, "IDAT" and len zero bytes; the data's own contributions are XORed in below
  uint32_t s0 = 0xFFFFFFFFu;
  for (int k = 0; k < 4; ++k) s0 = tab[(s0 ^ "IDAT"[k]) & 255] ^ (s0 >> 8);
  for (int k = tid; k < d.nidat; k += PNG_CHECK_T) acc[k] = crc_shift(x2n, s0, id[k].len);
  if (tid < 16) z[d.zlen + tid] = 0;
  __syncthreads();
  for (int64_t g = tid; g < d.nslice; g += PNG_CHECK_T) {
    int lo = 0, hi = d.nidat - 1;  // the IDAT holding slice g: last one with slice0 <= g
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (id[mid].slice0 <= g) lo = mid; else hi = mid - 1;
    }
    const PIdat e = id[lo];
    const int64_t a = (g - e.slice0) * PNG_SLICE, b = min(a + (int64_t)PNG_SLICE, (int64_t)e.len);
    const uint8_t *src = bytes + e.data;
    uint32_t c = 0;
    for (int64_t i = a; i < b; ++i) {
      const uint8_t v = src[i];
      c = tab[(c ^ v) & 255] ^ (c >> 8);
      z[e.zoff + i] = v;
    }
    atomicXor(&acc[lo], crc_shift(x2n, c, e.len - b));
  }
  __syncthreads();
  for (int k = tid; k < d.nidat; k += PNG_CHECK_T) {
    const uint8_t *q = bytes + id[k].data + id[k].len;
    const uint32_t stored = (uint32_t)q[0] << 24 | q[1] << 16 | q[2] << 8 | q[3];
    if ((acc[k] ^ 0xFFFFFFFFu) != stored) s_bad = 1;
  }
  __syncthreads();
  if (tid == 0) status[f] = s_bad ? SFE_PNG_CORRUPT : SFE_PNG_OK;
}

// ------------------------------------------------------------------ device: inflate
__constant__ uint16_t c_lbase[29] = {3,  4,  5,  6,  7,  8,  9,  10, 11,  13,  15,  17,  19,  23, 27,
                                     31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258};
__constant__ uint8_t c_lext[29] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0};
__constant__ uint16_t c_dbase[30] = {1,    2,    3,    4,    5,    7,     9,     13,    17,  25,   33,   49,   65,   97,  129,
                                     193,  257,  385,  513,  769,  1025,  1537,  2049,  3073, 4097, 6145, 8193, 12289, 16385, 24577};
__constant__ uint8_t c_dext[30] = {0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13};
__constant__ uint8_t c_clorder[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};

struct WarpTables {          // one warp's Huffman tables
  uint16_t ll[1 << PNG_LBITS];  // literal / length lookahead: symbol | length << 9; 0 = longer code or none
  uint16_t dl[1 << PNG_DBITS];  // distance lookahead (the code-length code uses its first 128 entries)
  uint16_t lsym[320], dsym[32]; // symbols in canonical order
  uint16_t lcnt[16], dcnt[16];  // codes per length
  uint16_t code[320];
  uint8_t lens[320];            // literal / length then distance code lengths of the block
};

// Canonical code of n lengths -> lookahead table of `bits` bits, counts and sorted symbols.  Returns false on an
// over-subscribed set, or an incomplete one unless zlib accepts it (a lone code of length 1, or no code at all for
// distances: `allow_empty`).  Called by the whole warp.
__device__ bool build_table(const uint8_t *len, int n, int bits, uint16_t *lut, uint16_t *cnt, uint16_t *sym,
                            uint16_t *code, bool complete_only, bool allow_empty) {
  const int lane = threadIdx.x & 31;
  int ok = 1;
  if (lane == 0) {
    for (int l = 0; l < 16; ++l) cnt[l] = 0;
    for (int s = 0; s < n; ++s) cnt[len[s]]++;
    cnt[0] = 0;
    int left = 1, maxl = 0;
    for (int l = 1; l < 16; ++l) {
      left = (left << 1) - cnt[l];
      if (left < 0) ok = 0;
      if (cnt[l]) maxl = l;
    }
    if (maxl == 0) {
      if (!allow_empty) ok = 0;
    } else if (left > 0 && (complete_only || maxl != 1)) {
      ok = 0;
    }
    uint16_t offs[16], next[16];
    int o = 0, c = 0;
    for (int l = 1; l < 16; ++l) offs[l] = o, o += cnt[l], next[l] = c, c = (c + cnt[l]) << 1;
    for (int s = 0; s < n; ++s)
      if (len[s]) sym[offs[len[s]]++] = s, code[s] = next[len[s]]++;
  }
  ok = __shfl_sync(0xffffffffu, ok, 0);
  if (!ok) return false;
  for (int e = lane; e < (1 << bits); e += 32) lut[e] = 0;
  __syncwarp();
  for (int s = lane; s < n; s += 32) {
    const int l = len[s];
    if (l == 0 || l > bits) continue;
    const uint32_t r = __brev((uint32_t)code[s]) >> (32 - l);
    for (uint32_t e = r; e < (1u << bits); e += 1u << l) lut[e] = (uint16_t)(s | l << 9);
  }
  __syncwarp();
  return true;
}

struct BitIn {                // the zlib stream, least significant bit first
  const uint32_t *w;
  int64_t k, kmax;            // next word, words readable (zero padding included)
  uint64_t bb;
  int bc;
  __device__ void refill() {
    if (bc < 32) {
      bb |= (uint64_t)(k < kmax ? w[k] : 0u) << bc;
      ++k, bc += 32;
    }
  }
  __device__ uint32_t take(int n) {  // n <= 32 bits, after a refill
    const uint32_t v = (uint32_t)(bb & ((1ull << n) - 1));
    bb >>= n, bc -= n;
    return v;
  }
  __device__ int64_t consumed() const { return k * 32 - bc; }
  __device__ void seek_byte(int64_t pos) {
    k = pos >> 2, bb = 0, bc = 0;
    const int sh = (int)(pos & 3) * 8;
    if (sh) {
      bb = (uint64_t)(k < kmax ? w[k] : 0u) >> sh;
      ++k, bc = 32 - sh;
    }
    refill();
  }
};

__device__ __forceinline__ int decode_sym(BitIn &in, const uint16_t *lut, int bits, const uint16_t *cnt,
                                          const uint16_t *sym) {
  const uint32_t e = lut[in.bb & ((1u << bits) - 1)];
  if (e) {
    const int l = e >> 9;
    in.bb >>= l, in.bc -= l;
    return e & 511;
  }
  int code = 0, first = 0, index = 0;  // canonical decoding, one bit at a time
  uint64_t b = in.bb;
  for (int l = 1; l < 16; ++l) {
    code |= (int)(b & 1);
    b >>= 1;
    const int count = cnt[l];
    if (code - count < first) {
      in.bb >>= l, in.bc -= l;
      return sym[index + (code - first)];
    }
    index += count, first += count;
    first <<= 1, code <<= 1;
  }
  return -1;
}

__global__ void __launch_bounds__(32 * PNG_WARPS) png_inflate_kernel(const PDesc *__restrict__ desc, int nf,
                                                                     uint8_t *__restrict__ scr,
                                                                     int32_t *__restrict__ status) {
  __shared__ WarpTables tables[PNG_WARPS];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int f = blockIdx.x * PNG_WARPS + wid;
  if (f >= nf || status[f] != SFE_PNG_OK) return;  // whole warps leave together
  const PDesc &d = desc[f];
  WarpTables &T = tables[wid];
  const PLayout L = playout(d);
  const uint8_t *zb = scr + L.zbuf;
  uint8_t *o = scr + L.img;
  const int64_t cap = d.img, zbits = d.zlen * 8;
  BitIn in{reinterpret_cast<const uint32_t *>(zb), 0, (d.zlen + 16) >> 2, 0, 0};
  int64_t p = 0;
  uint64_t ex_sum = 0, ex_isum = 0;  // this lane's writes past cap
  auto put = [&](int64_t q, uint8_t v) {
    if (q < cap) {
      o[q] = v;
    } else {
      o[cap + (q & (PNG_RING - 1))] = v;
      ex_sum += v, ex_isum += (uint64_t)(q % kAdlerMod) * v;
    }
  };
  auto get = [&](int64_t q) -> uint8_t { return q < cap ? o[q] : o[cap + (q & (PNG_RING - 1))]; };
  bool bad = d.zlen < 2;
  int window = 0;
  if (!bad) {
    const int cmf = zb[0], flg = zb[1];
    // RFC 1950: deflate, window <= 32 KB, check bits, no preset dictionary
    bad = (cmf & 15) != 8 || (cmf >> 4) > 7 || ((cmf << 8) | flg) % 31 != 0 || (flg & 0x20);
    window = 1 << ((cmf >> 4) + 8);
  }
  if (!bad) in.seek_byte(2);
  int loaded = 0;  // 1: the fixed tables are in T
  bool last = bad;
  while (!last) {
    in.refill();
    last = in.take(1);
    const int type = in.take(2);
    if (type == 0) {  // stored
      in.take(in.bc & 7);
      const int64_t q = in.consumed() >> 3;
      if (q + 4 > d.zlen) { bad = true; break; }
      const int len = zb[q] | zb[q + 1] << 8, nlen = zb[q + 2] | zb[q + 3] << 8;
      if ((len ^ 0xFFFF) != nlen || q + 4 + len > d.zlen) { bad = true; break; }
      for (int i = lane; i < len; i += 32) put(p + i, zb[q + 4 + i]);
      p += len;
      in.seek_byte(q + 4 + len);
      __syncwarp();
      continue;
    }
    if (type == 3) { bad = true; break; }
    if (type == 1) {
      if (!loaded) {
        for (int s = lane; s < 320; s += 32)
          T.lens[s] = s < 144 ? 8 : s < 256 ? 9 : s < 280 ? 7 : s < 288 ? 8 : 5;
        __syncwarp();
        // complete codes over 288 / 32 symbols; 286, 287 and distances 30, 31 are rejected when they occur
        build_table(T.lens, 288, PNG_LBITS, T.ll, T.lcnt, T.lsym, T.code, false, false);
        build_table(T.lens + 288, 32, PNG_DBITS, T.dl, T.dcnt, T.dsym, T.code, false, false);
        loaded = 1;
      }
    } else {  // dynamic
      loaded = 0;
      const int nlen = in.take(5) + 257, ndist = in.take(5) + 1, ncode = in.take(4) + 4;
      if (nlen > 286 || ndist > 30) { bad = true; break; }
      in.refill();
      if (lane < 19) T.lens[lane] = 0;
      __syncwarp();
      for (int s = 0; s < ncode; ++s) {
        if (s == 10) in.refill();
        const uint8_t v = (uint8_t)in.take(3);
        if (lane == 0) T.lens[c_clorder[s]] = v;
      }
      __syncwarp();
      if (!build_table(T.lens, 19, 7, T.dl, T.dcnt, T.dsym, T.code, true, false)) { bad = true; break; }
      // the literal / length and distance code lengths, one run-length alphabet: length n goes to T.lens[n]
      // (literal / length) or T.lens[288 + n - nlen] (distance); the code-length code is in T.dl by now
      for (int s = lane; s < 320; s += 32) T.lens[s] = 0;
      __syncwarp();
      int n = 0, prev = -1;
      while (n < nlen + ndist) {
        in.refill();
        const int s = decode_sym(in, T.dl, 7, T.dcnt, T.dsym);
        if (s < 0) { bad = true; break; }
        int rep = 1, v = s;
        if (s == 16) {
          if (prev < 0) { bad = true; break; }
          rep = 3 + in.take(2), v = prev;
        } else if (s == 17) {
          rep = 3 + in.take(3), v = 0;
        } else if (s == 18) {
          rep = 11 + in.take(7), v = 0;
        }
        if (n + rep > nlen + ndist) { bad = true; break; }
        if (lane == 0)
          for (int j = n; j < n + rep; ++j) T.lens[j < nlen ? j : 288 + j - nlen] = (uint8_t)v;
        n += rep, prev = v;
      }
      if (bad) break;
      __syncwarp();
      if (T.lens[256] == 0) { bad = true; break; }  // no end-of-block code
      if (!build_table(T.lens, nlen, PNG_LBITS, T.ll, T.lcnt, T.lsym, T.code, false, false) ||
          !build_table(T.lens + 288, ndist, PNG_DBITS, T.dl, T.dcnt, T.dsym, T.code, false, true)) {
        bad = true;
        break;
      }
    }
    // the block's symbols
    for (;;) {
      if (in.consumed() > zbits) { bad = true; break; }  // ran past the stream's end
      in.refill();
      const int s = decode_sym(in, T.ll, PNG_LBITS, T.lcnt, T.lsym);
      if (s < 256) {
        if (s < 0) { bad = true; break; }
        if (lane == 0) put(p, (uint8_t)s);
        ++p;
        continue;
      }
      if (s == 256) break;
      if (s > 285) { bad = true; break; }
      const int len = c_lbase[s - 257] + (int)in.take(c_lext[s - 257]);
      in.refill();
      const int ds = decode_sym(in, T.dl, PNG_DBITS, T.dcnt, T.dsym);
      if (ds < 0 || ds > 29) { bad = true; break; }
      const int dist = c_dbase[ds] + (int)in.take(c_dext[ds]);
      if (dist > p || dist > window) { bad = true; break; }
      __syncwarp();
      for (int i = lane; i < len; i += 32) put(p + i, get(p - dist + (dist >= len ? i : i % dist)));
      p += len;
    }
    __syncwarp();
    if (bad) break;
  }
  if (!bad) {  // the Adler-32 after the last block, byte aligned
    in.take(in.bc & 7);
    const int64_t q = in.consumed() >> 3;
    if (q + 4 > d.zlen || p < cap) {
      bad = true;
    } else if (lane == 0) {
      PRes *r = reinterpret_cast<PRes *>(scr + L.res);
      r->olen = p;
      r->adler = (uint32_t)zb[q] << 24 | zb[q + 1] << 16 | zb[q + 2] << 8 | zb[q + 3];
    }
  }
  ex_sum %= kAdlerMod, ex_isum %= kAdlerMod;
#pragma unroll
  for (int m = 16; m; m >>= 1) {
    ex_sum += __shfl_xor_sync(0xffffffffu, ex_sum, m);
    ex_isum += __shfl_xor_sync(0xffffffffu, ex_isum, m);
  }
  if (lane == 0) {
    if (bad) {
      status[f] = SFE_PNG_CORRUPT;
    } else {
      PRes *r = reinterpret_cast<PRes *>(scr + L.res);
      r->ex_sum = (uint32_t)(ex_sum % kAdlerMod), r->ex_isum = (uint32_t)(ex_isum % kAdlerMod);
    }
  }
}

// ------------------------------------------------------------------ device: unfilter, gray, Adler-32
__device__ __forceinline__ int paeth(int a, int b, int c) {
  const int pa = abs(b - c), pb = abs(a - c), pc = abs(a + b - 2 * c);
  return (pa <= pb && pa <= pc) ? a : (pb <= pc ? b : c);
}

// Rows of one frame (C channels): unfilter in place, gray into fo, this lane's Adler-32 sums.  False on a filter
// byte above 4.  Called by the whole warp; everything that decides control flow is uniform across it.
template <int C>
__device__ bool unfilter_rows(const PDesc &d, uint8_t *img, uint8_t *fo, uint64_t &sum, uint64_t &isum) {
  const int lane = threadIdx.x & 31;
  const int W = d.W, stride = 1 + W * C;
  for (int y = 0; y < d.H; ++y) {
    uint8_t *row = img + (int64_t)y * stride;
    const uint8_t *up_row = y ? row - stride : nullptr;
    const int ft = row[0];
    if (ft > 4) return false;
    uint32_t rs = lane == 0 ? ft : 0;  // this row's sum b and sum offset * b
    uint64_t ro = 0;
    int carry[C], carry_up[C];
#pragma unroll
    for (int c = 0; c < C; ++c) carry[c] = carry_up[c] = 0;
    for (int x0 = 0; x0 < W; x0 += 32) {
      const int x = x0 + lane, nv = min(32, W - x0);
      const bool valid = lane < nv;
      int v[C], raw[C], up[C];
#pragma unroll
      for (int c = 0; c < C; ++c) {
        const int off = 1 + x * C + c;
        raw[c] = valid ? row[off] : 0;
        up[c] = valid && up_row ? up_row[off] : 0;
        rs += raw[c], ro += (uint64_t)off * raw[c];
      }
#pragma unroll
      for (int c = 0; c < C; ++c) {
        if (ft == 0) {
          v[c] = raw[c];
        } else if (ft == 2) {
          v[c] = raw[c] + up[c];
        } else if (ft == 1) {
          int s = raw[c];
#pragma unroll
          for (int m = 1; m < 32; m <<= 1) {
            const int t = __shfl_up_sync(0xffffffffu, s, m);
            if (lane >= m) s += t;
          }
          v[c] = s + carry[c];
        } else {  // Average / Paeth: the left pixel passes from lane to lane
          int left = carry[c], ul = carry_up[c], mine = 0;
          for (int j = 0; j < nv; ++j) {
            const int r = __shfl_sync(0xffffffffu, raw[c], j), u = __shfl_sync(0xffffffffu, up[c], j);
            const int pred = ft == 3 ? (left + u) >> 1 : paeth(left, u, ul);
            const int val = (r + pred) & 255;
            if (lane == j) mine = val;
            left = val, ul = u;
          }
          v[c] = mine;
        }
        v[c] &= 255;
        carry[c] = __shfl_sync(0xffffffffu, v[c], nv - 1);
        carry_up[c] = __shfl_sync(0xffffffffu, up[c], nv - 1);
        if (valid) row[1 + x * C + c] = (uint8_t)v[c];
      }
      if (valid) fo[(int64_t)y * W + x] = C == 1 ? (uint8_t)v[0] : bgr2gray(v[C - 1], v[1 % C], v[0]);
    }
    const uint64_t base = ((uint64_t)y * stride) % kAdlerMod;
    sum += rs;
    isum = (isum + base * rs + ro) % kAdlerMod;
    __syncwarp();  // this row, unfiltered in place, is the next row's "up"
  }
  return true;
}

__global__ void __launch_bounds__(32 * PNG_WARPS) png_unfilter_kernel(const PDesc *__restrict__ desc, int nf,
                                                                      uint8_t *__restrict__ scr,
                                                                      int32_t *__restrict__ status,
                                                                      uint8_t *__restrict__ out, int64_t fstride) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int f = blockIdx.x * PNG_WARPS + wid;
  if (f >= nf) return;
  const PDesc &d = desc[f];
  uint8_t *fo = out + (int64_t)f * fstride;
  bool bad = status[f] != SFE_PNG_OK;
  if (!bad) {
    const PLayout L = playout(d);
    uint64_t sum = 0, isum = 0;  // this lane's sum b_i and sum i * b_i (mod 65521)
    bad = !(d.C == 1 ? unfilter_rows<1>(d, scr + L.img, fo, sum, isum) : unfilter_rows<3>(d, scr + L.img, fo, sum, isum));
    if (!bad) {
      sum %= kAdlerMod;
#pragma unroll
      for (int m = 16; m; m >>= 1) {
        sum += __shfl_xor_sync(0xffffffffu, sum, m);
        isum += __shfl_xor_sync(0xffffffffu, isum, m);
      }
      const PRes *r = reinterpret_cast<const PRes *>(scr + L.res);
      const uint64_t Lm = (uint64_t)(r->olen % kAdlerMod);
      const uint64_t S = (sum + r->ex_sum) % kAdlerMod, IS = (isum + r->ex_isum) % kAdlerMod;
      const uint32_t s1 = (uint32_t)((1 + S) % kAdlerMod);
      const uint32_t s2 = (uint32_t)((Lm + Lm * S + kAdlerMod - IS) % kAdlerMod);
      bad = ((s2 << 16) | s1) != r->adler;
    }
    if (bad && lane == 0) status[f] = SFE_PNG_CORRUPT;
  }
  if (bad)
    for (int64_t i = lane; i < fstride; i += 32) fo[i] = 0;
}

// ------------------------------------------------------------------ host: batches of streams
static uint32_t multmodp_host(uint32_t a, uint32_t b) {
  uint32_t m = 1u << 31, p = 0;
  for (;;) {
    if (a & m) {
      p ^= b;
      if ((a & (m - 1)) == 0) break;
    }
    m >>= 1;
    b = b & 1 ? (b >> 1) ^ 0xEDB88320u : b >> 1;
  }
  return p;
}

// the device-side bytes of a chunk of frames [f0, f0 + nf): descriptors, IDAT table, IDAT spans
struct PngPlan {
  std::vector<PDesc> desc;
  std::vector<PIdat> idat;
  std::vector<int64_t> src;       // span start in the chunk's byte buffer, per frame
  int64_t span_bytes = 0, scr_bytes = 0;
  size_t off_idat = 0, off_bytes = 0, total = 0;
};

static void plan_png_chunk(const StreamBatch<PHeader> &bt, int f0, int nf, PngPlan &p) {
  p = PngPlan();
  p.desc.resize(nf);
  p.src.assign(nf, 0);
  for (int i = 0; i < nf; ++i) {
    const PHeader &h = bt.hdr[f0 + i];
    PDesc &d = p.desc[i];
    memset(&d, 0, sizeof(d));
    d.status = h.status;
    if (h.status != SFE_PNG_OK) continue;
    d.H = h.H, d.W = h.W, d.C = h.ctype == 2 ? 3 : 1;
    d.img = (int64_t)d.H * (1 + (int64_t)d.W * d.C);
    d.idat0 = (int32_t)p.idat.size(), d.nidat = (int32_t)h.idat.size();
    p.src[i] = p.span_bytes;
    for (const auto &e : h.idat) {
      PIdat q;
      q.data = p.span_bytes + (e.first - h.span0), q.len = e.second, q.pad = 0;
      q.zoff = d.zlen, q.slice0 = d.nslice;
      d.zlen += e.second, d.nslice += (e.second + PNG_SLICE - 1) / PNG_SLICE;
      p.idat.push_back(q);
    }
    p.span_bytes += pal16(h.span1 - h.span0);
    d.scr = p.scr_bytes;
    p.scr_bytes += playout(d).total;
  }
  if (p.idat.empty()) p.idat.emplace_back();
  p.off_idat = pal16(sizeof(PDesc) * nf);
  p.off_bytes = p.off_idat + pal16(sizeof(PIdat) * p.idat.size());
  p.total = p.off_bytes + p.span_bytes + 16;
}

struct PngState final : StreamDecoder {
  StreamBatch<PHeader> bt;
  Buffer scr;
  X2N x2n;

  PngState() {
    x2n.t[0] = 1u << 30;  // x^1
    for (int k = 1; k < 32; ++k) x2n.t[k] = multmodp_host(x2n.t[k - 1], x2n.t[k - 1]);
  }
  ~PngState() override {
    if (scr.ptr) cudaFree(scr.ptr);
  }
  // Inflate is serial within a frame and latency-bound: a chunk of 32 frames (warps) per SM keeps every scheduler
  // busy.  A 512 x 512 ping takes about 0.5 MB of scratch, so a chunk of ~4k frames takes about 2 GB.
  int chunk_frames(const sfe_ctx *ctx) const override { return std::max(256, ctx->sm_count * 32); }
  void parse(const uint8_t *bytes, const int64_t *offsets, int n, int R, int B, const int32_t *shape) override {
    bt.parse(bytes, offsets, n, R, B, shape, parse_png, SFE_PNG_SIZE);
  }
  int frame_status(int i) const override { return bt.hdr[i].status; }
  const char *message(int status) const override { return sfe_png_status_message(status); }
  int reserve(sfe_ctx *ctx, int chunk, size_t out_bytes) override;
  int decode_chunk(sfe_ctx *ctx, int f0, int nf, uint8_t *out_dev) override;
};

StreamDecoder *png_decoder(sfe_ctx *ctx) {
  if (!ctx->png) ctx->png = new PngState();
  return ctx->png;
}
void destroy(PngState *s) { delete s; }

int PngState::reserve(sfe_ctx *ctx, int chunk, size_t out_bytes) {
  size_t in_max = 0, scr_max = 0;
  PngPlan p;
  for (int f0 = 0; f0 < bt.n; f0 += chunk) {
    plan_png_chunk(bt, f0, std::min(chunk, bt.n - f0), p);
    in_max = std::max(in_max, p.total);
    scr_max = std::max(scr_max, (size_t)p.scr_bytes);
  }
  const int rc = ensure(ctx, scr, scr_max + 16);
  return rc == SFE_OK ? reserve_common(ctx, bt.n, in_max, out_bytes) : rc;
}

int PngState::decode_chunk(sfe_ctx *ctx, int f0, int nf, uint8_t *out_dev) {
  PngPlan p;
  plan_png_chunk(bt, f0, nf, p);
  uint8_t *pin, *dev;
  int rc = stager.acquire(&pin);
  if (rc != SFE_OK) return rc;
  memcpy(pin, p.desc.data(), sizeof(PDesc) * nf);
  memcpy(pin + p.off_idat, p.idat.data(), sizeof(PIdat) * p.idat.size());
  for (int i = 0; i < nf; ++i) {
    if (p.desc[i].status != SFE_PNG_OK) continue;
    const PHeader &h = bt.hdr[f0 + i];
    memcpy(pin + p.off_bytes + p.src[i], bt.bytes + bt.offsets[f0 + i] + h.span0, h.span1 - h.span0);
  }
  rc = stager.upload(ctx, p.off_bytes + p.span_bytes, &dev);
  if (rc != SFE_OK) return rc;
  const PDesc *desc = reinterpret_cast<const PDesc *>(dev);
  const PIdat *idat = reinterpret_cast<const PIdat *>(dev + p.off_idat);
  uint8_t *s = static_cast<uint8_t *>(scr.ptr);
  int32_t *st = static_cast<int32_t *>(status.ptr) + f0;
  const int wblocks = (nf + PNG_WARPS - 1) / PNG_WARPS;
  timer.tic(ctx->stream, SFE_PNG_T_CHECK);
  png_check_kernel<<<nf, PNG_CHECK_T, 0, ctx->stream>>>(desc, idat, dev + p.off_bytes, s, st, x2n);
  timer.toc(ctx->stream);
  timer.tic(ctx->stream, SFE_PNG_T_INFLATE);
  png_inflate_kernel<<<wblocks, 32 * PNG_WARPS, 0, ctx->stream>>>(desc, nf, s, st);
  timer.toc(ctx->stream);
  timer.tic(ctx->stream, SFE_PNG_T_UNFILTER);
  png_unfilter_kernel<<<wblocks, 32 * PNG_WARPS, 0, ctx->stream>>>(desc, nf, s, st, out_dev, (int64_t)bt.R_of(f0) * bt.B_of(f0));
  timer.toc(ctx->stream);
  ctx->launches += 3;
  SFE_CUDA(cudaGetLastError());
  return stager.done(ctx);
}

}  // namespace sfe

using namespace sfe;

extern "C" {

const char *sfe_png_status_message(int status) {
  switch (status) {
    case SFE_PNG_OK: return "ok";
    case SFE_PNG_NOT_PNG: return "not a PNG stream (no PNG signature)";
    case SFE_PNG_TRUNCATED: return "chunk list truncated before IEND";
    case SFE_PNG_BAD_HEADER: return "malformed IHDR or chunk order (IDATs not consecutive, unknown critical chunk)";
    case SFE_PNG_DEPTH: return "bit depth other than 8 is not supported";
    case SFE_PNG_COLORTYPE: return "colour type other than gray or truecolour (palette, alpha) is not supported";
    case SFE_PNG_INTERLACED: return "interlaced (Adam7) PNG is not supported";
    case SFE_PNG_ORIENTATION: return "eXIf orientation other than 1 (imdecode would rotate the image)";
    case SFE_PNG_ANIMATED: return "animated PNG (acTL) is not supported";
    case SFE_PNG_SIZE: return "frame size differs from the call's R x B";
    case SFE_PNG_CORRUPT: return "corrupt image data (CRC, zlib / deflate, Adler-32, filter byte or too little data)";
    default: return "unknown status";
  }
}

int sfe_png_inspect_host(const uint8_t *bytes, const int64_t *offsets, int n, int32_t *info) {
  SFE_REQUIRE(bytes && offsets && info, "sfe_png_inspect_host: null argument");
  SFE_REQUIRE(n >= 0, "sfe_png_inspect_host: negative count");
  SFE_REQUIRE(offsets_ok(offsets, n), "sfe_png_inspect_host: offsets must be non-decreasing");
  for (int i = 0; i < n; ++i) {
    PHeader h;
    parse_png(bytes + offsets[i], offsets[i + 1] - offsets[i], h);
    int32_t *o = info + (size_t)SFE_PNG_INFO * i;
    o[0] = h.status, o[1] = h.H, o[2] = h.W, o[3] = h.ctype, o[4] = (int32_t)h.idat.size();
  }
  return SFE_OK;
}

int sfe_png_decode_host(sfe_ctx *ctx, const uint8_t *bytes, const int64_t *offsets, int n, int R, int B,
                        uint8_t *out_host, int32_t *status_host) {
  SFE_REQUIRE(out_host, "sfe_png_decode_host: null output");
  return decode_all(ctx, png_decoder, bytes, offsets, n, R, B, nullptr, out_host, status_host, "sfe_png_decode_host");
}

int sfe_png_decode_to_dev(sfe_ctx *ctx, const uint8_t *bytes_host, const int64_t *offsets_host, int n, int R, int B,
                          uint8_t *out_dev, int32_t *status_host) {
  SFE_REQUIRE(out_dev, "sfe_png_decode_to_dev: null output");
  return decode_all(ctx, png_decoder, bytes_host, offsets_host, n, R, B, out_dev, nullptr, status_host,
                    "sfe_png_decode_to_dev");
}

int sfe_png_set_timing(sfe_ctx *ctx, int enable) {
  SFE_REQUIRE(ctx != nullptr, "sfe_png_set_timing: null context");
  SFE_CUDA(cudaSetDevice(ctx->device));
  png_decoder(ctx)->timer.reset(enable != 0);
  return SFE_OK;
}

int sfe_png_get_timing(sfe_ctx *ctx, double *stage_ms, int64_t *stage_calls) {
  SFE_REQUIRE(ctx && stage_ms, "sfe_png_get_timing: null argument");
  SFE_CUDA(cudaSetDevice(ctx->device));
  return png_decoder(ctx)->timer.collect(ctx->stream, SFE_PNG_STAGES, stage_ms, stage_calls);
}

}  // extern "C"
