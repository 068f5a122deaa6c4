"""TEST INFRASTRUCTURE ONLY: a from-scratch numpy restatement of what the device PNG decoder computes (csrc/png.cu) for
the subset it accepts -- 8-bit gray (colour type 0) or truecolour (type 2), not interlaced, any deflate content, any
per-row filter -- plus a PNG writer that controls what cv2.imencode does not (per-row filters, zlib strategy / level /
window, the IDAT split) and builders for the edge-case, rejected and corrupt streams.

    chunks         PNG specification section 5 (signature, length / type / data / CRC-32)
    inflate        Python's zlib (RFC 1950 / 1951) serves as the inflate oracle
    unfilter       PNG specification section 9: None, Sub, Up, Average, Paeth, bytes per pixel = channels
    gray           gray samples are the image (B = G = R); truecolour goes through OpenCV 4.x's 8-bit BGR2GRAY,
                   (3735 B + 19235 G + 9798 R + 2^14) >> 15

decode(buf) returns the uint8 [H, W] image; a stream outside the subset raises Unsupported.  The CPU suite pins this
model against cv2.imdecode(IMREAD_COLOR) + BGR2GRAY; the GPU suite compares the device with cv2 and this model.
"""
import struct
import zlib

import numpy as np

SIG = b"\x89PNG\r\n\x1a\n"
NONE, SUB, UP, AVERAGE, PAETH = range(5)


class Unsupported(ValueError):
    pass


# ------------------------------------------------------------------ reading
def chunks(buf):
    """[(type, data, stored crc)] up to and including IEND."""
    b = bytes(buf)
    if b[:8] != SIG:
        raise Unsupported("not a PNG")
    i, out = 8, []
    while True:
        if i + 8 > len(b):
            raise Unsupported("truncated")
        n, t = struct.unpack(">I", b[i:i + 4])[0], b[i + 4:i + 8]
        if i + 12 + n > len(b):
            raise Unsupported("truncated")
        out.append((t, b[i + 8:i + 8 + n], struct.unpack(">I", b[i + 8 + n:i + 12 + n])[0]))
        i += 12 + n
        if t == b"IEND":
            return out


def _paeth(a, b, c):
    p = a + b - c
    pa, pb, pc = abs(p - a), abs(p - b), abs(p - c)
    return a if pa <= pb and pa <= pc else (b if pb <= pc else c)


def unfilter(data, h, w, c):
    """Filtered scanlines (h rows of 1 + w * c bytes) -> uint8 [h, w * c]."""
    stride = 1 + w * c
    raw = np.frombuffer(data, np.uint8)[:h * stride].reshape(h, stride)
    out = np.zeros((h, w * c), np.uint8)
    prev = np.zeros(w * c, np.int64)
    for y in range(h):
        f, x = int(raw[y, 0]), raw[y, 1:].astype(np.int64)
        if f == NONE:
            row = x
        elif f == SUB:
            row = np.cumsum(x.reshape(w, c), axis=0).reshape(-1)
        elif f == UP:
            row = x + prev
        elif f in (AVERAGE, PAETH):
            row = np.zeros(w * c, np.int64)
            for i in range(w * c):
                a = int(row[i - c]) if i >= c else 0
                b = int(prev[i])
                pc = int(prev[i - c]) if i >= c else 0
                pred = (a + b) >> 1 if f == AVERAGE else _paeth(a, b, pc)
                row[i] = (int(x[i]) + pred) & 255
        else:
            raise Unsupported("bad filter byte")
        row = row & 255
        out[y] = row
        prev = row
    return out


def to_gray(pixels, h, w, c):
    if c == 1:
        return np.ascontiguousarray(pixels.reshape(h, w))
    p = pixels.reshape(h, w, 3).astype(np.int64)
    r, g, b = p[..., 0], p[..., 1], p[..., 2]
    return ((3735 * b + 19235 * g + 9798 * r + (1 << 14)) >> 15).astype(np.uint8)


def decode(buf):
    cs = chunks(buf)
    t, d, _ = cs[0]
    if t != b"IHDR" or len(d) != 13:
        raise Unsupported("bad IHDR")
    w, h, depth, ctype, comp, filt, inter = struct.unpack(">IIBBBBB", d)
    if depth != 8 or ctype not in (0, 2) or comp or filt or inter:
        raise Unsupported("outside the subset")
    c = 1 if ctype == 0 else 3
    z = b"".join(d for t, d, _ in cs if t == b"IDAT")
    data = zlib.decompressobj().decompress(z)
    if len(data) < h * (1 + w * c):
        raise Unsupported("not enough image data")
    return to_gray(unfilter(data, h, w, c), h, w, c)


def cv2_gray(buf):
    """What the reference computes (feature_extraction.py:210-213)."""
    import cv2
    if not buf:
        return None
    dec = cv2.imdecode(np.frombuffer(bytes(buf), np.uint8), cv2.IMREAD_COLOR)
    return None if dec is None else cv2.cvtColor(dec, cv2.COLOR_BGR2GRAY)


# ------------------------------------------------------------------ writing
def chunk(t, data, crc=None):
    crc = zlib.crc32(t + data) if crc is None else crc
    return struct.pack(">I", len(data)) + t + data + struct.pack(">I", crc & 0xFFFFFFFF)


def ihdr(h, w, ctype=0, depth=8, interlace=0):
    return chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, depth, ctype, 0, 0, interlace))


def filter_rows(px, filters, c):
    """uint8 [h, w * c] -> filtered scanlines; filters: one filter type or one per row."""
    h, n = px.shape
    filters = [filters] * h if np.isscalar(filters) else list(filters)
    out, prev = bytearray(), np.zeros(n, np.int64)
    for y in range(h):
        x, f = px[y].astype(np.int64), int(filters[y])
        left = np.concatenate([np.zeros(c, np.int64), x[:-c]]) if n else x
        ul = np.concatenate([np.zeros(c, np.int64), prev[:-c]]) if n else prev
        if f == NONE:
            r = x
        elif f == SUB:
            r = x - left
        elif f == UP:
            r = x - prev
        elif f == AVERAGE:
            r = x - ((left + prev) >> 1)
        else:
            r = x - np.array([_paeth(int(a), int(b), int(cc)) for a, b, cc in zip(left, prev, ul)], np.int64)
        out.append(f)
        out += (r & 255).astype(np.uint8).tobytes()
        prev = x
    return bytes(out)


STRATEGIES = {"default": zlib.Z_DEFAULT_STRATEGY, "filtered": zlib.Z_FILTERED, "huffman": zlib.Z_HUFFMAN_ONLY,
              "rle": zlib.Z_RLE, "fixed": zlib.Z_FIXED}


def deflate(data, level=6, strategy="default", wbits=15):
    co = zlib.compressobj(level, zlib.DEFLATED, wbits, 9, STRATEGIES[strategy])
    return co.compress(data) + co.flush()


def split(z, idat):
    """IDAT payloads: idat = None (one chunk), an int k > 0 (chunks of k bytes) or -k (k chunks of about equal size)."""
    if idat is None:
        return [z]
    if idat > 0:
        return [z[i:i + idat] for i in range(0, len(z), idat)] or [b""]
    k = -idat
    cuts = [len(z) * j // k for j in range(k + 1)]
    return [z[cuts[j]:cuts[j + 1]] for j in range(k)]


def assemble(h, w, z, ctype=0, idat=None, before=(), after=(), depth=8, interlace=0):
    """A PNG around a ready zlib stream; before / after: extra chunk bytes placed before / after the IDATs."""
    return (SIG + ihdr(h, w, ctype, depth, interlace) + b"".join(before)
            + b"".join(chunk(b"IDAT", p) for p in split(z, idat)) + b"".join(after) + chunk(b"IEND", b""))


def write(img, filters=SUB, level=6, strategy="default", wbits=15, idat=None, before=(), after=()):
    """uint8 [H, W] (gray) or [H, W, 3] (RGB) -> PNG bytes."""
    img = np.ascontiguousarray(img, np.uint8)
    h, w = img.shape[:2]
    c = 1 if img.ndim == 2 else 3
    z = deflate(filter_rows(img.reshape(h, w * c), filters, c), level, strategy, wbits)
    return assemble(h, w, z, 0 if c == 1 else 2, idat, before, after)


def rgb_of(img):
    """The three-channel test image built from a ping (distinct channels)."""
    return np.dstack([img, np.roll(img, 3, 1), 255 - img])


# ------------------------------------------------------------------ a minimal deflate writer for what zlib will not emit
class BitWriter:
    def __init__(self):
        self.bits, self.n = 0, 0

    def put(self, v, k):            # k bits of v, least significant first
        self.bits |= (v & ((1 << k) - 1)) << self.n
        self.n += k

    def huff(self, code, k):        # a Huffman code, most significant bit first
        self.put(int(format(code, f"0{k}b")[::-1], 2) if k else 0, k)

    def align(self):
        self.n = (self.n + 7) & ~7

    def bytes(self):
        return self.bits.to_bytes((self.n + 7) // 8, "little")


def canonical(lengths):
    """Code lengths -> canonical codes (RFC 1951 3.2.2)."""
    bl = [0] * 16
    for l in lengths:
        bl[l] += 1
    bl[0] = 0
    code, nxt = 0, [0] * 16
    for b in range(1, 16):
        code = (code + bl[b - 1]) << 1
        nxt[b] = code
    out = []
    for l in lengths:
        out.append(nxt[l] if l else 0)
        if l:
            nxt[l] += 1
    return out


FIXED_LIT = [8] * 144 + [9] * 112 + [7] * 24 + [8] * 8
LBASE = [3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258]
LEXT = [0] * 8 + [1] * 4 + [2] * 4 + [3] * 4 + [4] * 4 + [5] * 4 + [0]
DBASE = [1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073,
         4097, 6145, 8193, 12289, 16385, 24577]
DEXT = [0, 0, 0, 0] + [k // 2 for k in range(2, 28)]


def _tokens(bw, tokens, lit_len, lit_code, d_len, d_code):
    for t in tokens:
        if isinstance(t, int):
            bw.huff(lit_code[t], lit_len[t])
            continue
        length, dist = t
        s = max(i for i in range(29) if LBASE[i] <= length)
        if length == 258:
            s = 28
        bw.huff(lit_code[257 + s], lit_len[257 + s])
        bw.put(length - LBASE[s], LEXT[s])
        ds = max(i for i in range(30) if DBASE[i] <= dist)
        bw.huff(d_code[ds], d_len[ds])
        bw.put(dist - DBASE[ds], DEXT[ds])
    bw.huff(lit_code[256], lit_len[256])


def raw_deflate(blocks):
    """blocks: [("stored", payload bytes) | ("fixed", tokens) | ("dynamic1", tokens, dist symbol)], the last one final.
    tokens: ints (literals) and (length, distance) pairs.  "dynamic1" is a dynamic block with (nearly) the fixed literal /
    length code lengths and a single distance code (one symbol, length 1: an incomplete code zlib accepts)."""
    bw = BitWriter()
    fl = canonical(FIXED_LIT)
    fd_len = [5] * 30
    fd = canonical(fd_len)
    for k, blk in enumerate(blocks):
        bw.put(1 if k == len(blocks) - 1 else 0, 1)
        if blk[0] == "stored":
            bw.put(0, 2)
            bw.align()
            p = blk[1]
            bw.put(len(p), 16)
            bw.put(len(p) ^ 0xFFFF, 16)
            for byte in p:
                bw.put(byte, 8)
        elif blk[0] == "fixed":
            bw.put(1, 2)
            _tokens(bw, blk[1], FIXED_LIT, fl, fd_len, fd)
        else:
            ds = blk[2]
            d_len = [0] * (ds + 1)
            d_len[ds] = 1
            bw.put(2, 2)
            bw.put(286 - 257, 5)
            bw.put(len(d_len) - 1, 5)
            bw.put(19 - 4, 4)
            cl_len = [4] * 16 + [0] * 3                     # code-length symbols 0..15 of length 4: complete
            order = [16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15]
            for s in order:
                bw.put(cl_len[s], 3)
            cl = canonical(cl_len)
            lit = FIXED_LIT[:284] + [7, 7]                  # 286 symbols, still a complete code
            for l in lit + d_len:
                bw.huff(cl[l], 4)
            _tokens(bw, blk[1], lit, canonical(lit), d_len, canonical(d_len))
    return bw.bytes()


def zwrap(deflated, data, cinfo=7):
    """RFC 1950 framing: CMF / FLG (window 2^(cinfo + 8)) + deflate data + Adler-32 of `data`."""
    cmf = (cinfo << 4) | 8
    flg = (31 - (cmf * 256) % 31) % 31
    return bytes([cmf, flg]) + deflated + struct.pack(">I", zlib.adler32(data))


def edge_streams():
    """name -> (h, w, PNG bytes) for deflate features zlib does not emit on demand; each inflates to what it says."""
    out = {}
    # a length-258 match at distance 32768, and overlapping copies (distance 1 and 3)
    h, w = 130, 511
    rng = np.random.default_rng(11)
    lit = rng.integers(0, 256, 32768, dtype=np.uint8)
    tokens = [int(v) for v in lit] + [(258, 32768)] * 3 + [(258, 1), (100, 3)]
    data = bytearray(lit.tobytes())
    for length, dist in [(258, 32768)] * 3 + [(258, 1), (100, 3)]:
        for _ in range(length):
            data.append(data[-dist])
    need = h * (1 + w)
    tail = bytes((j * 7) & 255 for j in range(need - len(data)))
    data += tail
    data = bytearray(data[:need])
    for y in range(h):
        data[y * (1 + w)] = y % 5                         # every filter, set on the already-built bytes
    blocks_data = bytes(data)
    # the filter bytes overwrote some literals / copies: re-derive tokens as literals + the long matches where intact
    toks = _tokens_for(blocks_data)
    z = zwrap(raw_deflate([("fixed", toks)]), blocks_data)
    out["fixed_258_at_32768"] = (h, w, assemble(h, w, z, 0))
    # empty stored blocks, and a stored block straddling IDAT chunks
    h, w = 9, 13
    px = rng.integers(0, 256, (h, w), dtype=np.uint8)
    raw = filter_rows(px, [y % 5 for y in range(h)], 1)
    z = zwrap(raw_deflate([("stored", b""), ("stored", raw[:50]), ("stored", b""), ("fixed", list(raw[50:]))]), raw)
    out["stored_empty_and_straddling"] = (h, w, assemble(h, w, z, 0, idat=7))
    # a dynamic block whose distance code has one symbol
    h, w = 16, 24
    row = bytes(range(24))
    raw = b"".join(b"\x00" + row for _ in range(h))
    toks = [0] + list(row) + [(25, 25)] * (h - 1)
    z = zwrap(raw_deflate([("dynamic1", toks, 9)]), raw)    # distance symbol 9: 25..32, 3 extra bits
    out["dynamic_single_distance_code"] = (h, w, assemble(h, w, z, 0))
    return out


def _tokens_for(data):
    """A greedy tokenisation: matches at distance 32768 / 1 / 3 where they hold, otherwise literals."""
    toks, i, n = [], 0, len(data)
    while i < n:
        best = None
        for dist in (32768, 1, 3):
            if i >= dist:
                k = 0
                while k < 258 and i + k < n and data[i + k] == data[i + k - dist]:
                    k += 1
                if k >= 3 and (best is None or k > best[0]):
                    best = (k, dist)
        if best:
            toks.append(best)
            i += best[0]
        else:
            toks.append(data[i])
            i += 1
    return toks


# ------------------------------------------------------------------ rejected and corrupt variants
def _exif(orientation):
    return (b"II*\x00" + (8).to_bytes(4, "little") + (1).to_bytes(2, "little") + (0x0112).to_bytes(2, "little")
            + (3).to_bytes(2, "little") + (1).to_bytes(4, "little") + orientation.to_bytes(2, "little") + b"\x00\x00"
            + (0).to_bytes(4, "little"))


def rejected_variants(img):
    """name -> (PNG bytes, expected status name) for streams the decoder refuses before decoding, plus accepted
    header variants (status "OK")."""
    h, w = img.shape
    z = deflate(filter_rows(img, SUB, 1))
    base = assemble(h, w, z)
    ih = base[8:33]
    out = {
        "jpeg": (b"\xff\xd8\xff\xe0" + b"\x00" * 40, "NOT_PNG"),
        "empty": (b"", "NOT_PNG"),
        "signature_only": (SIG, "TRUNCATED"),
        "cut_in_ihdr": (base[:20], "TRUNCATED"),
        "no_iend": (base[:-12], "TRUNCATED"),
        "cut_in_idat": (base[:len(base) // 2], "TRUNCATED"),
        "ihdr_not_first": (SIG + chunk(b"tEXt", b"a\x00b") + base[8:], "BAD_HEADER"),
        "ihdr_crc": (SIG + ih[:-4] + b"\x00\x00\x00\x00" + base[33:], "BAD_HEADER"),
        "ihdr_zero_width": (assemble(h, 0, z), "BAD_HEADER"),
        "compression_1": (SIG + chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, 8, 0, 1, 0, 0)) + base[33:], "BAD_HEADER"),
        "no_idat": (SIG + ih + chunk(b"IEND", b""), "BAD_HEADER"),
        "idat_split_by_text": (_split_by(h, w, z), "BAD_HEADER"),
        "unknown_critical": (assemble(h, w, z, before=[chunk(b"ABCD", b"xx")]), "BAD_HEADER"),
        "depth_16": (assemble(h, w, z, depth=16), "DEPTH"),
        "depth_4": (assemble(h, w, z, depth=4), "DEPTH"),
        "palette": (assemble(h, w, z, ctype=3, before=[chunk(b"PLTE", bytes(range(6)))]), "COLORTYPE"),
        "gray_alpha": (assemble(h, w, z, ctype=4), "COLORTYPE"),
        "rgba": (assemble(h, w, z, ctype=6), "COLORTYPE"),
        "adam7": (assemble(h, w, z, interlace=1), "INTERLACED"),
        "exif6": (assemble(h, w, z, before=[chunk(b"eXIf", _exif(6))]), "ORIENTATION"),
        "exif6_after_idat": (assemble(h, w, z, after=[chunk(b"eXIf", _exif(6))]), "ORIENTATION"),
        "actl": (assemble(h, w, z, before=[chunk(b"acTL", struct.pack(">II", 1, 0))]), "ANIMATED"),
        # accepted: ancillary chunks are ignored (a bad ancillary CRC is only a warning), IEND's CRC is not read
        "exif1": (assemble(h, w, z, before=[chunk(b"eXIf", _exif(1))]), "OK"),
        "text_bad_crc": (assemble(h, w, z, before=[chunk(b"tEXt", b"a\x00b", 5)]), "OK"),
        "trns_gama": (assemble(h, w, z, before=[chunk(b"gAMA", struct.pack(">I", 100000)),
                                                chunk(b"tRNS", b"\x00\x05")]), "OK"),
        "plte_in_gray": (assemble(h, w, z, before=[chunk(b"PLTE", bytes(range(6)))]), "OK"),
        "iend_bad_crc": (base[:-4] + b"\x00\x00\x00\x00", "OK"),
        "after_iend": (base + b"garbage", "OK"),
    }
    return out


def _split_by(h, w, z):
    """IDAT chunks that are not consecutive (libpng: "Not enough image data")."""
    parts = split(z, -2)
    return (SIG + ihdr(h, w) + chunk(b"IDAT", parts[0]) + chunk(b"tEXt", b"a\x00b") + chunk(b"IDAT", parts[1])
            + chunk(b"IEND", b""))


def corrupt_variants(img):
    """name -> PNG bytes whose headers are fine but whose data cv2 refuses (decode-time failures)."""
    h, w = img.shape
    raw = filter_rows(img, SUB, 1)
    z = deflate(raw)
    out = {}
    good = assemble(h, w, z)
    k = good.index(b"IDAT")
    crc_at = k + 4 + len(z)
    out["idat_crc"] = good[:crc_at] + bytes([good[crc_at] ^ 1]) + good[crc_at + 1:]
    out["adler"] = assemble(h, w, z[:-1] + bytes([z[-1] ^ 1]))
    out["zlib_header"] = assemble(h, w, bytes([z[0], z[1] ^ 1]) + z[2:])
    out["window_too_big"] = assemble(h, w, zwrap(deflate(raw)[2:-4], raw, cinfo=8)[:2] + z[2:])
    out["reserved_block_type"] = assemble(h, w, z[:2] + bytes([z[2] | 6]) + z[3:])
    out["stored_nlen"] = assemble(h, w, zwrap(b"\x01" + struct.pack("<HH", len(raw[:100]), 0) + raw[:100], raw[:100]))
    out["invalid_symbol"] = assemble(h, w, zwrap(raw_deflate_invalid_symbol(), b""))
    out["over_subscribed"] = assemble(h, w, zwrap(_over_subscribed(), b""))
    out["distance_too_far"] = assemble(h, w, zwrap(raw_deflate([("fixed", [1, 2, (3, 5)])]), b"\x01\x02\x01\x02\x01"))
    bf = bytearray(raw)
    bf[(h // 2) * (1 + w)] = 5
    out["filter_byte_5"] = assemble(h, w, deflate(bytes(bf)))
    out["not_enough_data"] = assemble(h, w, deflate(raw[:-w]))
    out["deflate_truncated"] = assemble(h, w, z[:len(z) // 2])
    return out


def raw_deflate_invalid_symbol():
    """A fixed block that uses literal / length symbol 286 (invalid)."""
    bw = BitWriter()
    bw.put(1, 1)
    bw.put(1, 2)
    fl = canonical(FIXED_LIT)
    bw.huff(fl[286], FIXED_LIT[286])
    bw.huff(fl[256], FIXED_LIT[256])
    return bw.bytes()


def _over_subscribed():
    """A dynamic block whose code-length code is over-subscribed (every symbol of length 1)."""
    bw = BitWriter()
    bw.put(1, 1)
    bw.put(2, 2)
    bw.put(0, 5)
    bw.put(0, 5)
    bw.put(15, 4)
    for _ in range(19):
        bw.put(1, 3)
    bw.put(0, 32)
    return bw.bytes()


def over_long(img, extra_rows=7):
    """A stream whose inflated data runs past the last row (IHDR height lowered): libpng warns and skips the rest."""
    h, w = img.shape
    tall = np.concatenate([img, img[:extra_rows]])
    z = deflate(filter_rows(tall, SUB, 1))
    return assemble(h, w, z)
