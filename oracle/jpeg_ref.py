"""TEST INFRASTRUCTURE ONLY: a from-scratch numpy restatement of what the device JPEG decoder computes (csrc/jpeg.cu)
for the subset it accepts -- baseline / extended sequential Huffman, 8-bit, 1 or 3 (YCbCr) components, 4:4:4, 4:2:2,
4:2:0, restart intervals -- written from the JPEG specification (ITU-T T.81) and the arithmetic libjpeg-turbo's
documentation and headers state:

    entropy decoding      T.81 F.2.2 (Huffman decoding, DC prediction restarted at every RSTn)
    IDCT                  JDCT_ISLOW: CONST_BITS 13, PASS1_BITS 2, the twelve FIX_* constants, a 10-bit wrap into the
                          post-IDCT range-limit table
    upsampling            "fancy" triangular h2v1 / h2v2 (3/4 nearer + 1/4 further sample, context rows repeated at
                          the image edges), plain replication for components at most 2 samples wide
    colour                YCbCr -> RGB with 16-bit fixed-point tables, then OpenCV 4.x's 8-bit BGR2GRAY
                          (3735 B + 19235 G + 9798 R + 2^14) >> 15

decode(buf) returns dict(image=uint8 [H, W], coefficients=int32 [n_blocks, 64] (dequantised, natural order, blocks in
decode order)); a stream outside the subset raises Unsupported.  The CPU suite pins this model against
cv2.imdecode + BGR2GRAY; the GPU suite compares the device's image and coefficients with it.
"""
import numpy as np

ZIGZAG = np.array([0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20,
                   13, 6, 7, 14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52,
                   45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63])


class Unsupported(ValueError):
    pass


def _segments(buf):
    """(marker, payload) pairs up to and including SOS; returns them and the offset of the entropy-coded data."""
    b = bytes(buf)
    if len(b) < 2 or b[0] != 0xFF or b[1] != 0xD8:
        raise Unsupported("not a JPEG stream")
    i, out = 2, []
    while True:
        while i < len(b) and b[i] != 0xFF:
            i += 1
        while i < len(b) and b[i] == 0xFF:
            i += 1
        if i >= len(b):
            raise Unsupported("truncated header")
        m = b[i]
        i += 1
        if m in (0x00, 0x01) or 0xD0 <= m <= 0xD7:
            continue
        if i + 2 > len(b):
            raise Unsupported("truncated header")
        n = b[i] << 8 | b[i + 1]
        if i + n > len(b):
            raise Unsupported("truncated header")
        out.append((m, b[i + 2:i + n]))
        i += n
        if m == 0xDA:
            return out, i


def _huff_table(bits, vals):
    """code -> (length, symbol) dictionary of a canonical Huffman table (T.81 Annex C)."""
    table, code, k = {}, 0, 0
    for length in range(1, 17):
        for _ in range(bits[length - 1]):
            table[(length, code)] = vals[k]
            code += 1
            k += 1
        code <<= 1
    return table


class _Bits:
    def __init__(self, data):
        self.data, self.pos = data, 0
        self.nbits = 8 * len(data)

    def get(self, n):
        if self.pos + n > self.nbits:
            raise Unsupported("corrupt entropy-coded data: out of bits")
        v = 0
        for _ in range(n):
            v = (v << 1) | ((self.data[self.pos >> 3] >> (7 - (self.pos & 7))) & 1)
            self.pos += 1
        return v

    def huff(self, table):
        code = 0
        for length in range(1, 17):
            code = (code << 1) | self.get(1)
            sym = table.get((length, code))
            if sym is not None:
                return sym
        raise Unsupported("corrupt entropy-coded data: invalid Huffman code")


def _extend(v, s):
    return v - (1 << s) + 1 if v < (1 << (s - 1)) else v


def _unstuff(b):
    """entropy-coded bytes -> list of restart segments (stuffed zeros removed), up to the first other marker"""
    segs, cur, i = [], bytearray(), 0
    while i < len(b):
        c = b[i]
        if c != 0xFF:
            cur.append(c)
            i += 1
            continue
        nxt = b[i + 1] if i + 1 < len(b) else None
        if nxt == 0x00:
            cur.append(0xFF)
            i += 2
        elif nxt == 0xFF:
            i += 1
        elif nxt is not None and 0xD0 <= nxt <= 0xD7:
            segs.append(bytes(cur))
            cur = bytearray()
            i += 2
        else:
            break
    segs.append(bytes(cur))
    return segs


def parse(buf):
    """Header facts: dict(H, W, nc, h, v, q (per component, natural order), dc, ac (tables per component), Ri, ecs)."""
    segs, ecs = _segments(buf)
    q, dcs, acs, Ri, sof, jfif, adobe = {}, {}, {}, 0, None, False, None
    for m, p in segs:
        if m in (0xC0, 0xC1):
            if p[0] != 8:
                raise Unsupported("precision")
            H, W, nc = p[1] << 8 | p[2], p[3] << 8 | p[4], p[5]
            comps = [(p[6 + 3 * c], p[7 + 3 * c] >> 4, p[7 + 3 * c] & 15, p[8 + 3 * c]) for c in range(nc)]
            sof = (H, W, nc, comps)
        elif 0xC2 <= m <= 0xCF and m not in (0xC4, 0xCC):
            raise Unsupported("not a baseline / extended sequential Huffman stream")
        elif m == 0xC4:
            o = 0
            while o < len(p):
                tc, th = p[o] >> 4, p[o] & 15
                bits = list(p[o + 1:o + 17])
                n = sum(bits)
                (acs if tc else dcs)[th] = _huff_table(bits, list(p[o + 17:o + 17 + n]))
                o += 17 + n
        elif m == 0xDB:
            o = 0
            while o < len(p):
                pq, tq = p[o] >> 4, p[o] & 15
                if pq:
                    zz = np.frombuffer(p[o + 1:o + 129], ">u2").astype(np.int64)
                else:
                    zz = np.frombuffer(p[o + 1:o + 65], np.uint8).astype(np.int64)
                nat = np.zeros(64, np.int64)
                nat[ZIGZAG] = zz
                q[tq] = nat
                o += 1 + 64 * (2 if pq else 1)
        elif m == 0xDD:
            Ri = p[0] << 8 | p[1]
        elif m == 0xE0 and p[:5] == b"JFIF\0":
            jfif = True
        elif m == 0xEE and p[:5] == b"Adobe" and len(p) >= 12:
            adobe = p[11]
        elif m == 0xDA:
            ns = p[0]
            scan = [(p[1 + 2 * c], p[2 + 2 * c] >> 4, p[2 + 2 * c] & 15) for c in range(ns)]
    if sof is None:
        raise Unsupported("no frame header")
    H, W, nc, comps = sof
    if nc not in (1, 3) or len(scan) != nc:
        raise Unsupported("component layout")
    if nc == 3 and not jfif and (adobe == 0 or (adobe is None and [c[0] for c in comps] == [82, 71, 66])):
        raise Unsupported("RGB")
    h = [1] * nc if nc == 1 else [c[1] for c in comps]
    v = [1] * nc if nc == 1 else [c[2] for c in comps]
    if nc == 3 and (h[1:] != [1, 1] or v[1:] != [1, 1] or (h[0], v[0]) not in ((1, 1), (2, 1), (2, 2))):
        raise Unsupported("sampling")
    return dict(H=H, W=W, nc=nc, h=h, v=v, q=[q[c[3]] for c in comps], dc=[dcs[s[1]] for s in scan],
                ac=[acs[s[2]] for s in scan], Ri=Ri, ecs=ecs)


def coefficients(buf):
    """Dequantised coefficient blocks in decode order: int64 [n_blocks, 64] (natural order) and the header facts."""
    hd = parse(buf)
    H, W, nc, h, v = hd["H"], hd["W"], hd["nc"], hd["h"], hd["v"]
    hmax, vmax = max(h), max(v)
    mcux, mcuy = -(-W // (8 * hmax)), -(-H // (8 * vmax))
    layout = [c for c in range(nc) for _ in range(h[c] * v[c])]    # component of every block of an MCU
    nmcu = mcux * mcuy
    Ri = hd["Ri"] or nmcu
    segs = _unstuff(bytes(buf)[hd["ecs"]:])
    if len(segs) < -(-nmcu // Ri):
        raise Unsupported("corrupt entropy-coded data: missing restart segment")
    blocks = np.zeros((nmcu * len(layout), 64), np.int64)
    k = 0
    for s in range(-(-nmcu // Ri)):
        bits, pred = _Bits(segs[s]), [0] * nc
        for _ in range(min(Ri, nmcu - s * Ri)):
            for c in layout:
                t = bits.huff(hd["dc"][c])
                d = _extend(bits.get(t), t) if t else 0
                pred[c] += d
                blk = np.zeros(64, np.int64)
                blk[0] = np.int16(np.int64(pred[c]).astype(np.int16))
                z = 1
                while z < 64:
                    rs = bits.huff(hd["ac"][c])
                    r, sz = rs >> 4, rs & 15
                    if sz == 0:
                        if r != 15:
                            break
                        z += 16
                        if z > 64:
                            raise Unsupported("corrupt entropy-coded data: run past coefficient 63")
                        continue
                    z += r
                    if z > 63:
                        raise Unsupported("corrupt entropy-coded data: run past coefficient 63")
                    blk[ZIGZAG[z]] = _extend(bits.get(sz), sz)
                    z += 1
                blocks[k] = blk * hd["q"][c]
                k += 1
    hd.update(mcux=mcux, mcuy=mcuy, layout=layout)
    return blocks, hd


_FIX = dict(a=2446, b=3196, c=4433, d=6270, e=7373, f=9633, g=12299, h=15137, i=16069, j=16819, k=20995, l=25172)


def _idct_1d(x):
    """x[..., 8] int64 -> the eight un-descaled sums of one ISLOW pass (outputs 0..7)."""
    F = _FIX
    z2, z3 = x[..., 2], x[..., 6]
    z1 = (z2 + z3) * F["c"]
    t2 = z1 - z3 * F["h"]
    t3 = z1 + z2 * F["d"]
    t0 = (x[..., 0] + x[..., 4]) << 13
    t1 = (x[..., 0] - x[..., 4]) << 13
    t10, t13, t11, t12 = t0 + t3, t0 - t3, t1 + t2, t1 - t2
    o0, o1, o2, o3 = x[..., 7], x[..., 5], x[..., 3], x[..., 1]
    z1, z2, z3, z4 = o0 + o3, o1 + o2, o0 + o2, o1 + o3
    z5 = (z3 + z4) * F["f"]
    o0, o1, o2, o3 = o0 * F["a"], o1 * F["j"], o2 * F["l"], o3 * F["g"]
    z1, z2, z3, z4 = -z1 * F["e"], -z2 * F["k"], -z3 * F["i"] + z5, -z4 * F["b"] + z5
    o0, o1, o2, o3 = o0 + z1 + z3, o1 + z2 + z4, o2 + z2 + z3, o3 + z1 + z4
    return np.stack([t10 + o3, t11 + o2, t12 + o1, t13 + o0, t13 - o0, t12 - o1, t11 - o2, t10 - o3], -1)


def _descale(x, n):
    return (x + (1 << (n - 1))) >> n


def idct_islow(blocks):
    """dequantised blocks [n, 64] (natural order) -> uint8 samples [n, 8, 8]"""
    c = blocks.reshape(-1, 8, 8).astype(np.int64)
    ws = _descale(_idct_1d(c.transpose(0, 2, 1)), 11).astype(np.int32).astype(np.int64)   # columns: [n, col, row]
    out = _descale(_idct_1d(ws.transpose(0, 2, 1)), 18)                                     # rows: [n, row, col]
    v = out & 1023
    return np.where(v < 128, v + 128, np.where(v < 512, 255, np.where(v < 896, 0, v - 896))).astype(np.uint8)


def _upsample(p, w, h, mode):
    """component plane p (whole MCUs) of real size h x w -> full-resolution plane (h2 = 2 rows per row for 4:2:0)"""
    p = p.astype(np.int64)
    if mode == 1:
        return p
    ys = np.arange(p.shape[0] * (2 if mode == 3 else 1))
    xs = np.arange(2 * p.shape[1])
    cx = xs >> 1
    if w <= 2:                                                   # replication
        return p[(ys >> 1) if mode == 3 else ys][:, cx]
    xn = np.where(xs & 1, np.minimum(cx + 1, w - 1), np.maximum(cx - 1, 0))
    if mode == 2:
        near, far = p[:, cx], p[:, xn]
        return np.where(xs & 1, (3 * near + far + 2) >> 2, (3 * near + far + 1) >> 2)
    cy = ys >> 1
    yn = np.where(ys & 1, np.minimum(cy + 1, h - 1), np.maximum(cy - 1, 0))
    colsum = 3 * p[cy] + p[yn]                                   # [rows, cols]
    return np.where(xs & 1, (3 * colsum[:, cx] + colsum[:, xn] + 7) >> 4, (3 * colsum[:, cx] + colsum[:, xn] + 8) >> 4)


def decode(buf):
    blocks, hd = coefficients(buf)
    H, W, nc, h, v, mcux, mcuy = hd["H"], hd["W"], hd["nc"], hd["h"], hd["v"], hd["mcux"], hd["mcuy"]
    px = idct_islow(blocks)
    bpm = len(hd["layout"])
    planes = []
    for c in range(nc):
        plane = np.zeros((mcuy * v[c] * 8, mcux * h[c] * 8), np.uint8)
        idx = [j for j, cc in enumerate(hd["layout"]) if cc == c]
        for m in range(mcux * mcuy):
            my, mx = divmod(m, mcux)
            for j, b in enumerate(idx):
                dy, dx = divmod(j, h[c])
                y0, x0 = (my * v[c] + dy) * 8, (mx * h[c] + dx) * 8
                plane[y0:y0 + 8, x0:x0 + 8] = px[m * bpm + b]
        planes.append(plane)
    if nc == 1:
        img = planes[0][:H, :W]
    else:
        mode = {(1, 1): 1, (2, 1): 2, (2, 2): 3}[(h[0], v[0])]
        Y = planes[0][:H, :W].astype(np.int64)
        cw, ch = -(-W // h[0]), -(-H // v[0])
        cb = _upsample(planes[1], cw, ch, mode)[:H, :W] - 128
        cr = _upsample(planes[2], cw, ch, mode)[:H, :W] - 128
        r = np.clip(Y + ((91881 * cr + 32768) >> 16), 0, 255)
        g = np.clip(Y + ((-22554 * cb + 32768 - 46802 * cr) >> 16), 0, 255)
        b = np.clip(Y + ((116130 * cb + 32768) >> 16), 0, 255)
        img = ((3735 * b + 19235 * g + 9798 * r + (1 << 14)) >> 15).astype(np.uint8)
    return dict(image=np.ascontiguousarray(img), coefficients=blocks.astype(np.int32))


# ------------------------------------------------------------------ test streams (cv2 is the encoder and the judge)
SAMPLINGS = ("gray", "444", "422", "420")


def encode(img, quality=80, sampling="gray", optimize=False, restart=0):
    """cv2.imencode('.jpg') of a uint8 [H, W] ping; colour samplings encode a 3-channel image built from it."""
    import cv2
    params = [cv2.IMWRITE_JPEG_QUALITY, int(quality), cv2.IMWRITE_JPEG_OPTIMIZE, int(bool(optimize)),
              cv2.IMWRITE_JPEG_RST_INTERVAL, int(restart)]
    if sampling != "gray":
        img = np.dstack([img, np.roll(img, 3, 1), 255 - img])
        params += [cv2.IMWRITE_JPEG_SAMPLING_FACTOR, {"444": cv2.IMWRITE_JPEG_SAMPLING_FACTOR_444,
                                                      "422": cv2.IMWRITE_JPEG_SAMPLING_FACTOR_422,
                                                      "420": cv2.IMWRITE_JPEG_SAMPLING_FACTOR_420}[sampling]]
    ok, buf = cv2.imencode(".jpg", np.ascontiguousarray(img), params)
    assert ok
    return buf.tobytes()


def cv2_gray(buf):
    """What the reference computes (feature_extraction.py:210-213)."""
    import cv2
    return cv2.cvtColor(cv2.imdecode(np.frombuffer(bytes(buf), np.uint8), cv2.IMREAD_COLOR), cv2.COLOR_BGR2GRAY)


def contents(h, w, seed=0):
    """The test images: a synthetic ping crop, uniform noise, constant 0 / 255, an 8-pixel checkerboard."""
    from sonar_slam_b200 import synth
    rng = np.random.default_rng(seed)
    frame = synth.make_frame(seed + 1)
    reps = (-(-h // frame.shape[0]), -(-w // frame.shape[1]))
    yy, xx = np.mgrid[:h, :w]
    return {"synth": np.ascontiguousarray(np.tile(frame, reps)[:h, :w]),
            "noise": rng.integers(0, 256, (h, w), dtype=np.uint8),
            "zero": np.zeros((h, w), np.uint8), "full": np.full((h, w), 255, np.uint8),
            "checker": (((yy // 8 + xx // 8) % 2) * 255).astype(np.uint8)}


# ------------------------------------------------------------------ hand-edited streams (header variants cv2 never writes)
def _header_segments(buf):
    """[(offset of the 0xFF, marker, segment length incl. the length field)] of the headers up to and including SOS"""
    b, i, out = bytes(buf), 2, []
    while True:
        m, n = b[i + 1], b[i + 2] << 8 | b[i + 3]
        out.append((i, m, n))
        if m == 0xDA:
            return out
        i += 2 + n


def _segment(marker, payload):
    return bytes([0xFF, marker]) + (len(payload) + 2).to_bytes(2, "big") + payload


def drop_jfif(buf):
    """the stream without its JFIF APP0 segment"""
    b = bytes(buf)
    for o, m, n in _header_segments(b):
        if m == 0xE0:
            return b[:o] + b[o + 2 + n:]
    return b


def with_segment(buf, marker, payload):
    """a segment inserted right after SOI"""
    b = bytes(buf)
    return b[:2] + _segment(marker, payload) + b[2:]


def adobe(buf, transform):
    """an Adobe APP14 segment with the given colour transform, JFIF APP0 removed"""
    return with_segment(drop_jfif(buf), 0xEE, b"Adobe" + bytes([0, 100, 0, 0, 0, 0, transform]))


def with_component_ids(buf, ids):
    """SOF and SOS component ids replaced (JFIF APP0 removed, so only the ids speak for the colour space)"""
    b = bytearray(drop_jfif(buf))
    for o, m, n in _header_segments(b):
        if m in (0xC0, 0xC1):
            for c, cid in enumerate(ids):
                b[o + 10 + 3 * c] = cid
        elif m == 0xDA:
            for c, cid in enumerate(ids):
                b[o + 5 + 2 * c] = cid
    return bytes(b)


def dqt_16bit(buf):
    """every quantisation table rewritten with 16-bit entries (same values)"""
    b = bytes(buf)
    out, last = bytearray(), 0
    for o, m, n in _header_segments(b):
        if m != 0xDB:
            continue
        p, q, payload = b[o + 4:o + 2 + n], 0, bytearray()
        while q < len(p):
            pq, tq = p[q] >> 4, p[q] & 15
            vals = np.frombuffer(p[q + 1:q + 129], ">u2") if pq else np.frombuffer(p[q + 1:q + 65], np.uint8)
            payload += bytes([0x10 | tq]) + vals.astype(">u2").tobytes()
            q += 1 + 64 * (2 if pq else 1)
        out += b[last:o] + _segment(0xDB, bytes(payload))
        last = o + 2 + n
    return bytes(out + b[last:])


def six_tables(buf):
    """a 3-component stream whose third component uses its own DC and AC tables (ids 2, copies of tables 1): six
    distinct table selectors in one scan"""
    b = bytes(buf)
    tabs = {}
    for o, m, n in _header_segments(b):
        if m == 0xC4:
            p, q = b[o + 4:o + 2 + n], 0
            while q < len(p):
                k = 17 + sum(p[q + 1:q + 17])
                tabs[p[q]] = p[q:q + k]
                q += k
    extra = bytes([0x02]) + tabs[0x01][1:] + bytes([0x12]) + tabs[0x11][1:]
    out = bytearray(with_segment(b, 0xC4, extra))
    sos = [o for o, m, n in _header_segments(out) if m == 0xDA][0]
    out[sos + 10] = 0x22
    return bytes(out)


def with_sof_size(buf, height, width=None):
    """SOF height (and width) replaced"""
    b = bytearray(buf)
    for o, m, n in _header_segments(b):
        if m in (0xC0, 0xC1):
            b[o + 5:o + 7] = int(height).to_bytes(2, "big")
            if width is not None:
                b[o + 7:o + 9] = int(width).to_bytes(2, "big")
    return bytes(b)


def header_variants():
    """name -> (stream, expected status name of sonar_slam_b200.jpeg): header forms cv2.imencode never writes"""
    img = contents(64, 48)["synth"]
    c444, c420, g = encode(img, 80, "444", True), encode(img, 75, "420"), encode(img, 50)
    sof = [o for o, m, n in _header_segments(c444) if m == 0xC0][0]
    cmyk = bytearray(c444)
    cmyk[sof + 9] = 4
    return {"dqt16_gray": (dqt_16bit(g), "OK"), "dqt16_420": (dqt_16bit(c420), "OK"),
            "adobe_ycc": (adobe(c420, 1), "OK"), "ids_123": (with_component_ids(c444, [1, 2, 3]), "OK"),
            "six_tables_444": (six_tables(c444), "OK"), "six_tables_420": (six_tables(c420), "OK"),
            "adobe_rgb": (adobe(c420, 0), "COLORSPACE"), "ids_rgb": (with_component_ids(c444, [82, 71, 66]), "COLORSPACE"),
            "cmyk": (bytes(cmyk), "COLORSPACE")}
