"""An integer restatement of imread(path, IMREAD_GRAYSCALE) for the JPEG subset l3d_decode_jpeg_gray_u8 reads (DESIGN.md §4c), and a
small baseline JPEG writer that emits chosen quantised coefficients, tables, sampling factors, restart intervals, scan layouts and
marker blocks.  No floating point anywhere: the writer never runs a forward DCT, it writes the coefficients it is given.

  parse(data)           markers -> dict (size, components, tables, scans, restart segments, EXIF orientation); raises JpegError
  decode_gray(data)     the grey bytes OpenCV returns: Y's coefficients, libjpeg-turbo's accurate integer IDCT as its x86 SIMD
                        code computes it (16-bit lanes, saturating), then OpenCV's EXIF orientation
  write_jpeg(...)       the file bytes
"""
from __future__ import annotations

import struct

import numpy as np

# zig-zag position k -> natural (row-major) index
ZIGZAG = np.array([0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14, 21, 28,
                   35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55,
                   62, 63], np.int64)

MAX_SIDE = 32767


class JpegError(ValueError):
    pass


# ------------------------------------------------------------------------------------------------ markers
def _exif_orientation(p):
    """OpenCV's ExifReader on an APP1 payload after "Exif\\0\\0": IFD0's tag 0x0112 as a u16 in the TIFF byte order; 0 when absent or
    broken"""
    if len(p) < 8 or p[:2] not in (b"II", b"MM"):
        return 0
    e = "<" if p[:2] == b"II" else ">"
    if struct.unpack(e + "H", p[2:4])[0] != 0x2A:
        return 0
    off = struct.unpack(e + "I", p[4:8])[0]
    if off + 2 > len(p):
        return 0
    n = struct.unpack(e + "H", p[off:off + 2])[0]
    for i in range(n):
        q = off + 2 + 12 * i
        if q + 12 > len(p):
            return 0
        if struct.unpack(e + "H", p[q:q + 2])[0] == 0x0112:
            return struct.unpack(e + "H", p[q + 8:q + 10])[0]
    return 0


def _huff_table(bits, vals, is_dc):
    """checks of libjpeg's jpeg_make_d_derived_tbl; returns (bits, vals)"""
    code, k = 0, 0
    for ln in range(1, 17):
        code += bits[ln - 1]
        if code >= (1 << ln):
            raise JpegError("corrupt Huffman table")
        code <<= 1
    if is_dc and any(v > 15 for v in vals):
        raise JpegError("corrupt Huffman table")
    return list(bits), list(vals)


def _scan_segments(data, pos):
    """entropy-coded bytes from pos: [(start, end)] split at RSTn, the RST numbers, and the position of the marker that ends the scan
    (its 0xFF).  Fill bytes (0xFF runs) before a marker are not part of a segment."""
    segs, rst, start, i, n = [], [], pos, pos, len(data)
    while True:
        if i >= n:
            raise JpegError("truncated entropy-coded data")
        if data[i] != 0xFF:
            i += 1
            continue
        j = i + 1
        while j < n and data[j] == 0xFF:
            j += 1
        if j >= n:
            raise JpegError("truncated entropy-coded data")
        if data[j] == 0x00:
            i = j + 1
            continue
        segs.append((start, i))
        if 0xD0 <= data[j] <= 0xD7:
            rst.append(data[j] - 0xD0)
            start = i = j + 1
            continue
        return segs, rst, i


REJECT = {0xC2: "progressive JPEG is not supported", 0xC6: "progressive JPEG is not supported", 0xCA: "progressive JPEG is not supported",
          0xCE: "progressive JPEG is not supported", 0xC3: "lossless JPEG is not supported", 0xC7: "lossless JPEG is not supported",
          0xCB: "lossless JPEG is not supported", 0xCF: "lossless JPEG is not supported", 0xC5: "hierarchical JPEG is not supported",
          0xDE: "hierarchical JPEG is not supported", 0xDF: "hierarchical JPEG is not supported", 0xC9: "arithmetic coding is not supported",
          0xCC: "arithmetic coding is not supported", 0xDC: "DNL markers are not supported"}
for _m in (0xC6, 0xC7, 0xCD, 0xCE, 0xCF, 0xC5):
    REJECT.setdefault(_m, "hierarchical JPEG is not supported")
REJECT[0xCD] = "arithmetic coding is not supported"


def parse(data):
    data = bytes(data)
    n = len(data)
    if n < 2 or data[0] != 0xFF or data[1] != 0xD8:
        raise JpegError("not a JPEG file (no SOI marker)")
    q = [None] * 4
    dc, ac = [None] * 4, [None] * 4
    ri, orient, jfif, adobe, sof = 0, 0, False, -1, None
    scans, exif_seen = [], False
    pos = 2
    while True:
        if pos >= n:
            raise JpegError("missing EOI marker")
        if data[pos] != 0xFF:
            raise JpegError("corrupt data between markers")
        while pos < n and data[pos] == 0xFF:
            pos += 1
        if pos >= n:
            raise JpegError("missing EOI marker")
        m = data[pos]
        pos += 1
        if m == 0xD9:
            break
        if m in REJECT:
            raise JpegError(REJECT[m])
        if m == 0xD8 or 0xD0 <= m <= 0xD7 or m == 0x01:
            raise JpegError(f"unexpected marker 0x{m:02X}")
        if pos + 2 > n:
            raise JpegError("truncated marker segment")
        ln = (data[pos] << 8) | data[pos + 1]
        if ln < 2 or pos + ln > n:
            raise JpegError("truncated marker segment")
        p = data[pos + 2:pos + ln]
        seg_end = pos + ln
        pos = seg_end
        if 0xE0 <= m <= 0xEF:
            if m == 0xE0 and len(p) >= 14 and p[:5] == b"JFIF\0":
                jfif = True
            elif m == 0xE1 and not exif_seen and len(p) >= 6 and p[:6] == b"Exif\0\0":
                exif_seen, orient = True, _exif_orientation(p[6:])
            elif m == 0xEE and len(p) >= 12 and p[:5] == b"Adobe":
                adobe = p[11]
        elif m == 0xFE:
            pass
        elif m == 0xDB:
            i = 0
            while i < len(p):
                pq, tq = p[i] >> 4, p[i] & 15
                sz = 64 * (pq + 1)
                if pq > 1 or tq > 3 or i + 1 + sz > len(p):
                    raise JpegError("corrupt quantisation table")
                raw = np.frombuffer(p[i + 1:i + 1 + sz], ">u2" if pq else "u1").astype(np.int64)
                t = np.zeros(64, np.int64)
                t[ZIGZAG] = raw
                q[tq] = t
                i += 1 + sz
        elif m == 0xC4:
            i = 0
            while i < len(p):
                if i + 17 > len(p):
                    raise JpegError("corrupt Huffman table")
                tc, th = p[i] >> 4, p[i] & 15
                bits = list(p[i + 1:i + 17])
                cnt = sum(bits)
                if tc > 1 or th > 3 or cnt > 256 or i + 17 + cnt > len(p):
                    raise JpegError("corrupt Huffman table")
                t = _huff_table(bits, p[i + 17:i + 17 + cnt], tc == 0)
                (dc if tc == 0 else ac)[th] = t
                i += 17 + cnt
        elif m == 0xDD:
            if ln != 4:
                raise JpegError("corrupt DRI marker")
            ri = (p[0] << 8) | p[1]
        elif m in (0xC0, 0xC1):
            if sof is not None:
                raise JpegError("more than one frame header")
            if len(p) < 6:
                raise JpegError("corrupt frame header")
            prec, h, w, nc = p[0], (p[1] << 8) | p[2], (p[3] << 8) | p[4], p[5]
            if prec != 8:
                raise JpegError(f"{prec}-bit precision is not supported")
            if h == 0:
                raise JpegError("DNL markers are not supported")
            if nc not in (1, 3):
                raise JpegError(f"{nc} components are not supported (only grey and YCbCr)")
            if len(p) != 6 + 3 * nc:
                raise JpegError("corrupt frame header")
            if w < 1 or w > MAX_SIDE or h < 1 or h > MAX_SIDE:
                raise JpegError("image side outside [1, 32767]")
            comps = []
            for c in range(nc):
                cid, hv, tq = p[6 + 3 * c], p[7 + 3 * c], p[8 + 3 * c]
                if not (1 <= hv >> 4 <= 4 and 1 <= hv & 15 <= 4) or tq > 3:
                    raise JpegError("corrupt frame header")
                comps.append(dict(id=cid, h=hv >> 4, v=hv & 15, tq=tq, q=None, scanned=False))
            sof = dict(width=w, height=h, comps=comps)
        elif m == 0xDA:
            if sof is None:
                raise JpegError("scan before the frame header")
            ns = p[0] if p else 0
            if ns < 1 or ns > 4 or len(p) != 4 + 2 * ns:
                raise JpegError("corrupt scan header")
            ss, se, ahl = p[1 + 2 * ns], p[2 + 2 * ns], p[3 + 2 * ns]
            if ss != 0 or se != 63 or ahl != 0:
                raise JpegError("corrupt scan header")
            sc = []
            for k in range(ns):
                cid, t = p[1 + 2 * k], p[2 + 2 * k]
                ci = [c for c in range(len(sof["comps"])) if sof["comps"][c]["id"] == cid]
                if len(ci) != 1 or ci[0] in [s["ci"] for s in sc] or sof["comps"][ci[0]]["scanned"]:
                    raise JpegError("corrupt scan header")
                comp = sof["comps"][ci[0]]
                td, ta = t >> 4, t & 15
                if td > 3 or ta > 3 or dc[td] is None or ac[ta] is None:
                    raise JpegError("missing Huffman table")
                if q[comp["tq"]] is None:
                    raise JpegError("missing quantisation table")
                comp["scanned"], comp["q"] = True, q[comp["tq"]].copy()
                sc.append(dict(ci=ci[0], dc=dc[td], ac=ac[ta]))
            if ns > 1 and sum(sof["comps"][s["ci"]]["h"] * sof["comps"][s["ci"]]["v"] for s in sc) > 10:
                raise JpegError("corrupt scan header")
            segs, rst, pos = _scan_segments(data, seg_end)
            scans.append(dict(comps=sc, segs=segs, rst=rst, ri=ri))
        else:
            raise JpegError(f"unexpected marker 0x{m:02X}")
    if sof is None:
        raise JpegError("no frame header")
    if not all(c["scanned"] for c in sof["comps"]):
        raise JpegError("a component has no scan")
    comps = sof["comps"]
    if len(comps) == 3:
        ids = tuple(c["id"] for c in comps)
        if not jfif and (adobe == 0 or (adobe < 0 and ids == (82, 71, 66))):
            raise JpegError("RGB JPEG is not supported")
    hmax, vmax = max(c["h"] for c in comps), max(c["v"] for c in comps)
    if comps[0]["h"] != hmax or comps[0]["v"] != vmax:
        raise JpegError("Y is not at the largest sampling factors (it would need upsampling)")
    W, H = sof["width"], sof["height"]
    for s in scans:
        geo = _scan_geometry(W, H, hmax, vmax, [comps[c["ci"]] for c in s["comps"]])
        s.update(geo)
        need = -(-s["mcus"] // s["ri"]) if s["ri"] else 1
        if len(s["segs"]) != need or s["rst"] != [k % 8 for k in range(need - 1)]:
            raise JpegError("corrupt restart markers")
    return dict(width=W, height=H, comps=comps, hmax=hmax, vmax=vmax, scans=scans, orientation=orient if 1 <= orient <= 8 else 1)


def _scan_geometry(W, H, hmax, vmax, comps):
    if len(comps) == 1:
        c = comps[0]
        cw, ch = -(-W * c["h"] // hmax), -(-H * c["v"] // vmax)
        bw, bh = -(-cw // 8), -(-ch // 8)
        return dict(mcus_x=bw, mcus_y=bh, mcus=bw * bh)
    mx, my = -(-W // (8 * hmax)), -(-H // (8 * vmax))
    return dict(mcus_x=mx, mcus_y=my, mcus=mx * my)


def out_size(info):
    W, H = info["width"], info["height"]
    return (H, W) if info["orientation"] >= 5 else (W, H)


# ------------------------------------------------------------------------------------------------ entropy decoding
def _lookup16(table):
    """(length, symbol) for every 16-bit window; length 0 where no code matches"""
    bits, vals = table
    ln = np.zeros(65536, np.int64)
    sym = np.zeros(65536, np.int64)
    code, k = 0, 0
    for L in range(1, 17):
        for _ in range(bits[L - 1]):
            lo, hi = code << (16 - L), (code + 1) << (16 - L)
            ln[lo:hi], sym[lo:hi] = L, vals[k]
            code, k = code + 1, k + 1
        code <<= 1
    return ln, sym


def _windows(seg):
    """un-stuffed bytes of a segment as bits; win[p] = the 32 bits from bit p (zeros past the end), n = the bit count"""
    out, i = bytearray(), 0
    while i < len(seg):
        b = seg[i]
        out.append(b)
        if b == 0xFF:
            i += 1
            while seg[i] == 0xFF:
                i += 1
            assert seg[i] == 0
        i += 1
    bits = np.unpackbits(np.frombuffer(bytes(out), np.uint8)).astype(np.int64)
    nb = len(bits)
    bits = np.concatenate([bits, np.zeros(64, np.int64)])
    win = np.zeros(nb + 32, np.int64)
    for i in range(32):
        win += bits[i:i + nb + 32] << (31 - i)
    return win, nb


def _extend(v, s):
    return v - (1 << s) + 1 if s and v < (1 << (s - 1)) else v


def decode_y_coefs(data, info):
    """Y's quantised coefficients [bh, bw, 64] in natural order as int16 (the JCOEF store; the DC predictor is an int)"""
    data = bytes(data)
    scan = next(s for s in info["scans"] if any(c["ci"] == 0 for c in s["comps"]))
    comps = info["comps"]
    inter = len(scan["comps"]) > 1
    ybw = scan["mcus_x"] * (comps[0]["h"] if inter else 1)
    ybh = scan["mcus_y"] * (comps[0]["v"] if inter else 1)
    out = np.zeros((ybh, ybw, 64), np.int16)
    tabs = [(_lookup16(c["dc"]), _lookup16(c["ac"])) for c in scan["comps"]]
    per_mcu = []
    for k, c in enumerate(scan["comps"]):
        cc = comps[c["ci"]]
        for by in range(cc["v"] if inter else 1):
            for bx in range(cc["h"] if inter else 1):
                per_mcu.append((k, c["ci"] == 0, bx, by))
    ri = scan["ri"] or scan["mcus"]
    for si, (a, b) in enumerate(scan["segs"]):
        win, nb = _windows(data[a:b])
        p = 0
        pred = [0] * len(scan["comps"])
        for m in range(si * ri, min(scan["mcus"], (si + 1) * ri)):
            mx, my = m % scan["mcus_x"], m // scan["mcus_x"]
            for k, is_y, bx, by in per_mcu:
                (dl, ds), (al, as_) = tabs[k]
                w = int(win[p]) >> 16
                L = int(dl[w])
                if L == 0:
                    raise JpegError("corrupt Huffman code")
                s = int(ds[w])
                p += L
                v = (int(win[p]) >> (32 - s)) if s else 0
                p += s
                pred[k] += _extend(v, s)
                blk = np.zeros(64, np.int64)
                blk[0] = pred[k]
                kk = 1
                while kk < 64:
                    w = int(win[p]) >> 16
                    L = int(al[w])
                    if L == 0:
                        raise JpegError("corrupt Huffman code")
                    rs = int(as_[w])
                    p += L
                    r, s = rs >> 4, rs & 15
                    if s:
                        kk += r
                        if kk > 63:
                            raise JpegError("corrupt AC coefficients")
                        v = int(win[p]) >> (32 - s)
                        p += s
                        blk[ZIGZAG[kk]] = _extend(v, s)
                        kk += 1
                    elif r == 15:
                        kk += 16
                    else:
                        break
                if p > nb:
                    raise JpegError("corrupt entropy-coded data (a segment ends early)")
                if is_y:
                    gx = mx * (comps[0]["h"] if inter else 1) + bx
                    gy = my * (comps[0]["v"] if inter else 1) + by
                    out[gy, gx] = ((blk + 32768) & 0xFFFF) - 32768
    return out


# ------------------------------------------------------------------------------------------------ IDCT and output
# libjpeg-turbo's accurate integer IDCT as its x86 SIMD code computes it (jsimd_idct_islow_sse2 / _avx2, which OpenCV's build uses):
# the jpeg_idct_islow algorithm (13-bit constants, two passes, PASS1_BITS 2) on 16-bit lanes.  Where that differs from the C routine:
#   - dequantisation keeps the low 16 bits of coef * q (pmullw);
#   - in0 + in4, in0 - in4, in7 + in3 and in5 + in1 are 16-bit sums (paddw / psubw);
#   - the pass-1 results are saturated to 16 bits (packssdw), and so are the pass-2 results before the final 8-bit saturation
#     (packsswb) and the +128 centring: the output is clamp(x, -128, 127) + 128, not the C range-limit table's & 1023 wrap;
#   - pass 1 takes the DC-only shortcut for the whole block when rows 1..7 are all zero, and it shifts in 16 bits (psllw);
#     pass 2 has no shortcut.
# Every 32-bit sum stays below 2^31 for 16-bit inputs, so plain integers restate the rest exactly.
CONST_BITS, PASS1_BITS = 13, 2
F0298, F0390, F0541, F0765, F0899, F1175, F1501, F1847, F1961, F2053, F2562, F3072 = (2446, 3196, 4433, 6270, 7373, 9633, 12299, 15137,
                                                                                        16069, 16819, 20995, 25172)


def _i16(x):
    return ((np.asarray(x, np.int64) + 32768) & 0xFFFF) - 32768


def _sat16(x):
    return np.clip(x, -32768, 32767)


def _descale(x, n):
    return (x + (1 << (n - 1))) >> n


def _idct_1d(s0, s1, s2, s3, s4, s5, s6, s7, shift):
    """one pass on int64 arrays of 16-bit values: the 8 outputs, descaled by `shift` and saturated to 16 bits"""
    tmp2 = s2 * F0541 + s6 * (F0541 - F1847)
    tmp3 = s2 * (F0541 + F0765) + s6 * F0541
    tmp0 = _i16(s0 + s4) << CONST_BITS
    tmp1 = _i16(s0 - s4) << CONST_BITS
    t10, t13, t11, t12 = tmp0 + tmp3, tmp0 - tmp3, tmp1 + tmp2, tmp1 - tmp2
    z3, z4 = _i16(s7 + s3), _i16(s5 + s1)
    Z3 = z3 * (F1175 - F1961) + z4 * F1175
    Z4 = z3 * F1175 + z4 * (F1175 - F0390)
    T0 = s7 * (F0298 - F0899) + s1 * -F0899 + Z3
    T3 = s7 * -F0899 + s1 * (F1501 - F0899) + Z4
    T1 = s5 * (F2053 - F2562) + s3 * -F2562 + Z4
    T2 = s5 * -F2562 + s3 * (F3072 - F2562) + Z3
    return [_sat16(_descale(v, shift)) for v in (t10 + T3, t11 + T2, t12 + T1, t13 + T0, t13 - T0, t12 - T1, t11 - T2, t10 - T3)]


def idct_islow(coefs, q):
    """coefs [..., 64] natural order (int16), q [64] (the table's entries as 16-bit words): pixels [..., 8, 8] uint8"""
    raw = coefs.astype(np.int64).reshape(-1, 8, 8)
    c = _i16(raw * np.asarray(q, np.int64).reshape(8, 8))
    ws = np.stack(_idct_1d(*[c[:, k, :] for k in range(8)], CONST_BITS - PASS1_BITS), axis=1)       # [N, row, col]
    dc_only = ~np.any(raw[:, 1:, :], axis=(1, 2))                    # tested on the coefficients, before dequantisation
    ws[dc_only] = _i16(c[dc_only, 0:1, :] << PASS1_BITS)
    o = np.stack(_idct_1d(*[ws[:, :, k] for k in range(8)], CONST_BITS + PASS1_BITS + 3), axis=2)
    return (np.clip(o, -128, 127) + 128).astype(np.uint8).reshape(coefs.shape[:-1] + (8, 8))


def orient(img, o):
    """OpenCV's ExifTransform"""
    if o == 2:
        return img[:, ::-1]
    if o == 3:
        return img[::-1, ::-1]
    if o == 4:
        return img[::-1, :]
    if o == 5:
        return img.T
    if o == 6:
        return img.T[:, ::-1]
    if o == 7:
        return img.T[::-1, ::-1]
    if o == 8:
        return img.T[::-1, :]
    return img


def decode_gray(data):
    info = parse(data)
    co = decode_y_coefs(data, info)
    px = idct_islow(co, info["comps"][0]["q"])                       # [bh, bw, 8, 8]
    bh, bw = co.shape[:2]
    img = px.transpose(0, 2, 1, 3).reshape(bh * 8, bw * 8)[:info["height"], :info["width"]]
    return np.ascontiguousarray(orient(img, info["orientation"]))


# ------------------------------------------------------------------------------------------------ writer
def _code_lengths(freq):
    """JPEG Annex K.2 code lengths (at most 16 bits, the all-ones code reserved) for {symbol: count}: (bits[16], vals)"""
    syms = sorted(freq)
    f = {s: freq[s] for s in syms}
    f[256] = 1
    size = {s: 0 for s in f}
    nodes = [(f[s], [s]) for s in f]
    while len(nodes) > 1:
        nodes.sort(key=lambda t: (t[0], -len(t[1]), t[1][0]))
        (fa, a), (fb, b) = nodes[0], nodes[1]
        for s in a + b:
            size[s] += 1
        nodes = nodes[2:] + [(fa + fb, a + b)]
    bits = [0] * 300
    for s in f:
        bits[max(size[s], 1)] += 1
    for i in range(299, 16, -1):
        while bits[i] > 0:
            j = i - 2
            while bits[j] == 0:
                j -= 1
            bits[i] -= 2
            bits[i - 1] += 1
            bits[j + 1] += 2
            bits[j] -= 1
    i = 16
    while bits[i] == 0:
        i -= 1
    bits[i] -= 1
    order = sorted(syms, key=lambda s: (size[s], s))
    return bits[1:17], order


def _codes(bits, vals):
    out, code, k = {}, 0, 0
    for L in range(1, 17):
        for _ in range(bits[L - 1]):
            out[vals[k]] = (code, L)
            code, k = code + 1, k + 1
        code <<= 1
    return out


class _Bits:
    def __init__(self):
        self.out, self.acc, self.n = bytearray(), 0, 0

    def put(self, v, n):
        self.acc = (self.acc << n) | (v & ((1 << n) - 1))
        self.n += n
        while self.n >= 8:
            b = (self.acc >> (self.n - 8)) & 0xFF
            self.out.append(b)
            if b == 0xFF:
                self.out.append(0)
            self.n -= 8
        self.acc &= (1 << self.n) - 1

    def flush(self):
        if self.n:
            self.put((1 << (8 - self.n)) - 1, 8 - self.n)
        b, self.out = bytes(self.out), bytearray()
        return b


def _size(v):
    return int(abs(v)).bit_length()


def _block_symbols(blk, pred):
    """[(kind, symbol, value bits, bit count)] of one block (zig-zag from natural order); kind 0 DC, 1 AC"""
    z = [int(blk[ZIGZAG[k]]) for k in range(64)]
    d = z[0] - pred
    s = _size(d)
    out = [(0, s, d if d >= 0 else d + (1 << s) - 1, s)]
    last = max([k for k in range(1, 64) if z[k]] or [0])
    r = 0
    for k in range(1, last + 1):
        if z[k] == 0:
            r += 1
            continue
        while r > 15:
            out.append((1, 0xF0, 0, 0))
            r -= 16
        s = _size(z[k])
        out.append((1, (r << 4) | s, z[k] if z[k] >= 0 else z[k] + (1 << s) - 1, s))
        r = 0
    if last < 63:
        out.append((1, 0x00, 0, 0))
    return out


def _seg(marker, payload):
    return bytes([0xFF, marker]) + struct.pack(">H", len(payload) + 2) + payload


def exif_block(orientation, big_endian=False, first=True):
    """an APP1 payload "Exif\\0\\0" + TIFF header + IFD0 with the orientation tag, first or after two other tags"""
    e = ">" if big_endian else "<"
    tags = [(0x010F, 2, 4, b"cam\0"), (0x0110, 2, 4, b"mod\0")]
    ori = (0x0112, 3, 1, struct.pack(e + "H", orientation) + b"\0\0")
    tags = [ori] + tags if first else tags + [ori]
    ifd = struct.pack(e + "H", len(tags)) + b"".join(struct.pack(e + "HHI", t, ty, c) + v for t, ty, c, v in tags) + struct.pack(e + "I", 0)
    return b"Exif\0\0" + (b"MM" if big_endian else b"II") + struct.pack(e + "HI", 0x2A, 8) + ifd


def write_jpeg(width, height, comps, coefs, qtables, scans=None, restart=0, sof=0xC0, huff="optimal", app=(), fill=0, ids=None,
               adobe=None, jfif=True, dqt16=False):
    """A baseline / extended-sequential JPEG.
    comps: [(h, v, tq)] per component; coefs: per component int [bh, bw, 64] natural-order quantised coefficients over the
    interleaved (MCU-padded) block grid; qtables: {tq: 64 values, natural order}; scans: lists of component indices (default one
    interleaved scan); restart: DRI interval in MCUs; huff: "optimal" (K.2 from the data) or "skewed" (long codes, up to 16 bits);
    app: [(marker, payload)] written after SOI/JFIF; fill: 0xFF fill bytes before every marker after the first scan starts;
    ids: component ids (default 1, 2, 3); adobe: APP14 transform byte; dqt16: 16-bit DQT entries."""
    nc = len(comps)
    ids = ids or list(range(1, nc + 1))
    scans = scans or [list(range(nc))]
    hmax, vmax = max(c[0] for c in comps), max(c[1] for c in comps)
    out = bytearray(b"\xFF\xD8")
    if jfif:
        out += _seg(0xE0, b"JFIF\0\x01\x01\0\0\x01\0\x01\0\0")
    if adobe is not None:
        out += _seg(0xEE, b"Adobe\0\x64\0\0\0\0" + bytes([adobe]))
    for m, pl in app:
        out += _seg(m, pl)
    for tq, t in sorted(qtables.items()):
        t = np.asarray(t, np.int64)[ZIGZAG]
        out += _seg(0xDB, bytes([(16 if dqt16 else 0) | tq]) + (b"".join(struct.pack(">H", int(v)) for v in t) if dqt16 else bytes(int(v) for v in t)))
    out += _seg(sof, bytes([8]) + struct.pack(">HHB", height, width, nc) + b"".join(bytes([ids[i], (c[0] << 4) | c[1], c[2]]) for i, c in enumerate(comps)))
    if restart:
        out += _seg(0xDD, struct.pack(">H", restart))
    fb = b"\xFF" * fill
    for sc in scans:
        inter = len(sc) > 1
        if inter:
            mx, my = -(-width // (8 * hmax)), -(-height // (8 * vmax))
        else:
            c = comps[sc[0]]
            mx, my = -(-(-(-width * c[0] // hmax)) // 8), -(-(-(-height * c[1] // vmax)) // 8)
        # the symbol stream per MCU, then tables from its statistics
        mcus, pred = [], [0] * len(sc)
        for m in range(mx * my):
            if restart and m % restart == 0:
                pred = [0] * len(sc)
            syms = []
            for k, ci in enumerate(sc):
                h, v = (comps[ci][0], comps[ci][1]) if inter else (1, 1)
                for by in range(v):
                    for bx in range(h):
                        blk = coefs[ci][(m // mx) * v + by, (m % mx) * h + bx]
                        syms += [(k,) + t for t in _block_symbols(blk, pred[k])]
                        pred[k] = int(blk[0])
            mcus.append(syms)
        tabs = []
        for k in range(len(sc)):
            tk = []
            for kind in (0, 1):
                freq = {}
                for syms in mcus:
                    for kk, kd, s, _, _ in syms:
                        if kk == k and kd == kind:
                            freq[s] = freq.get(s, 0) + 1
                freq = freq or {0: 1}
                if huff == "skewed":
                    freq = {s: 1 << max(0, 40 - i) for i, s in enumerate(sorted(freq, key=lambda s: -freq[s]))}
                tk.append(_code_lengths(freq))
            tabs.append(tk)
        # each scan component gets its own table slot: DC / AC tables k
        for k in range(len(sc)):
            for kind in (0, 1):
                bits, vals = tabs[k][kind]
                out += _seg(0xC4, bytes([(kind << 4) | k]) + bytes(bits) + bytes(vals))
        out += _seg(0xDA, bytes([len(sc)]) + b"".join(bytes([ids[ci], (k << 4) | k]) for k, ci in enumerate(sc)) + b"\x00\x3F\x00")
        codes = [[_codes(*tabs[k][0]), _codes(*tabs[k][1])] for k in range(len(sc))]
        bw = _Bits()
        for m, syms in enumerate(mcus):
            if restart and m and m % restart == 0:
                out += bw.flush() + fb + bytes([0xFF, 0xD0 + (m // restart - 1) % 8])
            for k, kind, s, v, nb in syms:
                code, L = codes[k][kind][s]
                bw.put(code, L)
                if nb:
                    bw.put(v, nb)
        out += bw.flush() + fb
    out += b"\xFF\xD9"
    return bytes(out)


def random_coefs(rng, width, height, comps, amp=40, ac_terms=12, dc_step=8):
    """per component int [bh, bw, 64] over the MCU-padded grid: DC a random walk, a few low-frequency AC terms"""
    hmax, vmax = max(c[0] for c in comps), max(c[1] for c in comps)
    mx, my = -(-width // (8 * hmax)), -(-height // (8 * vmax))
    out = []
    for h, v, _ in comps:
        bh, bw = my * v, mx * h
        c = np.zeros((bh, bw, 64), np.int64)
        c[:, :, 0] = np.clip(np.cumsum(rng.integers(-dc_step, dc_step + 1, (bh, bw)), axis=1), -120, 120)
        k = rng.integers(1, 64, (bh, bw, ac_terms))
        val = rng.integers(-amp, amp + 1, (bh, bw, ac_terms)) * (rng.random((bh, bw, ac_terms)) < 0.5)
        for t in range(ac_terms):
            np.put_along_axis(c, ZIGZAG[k[:, :, t:t + 1]], val[:, :, t:t + 1], axis=2)
        out.append(c)
    return out


def std_q(quality=75):
    """a luminance-like quantisation table (natural order), integer-scaled"""
    base = np.array([16, 11, 10, 16, 24, 40, 51, 61, 12, 12, 14, 19, 26, 58, 60, 55, 14, 13, 16, 24, 40, 57, 69, 56, 14, 17, 22, 29, 51, 87,
                     80, 62, 18, 22, 37, 56, 68, 109, 103, 77, 24, 35, 55, 64, 81, 104, 113, 92, 49, 64, 78, 87, 103, 121, 120, 101, 72, 92,
                     95, 98, 112, 100, 103, 99], np.int64)
    s = 5000 // quality if quality < 50 else 200 - 2 * quality
    return np.clip((base * s + 50) // 100, 1, 255)


# ------------------------------------------------------------------------------------------------ the synthetic fixtures
SAMPLING = {"444": [(1, 1, 0), (1, 1, 1), (1, 1, 1)], "422": [(2, 1, 0), (1, 1, 1), (1, 1, 1)], "440": [(1, 2, 0), (1, 1, 1), (1, 1, 1)],
            "420": [(2, 2, 0), (1, 1, 1), (1, 1, 1)], "411": [(4, 1, 0), (1, 1, 1), (1, 1, 1)], "4x2": [(4, 2, 0), (1, 1, 1), (1, 1, 1)],
            "grey": [(1, 1, 0)], "grey22": [(2, 2, 0)]}


def build_case(p):
    """the bytes of a writer-made fixture from its parameters (a dict; everything derives from p["seed"])"""
    rng = np.random.default_rng(p["seed"])
    w, h = p["w"], p["h"]
    comps = SAMPLING[p.get("sampling", "grey")]
    coefs = random_coefs(rng, w, h, comps, amp=p.get("amp", 40), ac_terms=p.get("ac_terms", 12))
    kind = p.get("coefs", "")
    if kind == "dc11":                      # DC differences of size 11: alternating +-1023
        for c in coefs:
            c[:, :, 0] = np.where((np.arange(c.shape[1])[None, :] + np.arange(c.shape[0])[:, None]) % 2, 1023, -1023)
    elif kind == "extreme":                 # IDCT inputs far outside the 8-bit range, DC-only blocks with a wrapping 16-bit shift
        for c in coefs:
            c[:, :, 0] = rng.integers(-2047, 2048, c.shape[:2])
            c[::2, ::3, 1:] = 0
            c[1::2, :, 8:] = rng.integers(-1023, 1024, c[1::2, :, 8:].shape) * (rng.random(c[1::2, :, 8:].shape) < 0.2)
    q = {0: std_q(p.get("quality", 75)), 1: std_q(max(1, p.get("quality", 75) - 25))}
    if p.get("qtable") == "big":           # 16-bit entries, some above 32767
        q = {0: rng.integers(1, 65536, 64), 1: rng.integers(1, 300, 64)}
    elif p.get("qtable") == "255":
        q = {0: np.full(64, 255), 1: np.full(64, 255)}
    if len(comps) == 1:
        q = {0: q[0]}
    app = []
    for a in p.get("app", ()):
        if a[0] == "exif":
            app.append((0xE1, exif_block(a[1], a[2], a[3])))
        elif a[0] == "exif_broken":
            app.append((0xE1, exif_block(a[1])[:20]))
        elif a[0] == "com":
            app.append((0xFE, b"a comment \xff\xd9 inside"))
        elif a[0] == "xmp":
            app.append((0xE1, b"http://ns.adobe.com/xap/1.0/\0<x:xmpmeta/>"))
        elif a[0] == "app":
            app.append((a[1], bytes(rng.integers(0, 256, 40, dtype=np.uint8))))
    scans = p.get("scans")
    return write_jpeg(w, h, comps, coefs, q, scans=scans, restart=p.get("restart", 0), sof=p.get("sof", 0xC0), huff=p.get("huff", "optimal"),
                      app=app, fill=p.get("fill", 0), ids=p.get("ids"), adobe=p.get("adobe"), jfif=p.get("jfif", True),
                      dqt16=p.get("dqt16", False))


def writer_cases():
    """name -> parameters of every writer-made fixture"""
    c = {}
    for w, h in [(1, 1), (7, 7), (8, 8), (9, 9), (15, 15), (16, 16), (17, 17), (7, 16), (17, 8), (33, 15)]:
        c[f"grey_{w}x{h}"] = dict(w=w, h=h, seed=w * 100 + h)
    for w, h in [(1, 1), (9, 7), (17, 9), (31, 33), (16, 17)]:
        c[f"420_{w}x{h}"] = dict(w=w, h=h, sampling="420", seed=1000 + w * 100 + h)
    c["grey22_19x21"] = dict(w=19, h=21, sampling="grey22", seed=5)
    for s in ("444", "422", "440", "420", "411", "4x2"):
        c[f"sampling_{s}"] = dict(w=45, h=37, sampling=s, seed=int(s.replace("x", "")))
    c["restart1_420"] = dict(w=41, h=35, sampling="420", restart=1, seed=11)
    c["restart3_grey"] = dict(w=40, h=24, restart=3, seed=12)          # 5 MCUs per row: 3 does not divide a row
    c["restart7_422"] = dict(w=57, h=30, sampling="422", restart=7, seed=13)
    c["restart2_411_fill"] = dict(w=70, h=20, sampling="411", restart=2, fill=3, seed=14)
    c["nonint_y_first"] = dict(w=43, h=29, sampling="420", scans=[[0], [1], [2]], seed=15)
    c["nonint_chroma_first"] = dict(w=43, h=29, sampling="420", scans=[[1], [2], [0]], seed=16)
    c["nonint_mixed_restart"] = dict(w=50, h=26, sampling="422", scans=[[1, 2], [0]], restart=5, seed=17)
    c["nonint_restart_y"] = dict(w=27, h=45, sampling="440", scans=[[0], [2], [1]], restart=4, seed=18)
    c["sof1_dqt16"] = dict(w=30, h=22, sampling="420", sof=0xC1, dqt16=True, seed=19)
    c["dc_size11"] = dict(w=48, h=24, sampling="420", coefs="dc11", seed=20)
    c["huff16"] = dict(w=64, h=40, huff="skewed", seed=21)
    c["huff16_420_restart"] = dict(w=39, h=41, sampling="420", huff="skewed", restart=2, seed=22)
    c["zrl_sparse"] = dict(w=40, h=40, ac_terms=2, amp=200, seed=23)
    c["stuffing_restart1"] = dict(w=96, h=64, restart=1, amp=300, quality=95, seed=24)
    c["markers_com_app"] = dict(w=23, h=18, sampling="420", app=[("com",), ("app", 0xE2), ("xmp",), ("app", 0xED)], fill=2, seed=25)
    c["extreme_q255"] = dict(w=64, h=48, coefs="extreme", qtable="255", seed=26)
    c["extreme_q16bit"] = dict(w=64, h=48, sampling="420", coefs="extreme", qtable="big", sof=0xC1, dqt16=True, seed=27)
    c["extreme_amp"] = dict(w=40, h=40, amp=1023, qtable="255", seed=28)
    for o in range(10):
        for be in (False, True):
            c[f"exif_{o}_{'mm' if be else 'ii'}"] = dict(w=21, h=13, sampling="420" if o % 2 else "grey", app=[("exif", o, be, True)],
                                                          seed=30 + 2 * o + be)
    c["exif_6_not_first"] = dict(w=19, h=11, app=[("exif", 6, False, False)], seed=50)
    c["exif_8_not_first_mm"] = dict(w=19, h=11, sampling="420", app=[("exif", 8, True, False)], seed=51)
    c["exif_broken"] = dict(w=19, h=11, app=[("exif_broken", 6)], seed=52)
    c["exif_then_xmp"] = dict(w=25, h=9, app=[("exif", 5, True, True), ("xmp",)], seed=53)
    c["adobe1_rgb_ids"] = dict(w=20, h=20, sampling="420", jfif=False, adobe=1, ids=[82, 71, 66], seed=54)
    c["jfif_rgb_ids"] = dict(w=20, h=20, sampling="444", ids=[82, 71, 66], seed=55)
    c["nojfif_ids_0_1_2"] = dict(w=20, h=20, sampling="422", jfif=False, ids=[0, 1, 2], seed=56)
    return c
