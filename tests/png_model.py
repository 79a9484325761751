"""A numpy restatement of imread(path, IMREAD_GRAYSCALE) for the PNG subset l3d_decode_png_gray_u8 reads (DESIGN.md §4d), and a PNG
writer with its own small DEFLATE encoder, so that fixtures can hold what zlib never emits (stored blocks of 0 and 65,535 bytes, fixed
blocks, 15-bit codes, a single distance code or none, chosen matches, IDAT splits anywhere).

  parse(data)           chunks -> dict (IHDR fields, palette, gamma, EXIF orientation, the IDAT payload); raises PngError naming the
                        reason for anything outside the subset
  decode_gray(data)     the grey bytes OpenCV returns: zlib.decompress, unfiltering, Adam7, libpng's conversion to grey (with its gamma
                        tables when the file has gAMA / sRGB), then OpenCV's EXIF orientation
  write_png(...)        the file bytes
"""
from __future__ import annotations

import heapq
import math
import struct
import zlib

import numpy as np

SIG = b"\x89PNG\r\n\x1a\n"
MAX_SIDE = 1000000            # libpng's default user limits (PNG_USER_WIDTH_MAX / PNG_USER_HEIGHT_MAX)
MAX_PIXELS = 1 << 30          # OpenCV's CV_IO_MAX_IMAGE_PIXELS
LEGAL = {0: (1, 2, 4, 8, 16), 2: (8, 16), 3: (1, 2, 4, 8), 4: (8, 16), 6: (8, 16)}
CHANNELS = {0: 1, 2: 3, 3: 1, 4: 2, 6: 4}
# Adam7: (x0, y0, dx, dy) of each pass
ADAM7 = [(0, 0, 8, 8), (4, 0, 8, 8), (0, 4, 4, 8), (2, 0, 4, 4), (0, 2, 2, 4), (1, 0, 2, 2), (0, 1, 1, 2)]
RC, GC, BC = 9797, 19234, 3737   # libpng's png_set_rgb_to_gray(…, 0.299, 0.587) in 15-bit fixed point (blue = 32768 - red - green)


class PngError(ValueError):
    pass


# ------------------------------------------------------------------------------------------------ EXIF
def exif_orientation(p):
    """OpenCV's ExifReader on a TIFF block: IFD0's tag 0x0112 as a u16 in the TIFF byte order; 0 when absent or broken"""
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


def orient(img, o):
    """OpenCV's ExifTransform of a 2-D array"""
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


# ------------------------------------------------------------------------------------------------ gamma
def reciprocal(a):
    """libpng's png_reciprocal: 1/a in its 1e5 fixed point, rounded"""
    return int(math.floor(1e10 / a + .5))


def significant(g):
    """libpng's png_gamma_significant"""
    return g < 100000 - 5000 or g > 100000 + 5000


def table8(g):
    """libpng's png_build_8bit_table with png_gamma_8bit_correct (floating-point arithmetic)"""
    if not significant(g):
        return np.arange(256, dtype=np.uint8)
    t = [0] + [int(math.floor(255 * math.pow(v / 255., g * .00001) + .5)) for v in range(1, 255)] + [255]
    return np.array(t, np.uint8)


def gamma_tables(file_gamma):
    """(to_1, from_1) of libpng's rgb_to_gray with a file gamma (1e5 fixed point) and no screen gamma set, or None when libpng builds
    no tables (the plain formula applies).  libpng then takes the screen gamma as the file gamma's reciprocal, so the overall
    correction is identity: grey triples pass unchanged."""
    if not file_gamma:
        return None
    screen = reciprocal(file_gamma)
    if not significant(file_gamma) and not significant(screen):
        return None
    return table8(reciprocal(file_gamma)), table8(reciprocal(screen))


def rgb_to_gray8(r, g, b, tables=None):
    r, g, b = (np.asarray(v, np.int64) for v in (r, g, b))
    eq = (r == g) & (r == b)
    if tables is None:
        y = (RC * r + GC * g + BC * b) >> 15
    else:
        to1, fr1 = (t.astype(np.int64) for t in tables)
        y = fr1[(RC * to1[r] + GC * to1[g] + BC * to1[b] + 16384) >> 15]
    return np.where(eq, r, y).astype(np.uint8)


def rgb_to_gray16(r, g, b):
    r, g, b = (np.asarray(v, np.int64) for v in (r, g, b))
    eq = (r == g) & (r == b)
    y = (RC * r + GC * g + BC * b + 16384) >> 15
    return (np.where(eq, r, y) >> 8).astype(np.uint8)


# ------------------------------------------------------------------------------------------------ parsing
def _u32(b, o):
    return struct.unpack(">I", b[o:o + 4])[0]


def row_bytes(width, ct, depth):
    return (width * CHANNELS[ct] * depth + 7) // 8


def passes(w, h, interlace):
    """(pass width, pass height) of each pass that has bytes"""
    if not interlace:
        return [(w, h)]
    out = []
    for x0, y0, dx, dy in ADAM7:
        pw, ph = (w - x0 + dx - 1) // dx if w > x0 else 0, (h - y0 + dy - 1) // dy if h > y0 else 0
        out.append((pw, ph))
    return out


def raw_size(w, h, ct, depth, interlace):
    return sum(ph * (row_bytes(pw, ct, depth) + 1) for pw, ph in passes(w, h, interlace) if pw and ph)


def parse(data):
    """the file's chunks -> dict; PngError(reason) for anything outside the subset (the same reasons, in the same order, as
    l3d_png_parse of csrc/line3d_png.cc)"""
    d = bytes(data)
    if len(d) < 8 or d[:8] != SIG:
        raise PngError("not a PNG file (no PNG signature)")
    pos, first = 8, True
    h = dict(palette=None, gamma=0, srgb=False, orientation=1, idat=[], exif=False)
    seen_idat = ended_idat = False
    while True:
        if pos + 8 > len(d):
            raise PngError("truncated chunk")
        n, t = _u32(d, pos), d[pos + 4:pos + 8]
        if n > 0x7FFFFFFF or pos + 12 + n > len(d):
            raise PngError("truncated chunk")
        body = d[pos + 8:pos + 8 + n]
        if zlib.crc32(t + body) != _u32(d, pos + 8 + n):
            raise PngError("bad CRC in chunk " + t.decode("latin-1"))
        pos += 12 + n
        if not all(65 <= c <= 90 or 97 <= c <= 122 for c in t):
            raise PngError("bad chunk type")
        if first != (t == b"IHDR"):
            raise PngError("IHDR is not the first chunk")
        first = False
        if t != b"IDAT" and seen_idat:
            ended_idat = True
        if t == b"IHDR":
            if n != 13:
                raise PngError("corrupt IHDR")
            w, hh, depth, ct, cm, fm, il = struct.unpack(">IIBBBBB", body)
            if ct not in LEGAL or depth not in LEGAL[ct]:
                raise PngError("invalid colour type and bit depth")
            if cm != 0 or fm != 0 or il > 1:
                raise PngError("invalid compression, filter or interlace method")
            if w < 1 or hh < 1 or w > MAX_SIDE or hh > MAX_SIDE or w * hh > MAX_PIXELS:
                raise PngError("image size outside the supported limits")
            h.update(width=w, height=hh, depth=depth, ct=ct, interlace=il)
        elif t == b"PLTE":
            if h["palette"] is not None or seen_idat or n % 3 or n == 0 or n > 768:
                raise PngError("corrupt PLTE")
            if h["ct"] in (0, 4):
                raise PngError("PLTE in a grey image")
            if h["ct"] == 3 and n // 3 > (1 << h["depth"]):
                raise PngError("PLTE longer than the bit depth allows")
            h["palette"] = np.frombuffer(body, np.uint8).reshape(-1, 3)
        elif t == b"IDAT":
            if ended_idat:
                raise PngError("IDAT chunks are not consecutive")
            seen_idat = True
            h["idat"].append(body)
        elif t == b"IEND":
            break
        elif t == b"tRNS":
            if seen_idat:
                raise PngError("tRNS out of place")
        elif t == b"gAMA":
            if n != 4 or seen_idat or h["palette"] is not None:
                raise PngError("gAMA out of place or corrupt")
            if h["gamma"]:
                raise PngError("more than one gAMA")
            h["gamma"] = _u32(body, 0)
            if h["gamma"] < 16 or h["gamma"] > 625000000:
                raise PngError("gAMA value out of range")
        elif t == b"sRGB":
            if n != 1 or seen_idat or h["palette"] is not None:
                raise PngError("sRGB out of place or corrupt")
            if h["srgb"]:
                raise PngError("more than one sRGB")
            if body[0] > 3:
                raise PngError("sRGB rendering intent out of range")
            h["srgb"] = True
        elif t == b"iCCP":
            raise PngError("iCCP colour profiles are not supported")
        elif t == b"cHRM":
            raise PngError("cHRM chromaticities are not supported")
        elif t == b"cICP":
            raise PngError("cICP colour information is not supported")
        elif t in (b"acTL", b"fcTL", b"fdAT"):
            raise PngError("animated PNG is not supported")
        elif t == b"eXIf":
            if not h["exif"]:
                h["exif"] = True
                h["orientation"] = exif_orientation(body)
        elif not (t[0] & 32):
            raise PngError("unknown critical chunk " + t.decode("latin-1"))
    if pos != len(d):
        raise PngError("data after IEND")
    if "width" not in h:
        raise PngError("IHDR is not the first chunk")
    if not h["idat"]:
        raise PngError("no IDAT chunk")
    if h["ct"] == 3 and h["palette"] is None:
        raise PngError("palette image without PLTE")
    if h["srgb"] and h["gamma"] and h["gamma"] != 45455:
        raise PngError("gAMA and sRGB disagree")
    fg = 45455 if h["srgb"] else h["gamma"]
    h["tables"] = gamma_tables(fg) if h["ct"] in (2, 3, 6) else None
    if h["tables"] is not None and h["depth"] == 16:
        raise PngError("gamma correction of 16-bit colour is not supported")
    z = b"".join(h["idat"])
    if len(z) < 2 or (z[0] & 15) != 8 or (z[0] >> 4) > 7 or ((z[0] << 8) | z[1]) % 31:
        raise PngError("corrupt zlib header")
    if z[1] & 32:
        raise PngError("zlib preset dictionary")
    h["zlib"] = z
    o = h["orientation"]
    h["orientation"] = o if 1 <= o <= 8 else 1
    W, H = h["width"], h["height"]
    h["out_width"], h["out_height"] = (H, W) if h["orientation"] >= 5 else (W, H)
    h["raw_size"] = raw_size(W, H, h["ct"], h["depth"], h["interlace"])
    return h


def info(data):
    h = parse(data)
    return h["out_width"], h["out_height"]


# ------------------------------------------------------------------------------------------------ decoding
def inflate(z, size):
    """the zlib stream's output, checked as the GPU checks it: exactly `size` bytes, a correct Adler-32, nothing after the stream"""
    dec = zlib.decompressobj()
    try:
        out = dec.decompress(z, size + 1)
    except zlib.error as e:
        raise PngError("corrupt deflate stream (%s)" % e)
    if len(out) > size:
        raise PngError("corrupt deflate stream (more data than the image holds)")
    if not dec.eof:
        raise PngError("corrupt deflate stream (it ends early)")
    if dec.unused_data:
        raise PngError("data after the zlib stream")
    if len(out) < size:
        raise PngError("corrupt deflate stream (less data than the image holds)")
    if (z[0] >> 4) < 7 and max_distance(z) > 1 << ((z[0] >> 4) + 8):
        raise PngError("corrupt deflate stream (distance too far back)")
    return np.frombuffer(out, np.uint8)


def max_distance(z):
    """the longest match distance of a valid zlib stream (zlib never checks it against the header's window when the output buffer
    holds the bytes; the GPU rejects any distance beyond that window, and libpng, which inflates row by row, rejects most)"""
    bits = int.from_bytes(z[2:], "little")
    pos = [0]

    def get(k):
        v = (bits >> pos[0]) & ((1 << k) - 1)
        pos[0] += k
        return v

    def table(lens):
        codes = canonical(lens)
        return {(ln, c): s for s, (ln, c) in enumerate(zip(lens, codes)) if ln}

    def sym(t):
        c = ln = 0
        while (ln, c) not in t:
            c = c << 1 | get(1)
            ln += 1
        return t[(ln, c)]
    far, last = 0, 0
    while not last:
        last, kind = get(1), get(2)
        if kind == 0:
            pos[0] = (pos[0] + 7) // 8 * 8
            n = get(16)
            get(16)
            pos[0] += 8 * n
            continue
        if kind == 1:
            lt, dt = table(FIXED_LIT), table(FIXED_DIST)
        else:
            nl, nd, nc = get(5) + 257, get(5) + 1, get(4) + 4
            cl = [0] * 19
            for k in range(nc):
                cl[CL_ORDER[k]] = get(3)
            ct, lens = table(cl), []
            while len(lens) < nl + nd:
                s = sym(ct)
                if s < 16:
                    lens.append(s)
                elif s == 16:
                    lens += [lens[-1]] * (3 + get(2))
                else:
                    lens += [0] * ((3 + get(3)) if s == 17 else (11 + get(7)))
            lt, dt = table(lens[:nl]), table(lens[nl:])
        while True:
            s = sym(lt)
            if s == 256:
                break
            if s > 256:
                get(LEN_EXTRA[s - 257])
                d = sym(dt)
                far = max(far, DIST_BASE[d] + get(DIST_EXTRA[d]))
    return far


def unfilter(raw, pw, ph, bpp, rb):
    """filtered rows (filter byte + rb bytes each) -> [ph, rb] uint8"""
    rows = raw.reshape(ph, rb + 1).astype(np.int64)
    out = np.zeros((ph, rb), np.int64)
    prev = np.zeros(rb, np.int64)
    for y in range(ph):
        f, cur = int(rows[y, 0]), rows[y, 1:].copy()
        if f == 0:
            pass
        elif f == 1:
            for x in range(bpp, rb):
                cur[x] = (cur[x] + cur[x - bpp]) & 255
        elif f == 2:
            cur = (cur + prev) & 255
        elif f == 3:
            for x in range(rb):
                a = cur[x - bpp] if x >= bpp else 0
                cur[x] = (cur[x] + ((a + prev[x]) >> 1)) & 255
        elif f == 4:
            for x in range(rb):
                a = cur[x - bpp] if x >= bpp else 0
                c = prev[x - bpp] if x >= bpp else 0
                b = prev[x]
                p = a + b - c
                pa, pb, pc = abs(p - a), abs(p - b), abs(p - c)
                pr = a if pa <= pb and pa <= pc else (b if pb <= pc else c)
                cur[x] = (cur[x] + pr) & 255
        else:
            raise PngError("corrupt image data (bad filter type)")
        out[y] = cur
        prev = cur
    return out.astype(np.uint8)


def samples(rows, pw, ch, depth):
    """unfiltered rows -> [ph, pw, ch] int64 samples"""
    if depth == 16:
        s = rows.astype(np.int64)
        s = (s[:, 0::2] << 8) | s[:, 1::2]
    elif depth == 8:
        s = rows.astype(np.int64)
    else:
        bits = np.unpackbits(rows, axis=1).reshape(rows.shape[0], -1, depth)
        s = np.zeros(bits.shape[:2], np.int64)
        for k in range(depth):
            s = (s << 1) | bits[:, :, k]
    return s[:, :pw * ch].reshape(rows.shape[0], pw, ch)


def to_gray(s, h):
    """libpng's transforms as OpenCV sets them for IMREAD_GRAYSCALE: strip alpha, palette -> RGB (indices past PLTE read black),
    1/2/4-bit grey by bit replication, rgb_to_gray, 16 -> 8 bits by the high byte"""
    ct, depth = h["ct"], h["depth"]
    if ct in (0, 4):
        g = s[..., 0]
        if depth == 16:
            return (g >> 8).astype(np.uint8)
        return (g * (255 // ((1 << depth) - 1))).astype(np.uint8)
    if ct == 3:
        pal = np.zeros((256, 3), np.int64)
        pal[:len(h["palette"])] = h["palette"]
        rgb = pal[s[..., 0]]
        return rgb_to_gray8(rgb[..., 0], rgb[..., 1], rgb[..., 2], h["tables"])
    if depth == 16:
        return rgb_to_gray16(s[..., 0], s[..., 1], s[..., 2])
    return rgb_to_gray8(s[..., 0], s[..., 1], s[..., 2], h["tables"])


def decode_gray(data):
    h = parse(data)
    W, H, ct, depth = h["width"], h["height"], h["ct"], h["depth"]
    raw = inflate(h["zlib"], h["raw_size"])
    ch = CHANNELS[ct]
    bpp = max(1, ch * depth // 8)
    img = np.zeros((H, W), np.uint8)
    off = 0
    for k, (pw, ph) in enumerate(passes(W, H, h["interlace"])):
        if not pw or not ph:
            continue
        rb = row_bytes(pw, ct, depth)
        rows = unfilter(raw[off:off + ph * (rb + 1)], pw, ph, bpp, rb)
        off += ph * (rb + 1)
        g = to_gray(samples(rows, pw, ch, depth), h)
        if h["interlace"]:
            x0, y0, dx, dy = ADAM7[k]
            img[y0::dy, x0::dx] = g
        else:
            img[:] = g
    return np.ascontiguousarray(orient(img, h["orientation"]))


# ------------------------------------------------------------------------------------------------ DEFLATE encoder
class BitWriter:
    def __init__(self):
        self.acc, self.n, self.out = 0, 0, bytearray()

    def bits(self, v, k):
        self.acc |= v << self.n
        self.n += k
        while self.n >= 8:
            self.out.append(self.acc & 255)
            self.acc >>= 8
            self.n -= 8

    def code(self, c, ln):
        """a Huffman code, most significant bit first"""
        r = 0
        for i in range(ln):
            r |= ((c >> i) & 1) << (ln - 1 - i)
        self.bits(r, ln)

    def align(self):
        if self.n:
            self.bits(0, 8 - self.n)


LEN_BASE = [3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258]
LEN_EXTRA = [0] * 8 + [1] * 4 + [2] * 4 + [3] * 4 + [4] * 4 + [5] * 4 + [0]
DIST_BASE = [1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097, 6145, 8193,
             12289, 16385, 24577]
DIST_EXTRA = [0, 0, 0, 0] + [i // 2 for i in range(2, 28)]
CL_ORDER = [16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15]


def _len_code(n):
    for i in range(28, -1, -1):
        if n >= LEN_BASE[i]:
            return i
    raise ValueError(n)


def _dist_code(d):
    for i in range(29, -1, -1):
        if d >= DIST_BASE[i]:
            return i
    raise ValueError(d)


def lz77(data, start=0, window=32768, min_len=3):
    """greedy tokens of data[start:] (literals as ints, matches as (length, distance)); matches may reach back before start"""
    toks, head, i, n = [], {}, start, len(data)
    for j in range(max(0, start - window), start):
        if j + 3 <= n:
            head.setdefault(bytes(data[j:j + 3]), []).append(j)
    while i < n:
        best = (0, 0)
        if i + 3 <= n:
            key = bytes(data[i:i + 3])
            for j in reversed(head.get(key, [])[-16:]):
                if i - j > window:
                    break
                k = 0
                while k < 258 and i + k < n and data[j + k] == data[i + k]:
                    k += 1
                if k > best[0]:
                    best = (k, i - j)
        step = best[0] if best[0] >= min_len else 1
        for j in range(i, i + step):
            if j + 3 <= n:
                head.setdefault(bytes(data[j:j + 3]), []).append(j)
        toks.append(best if best[0] >= min_len else int(data[i]))
        i += step
    return toks


def huffman_lengths(freq, limit=15):
    """code lengths (<= limit) of a Huffman code for the nonzero frequencies; one used symbol gets length 1"""
    used = [i for i, f in enumerate(freq) if f]
    lens = [0] * len(freq)
    if len(used) == 1:
        lens[used[0]] = 1
        return lens
    scale = 1
    while True:
        h = [(max(1, freq[i] // scale), k, [i]) for k, i in enumerate(used)]
        heapq.heapify(h)
        cnt = len(h)
        depth = {i: 0 for i in used}
        while len(h) > 1:
            a, b = heapq.heappop(h), heapq.heappop(h)
            for s in a[2] + b[2]:
                depth[s] += 1
            heapq.heappush(h, (a[0] + b[0], cnt, a[2] + b[2]))
            cnt += 1
        if max(depth.values()) <= limit:
            for i in used:
                lens[i] = depth[i]
            return lens
        scale *= 2


def canonical(lens):
    """the canonical codes of a length list (RFC 1951 3.2.2)"""
    mx = max(lens) if lens else 0
    bl = [0] * (mx + 2)
    for ln in lens:
        if ln:
            bl[ln] += 1
    code, nxt = 0, [0] * (mx + 2)
    for b in range(1, mx + 1):
        code = (code + bl[b - 1]) << 1
        nxt[b] = code
    out = [0] * len(lens)
    for i, ln in enumerate(lens):
        if ln:
            out[i] = nxt[ln]
            nxt[ln] += 1
    return out


FIXED_LIT = [8] * 144 + [9] * 112 + [7] * 24 + [8] * 8
FIXED_DIST = [5] * 30


def _symbols(toks):
    for t in toks:
        if isinstance(t, tuple):
            ln, dist = t
            lc, dc = _len_code(ln), _dist_code(dist)
            yield 257 + lc, (ln - LEN_BASE[lc], LEN_EXTRA[lc]), dc, (dist - DIST_BASE[dc], DIST_EXTRA[dc])
        else:
            yield t, None, None, None


def _rle_lengths(lens):
    """code-length symbols (symbol, extra value, extra bits) with 16/17/18 runs"""
    out, i = [], 0
    while i < len(lens):
        v, r = lens[i], 1
        while i + r < len(lens) and lens[i + r] == v:
            r += 1
        if v == 0 and r >= 11:
            k = min(r, 138)
            out.append((18, k - 11, 7))
        elif v == 0 and r >= 3:
            k = min(r, 10)
            out.append((17, k - 3, 3))
        elif v and r >= 4:
            out.append((v, 0, 0))
            k = min(r - 1, 6)
            out.append((16, k - 3, 2))
            k += 1
        else:
            out.append((v, 0, 0))
            k = 1
        i += k
    return out


def _write_tokens(bw, toks, lit_lens, dist_lens):
    lc_, dc_ = canonical(lit_lens), canonical(dist_lens)
    for sym, lx, dsym, dx in _symbols(toks):
        bw.code(lc_[sym], lit_lens[sym])
        if lx is not None:
            bw.bits(*lx)
            bw.code(dc_[dsym], dist_lens[dsym])
            bw.bits(*dx)
    bw.code(lc_[256], lit_lens[256])


def deflate_blocks(blocks):
    """raw DEFLATE of a list of blocks; each block is (kind, payload, opts):
      ("stored", bytes)                      one stored block (any length up to 65,535, 0 allowed)
      ("fixed", tokens)                      the fixed codes
      ("dynamic", tokens, opts)              Huffman codes from the tokens' frequencies; opts: chain=True gives the used literal /
                                             length symbols the lengths 1, 2, .., k-1, k-1 (15-bit codes for 16 symbols);
                                             no_dist=True writes one distance code of length 0 (no matches allowed)
    The last block is marked final."""
    bw = BitWriter()
    for bi, blk in enumerate(blocks):
        kind, payload = blk[0], blk[1]
        opts = blk[2] if len(blk) > 2 else {}
        final = 1 if bi == len(blocks) - 1 else 0
        if kind == "stored":
            bw.bits(final, 1)
            bw.bits(0, 2)
            bw.align()
            n = len(payload)
            bw.bits(n, 16)
            bw.bits(n ^ 0xFFFF, 16)
            for c in payload:
                bw.bits(c, 8)
        elif kind == "fixed":
            bw.bits(final, 1)
            bw.bits(1, 2)
            _write_tokens(bw, payload, FIXED_LIT, FIXED_DIST)
        else:
            lf, df = [0] * 286, [0] * 30
            lf[256] = 1
            for sym, _, dsym, _ in _symbols(payload):
                lf[sym] += 1
                if dsym is not None:
                    df[dsym] += 1
            if opts.get("chain"):
                used = sorted((i for i in range(286) if lf[i]), key=lambda i: -lf[i])
                ll = [0] * 286
                for r, i in enumerate(used):
                    ll[i] = min(r + 1, len(used) - 1) if len(used) > 1 else 1
            else:
                ll = huffman_lengths(lf)
            dl = [0] if opts.get("no_dist") else (huffman_lengths(df) if any(df) else [0])
            nl = max(257, max(i for i in range(286) if ll[i]) + 1)
            nd = max(1, max([i for i in range(len(dl)) if dl[i]] or [0]) + 1)
            seq = _rle_lengths(ll[:nl] + dl[:nd])
            cf = [0] * 19
            for s, _, _ in seq:
                cf[s] += 1
            cl = huffman_lengths(cf, 7)
            ncl = max(4, max(k for k in range(19) if cl[CL_ORDER[k]]) + 1)
            bw.bits(final, 1)
            bw.bits(2, 2)
            bw.bits(nl - 257, 5)
            bw.bits(nd - 1, 5)
            bw.bits(ncl - 4, 4)
            for k in range(ncl):
                bw.bits(cl[CL_ORDER[k]], 3)
            cc = canonical(cl)
            for s, v, k in seq:
                bw.code(cc[s], cl[s])
                if k:
                    bw.bits(v, k)
            _write_tokens(bw, payload, ll + [0] * (288 - len(ll)), dl + [0] * (30 - len(dl)))
    bw.align()
    return bytes(bw.out)


def zlib_wrap(raw_deflate, data, adler=None, cmf=0x78):
    """a zlib stream: the header (cmf: method 8 and the window's CINFO), the DEFLATE data, the Adler-32 of data"""
    a = zlib.adler32(data) if adler is None else adler
    return bytes([cmf, (31 - (cmf << 8) % 31) % 31]) + raw_deflate + struct.pack(">I", a & 0xFFFFFFFF)


def tokens_of(data, start, end):
    """greedy tokens of data[start:end], matches allowed to reach back before start"""
    return lz77(data[:end], start)


# ------------------------------------------------------------------------------------------------ PNG writer
def chunk(t, body, bad_crc=False):
    c = zlib.crc32(t + body) ^ (1 if bad_crc else 0)
    return struct.pack(">I", len(body)) + t + body + struct.pack(">I", c)


def filter_rows(rows, bpp, filters):
    """[ph, rb] uint8 rows -> filtered bytes; filters: one type per row (cycled)"""
    out = bytearray()
    prev = np.zeros(rows.shape[1], np.int64)
    for y in range(rows.shape[0]):
        f = filters[y % len(filters)]
        cur = rows[y].astype(np.int64)
        a = np.concatenate([np.zeros(bpp, np.int64), cur[:-bpp] if bpp < len(cur) else np.zeros(0, np.int64)])[:len(cur)]
        c = np.concatenate([np.zeros(bpp, np.int64), prev[:-bpp] if bpp < len(prev) else np.zeros(0, np.int64)])[:len(cur)]
        if f == 0:
            r = cur
        elif f == 1:
            r = cur - a
        elif f == 2:
            r = cur - prev
        elif f == 3:
            r = cur - ((a + prev) >> 1)
        else:
            p = a + prev - c
            pa, pb, pc = np.abs(p - a), np.abs(p - prev), np.abs(p - c)
            pr = np.where((pa <= pb) & (pa <= pc), a, np.where(pb <= pc, prev, c))
            r = cur - pr
        out.append(f)
        out += (r & 255).astype(np.uint8).tobytes()
        prev = cur
    return bytes(out)


def pack_samples(s, depth):
    """[ph, pw, ch] int samples -> [ph, rb] uint8 rows"""
    ph = s.shape[0]
    flat = s.reshape(ph, -1).astype(np.int64)
    if depth == 16:
        return np.stack([flat >> 8, flat & 255], axis=2).reshape(ph, -1).astype(np.uint8)
    if depth == 8:
        return flat.astype(np.uint8)
    bits = ((flat[:, :, None] >> np.arange(depth - 1, -1, -1)) & 1).reshape(ph, -1).astype(np.uint8)
    return np.packbits(bits, axis=1)


def raw_image(s, ct, depth, interlace, filters=(0,)):
    """samples [H, W, ch] -> the filtered bytes of every pass"""
    H, W = s.shape[:2]
    ch = CHANNELS[ct]
    bpp = max(1, ch * depth // 8)
    out = b""
    if not interlace:
        return filter_rows(pack_samples(s, depth), bpp, filters)
    for x0, y0, dx, dy in ADAM7:
        p = s[y0::dy, x0::dx]
        if p.shape[0] and p.shape[1]:
            out += filter_rows(pack_samples(p, depth), bpp, filters)
    return out


def exif_block(o, big_endian=False):
    """a TIFF block with IFD0 holding only the orientation tag"""
    e = ">" if big_endian else "<"
    return (b"MM" if big_endian else b"II") + struct.pack(e + "HI", 0x2A, 8) + struct.pack(e + "H", 1) + \
        struct.pack(e + "HHIHH", 0x0112, 3, 1, o, 0) + struct.pack(e + "I", 0)


def write_png(s, ct, depth, interlace=0, filters=(0,), palette=None, zdata=None, compress=None, splits=None, pre=(), mid=(),
              post_idat=(), trailer=b"", idat_bad_crc=False):
    """samples [H, W, ch] (ints) -> file bytes.  zdata: the zlib stream to use as is; compress: a function raw -> zlib stream
    (default zlib level 6); splits: byte offsets where the zlib stream is cut into IDAT chunks; pre: (type, body) chunks between IHDR
    and PLTE; mid: chunks between PLTE and IDAT; post_idat: chunks between the last IDAT and IEND; trailer: bytes after IEND"""
    s = np.asarray(s)
    if s.ndim == 2:
        s = s[:, :, None]
    H, W = s.shape[:2]
    raw = raw_image(s, ct, depth, interlace, filters)
    if zdata is None:
        zdata = compress(raw) if compress else zlib.compress(raw, 6)
    out = SIG + chunk(b"IHDR", struct.pack(">IIBBBBB", W, H, depth, ct, 0, 0, interlace))
    for t, b in pre:
        out += chunk(t, b)
    if palette is not None:
        out += chunk(b"PLTE", np.asarray(palette, np.uint8).tobytes())
    for t, b in mid:
        out += chunk(t, b)
    cuts = [0] + list(splits or []) + [len(zdata)]
    for a, b in zip(cuts[:-1], cuts[1:]):
        out += chunk(b"IDAT", zdata[a:b], idat_bad_crc)
    for t, b in post_idat:
        out += chunk(t, b)
    return out + chunk(b"IEND", b"") + trailer


# ------------------------------------------------------------------------------------------------ fixtures
def rle_tokens(data):
    """literals and distance-1 matches only: one distance code in the whole block"""
    toks, i = [], 0
    while i < len(data):
        r = 0
        while i > 0 and i + r < len(data) and r < 258 and data[i + r] == data[i - 1]:
            r += 1
        if r >= 3:
            toks.append((r, 1))
            i += r
        else:
            toks.append(int(data[i]))
            i += 1
    return toks


def special_deflate(kind, raw):
    """the zlib stream of raw as one of the writer's DEFLATE layouts"""
    raw = bytes(raw)
    n = len(raw)
    if kind == "stored":          # an empty stored block, then blocks of 65,535 bytes and the rest
        blocks, i = [("stored", b"")], 0
        while i < n:
            blocks.append(("stored", raw[i:i + 65535]))
            i += 65535
    elif kind == "fixed":
        blocks = [("fixed", lz77(raw))]
    elif kind == "dyn_chain":     # 16 used literal/length symbols: codes of 1 .. 15 bits
        blocks = [("dynamic", [int(c) for c in raw], {"chain": True})]
    elif kind == "single_dist":
        blocks = [("dynamic", rle_tokens(raw))]
    elif kind == "no_dist":
        blocks = [("dynamic", [int(c) for c in raw], {"no_dist": True})]
    elif kind == "far":           # literals for the first 32,768 bytes, then matches of up to 258 at distance 32,768
        toks, i = [int(c) for c in raw[:32768]], 32768
        while i < n:
            k = min(258, n - i)
            toks += [(k, 32768)] if k >= 3 else [int(c) for c in raw[i:i + k]]
            i += k
        blocks = [("dynamic", toks)]
    elif kind == "overlap":       # matches at distances 1..31 only, mostly longer than their distance
        blocks = [("dynamic", lz77(raw, window=31))]
    elif kind == "block_in_row":  # block boundaries inside rows; matches reach across them
        cuts = [0, 37, 500, 1001, 1700, n]
        kinds = ["dynamic", "fixed", "stored", "dynamic", "fixed"]
        blocks = []
        for k, (a, b) in zip(kinds, zip(cuts[:-1], cuts[1:])):
            blocks.append(("stored", raw[a:b]) if k == "stored" else (k, tokens_of(raw, a, b)))
    elif kind == "small_window":  # a header announcing a 256-byte window, with matches farther back (zlib and libpng accept them)
        return zlib_wrap(deflate_blocks([("fixed", lz77(raw))]), raw, cmf=0x08)
    else:
        raise ValueError(kind)
    return zlib_wrap(deflate_blocks(blocks), raw)


def case_samples(p):
    """the samples [h, w, ch] of a writer case"""
    rng = np.random.default_rng(p["seed"])
    ct, depth, w, h = p["ct"], p["depth"], p["w"], p["h"]
    ch = CHANNELS[ct]
    hi = (1 << depth) if ct != 3 else min(1 << depth, p.get("pal_n", 1 << depth) + p.get("pal_over", 0))
    pat = p.get("pattern", "random")
    if pat == "levels":
        return rng.integers(0, p["levels"], (h, w, ch))
    if pat == "smooth":
        y, x = np.mgrid[0:h, 0:w]
        s = ((x * 7 + y * 3) // 5 % hi)[:, :, None].repeat(ch, 2)
        return s + 0 * rng.integers(0, 1, s.shape)
    if pat == "repeat128":
        s = rng.integers(0, hi, (128, w, ch))
        return np.concatenate([s, s[:h - 128]], 0)
    if pat == "row_pairs":
        s = rng.integers(0, hi, ((h + 1) // 2, w, ch))
        return np.repeat(s, 2, 0)[:h]
    if pat == "periodic":
        per = rng.integers(1, 32, h)
        return np.stack([np.tile(rng.integers(0, hi, (per[y], ch)), (w // per[y] + 1, 1))[:w] for y in range(h)], 0)
    s = rng.integers(0, hi, (h, w, ch))
    if ct in (2, 6):
        g = rng.random((h, w)) < 0.25
        s[g, 1] = s[g, 0]
        s[g, 2] = s[g, 0]
    return s


def build_case(p):
    """the file bytes of a writer case (writer_cases)"""
    s = case_samples(p)
    rng = np.random.default_rng(p["seed"] + 1)
    pal = rng.integers(0, 256, (p.get("pal_n", 1 << p["depth"]), 3)) if p["ct"] == 3 else None
    chunks = lambda key: [(t.encode(), bytes.fromhex(b)) for t, b in p.get(key, [])]  # noqa: E731
    comp = None
    if p.get("deflate"):
        comp = lambda raw: special_deflate(p["deflate"], raw)  # noqa: E731
    elif p.get("level") is not None:
        comp = lambda raw: zlib.compress(raw, p["level"])  # noqa: E731
    return write_png(s, p["ct"], p["depth"], interlace=p.get("interlace", 0), filters=tuple(p.get("filters", (0,))), palette=pal,
                     compress=comp, splits=p.get("splits"), pre=chunks("pre"), mid=chunks("mid"), post_idat=chunks("post"))


def _gama(g):
    return ["gAMA", struct.pack(">I", g).hex()]


def writer_cases():
    """[(name, params)] of the writer's fixtures"""
    out, seed = [], 100
    F = [0, 1, 2, 3, 4]

    def add(name, **p):
        nonlocal seed
        p.setdefault("seed", seed)
        seed += 1
        out.append((name, p))
    for ct, depths in LEGAL.items():
        for d in depths:
            add(f"ct{ct}_d{d}", ct=ct, depth=d, w=29, h=13, filters=F)
            add(f"ct{ct}_d{d}_adam7", ct=ct, depth=d, w=23, h=19, filters=F, interlace=1)
    for k in range(1, 10):
        add(f"adam7_grey_{k}x{k}", ct=0, depth=8, w=k, h=k, interlace=1, filters=F)
        add(f"adam7_rgb_{k}x{k + 1}", ct=2, depth=8, w=k, h=k + 1, interlace=1, filters=F)
    for o in range(1, 9):
        for be in (0, 1):
            add(f"exif_{o}_{'mm' if be else 'ii'}", ct=0, depth=8, w=7, h=5, filters=F, pre=[["eXIf", exif_block(o, be).hex()]])
    add("exif_6_adam7_rgb", ct=2, depth=8, w=11, h=6, interlace=1, filters=F, pre=[["eXIf", exif_block(6).hex()]])
    add("exif_bad_value", ct=0, depth=8, w=7, h=5, pre=[["eXIf", exif_block(9).hex()]])
    add("exif_twice_first_wins", ct=0, depth=8, w=7, h=5, pre=[["eXIf", exif_block(6).hex()], ["eXIf", exif_block(3, 1).hex()]])
    for g in (100000, 45455, 220000, 96000, 94000, 104000, 106000, 50000):
        add(f"gamma_{g}_rgb", ct=2, depth=8, w=64, h=64, pre=[_gama(g)])
    add("gamma_45455_rgba", ct=6, depth=8, w=40, h=30, pre=[_gama(45455)], filters=F)
    add("gamma_45455_palette", ct=3, depth=8, w=40, h=30, pre=[_gama(45455)])
    add("gamma_45455_palette_2bit", ct=3, depth=2, w=40, h=30, pre=[_gama(45455)])
    add("gamma_45455_grey", ct=0, depth=8, w=40, h=30, pre=[_gama(45455)])
    add("gamma_45455_grey16", ct=0, depth=16, w=40, h=30, pre=[_gama(45455)])
    add("srgb_rgb", ct=2, depth=8, w=64, h=64, pre=[["sRGB", "00"]])
    add("srgb_gama_rgb", ct=2, depth=8, w=64, h=64, pre=[["sRGB", "00"], _gama(45455)])
    add("gamma_100000_rgb16", ct=2, depth=16, w=20, h=20, pre=[_gama(100000)])
    add("trns_grey", ct=0, depth=8, w=20, h=9, mid=[["tRNS", "0007"]])
    add("trns_grey_2bit", ct=0, depth=2, w=20, h=9, mid=[["tRNS", "0001"]])
    add("trns_rgb", ct=2, depth=8, w=20, h=9, mid=[["tRNS", "000700080009"]])
    add("trns_palette", ct=3, depth=4, w=20, h=9, mid=[["tRNS", "00ff80"]])
    add("trns_rgb_bad_length", ct=2, depth=8, w=20, h=9, mid=[["tRNS", "0007"]])
    add("trns_grey_bad_length", ct=0, depth=8, w=20, h=9, mid=[["tRNS", "000700"]])
    add("palette_short", ct=3, depth=8, w=20, h=9, pal_n=5, pal_over=40)
    add("palette_rgb_suggested", ct=2, depth=8, w=20, h=9, mid=[["PLTE", "102030405060"]])
    add("unknown_ancillary", ct=2, depth=8, w=20, h=9, pre=[["abCd", "68656c6c6f"]], post=[["zzZz", ""]])
    add("text_chunks", ct=0, depth=8, w=20, h=9, pre=[["tEXt", b"Title\0x".hex()], ["pHYs", "000000010000000100"]])
    add("idat_empty_and_split", ct=2, depth=8, w=40, h=20, splits=[0, 0, 1, 2, 2, 7, 100, 101])
    add("idat_split_in_header", ct=0, depth=8, w=40, h=20, splits=[1])
    add("idat_split_every_byte", ct=0, depth=4, w=17, h=5, splits=list(range(1, 60)), filters=F)
    for lv in (0, 1, 9):
        add(f"zlib_level{lv}_rgb", ct=2, depth=8, w=120, h=70, level=lv, filters=F, pattern="smooth")
    add("deflate_stored", ct=0, depth=8, w=300, h=300, deflate="stored")
    add("deflate_fixed", ct=2, depth=8, w=50, h=20, deflate="fixed", pattern="smooth", filters=F)
    add("deflate_dyn_15bit_codes", ct=0, depth=8, w=40, h=40, deflate="dyn_chain", pattern="levels", levels=15)
    add("deflate_single_distance", ct=0, depth=8, w=64, h=16, deflate="single_dist", pattern="levels", levels=2)
    add("deflate_no_distance", ct=0, depth=8, w=30, h=20, deflate="no_dist")
    add("deflate_258_at_32768", ct=0, depth=8, w=255, h=160, deflate="far", pattern="repeat128")
    add("deflate_overlaps_1_31", ct=0, depth=8, w=200, h=40, deflate="overlap", pattern="periodic")
    add("deflate_block_in_row", ct=2, depth=8, w=41, h=20, deflate="block_in_row", pattern="smooth", filters=F)
    add("deflate_block_in_row_adam7", ct=6, depth=8, w=33, h=17, deflate="block_in_row", interlace=1, filters=F)
    add("wide_16bit_rgba_adam7", ct=6, depth=16, w=301, h=37, interlace=1, filters=F, level=1)
    add("tall_1bit", ct=0, depth=1, w=3, h=700, filters=F)
    return out


def reject_files():
    """[(name, bytes, reason)] of files the parser must reject, each naming its reason"""
    rng = np.random.default_rng(7)
    img = rng.integers(0, 256, (20, 30, 3))
    ok = write_png(img, 2, 8)
    z = zlib.compress(raw_image(img, 2, 8, 0), 6)
    rows = [("not_png", b"GIF89a" + bytes(20), "not a PNG file (no PNG signature)"),
            ("bad_idat_crc", write_png(img, 2, 8, idat_bad_crc=True), "bad CRC in chunk IDAT"),
            ("bad_ancillary_crc", ok[:33] + chunk(b"tEXt", b"a\0b", bad_crc=True) + ok[33:], "bad CRC in chunk tEXt"),
            ("truncated", ok[:-20], "truncated chunk"),
            ("no_iend", ok[:-12], "truncated chunk"),
            ("after_iend", ok + b"\0", "data after IEND"),
            ("iccp", write_png(img, 2, 8, pre=[(b"iCCP", b"p\0\0" + zlib.compress(b"x"))]), "iCCP colour profiles are not supported"),
            ("chrm", write_png(img, 2, 8, pre=[(b"cHRM", bytes(32))]), "cHRM chromaticities are not supported"),
            ("cicp", write_png(img, 2, 8, pre=[(b"cICP", b"\x01\x0d\x00\x01")]), "cICP colour information is not supported"),
            ("apng", write_png(img, 2, 8, pre=[(b"acTL", struct.pack(">II", 1, 0))]), "animated PNG is not supported"),
            ("gamma_rgb16", write_png(rng.integers(0, 65536, (5, 6, 3)), 2, 16, pre=[(b"gAMA", struct.pack(">I", 45455))]),
             "gamma correction of 16-bit colour is not supported"),
            ("gama_srgb_disagree", write_png(img, 2, 8, pre=[(b"sRGB", b"\0"), (b"gAMA", struct.pack(">I", 50000))]), "gAMA and sRGB disagree"),
            ("gama_after_plte", write_png(rng.integers(0, 4, (5, 6)), 3, 8, palette=rng.integers(0, 256, (4, 3)),
                                          mid=[(b"gAMA", struct.pack(">I", 45455))]), "gAMA out of place or corrupt"),
            ("gama_zero", write_png(img, 2, 8, pre=[(b"gAMA", bytes(4))]), "gAMA value out of range"),
            ("palette_without_plte", write_png(rng.integers(0, 4, (5, 6)), 3, 8), "palette image without PLTE"),
            ("plte_in_grey", write_png(rng.integers(0, 4, (5, 6)), 0, 8, mid=[(b"PLTE", bytes(6))]), "PLTE in a grey image"),
            ("plte_too_long", write_png(rng.integers(0, 4, (5, 6)), 3, 1, palette=rng.integers(0, 256, (3, 3))),
             "PLTE longer than the bit depth allows"),
            ("unknown_critical", write_png(img, 2, 8, pre=[(b"ABCD", b"")]), "unknown critical chunk ABCD"),
            ("bad_depth", SIG + chunk(b"IHDR", struct.pack(">IIBBBBB", 4, 4, 3, 2, 0, 0, 0)) + chunk(b"IDAT", z) + chunk(b"IEND", b""),
             "invalid colour type and bit depth"),
            ("interlace_2", SIG + chunk(b"IHDR", struct.pack(">IIBBBBB", 30, 20, 8, 2, 0, 0, 2)) + chunk(b"IDAT", z) + chunk(b"IEND", b""),
             "invalid compression, filter or interlace method"),
            ("too_wide", SIG + chunk(b"IHDR", struct.pack(">IIBBBBB", 1000001, 1, 8, 0, 0, 0, 0)) + chunk(b"IDAT", z) + chunk(b"IEND", b""),
             "image size outside the supported limits"),
            ("too_many_pixels", SIG + chunk(b"IHDR", struct.pack(">IIBBBBB", 40000, 30000, 8, 0, 0, 0, 0)) + chunk(b"IDAT", z) + chunk(b"IEND", b""),
             "image size outside the supported limits"),
            ("no_idat", SIG + chunk(b"IHDR", struct.pack(">IIBBBBB", 30, 20, 8, 2, 0, 0, 0)) + chunk(b"IEND", b""), "no IDAT chunk"),
            ("ihdr_not_first", SIG + chunk(b"tEXt", b"a\0b") + ok[8:], "IHDR is not the first chunk"),
            ("zlib_bad_method", write_png(img, 2, 8, zdata=b"\x79" + z[1:]), "corrupt zlib header"),
            ("zlib_bad_fcheck", write_png(img, 2, 8, zdata=z[:1] + bytes([z[1] ^ 1]) + z[2:]), "corrupt zlib header"),
            ("zlib_dictionary", write_png(img, 2, 8, zdata=b"\x78\xbb" + z[2:]), "zlib preset dictionary")]
    # IDAT chunks with another chunk between them
    parts = write_png(img, 2, 8, splits=[10])
    i = parts.index(b"IDAT", parts.index(b"IDAT") + 4) - 4
    rows.append(("idat_not_consecutive", parts[:i] + chunk(b"tEXt", b"a\0b") + parts[i:], "IDAT chunks are not consecutive"))
    # gamma chunks libpng only warns about: it keeps the first gAMA, and ignores a second sRGB or one with an intent above 3
    g45, g100 = (b"gAMA", struct.pack(">I", 45455)), (b"gAMA", struct.pack(">I", 100000))
    rows += [("gama_twice_45455_first", write_png(img, 2, 8, pre=[g45, g100]), "more than one gAMA"),
             ("gama_twice_100000_first", write_png(img, 2, 8, pre=[g100, g45]), "more than one gAMA"),
             ("srgb_twice", write_png(img, 2, 8, pre=[(b"sRGB", b"\0"), (b"sRGB", b"\1")]), "more than one sRGB"),
             ("srgb_intent_9", write_png(img, 2, 8, pre=[(b"sRGB", b"\x09")]), "sRGB rendering intent out of range")]
    return rows


def corrupt_streams():
    """[(name, bytes, reason)] of files whose headers parse but whose zlib stream or filters are corrupt: found on the GPU"""
    rng = np.random.default_rng(11)
    img = rng.integers(0, 256, (40, 50, 3))
    raw = raw_image(img, 2, 8, 0, (0, 1, 2, 3, 4))
    z = zlib.compress(raw, 6)

    def png(zd, s=img):
        return write_png(s, 2, 8, zdata=zd)
    bad_filter = bytearray(raw)
    bad_filter[151 * 7] = 5
    # a dynamic block whose literal/length code set is over-subscribed: HLIT 257, HDIST 1, HCLEN 18 codes of length 1..
    bw = BitWriter()
    bw.bits(1, 1); bw.bits(2, 2); bw.bits(0, 5); bw.bits(0, 5); bw.bits(15, 4)
    for _ in range(19):
        bw.bits(1, 3)
    bw.align()
    overs = zlib_wrap(bytes(bw.out) + bytes(16), raw)
    # a match whose distance reaches before the start: fixed block, literal then (3, 2)
    far = zlib_wrap(deflate_blocks([("fixed", [0, (3, 2)])]), raw)
    # a dynamic block whose code-length code is incomplete: two code-length codes of length 2
    bw = BitWriter()
    bw.bits(1, 1); bw.bits(2, 2); bw.bits(0, 5); bw.bits(0, 5); bw.bits(0, 4)
    for ln in (2, 2, 0, 0):
        bw.bits(ln, 3)
    bw.align()
    incomplete = zlib_wrap(bytes(bw.out) + bytes(16), raw)

    def fixed_symbols(lit, dist=None):
        """a final fixed block: literal 0, then literal/length symbol lit (with distance symbol dist)"""
        lc, dc = canonical(FIXED_LIT), canonical(FIXED_DIST + [5, 5])
        bw = BitWriter()
        bw.bits(1, 1); bw.bits(1, 2)
        bw.code(lc[0], FIXED_LIT[0])
        bw.code(lc[lit], FIXED_LIT[lit])
        if dist is not None:
            bw.code(dc[dist], 5)
        bw.code(lc[256], 7)
        bw.align()
        return zlib_wrap(bytes(bw.out) + bytes(8), raw)
    return [("bad_code_set", png(overs), "corrupt deflate stream (bad code lengths)"),
            ("incomplete_code_length_code", png(incomplete), "corrupt deflate stream (bad code lengths)"),
            ("literal_length_286", png(fixed_symbols(286)), "corrupt deflate stream (invalid code)"),
            ("literal_length_287", png(fixed_symbols(287)), "corrupt deflate stream (invalid code)"),
            ("distance_code_30", png(fixed_symbols(257, 30)), "corrupt deflate stream (invalid code)"),
            ("distance_code_31", png(fixed_symbols(257, 31)), "corrupt deflate stream (invalid code)"),
            ("cut_mid_stream", png(z[:len(z) // 2]), "corrupt deflate stream (it ends early)"),
            ("distance_beyond_window", build_case(dict(seed=5, ct=0, depth=8, w=300, h=6, deflate="small_window", pattern="row_pairs")),
             "corrupt deflate stream (distance too far back)"),
            ("distance_before_start", png(far), "corrupt deflate stream (distance too far back)"),
            ("overlong", png(zlib.compress(raw + bytes(151), 6)), "corrupt deflate stream (more data than the image holds)"),
            ("short", png(z[:-30]), "corrupt deflate stream (it ends early)"),
            ("underlong", png(zlib.compress(raw[:-151], 6)), "corrupt deflate stream (less data than the image holds)"),
            ("trailing", png(z + b"\0\0"), "data after the zlib stream"),
            ("adler", png(z[:-1] + bytes([z[-1] ^ 1])), "corrupt deflate stream (Adler-32 mismatch)"),
            ("block_type_3", png(b"\x78\x01\x07" + bytes(8)), "corrupt deflate stream (invalid block type)"),
            ("stored_nlen", png(b"\x78\x01\x01\x05\x00\x00\x00" + bytes(8)), "corrupt deflate stream (stored block length does not match its complement)"),
            ("bad_filter", png(zlib.compress(bytes(bad_filter), 6)), "corrupt image data (bad filter type)")]
