"""numpy restatement of the image preparation in front of line detection (line3dpp_b200/csrc/l3d_image_prep.cu, DESIGN.md §4b): what
the reference's detectLineSegments (line3D.cc:249-289) does with OpenCV before it calls LSD, i.e. cvtColor(CV_RGB2GRAY) for 3-channel
input and, when max_img_width > 0 and the larger side exceeds it, cv::resize(gray, out, Size(), s, s) with INTER_LINEAR; and the
post-processing of the detections (line3D.cc:317-366).  TEST INFRASTRUCTURE: the arithmetic of OpenCV 4.13's x86 build, integer by
integer, so that the kernel can be checked byte for byte on machines without OpenCV."""
import hashlib

import numpy as np

# RGB2Gray<uchar>: channel 0 is R; 15-bit fixed point with rounding (checked against cv2 over all 2^24 triples)
GRAY_R, GRAY_G, GRAY_B, GRAY_SHIFT = 9798, 19235, 3735, 15
COEF_SCALE = 2048           # INTER_RESIZE_COEF_SCALE: 11-bit interpolation weights


def make_image(h, w, c, seed=0):
    """uint8 [h, w] or [h, w, 3] from a seeded generator"""
    img = np.random.default_rng(seed).integers(0, 256, size=(h, w, c), dtype=np.uint8)
    return img[:, :, 0] if c == 1 else img


def sha(*arrays):
    h = hashlib.sha256()
    for a in arrays:
        h.update(np.ascontiguousarray(a).tobytes())
    return h.hexdigest()


def gray(img):
    """cvtColor(CV_RGB2GRAY) of an [h, w, 3] image; a 2-D image is returned as it is (the reference's clone())"""
    if img.ndim == 2:
        return img.copy()
    r, g, b = (img[..., k].astype(np.int64) for k in range(3))
    return ((r * GRAY_R + g * GRAY_G + b * GRAY_B + (1 << (GRAY_SHIFT - 1))) >> GRAY_SHIFT).astype(np.uint8)


def prepared_size(w, h, max_img_width):
    """(w, h, resized) of the image LSD sees: the rounding of csrc/line3d_bin.cc preparedImageSize, i.e. the size
    cv::resize(img, out, Size(), s, s) gives with s = float(max_img_width) / float(max(w, h)) when the larger side exceeds it"""
    if max_img_width > 0 and max(w, h) > max_img_width:
        s = float(np.float32(max_img_width) / np.float32(max(w, h)))
        return int(np.rint(w * s)), int(np.rint(h * s)), True
    return w, h, False


def scale_of(w, h, max_img_width):
    """the double 1 / s OpenCV uses as its source step (s: the float scale widened to double)"""
    return 1.0 / float(np.float32(max_img_width) / np.float32(max(w, h)))


def _linear_taps(n_dst, n_src, scale):
    """per destination index: first tap, weight of tap 0 and of tap 1 (OpenCV's xofs / ialpha or yofs / ibeta for downscaling)"""
    d = np.arange(n_dst, dtype=np.float64)
    f = ((d + 0.5) * scale - 0.5).astype(np.float32)
    i = np.floor(f).astype(np.int64)
    f = (f - i.astype(np.float32)).astype(np.float32)
    w0 = np.rint((np.float32(1) - f).astype(np.float32) * np.float32(COEF_SCALE)).astype(np.int64)
    w1 = np.rint(f * np.float32(COEF_SCALE)).astype(np.int64)
    return i, w0, w1


def resize_linear(g, dw, dh, scale):
    """cv::resize INTER_LINEAR of an 8-bit grey image to (dw, dh), source step `scale` (> 1) in both directions"""
    H, W = g.shape
    sx, a0, a1 = _linear_taps(dw, W, scale)
    # horizontal: a column whose second tap lies outside the image takes its first tap (clamped to the last column) at full weight
    edge = sx + 1 >= W
    sx = np.minimum(sx, W - 1)
    a0 = np.where(edge, COEF_SCALE, a0)
    a1 = np.where(edge, 0, a1)
    G = g.astype(np.int64)
    rows = G[:, sx] * a0 + G[:, np.minimum(sx + 1, W - 1)] * a1            # [H, dw], at most 255 * 2048
    # vertical: rows sy and sy + 1, the second clamped to the last row with its weight kept; OpenCV's SIMD mix (v_mul_hi of the
    # values shifted right by 4, rounding shift by 2), which its x86 build applies to every column
    sy, b0, b1 = _linear_taps(dh, H, scale)
    S0, S1 = rows[np.minimum(sy, H - 1)] >> 4, rows[np.minimum(sy + 1, H - 1)] >> 4
    v = ((S0 * b0[:, None]) >> 16) + ((S1 * b1[:, None]) >> 16)
    return np.clip((v + 2) >> 2, 0, 255).astype(np.uint8)


def resize_area2(g, dw, dh):
    """cv::resize with a source step of exactly 2: INTER_LINEAR becomes the fast INTER_AREA 2x2 mean; a destination pixel whose
    2x2 block leaves the image averages the pixels inside with cvRound (half to even)"""
    H, W = g.shape
    G = g.astype(np.int64)
    out = np.zeros((dh, dw), np.int64)
    fh, fw = min(dh, H // 2), min(dw, W // 2)
    blk = G[:2 * fh, :2 * fw].reshape(fh, 2, fw, 2).sum(axis=(1, 3))
    out[:fh, :fw] = (blk + 2) >> 2
    for y in range(dh):
        for x in range(dw):
            if y < fh and x < fw:
                continue
            ys = [v for v in (2 * y, 2 * y + 1) if v < H]
            xs = [v for v in (2 * x, 2 * x + 1) if v < W]
            vals = [G[a, b] for a in ys for b in xs]
            out[y, x] = int(np.rint(np.float32(sum(vals)) / np.float32(len(vals)))) if vals else 0
    return out.astype(np.uint8)


def prepare(img, max_img_width):
    """the grey image detectLineSegments hands to LSD"""
    g = gray(img)
    H, W = g.shape
    dw, dh, resized = prepared_size(W, H, max_img_width)
    if not resized:
        return g
    scale = scale_of(W, H, max_img_width)
    if scale == 2.0:
        return resize_area2(g, dw, dh)
    return resize_linear(g, dw, dh, scale)


def postprocess(det, orig_w, orig_h, prep_w, prep_h, max_line_segments):
    """line3D.cc:317-360 on detections (x1, y1, x2, y2) in the prepared image: upscale, float length, keep length > diag * 0.005,
    longest first as std::priority_queue with SegmentData2D_comparison pops them, cut at max_line_segments.  Returns float32 [n, 4].
    The pop order of equal lengths is the heap's, so this replays std::push_heap / std::pop_heap exactly."""
    f = np.float32
    ux, uy = f(orig_w) / f(prep_w), f(orig_h) / f(prep_h)
    min_len = f(np.sqrt(f(orig_h * orig_h) + f(orig_w * orig_w))) * f(0.005)
    heap = []
    for d in np.asarray(det, np.float32).reshape(-1, 4):
        p = np.array([d[0] * ux, d[1] * uy, d[2] * ux, d[3] * uy], np.float32)
        dx, dy = f(p[0] - p[2]), f(p[1] - p[3])
        length = f(np.sqrt(f(f(dx * dx) + f(dy * dy))))
        if length > min_len:
            _push_heap(heap, (float(length), p))
    out = []
    n = len(heap) if len(heap) < max_line_segments else max_line_segments
    while heap and len(out) < n:
        out.append(_pop_heap(heap)[1])
    return np.array(out, np.float32).reshape(-1, 4)


# libstdc++'s std::push_heap / std::pop_heap (max-heap on length with operator<), so that ties pop in the same order
def _push_heap(h, item):
    h.append(item)
    i = len(h) - 1
    while i > 0:
        parent = (i - 1) // 2
        if not (h[parent][0] < item[0]):
            break
        h[i] = h[parent]
        i = parent
    h[i] = item


def _pop_heap(h):
    top, last = h[0], h.pop()
    if not h:
        return top
    # __adjust_heap: move the hole to a leaf along the larger children, then push `last` up from there
    n, hole = len(h), 0
    child = 2 * hole + 2
    while child < n:
        if h[child][0] < h[child - 1][0]:
            child -= 1
        h[hole] = h[child]
        hole = child
        child = 2 * hole + 2
    if child == n:
        h[hole] = h[child - 1]
        hole = child - 1
    while hole > 0:
        parent = (hole - 1) // 2
        if not (h[parent][0] < last[0]):
            break
        h[hole] = h[parent]
        hole = parent
    h[hole] = last
    return top

