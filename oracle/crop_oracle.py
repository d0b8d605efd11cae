"""Detection crops: a numpy restatement of ``aae_extract_square_patches`` (augmentedautoencoder_b200/csrc/crops.cu) from the
integer (x, y, w, h, size) table onward, and the reference's scalar box arithmetic it starts from.

The reference (auto_pose/m3_interface/ae_pose_estimator.py:106-131,157-162) pastes the truncated box centred into a black
square of side ``size`` and resizes that with ``cv2.resize(..., INTER_LINEAR)``.  OpenCV's 8-bit path computes, per output
pixel d along each axis, ``fx = float32((d + 0.5) * scale - 0.5)`` in double, ``sx = floor(fx)``, the fraction rounded to
11-bit fixed point, the horizontal taps clamped to the source (the vertical ones are clipped instead), and
``(((b0 * (S0 >> 4)) >> 16) + ((b1 * (S1 >> 4)) >> 16) + 2) >> 2`` with S = p0 * a0 + p1 * a1.  ``tests/test_crops_cpu.py``
pins this restatement to the cv2 the tests import."""
import numpy as np


def reference_box_ints(bb_xywh, pad_factor):
    """(x, y, w, h, size) exactly as the reference writes them, one box at a time (ae_pose_estimator.py:108-109)."""
    x, y, w, h = np.array(bb_xywh).astype(np.int32)
    size = int(np.maximum(h, w) * pad_factor)
    return int(x), int(y), int(w), int(h), size


def float32_box_ints(bb_xywh, pad_factor):
    """The same integers by way of float32 boxes and a float32 pad factor, the route the device crops took before the
    host computed them: a float64 side just below an integer rounds up to it, and float32(1.3) < 1.3 < float64(1.3)."""
    x, y, w, h = (int(v) for v in np.asarray(bb_xywh, dtype=np.float32))
    size = int(float(max(h, w)) * float(np.float32(pad_factor)))
    return x, y, w, h, size


def detector_box(xmin, ymin, xmax, ymax, W, H):
    """The float64 pixel box AePoseEstimator.process makes of a relative BoundingBox (ae_pose_estimator.py:152)."""
    return [xmin * W, ymin * H, (xmax - xmin) * W, (ymax - ymin) * H]


def whole_pixel_boxes(W, H, n, rng, stride=3, max_side=None):
    """n detector boxes from pixel x0 to pixel x1 > x0 (and y0 to y1) on a stride-``stride`` grid, normalised by the frame
    size and multiplied back as process() does: float64 values that often land just below an integer.  Boxes may end on
    the frame's right or bottom edge.  ``max_side`` bounds the box sides (default: the frame)."""
    def pairs(N):
        m = N if max_side is None else max_side
        return np.array([(a, b) for a in range(0, N, stride) for b in range(a + 1, min(N, a + m) + 1, stride)])
    px, py = pairs(W), pairs(H)
    ix, iy = rng.randint(0, len(px), n), rng.randint(0, len(py), n)
    return [detector_box(px[i, 0] / W, py[j, 0] / H, px[i, 1] / W, py[j, 1] / H, W, H) for i, j in zip(ix, iy)]


def two_decimal_boxes(W, H, n, rng, max_rel=1.0):
    """n detector boxes with two-decimal relative corners (0.2, 0.35, ...), as a detector that rounds its output gives;
    sides up to ``max_rel`` of the frame."""
    m = int(round(max_rel * 100))
    pairs = np.array([(a, b) for a in range(100) for b in range(a + 1, min(100, a + m) + 1)])
    ix, iy = rng.randint(0, len(pairs), n), rng.randint(0, len(pairs), n)
    return [detector_box(pairs[i, 0] / 100, pairs[j, 0] / 100, pairs[i, 1] / 100, pairs[j, 1] / 100, W, H) for i, j in zip(ix, iy)]


def smooth_scene(H, W):
    """A smooth BGR uint8 scene from integer arithmetic only (the same bytes on any machine): ramps and broad waves,
    different per channel, wrapping at 256."""
    yy, xx = np.mgrid[0:H, 0:W].astype(np.int64)
    b = (xx * 3 + yy * 2 + ((xx * yy) >> 9)) % 256
    g = (xx + yy * 3 + (((xx - W // 2) ** 2 + (yy - H // 2) ** 2) >> 8)) % 256
    r = (255 - (xx * 2 + yy) % 256 + ((xx * xx) >> 11)) % 256
    return np.stack([b, g, r], -1).astype(np.uint8)


def scene_crc(img):
    import zlib
    return zlib.crc32(np.ascontiguousarray(img).tobytes())


def lin_coef(n_out, src_n, size, clamp):
    """lin_coef of crops.cu for d = 0 .. n_out-1: source indices (s0, s1) and 11-bit weights (c0, c1), int64 arrays."""
    scale = 1.0 / (float(n_out) / float(size))
    f = ((np.arange(n_out, dtype=np.float64) + 0.5) * scale - 0.5).astype(np.float32)
    s = np.floor(f).astype(np.int64)
    f = (f - s.astype(np.float32)).astype(np.float32)
    if clamp:
        lo, hi = s < 0, s >= src_n - 1
        s = np.where(lo, 0, np.where(hi, src_n - 1, s))
        f = np.where(lo | hi, np.float32(0), f).astype(np.float32)
    c0 = np.rint((np.float32(1) - f) * np.float32(2048)).astype(np.int64)      # __float2int_rn: half to even
    c1 = np.rint(f * np.float32(2048)).astype(np.int64)
    return np.clip(s, 0, src_n - 1), np.clip(s + 1, 0, src_n - 1), c0, c1


def square_patch(img, box_xywhs, out):
    """One crop of extract_square_patches_kernel: img uint8 [H, W, 3], box_xywhs the table row (x, y, w, h, size).
    Pixels outside the frame read as black; an empty box or a square smaller than the box gives a black crop."""
    x, y, w, h, size = (int(v) for v in box_xywhs)
    res = np.zeros((out, out, 3), np.uint8)
    if size <= 0 or w <= 0 or h <= 0 or size < max(w, h):
        return res
    H, W = img.shape[:2]
    # the black square with the box pasted centred; box pixels outside the frame stay black (fetch() of crops.cu)
    square = np.zeros((size, size, 3), np.int32)
    oy, ox = (size - h) // 2, (size - w) // 2
    y0, y1, x0, x1 = max(y, 0), min(y + h, H), max(x, 0), min(x + w, W)
    if y0 < y1 and x0 < x1:
        square[oy + y0 - y:oy + y1 - y, ox + x0 - x:ox + x1 - x] = img[y0:y1, x0:x1]
    xs0, xs1, a0, a1 = lin_coef(out, size, size, True)
    ys0, ys1, b0, b1 = lin_coef(out, size, size, False)
    a0, a1 = a0.astype(np.int32)[None, :, None], a1.astype(np.int32)[None, :, None]
    r0, r1 = square[ys0], square[ys1]
    S0 = r0[:, xs0] * a0 + r0[:, xs1] * a1                 # int32, as in the kernel: at most 255 * 2048
    S1 = r1[:, xs0] * a0 + r1[:, xs1] * a1
    b0, b1 = b0.astype(np.int32)[:, None, None], b1.astype(np.int32)[:, None, None]
    v = (((b0 * (S0 >> 4)) >> 16) + ((b1 * (S1 >> 4)) >> 16) + 2) >> 2
    res[:] = np.clip(v, 0, 255)
    return res


def square_patches(img, table, out):
    """All crops of a table: uint8 [n, out, out, 3]."""
    return np.stack([square_patch(img, row, out) for row in np.asarray(table).reshape(-1, 5)])
