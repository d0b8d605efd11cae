"""Training input pipeline of auto_pose/ae/dataset.py:456-495 (``Dataset.batch``) with the image work on the GPU: background
paste by mask + the imgaug chain the training cfg names under ``[Augmentation] CODE`` (auto_pose/ae/cfg/train_template.cfg:26-37).

The cfg string is evaluated against recording stand-ins for the imgaug classes (imgaug itself is not needed), the per-image
random draws are made here with numpy (same distributions as imgaug's stochastic parameters, not its random stream), and
``aae_augment`` applies them: cv2.warpAffine / cv2.GaussianBlur / cv2.resize(NEAREST) arithmetic bit for bit, the
value ops as composed 256-entry tables (include/aae_b200.h).  At the tensor-core trainer's ~10 000 images/s the reference's
10 Python threads of imgaug would be the bottleneck by more than an order of magnitude.

Supported chain: any subset of the template's ops IN THE TEMPLATE'S ORDER (CropAndPad, Affine, CoarseDropout, GaussianBlur, Add,
Invert, Multiply, Multiply, ContrastNormalization; another order raises): Sometimes(p, CropAndPad(percent= or px=, pad_cval=,
sample_independently=)), Sometimes(p, Affine(scale=(a, b))), Sometimes(p, CoarseDropout(p=, size_percent=)),
Sometimes(p, GaussianBlur(sigma)), Sometimes(p, Add((a, b), per_channel=)), Sometimes(p, Invert(p, per_channel=True)),
Sometimes(p, Multiply((a, b), per_channel=)), Sometimes(p, ContrastNormalization((a, b), per_channel=)).  Anything else raises.
CropAndPad (the template's commented-out ``Sometimes(0.5, CropAndPad(percent=(-0.05, 0.1)))``) takes a scalar or a (low, high)
range for ``percent`` / ``px`` and ``pad_cval``, ``pad_mode="constant"`` and ``keep_size=True`` only; its image is resized
back to (H, W) with cv2.resize's INTER_CUBIC / INTER_AREA arithmetic (``crop_pad_rule`` and the helpers below it).

``Occlusion`` adds the two occlusion switches of the cfg's ``[Augmentation]`` section (REALISTIC_OCCLUSION, SQUARE_OCCLUSION,
dataset.py:421-454), which edit the masks before the paste; ``aae_occlusion`` applies them.
"""
import ctypes as C

import numpy as np
import torch

from .. import _lib

FLAG_AFFINE, FLAG_DROP, FLAG_BLUR, FLAG_CROP = 1, 2, 4, 8


# ----------------------------------------------------------------------------------------------------------- cfg parsing
class _Op(object):
    def __init__(self, kind, *args, **kw):
        self.kind, self.args, self.kw = kind, args, kw

    def __repr__(self):
        return "%s%r%r" % (self.kind, self.args, self.kw)


def _recorder(kind):
    return lambda *a, **k: _Op(kind, *a, **k)


def parse_code(code):
    """``CODE`` string of the training cfg -> list of (probability, _Op).  ``np`` inside the string is numpy (the template
    draws the blur sigma with np.random.rand() once, when the cfg is evaluated -- as the reference does)."""
    names = ["Affine", "CoarseDropout", "GaussianBlur", "Add", "Invert", "Multiply", "ContrastNormalization", "LinearContrast",
             "PerspectiveTransform", "CropAndPad", "Fliplr", "Flipud", "AdditiveGaussianNoise", "Dropout"]
    ns = {n: _recorder(n) for n in names}
    ns["np"] = np
    ns["Sometimes"] = lambda p, op, *a, **k: (float(p), op)
    ns["Sequential"] = lambda ops, random_order=False, **k: ("seq", list(ops), bool(random_order))
    tag, ops, random_order = eval(code, {"__builtins__": {}}, ns)    # the reference evals the same string against imgaug (dataset.py:60-64)
    if random_order:
        raise NotImplementedError("Sequential(random_order=True) is not supported")
    out = []
    for item in ops:
        p, op = item if isinstance(item, tuple) else (1.0, item)
        if op.kind not in ("CropAndPad", "Affine", "CoarseDropout", "GaussianBlur", "Add", "Invert", "Multiply", "ContrastNormalization",
                           "LinearContrast"):
            raise NotImplementedError("augmenter %s is not supported on the device pipeline" % op.kind)
        out.append((p, op))
    return out


def _range(v):
    if isinstance(v, (tuple, list)):
        return float(v[0]), float(v[1])
    return float(v), float(v)


# ----------------------------------------------------------------------------------------------------------- OpenCV tables
def bilinear_table():
    """OpenCV's INTER_LINEAR fixed-point weight table (initInterTab2D): [32*32][4] uint16 (the weight of an exact pixel hit is
    32768 itself), every row sums to 32768."""
    t = np.arange(32, dtype=np.float32) / np.float32(32)
    c = np.stack([np.float32(1) - t, t], 1).astype(np.float32)
    w = (c[:, None, :, None] * c[None, :, None, :]).astype(np.float32).reshape(32 * 32, 4)      # [fy][fx][(ky, kx)]
    it = np.rint(w * np.float32(32768)).astype(np.int32)
    for row in it:
        diff = int(row.sum()) - 32768
        if diff:
            mk, big = 0, 0
            for k in range(4):
                if row[k] < row[mk]:
                    mk = k
                elif row[k] > row[big]:
                    big = k
            if diff < 0:
                row[big] -= diff
            else:
                row[mk] -= diff
    return it.astype(np.uint16)


def affine_tables(M, h, w):
    """cv2.warpAffine's fixed-point coordinate tables for the forward matrix M [2,3]: adelta[w], bdelta[w], X0[h], Y0[h] (int32)."""
    M = np.array(M, np.float64).reshape(2, 3).copy()
    D = M[0, 0] * M[1, 1] - M[0, 1] * M[1, 0]
    D = 1.0 / D if D != 0 else 0.0
    a11, a22 = M[1, 1] * D, M[0, 0] * D
    M[0, 0] = a11
    M[0, 1] *= -D
    M[1, 0] *= -D
    M[1, 1] = a22
    b1 = -M[0, 0] * M[0, 2] - M[0, 1] * M[1, 2]
    b2 = -M[1, 0] * M[0, 2] - M[1, 1] * M[1, 2]
    M[0, 2], M[1, 2] = b1, b2
    xs, ys = np.arange(w, dtype=np.float64), np.arange(h, dtype=np.float64)
    adelta = np.rint(M[0, 0] * xs * 1024.0)
    bdelta = np.rint(M[1, 0] * xs * 1024.0)
    X0 = np.rint((M[0, 1] * ys + M[0, 2]) * 1024.0) + 16
    Y0 = np.rint((M[1, 1] * ys + M[1, 2]) * 1024.0) + 16
    return adelta.astype(np.int32), bdelta.astype(np.int32), X0.astype(np.int32), Y0.astype(np.int32)


def gaussian_taps_q8(sigma):
    """OpenCV's fixed-point 5-tap Gaussian (8 fractional bits): outer taps rounded with error diffusion, centre = 256 - 2 * (t0 + t1)."""
    x = np.arange(5, dtype=np.float64) - 2.0
    k = np.exp(-x * x / (2.0 * sigma * sigma))
    k /= k.sum()
    kq = np.zeros(5, np.int32)
    err = 0.0
    for i in range(2):
        adj = k[i] * 256.0 + err
        v0 = int(np.rint(adj))
        err = adj - v0
        kq[i] = kq[4 - i] = v0
    kq[2] = 256 - 2 * int(kq[0] + kq[1])
    return kq


def nearest_cells(dst, src):
    ifx = 1.0 / (float(dst) / float(src))
    return np.minimum(np.floor(np.arange(dst, dtype=np.float64) * ifx).astype(np.int64), src - 1).astype(np.uint8)


# CropAndPad (imgaug 0.4.0, the version the reference pins; its source is not available here).  Each rule below is imgaug as
# remembered: UNVERIFIED (DESIGN.md section 2).
CROP_PAD_SIDES = ("top", "right", "bottom", "left")     # draw order of the four sides with sample_independently=True


def crop_pad_pixels(size, value, percent):
    """Pixels of one side from its drawn value: in percent mode np.round(float32(size) * pct) (half to even) as int32; px
    values are used as drawn.  Negative = crop, positive = pad."""
    if not percent:
        return np.asarray(value).astype(np.int32)
    return np.round(np.float32(size) * np.asarray(value, np.float64)).astype(np.int32)


def crop_pad_limit_crops(size, start, end):
    """_prevent_zero_sizes_after_crops_: crops of one axis (start, end >= 0) reduced so that at least one pixel remains; the
    excess is taken back floor-half from the start and ceil-half from the end."""
    start, end = np.array(start, np.int32), np.array(end, np.int32)
    excess = np.maximum(start + end - (size - 1), 0)
    start, end = start - excess // 2, end - (excess - excess // 2)
    return np.maximum(start, 0) + np.minimum(end, 0), np.maximum(end, 0) + np.minimum(start, 0)


def crop_pad_rule(src_h, src_w, dst_h, dst_w):
    """imresize_single_image's default interpolation for keep_size: "cubic" when the target is larger than the source along
    either axis, else "area" (cv2.resize copies an image whose size did not change; area at ratio 1 is that copy)."""
    return "cubic" if dst_h > src_h or dst_w > src_w else "area"


def cubic_taps(dst, src):
    """cv2.resize(INTER_CUBIC) along one axis, uint8: source indices [dst, 4] (clamped to the image) and fixed-point weights
    [dst, 4] with 11 fractional bits (interpolateCubic, A = -0.75, float32 arithmetic, saturate_cast<short>)."""
    f = np.float32
    scale = 1.0 / (float(dst) / float(src))
    fx = ((np.arange(dst, dtype=np.float64) + 0.5) * scale - 0.5).astype(np.float32)
    sx = np.floor(fx).astype(np.int64)
    x = (fx - sx.astype(np.float32)).astype(np.float32)
    A = f(-0.75)
    x1, om = x + f(1), f(1) - x
    c0 = ((A * x1 - f(5) * A) * x1 + f(8) * A) * x1 - f(4) * A
    c1 = ((A + f(2)) * x - (A + f(3))) * x * x + f(1)
    c2 = ((A + f(2)) * om - (A + f(3))) * om * om + f(1)
    c3 = f(1) - c0 - c1 - c2
    w = np.rint(np.stack([c0, c1, c2, c3], 1).astype(np.float32) * f(2048)).astype(np.int32)
    idx = np.clip(sx[:, None] + np.arange(-1, 3)[None, :], 0, src - 1).astype(np.int32)
    return idx, w


def area_taps(dst, src, taps=4):
    """cv2.resize(INTER_AREA) along one axis for src >= dst (computeResizeAreaTab): per destination index the source indices
    and float32 weights in OpenCV's accumulation order, padded to ``taps`` with weight 0 on the last index (adding +0 leaves
    a float sum unchanged).  More taps than ``taps`` raise NotImplementedError."""
    scale = 1.0 / (float(dst) / float(src))
    idx, w = np.zeros((dst, taps), np.int32), np.zeros((dst, taps), np.float32)
    for dx in range(dst):
        f1 = dx * scale
        f2 = f1 + scale
        cell = min(scale, src - f1)
        s1, s2 = int(np.ceil(f1)), int(np.floor(f2))
        s2 = min(s2, src - 1)
        s1 = min(s1, s2)
        row = []
        if s1 - f1 > 1e-3:
            row.append((s1 - 1, np.float32((s1 - f1) / cell)))
        row += [(s, np.float32(1.0 / cell)) for s in range(s1, s2)]
        if f2 - s2 > 1e-3:
            row.append((s2, np.float32(min(min(f2 - s2, 1.0), cell) / cell)))
        if len(row) > taps:
            raise NotImplementedError("CropAndPad: INTER_AREA from %d to %d pixels needs %d taps (%d supported)" % (src, dst, len(row), taps))
        row += [(row[-1][0], np.float32(0))] * (taps - len(row))
        idx[dx], w[dx] = [r[0] for r in row], [r[1] for r in row]
    return idx, w


CROP_PAD_ROWS = 8              # output rows of one crop-pad CTA (csrc/augment.cu)
CROP_PAD_SMEM_LIMIT = 48 * 1024


_IDENT = np.arange(256, dtype=np.uint8)


def _lut_add(v):
    return np.clip(np.arange(256, dtype=np.int16) + int(v), 0, 255).astype(np.uint8)


def _lut_mul(m):
    return np.clip(np.arange(256, dtype=np.float32) * np.float32(m), 0, 255).astype(np.uint8)


def _lut_contrast(a):
    return np.clip(np.float32(127) + np.float32(a) * (np.arange(256, dtype=np.float32) - np.float32(127)), 0, 255).astype(np.uint8)


# ----------------------------------------------------------------------------------------------------------- augmenter
class Augmenter(object):
    def __init__(self, code, shape=(128, 128, 3), seed=None):
        self.h, self.w, self.c = int(shape[0]), int(shape[1]), int(shape[2])
        self.ops = parse_code(code) if isinstance(code, str) else list(code)
        canon = ["CropAndPad", "Affine", "CoarseDropout", "GaussianBlur", "Add", "Invert", "Multiply", "Multiply", "ContrastNormalization"]
        pos = 0
        for _, op in self.ops:                                  # the kernels apply the ops in the template's order
            kind = "ContrastNormalization" if op.kind == "LinearContrast" else op.kind
            while pos < len(canon) and canon[pos] != kind:
                pos += 1
            if pos == len(canon):
                raise NotImplementedError("augmenter order %s is not a sub-sequence of %s" % ([o.kind for _, o in self.ops], canon))
            pos += 1
        self.rng = np.random.RandomState(seed)
        self.sigma = 0.0
        self.low = (1, 1)
        for _, op in self.ops:
            if op.kind == "GaussianBlur":
                self.sigma = float(op.args[0] if op.args else op.kw.get("sigma", 0.0))
                if self.sigma >= 1.5:
                    raise NotImplementedError("GaussianBlur sigma >= 1.5 needs a kernel larger than 5 taps")
            if op.kind == "CoarseDropout":
                sp = float(op.kw.get("size_percent", 0.05))
                self.low = (max(int(self.h * sp), 4), max(int(self.w * sp), 4))     # FromLowerResolution(min_size=4)
                if self.low[0] * self.low[1] > 64:
                    raise NotImplementedError("CoarseDropout masks with more than 64 cells are not supported")
        self.crop = None
        for _, op in self.ops:
            if op.kind == "CropAndPad":
                self.crop = self._crop_pad_setup(op)
        self._dev = {}

    def _crop_pad_setup(self, op):
        """Checks CropAndPad's arguments and builds the resampling tables of every reachable source size: one int32 array of
        [dst][4 indices, 4 weights] blocks (weights int for cubic, float32 bits for area), with the offset of each block."""
        kw = dict(op.kw)
        if op.args:
            raise NotImplementedError("CropAndPad: positional arguments are not supported (use px= or percent=)")
        unknown = set(kw) - {"px", "percent", "pad_mode", "pad_cval", "keep_size", "sample_independently", "name", "deterministic",
                             "random_state"}
        if unknown:
            raise NotImplementedError("CropAndPad: argument %s is not supported" % sorted(unknown)[0])
        if (kw.get("px") is None) == (kw.get("percent") is None):
            raise NotImplementedError("CropAndPad: exactly one of px= and percent= is supported")
        percent = kw.get("percent") is not None
        value = kw["percent"] if percent else kw["px"]
        if isinstance(value, (tuple, list)) and (len(value) != 2 or any(isinstance(v, (tuple, list)) for v in value)):
            raise NotImplementedError("CropAndPad: %s as per-side tuples or lists is not supported (a scalar or one (low, high) range)"
                                      % ("percent" if percent else "px"))
        if kw.get("pad_mode", "constant") != "constant":
            raise NotImplementedError("CropAndPad: pad_mode=%r is not supported (only \"constant\")" % (kw["pad_mode"],))
        if not kw.get("keep_size", True):
            raise NotImplementedError("CropAndPad: keep_size=False is not supported (batch images must keep one shape)")
        cval = kw.get("pad_cval", 0)
        if isinstance(cval, (tuple, list)) and len(cval) != 2:
            raise NotImplementedError("CropAndPad: pad_cval as a list is not supported (a scalar or one (low, high) range)")
        lo, hi = _range(value)
        if not 0 <= _range(cval)[0] <= _range(cval)[1] <= 255:
            raise NotImplementedError("CropAndPad: pad_cval=%r is not a uint8 value or range" % (cval,))
        if not percent and (lo != int(lo) or hi != int(hi)):
            raise NotImplementedError("CropAndPad: px= needs integer pixel counts")
        cz = _range(cval)
        c = dict(percent=percent, lo=lo, hi=hi, cval=(int(cz[0]), int(cz[1])), independent=bool(kw.get("sample_independently", True)))
        # reachable source sizes per axis: every side between its smallest and its largest pixel count
        sizes = {}
        for axis, n in (("y", self.h), ("x", self.w)):
            a, b = (int(crop_pad_pixels(n, v, percent)) for v in (lo, hi))
            sizes[axis] = range(max(1, n + 2 * a), n + 2 * b + 1)
        blocks, off, rows = [], {}, 1
        pos = 0
        for axis, dst in (("y", self.h), ("x", self.w)):
            for n in sizes[axis]:
                if n > dst and n % dst == 0:
                    raise NotImplementedError("CropAndPad: %d -> %d pixels is an integer ratio, which cv2.resize's INTER_AREA takes "
                                              "through its separate fast path (not supported)" % (n, dst))
                kinds = [("cubic", cubic_taps(dst, n))] + ([("area", area_taps(dst, n))] if n >= dst else [])
                for kind, (idx, w) in kinds:
                    blk = np.concatenate([idx, w.view(np.int32) if w.dtype == np.float32 else w], 1).astype(np.int32)
                    off[(axis, kind, n)] = pos
                    blocks.append(blk.ravel())
                    pos += blk.size
                    if axis == "y":
                        first, last = idx[::CROP_PAD_ROWS, 0], idx[np.minimum(np.arange(CROP_PAD_ROWS - 1, dst + CROP_PAD_ROWS - 1,
                                                                                         CROP_PAD_ROWS), dst - 1), 3]
                        rows = max(rows, int((last - first).max()) + 1)
        c.update(sizes=sizes, table=np.concatenate(blocks), offsets=off, max_rows=rows, max_w=sizes["x"][-1])
        smem = rows * c["max_w"] * self.c
        if smem > CROP_PAD_SMEM_LIMIT:
            raise NotImplementedError("CropAndPad: source rows of %d x %d x %d bytes per CTA exceed the %d bytes of shared memory "
                                      "the crop-pad kernel uses" % (rows, c["max_w"], self.c, CROP_PAD_SMEM_LIMIT))
        return c

    # -- host: random draws (imgaug's distributions; numpy's stream) -------------------------------------------------
    def sample(self, B):
        """Per-image parameters of one batch: dict of arrays (``*_on`` = the Sometimes draw, values per image / channel)."""
        r, C_ = self.rng, self.c
        P = {"affine_on": np.zeros(B, bool), "affine_M": np.tile(np.array([[1.0, 0, 0], [0, 1.0, 0]]), (B, 1, 1)),
             "drop_on": np.zeros(B, bool), "drop_keep": np.ones((B,) + self.low, np.uint8), "blur_on": np.zeros(B, bool),
             "add_on": np.zeros(B, bool), "add_val": np.zeros((B, C_), np.int32), "invert_on": np.zeros(B, bool),
             "invert_ch": np.zeros((B, C_), bool), "mul1_on": np.zeros(B, bool), "mul1_val": np.ones((B, C_), np.float32),
             "mul2_on": np.zeros(B, bool), "mul2_val": np.ones((B, C_), np.float32), "contrast_on": np.zeros(B, bool),
             "contrast_val": np.ones((B, C_), np.float32)}
        n_mul = 0

        def per_channel(pc, draw):
            """value per channel: with probability pc (True = 1, False = 0) independent draws, else one draw repeated"""
            v = draw((B, C_))
            same = r.rand(B) >= float(pc)
            v[same] = v[same][:, :1]
            return v

        for p, op in self.ops:
            on = r.rand(B) < p
            if op.kind == "CropAndPad":
                c = self.crop
                if c["percent"]:
                    draw = lambda sz: r.uniform(c["lo"], c["hi"], sz)      # noqa: E731
                else:
                    draw = lambda sz: r.randint(int(c["lo"]), int(c["hi"]) + 1, sz)      # noqa: E731
                v = draw((B, 4)) if c["independent"] else np.repeat(draw(B)[:, None], 4, 1)
                px = np.stack([crop_pad_pixels(self.h if k % 2 == 0 else self.w, v[:, k], c["percent"]) for k in range(4)], 1)
                for a, b, n in ((0, 2, self.h), (3, 1, self.w)):
                    cs, ce = crop_pad_limit_crops(n, np.maximum(-px[:, a], 0), np.maximum(-px[:, b], 0))
                    px[:, a], px[:, b] = np.where(px[:, a] < 0, -cs, px[:, a]), np.where(px[:, b] < 0, -ce, px[:, b])
                P["crop_on"], P["crop_px"] = on, px.astype(np.int32)
                lo, hi = c["cval"]
                P["crop_cval"] = np.full(B, lo, np.int32) if lo == hi else r.randint(lo, hi + 1, B).astype(np.int32)
            elif op.kind == "Affine":
                lo, hi = _range(op.kw.get("scale", 1.0))
                s = r.uniform(lo, hi, B)
                cx, cy = self.w / 2.0 - 0.5, self.h / 2.0 - 0.5
                P["affine_on"] = on
                for b in range(B):
                    P["affine_M"][b] = [[s[b], 0.0, cx - s[b] * cx], [0.0, s[b], cy - s[b] * cy]]
            elif op.kind == "CoarseDropout":
                P["drop_on"] = on
                P["drop_keep"] = (r.rand(B, *self.low) >= float(op.kw.get("p", op.args[0] if op.args else 0.0))).astype(np.uint8)
            elif op.kind == "GaussianBlur":
                P["blur_on"] = on
            elif op.kind == "Add":
                lo, hi = _range(op.args[0] if op.args else op.kw.get("value", 0))
                P["add_on"] = on
                P["add_val"] = per_channel(op.kw.get("per_channel", False), lambda sz: r.randint(int(lo), int(hi) + 1, sz)).astype(np.int32)
            elif op.kind == "Invert":
                P["invert_on"] = on
                pi = float(op.args[0] if op.args else op.kw.get("p", 0.0))
                P["invert_ch"] = per_channel(op.kw.get("per_channel", False), lambda sz: (r.rand(*sz) < pi)).astype(bool)
            elif op.kind == "Multiply":
                lo, hi = _range(op.args[0] if op.args else op.kw.get("mul", 1.0))
                key = "mul1" if n_mul == 0 else "mul2"
                if n_mul > 1:
                    raise NotImplementedError("more than two Multiply stages")
                n_mul += 1
                P[key + "_on"] = on
                P[key + "_val"] = per_channel(op.kw.get("per_channel", False), lambda sz: r.uniform(lo, hi, sz)).astype(np.float32)
            else:  # ContrastNormalization / LinearContrast
                lo, hi = _range(op.args[0] if op.args else op.kw.get("alpha", 1.0))
                P["contrast_on"] = on
                P["contrast_val"] = per_channel(op.kw.get("per_channel", False), lambda sz: r.uniform(lo, hi, sz)).astype(np.float32)
        return P

    # -- host: pack the draws into the two device buffers ------------------------------------------------------------
    def pack(self, P):
        """-> geom int32 [B, 4 + 2W + 2H], lut uint8 [B, C, 256] (include/aae_b200.h: aae_augment_args); vectorised over the batch."""
        B = len(P["affine_on"])
        H, W, C_ = self.h, self.w, self.c
        geom = np.zeros((B, 4 + 2 * W + 2 * H), np.int32)
        blur = bool(self.sigma > 1e-3)
        geom[:, 0] = (P["affine_on"].astype(np.int32) * FLAG_AFFINE) | (P["drop_on"].astype(np.int32) * FLAG_DROP) | \
                     ((P["blur_on"] & blur).astype(np.int32) * FLAG_BLUR)
        if "crop_on" in P:
            geom[:, 0] |= P["crop_on"].astype(np.int32) * FLAG_CROP
        weights = (np.uint64(1) << np.arange(self.low[0] * self.low[1], dtype=np.uint64))
        keep = (P["drop_keep"].reshape(B, -1).astype(np.uint64) * weights[None, :]).sum(1, dtype=np.uint64)
        geom[:, 1] = (keep & np.uint64(0xFFFFFFFF)).astype(np.uint32).view(np.int32)
        geom[:, 2] = (keep >> np.uint64(32)).astype(np.uint32).view(np.int32)
        on = np.nonzero(P["affine_on"])[0]
        if len(on):
            # cv2.warpAffine: invert the forward matrix in double, then 10-bit fixed-point column / row tables (affine_tables, batched)
            M = np.array(P["affine_M"][on], np.float64)
            D = M[:, 0, 0] * M[:, 1, 1] - M[:, 0, 1] * M[:, 1, 0]
            D = np.where(D != 0, 1.0 / np.where(D != 0, D, 1.0), 0.0)
            a11, a22 = M[:, 1, 1] * D, M[:, 0, 0] * D
            m01, m10 = M[:, 0, 1] * -D, M[:, 1, 0] * -D
            b1 = -a11 * M[:, 0, 2] - m01 * M[:, 1, 2]
            b2 = -m10 * M[:, 0, 2] - a22 * M[:, 1, 2]
            xs, ys = np.arange(W, dtype=np.float64)[None, :], np.arange(H, dtype=np.float64)[None, :]
            geom[on, 4:4 + W] = np.rint(a11[:, None] * xs * 1024.0).astype(np.int32)
            geom[on, 4 + W:4 + 2 * W] = np.rint(m10[:, None] * xs * 1024.0).astype(np.int32)
            geom[on, 4 + 2 * W:4 + 2 * W + H] = (np.rint((m01[:, None] * ys + b1[:, None]) * 1024.0) + 16).astype(np.int32)
            geom[on, 4 + 2 * W + H:] = (np.rint((a22[:, None] * ys + b2[:, None]) * 1024.0) + 16).astype(np.int32)
        # value ops: one uint8 -> uint8 table per (image, channel) = the op chain evaluated on the 256 possible values, every op
        # with the arithmetic of its imgaug uint8 table (integer add + clip; float32 multiply, clip, truncate)
        t = np.broadcast_to(np.arange(256, dtype=np.int32)[None, None, :], (B, C_, 256))
        f127 = np.float32(127)

        def sel(on_b, new):
            m = on_b[:, None, None] if on_b.ndim == 1 else on_b[:, :, None]
            return np.where(m, new, t)

        if P["add_on"].any():
            t = sel(P["add_on"], np.clip(t + P["add_val"].astype(np.int32)[:, :, None], 0, 255))
        inv = P["invert_on"][:, None] & P["invert_ch"]
        if inv.any():
            t = sel(inv, 255 - t)
        for key in ("mul1", "mul2"):
            if P[key + "_on"].any():
                t = sel(P[key + "_on"], np.clip(t.astype(np.float32) * P[key + "_val"].astype(np.float32)[:, :, None], 0, 255).astype(np.uint8).astype(np.int32))
        if P["contrast_on"].any():
            c = f127 + P["contrast_val"].astype(np.float32)[:, :, None] * (t.astype(np.float32) - f127)
            t = sel(P["contrast_on"], np.clip(c, 0, 255).astype(np.uint8).astype(np.int32))
        # t may still be the stride-0 broadcast view (no value op fired): astype would keep a permuted memory order, and the
        # kernel reads raw [B][C][256] memory
        return np.ascontiguousarray(geom), np.ascontiguousarray(t, dtype=np.uint8)

    def pack_crop(self, P):
        """-> the CropAndPad table int32 [B, 8] (include/aae_b200.h: aae_augment): mode (0 off, 1 cubic, 2 area),
        source height and width after crop and pad, signed top and left pixels, pad value, offsets of the row and column
        resampling blocks in the Augmenter's table.  None for a chain without CropAndPad."""
        if self.crop is None:
            return None
        B, H, W = len(P["crop_on"]), self.h, self.w
        t = np.zeros((B, 8), np.int32)
        off = self.crop["offsets"]
        px = P["crop_px"]
        for b in np.nonzero(P["crop_on"])[0]:
            top, right, bottom, left = (int(v) for v in px[b])
            sh, sw = H + top + bottom, W + left + right
            kind = crop_pad_rule(sh, sw, H, W)
            t[b] = (1 if kind == "cubic" else 2, sh, sw, top, left, P["crop_cval"][b], off[("y", kind, sh)], off[("x", kind, sw)])
        return t

    # -- device ------------------------------------------------------------------------------------------------------
    def _constants(self, dev):
        key = str(dev)
        if key not in self._dev:
            k = self._dev[key] = {
                "tab": torch.from_numpy(bilinear_table().view(np.int16)).to(dev),     # raw 16-bit patterns (torch has no uint16 arithmetic)
                "rows": torch.from_numpy(nearest_cells(self.h, self.low[0])).to(dev),
                "cols": torch.from_numpy(nearest_cells(self.w, self.low[1])).to(dev),
                "to_float": torch.from_numpy((np.arange(256) / 255.).astype(np.float32)).to(dev),     # batch_x / 255. then the float32 feed
                "taps": gaussian_taps_q8(self.sigma).astype(np.int32) if self.sigma > 1e-3 else None,
                # the target's float32 y / 255. as torch computes it (Dataset.batch_device), for the indexed call's y output
                "y_to_float": torch.arange(256, dtype=torch.int32, device=dev).to(torch.uint8).to(torch.float32) / 255.0,
                # CropAndPad's resampling blocks of every reachable source size, built once per Augmenter
                "resample": torch.from_numpy(self.crop["table"]).to(dev) if self.crop is not None else None,
            }
            # the fields of aae_augment_args that stay the same from batch to batch; the tensors above keep them alive
            k["args"] = _lib.AugmentArgs(h=self.h, w=self.w, c=self.c, low_w=self.low[1], bilinear_tab=k["tab"], row_cell=k["rows"],
                                         col_cell=k["cols"], blur_kernel_q8=k["taps"], u8_to_float=k["to_float"],
                                         y_to_float=k["y_to_float"])
            if self.crop is not None:
                k["args"].set(resample=k["resample"], resample_len=int(k["resample"].numel()), max_src_rows=self.crop["max_rows"],
                              max_src_w=self.crop["max_w"])
            torch.cuda.current_stream(dev).synchronize()    # usable from any stream (the batch producer's) from here on
        return self._dev[key]

    def _launch(self, dev, stream, what, **batch):
        """aae_augment on ``stream`` with the device's constant fields and this batch's (``batch``: field -> tensor or value)."""
        a = self._constants(dev)["args"].copy().set(**batch)
        _lib.check(_lib.lib().aae_augment(C.byref(a), C.c_void_p(stream.cuda_stream)), what)

    def augment_device(self, x, mask, bg, params=None, want_u8=False):
        """x, bg: uint8 CUDA tensors [B,H,W,C]; mask: bool/uint8 CUDA tensor [B,H,W] (True = background).  Returns the float32
        batch in [0, 1] the training step consumes (and the uint8 image when want_u8)."""
        dev = x.device
        B = x.shape[0]
        P = params if params is not None else self.sample(B)
        geom, lut = self.pack(P)
        geom, lut = np.ascontiguousarray(geom, dtype=np.int32), np.ascontiguousarray(lut, dtype=np.uint8)
        if geom.shape != (B, 4 + 2 * self.w + 2 * self.h) or lut.shape != (B, self.c, 256):
            raise ValueError("augmentation tables have shapes %s / %s for a batch of %d" % (geom.shape, lut.shape, B))
        geom_d, lut_d = torch.from_numpy(geom).to(dev, non_blocking=True), torch.from_numpy(lut).to(dev, non_blocking=True)
        assert geom_d.is_contiguous() and lut_d.is_contiguous()
        x, bg, mask8 = x.contiguous(), bg.contiguous(), mask.to(torch.uint8).contiguous()
        out_f = torch.empty(x.shape, dtype=torch.float32, device=dev)
        out_u = torch.empty_like(x) if want_u8 else None
        crop = {}
        if self.crop is not None:
            crop = dict(crop=torch.from_numpy(self.pack_crop(P)).to(dev, non_blocking=True), crop_tmp=torch.empty_like(x))
        self._launch(dev, torch.cuda.current_stream(dev), "augment batch", batch=B, x=x, mask=mask8, bg=bg, geom=geom_d, lut=lut_d,
                     tmp=torch.empty_like(x), out_u8=out_u, out_f32=out_f, **crop)
        return (out_f, out_u) if want_u8 else out_f

    def augment_indexed(self, stacks, idx_d, idx_bg_d, geom_d, lut_d, out_f, y_out, stream, mask_batch=None, tmp=None, crop_d=None,
                        crop_tmp=None):
        """``augment_device`` on device-resident stacks (``aae_augment`` with idx / idx_bg): image b is row idx_d[b] of stacks["x"]
        / ["mask"] / ["y"] and row idx_bg_d[b] of stacks["bg"]; mask_batch (uint8 [B,H,W], e.g. an occlusion output) replaces the
        mask rows.  Writes the float32 input into out_f and the target y / 255. into y_out; geom_d / lut_d are ``pack``'s tables on
        the device; tmp (uint8 [B,H,W,C]) is the scratch of the geometry pass, allocated here when None.  With CropAndPad in the
        chain crop_d is ``pack_crop``'s table on the device and crop_tmp (uint8 [B,H,W,C], allocated here when None) the
        crop-pad output.  Asynchronous on ``stream``."""
        dev = out_f.device
        B = int(out_f.shape[0])
        shape = (B, self.h, self.w, self.c)
        if tmp is None:
            tmp = torch.empty(shape, dtype=torch.uint8, device=dev)
        crop = {}
        if self.crop is not None:
            if crop_d is None:
                raise ValueError("a chain with CropAndPad needs pack_crop's table (crop_d)")
            crop = dict(crop=crop_d, crop_tmp=crop_tmp if crop_tmp is not None else torch.empty(shape, dtype=torch.uint8, device=dev))
        self._launch(dev, stream, "augment batch (indexed)", batch=B, x=stacks["x"], mask=stacks["mask"], bg=stacks["bg"],
                     y=stacks["y"], idx=idx_d, idx_bg=idx_bg_d, n_images=len(stacks["x"]), n_bg=len(stacks["bg"]),
                     mask_batch=mask_batch, geom=geom_d, lut=lut_d, tmp=tmp, out_f32=out_f, y_out=y_out, **crop)


# ----------------------------------------------------------------------------------------------------------- occlusion
OCCLUSION_BANK_SIDE = 224                  # arbitrary_syn_masks_1000.bin: raw bits of 224 x 224 masks (dataset.py:405-418)
OCCLUSION_MIN_TRANS, OCCLUSION_MAX_TRANS = 0.2, 0.7      # augment_occlusion_mask's defaults (dataset.py:421)
SQUARE_P_ON, SQUARE_P_DROP, SQUARE_SIZE_PERCENT = 0.7, 0.4, 0.01    # Sometimes(0.7, CoarseDropout(p=0.4, size_percent=0.01))
# Cells per side of the square-occlusion dropout grid: max(int(side * 0.01), min_size) = min_size at 128.  min_size is a default
# of imgaug 0.4.0's CoarseDropout (the version the reference pins), whose source is not available here: 3 is that default as
# remembered (imgaug 0.2.x used 4).  UNVERIFIED.
SQUARE_OCCLUSION_MIN_SIZE = 3
# Candidates per image and step.  Taking the first accepted one in draw order is the reference's unbounded rejection loop
# conditioned on success within K.  An image whose draws pass with probability p falls back with probability (1 - p)^K:
# 1.2e-3 at p = 0.1, 6e-7 at p = 0.2.  The kernel stops at the first round of 8 candidates with an accept, so a larger K costs
# device time only on images that keep failing; on the host it costs 14 draws and 12 bytes of upload per candidate.
OCCLUSION_CANDIDATES = 64


def occlusion_limit(value):
    """``max_occl`` of an occlusion switch read as the reference reads it (dataset.py:468-471): the cfg string evaluated,
    as a float; ``False`` / ``0`` (or a missing key) = off."""
    if value is None:
        return 0.0
    return float(eval(str(value), {"__builtins__": {}}))


def square_grid(h, w):
    """Cells (rows, cols) of the square-occlusion dropout grid (imgaug's FromLowerResolution(size_percent, min_size))."""
    return max(int(h * SQUARE_SIZE_PERCENT), SQUARE_OCCLUSION_MIN_SIZE), max(int(w * SQUARE_SIZE_PERCENT), SQUARE_OCCLUSION_MIN_SIZE)


def load_occlusion_bank(path, shape):
    """The occluder bank of ``Dataset.random_syn_masks`` (dataset.py:405-418) bit-packed: uint32 [n, rows, cols / 32] with bit
    j of word w = column 32 w + j, as ``aae_occlusion`` reads it.  The reference unpacks the file with bitarray (default
    big-endian bit order, the order of np.unpackbits), reshapes to 224 x 224 masks and resizes each one with
    cv2.resize(mask, (shape[0], shape[1]), INTER_NEAREST) -- dsize is (width, height), so the result has shape[1] rows."""
    bits = np.unpackbits(np.fromfile(path, dtype=np.uint8))
    side = OCCLUSION_BANK_SIDE
    if bits.size == 0 or bits.size % (side * side):
        raise ValueError("%s holds %d bits, not a whole number of %d x %d masks" % (path, bits.size, side, side))
    rows, cols = int(shape[1]), int(shape[0])
    if cols % 32:
        raise NotImplementedError("occlusion masks %d pixels wide: the device step packs rows into 32-bit words" % cols)
    masks = bits.reshape(-1, side, side)
    masks = masks[:, nearest_cells(rows, side)][:, :, nearest_cells(cols, side)]
    return np.ascontiguousarray(np.packbits(masks, axis=-1, bitorder="little")).view("<u4").astype(np.uint32)


class Occlusion(object):
    """REALISTIC_OCCLUSION and SQUARE_OCCLUSION of Dataset.batch (dataset.py:468-471) on the device.  ``realistic`` / ``square``
    are the switches' ``max_occl`` (0 = off).  Draws come from a RandomState of their own, so the other streams of a batch are
    the same whether the switches are on or off."""

    def __init__(self, shape, realistic=0.0, square=0.0, seed=None, candidates=OCCLUSION_CANDIDATES):
        self.h, self.w = int(shape[0]), int(shape[1])
        if self.h != self.w:
            raise NotImplementedError("occlusion augmentation needs square crops (the reference mixes the two axes)")
        if self.w % 32:
            raise NotImplementedError("occlusion augmentation needs a crop width that is a multiple of 32")
        self.realistic, self.square = float(realistic), float(square)
        self.K = int(candidates)
        self.low = square_grid(self.h, self.w)
        if self.low[0] * self.low[1] > 32:
            raise NotImplementedError("square occlusion grids of more than 32 cells are not supported")
        self.rng = np.random.RandomState(None if seed is None else [int(seed), 1])     # not the Augmenter's RandomState(seed)
        self._dev = {}

    # -- host: random draws ------------------------------------------------------------------------------------------
    def sample(self, B, n_bank=0):
        """Candidates of one batch: occluder index [B] and shifts tx, ty [B, K] (realistic), Sometimes flags [B, K] and keep
        cells [B, K, rows, cols] (square), in the reference's distributions (dataset.py:424-430, 392-402)."""
        r, K, P = self.rng, self.K, {}
        if self.realistic:
            P["occluder"] = r.choice(n_bank, B)
            sx, ux, sy, uy = r.choice((-1, 1), (B, K)), r.rand(B, K), r.choice((-1, 1), (B, K)), r.rand(B, K)
            span = OCCLUSION_MAX_TRANS - OCCLUSION_MIN_TRANS
            P["tx"] = np.trunc(sx * (ux * span + OCCLUSION_MIN_TRANS) * self.h).astype(np.int32)     # int(): toward zero
            P["ty"] = np.trunc(sy * (uy * span + OCCLUSION_MIN_TRANS) * self.w).astype(np.int32)
        if self.square:
            P["square_on"] = r.rand(B, K) < SQUARE_P_ON
            P["square_keep"] = r.rand(B, K, *self.low) >= SQUARE_P_DROP
        return P

    def pack(self, P):
        """-> int32 [B, 1 + 3K]: occluder, tx[K], ty[K], keep bits[K] (include/aae_b200.h: aae_occlusion)."""
        K = self.K
        cells = self.low[0] * self.low[1]
        B = len(P["occluder"]) if "occluder" in P else len(P["square_on"])
        cand = np.zeros((B, 1 + 3 * K), np.int32)
        full = np.uint32((1 << cells) - 1)
        keep = np.full((B, K), full, np.uint32)
        if self.realistic:
            cand[:, 0] = P["occluder"]
            cand[:, 1:K + 1] = P["tx"]
            cand[:, K + 1:2 * K + 1] = P["ty"]
        if self.square:
            weights = np.uint64(1) << np.arange(cells, dtype=np.uint64)
            bits = (P["square_keep"].reshape(B, K, cells).astype(np.uint64) * weights).sum(-1, dtype=np.uint64).astype(np.uint32)
            keep = np.where(P["square_on"], bits, full)
        cand[:, 2 * K + 1:] = keep.view(np.int32)
        return cand

    # -- device ------------------------------------------------------------------------------------------------------
    def _state(self, dev):
        key = str(dev)
        if key not in self._dev:
            st = self._dev[key] = {
                "rows": torch.from_numpy(nearest_cells(self.h, self.low[0])).to(dev),
                "cols": torch.from_numpy(nearest_cells(self.w, self.low[1])).to(dev),
                "fallbacks": torch.zeros(2, dtype=torch.int32, device=dev),
                "bank_src": None, "bank": None,
            }
            # the fields of aae_occlusion_args that stay the same from batch to batch
            st["args"] = _lib.OcclusionArgs(h=self.h, w=self.w, realistic=int(self.realistic != 0), max_occl=self.realistic,
                                            square=int(self.square != 0), min_kept=1.0 - self.square,      # dataset.py:451: 1-max_occl
                                            n_cand=self.K, row_cell=st["rows"], col_cell=st["cols"], low_h=self.low[0],
                                            low_w=self.low[1], fallbacks=st["fallbacks"])
            torch.cuda.current_stream(dev).synchronize()    # usable from any stream (the batch producer's) from here on
        return self._dev[key]

    def _bank(self, st, dev, bank):
        if bank is None or bank.ndim != 3 or bank.shape[1:] != (self.h, self.w // 32):
            raise ValueError("realistic occlusion needs an occluder bank of [n, %d, %d] words" % (self.h, self.w // 32))
        if st["bank_src"] is not bank:                  # one upload per device and bank
            st["bank"], st["bank_src"] = torch.from_numpy(np.ascontiguousarray(bank, np.uint32).view(np.int32)).to(dev), bank
        return st["bank"]

    def _launch(self, st, stream, what, **batch):
        """aae_occlusion on ``stream`` with the device's constant fields, its bank, and this batch's (field -> tensor or value)."""
        bank_d = st["bank"] if self.realistic else None
        a = st["args"].copy().set(bank=bank_d, n_bank=len(bank_d) if bank_d is not None else 0, **batch)
        _lib.check(_lib.lib().aae_occlusion(C.byref(a), C.c_void_p(stream.cuda_stream)), what)

    def apply_device(self, mask, bank=None, params=None):
        """mask: bool / uint8 CUDA tensor [B,H,W] (True = background); bank: ``load_occlusion_bank`` array (realistic step).
        Returns the occluded uint8 mask [B,H,W] (1 = background).  Asynchronous; ``fallbacks()`` reads the counters."""
        dev = mask.device
        B = int(mask.shape[0])
        if tuple(mask.shape) != (B, self.h, self.w):
            raise ValueError("occlusion: mask of shape %s, expected [B, %d, %d]" % (tuple(mask.shape), self.h, self.w))
        st = self._state(dev)
        if self.realistic:
            self._bank(st, dev, bank)
        P = params if params is not None else self.sample(B, len(bank) if bank is not None else 0)
        cand = torch.from_numpy(self.pack(P)).to(dev, non_blocking=True)
        mask8 = mask.to(torch.uint8).contiguous()
        out = torch.empty_like(mask8)
        self._launch(st, torch.cuda.current_stream(dev), "augment occlusion", batch=B, mask=mask8, cand=cand, mask_out=out)
        return out

    def apply_indexed(self, mask_stack, idx_d, cand_d, bank, out, stream):
        """``apply_device`` on the masks mask_stack[idx_d[b]] of a device-resident stack (``aae_occlusion`` with idx): cand_d is
        ``pack``'s candidate table on the device, out the uint8 [B,H,W] result.  Asynchronous on ``stream``; counts into the same
        fallback counters."""
        st = self._state(out.device)
        if self.realistic:
            self._bank(st, out.device, bank)
        self._launch(st, stream, "augment occlusion (indexed)", batch=int(out.shape[0]), mask=mask_stack, idx=idx_d,
                     n_images=len(mask_stack), cand=cand_d, mask_out=out)

    def fallbacks(self):
        """Images that exhausted their K candidates since the last call, per step: {"realistic": n, "square": n}.  Clears the
        counters; synchronises the devices that ran the step."""
        n = np.zeros(2, np.int64)
        for key, st in self._dev.items():
            torch.cuda.synchronize(torch.device(key))
            n += st["fallbacks"].cpu().numpy()
            st["fallbacks"].zero_()
        return {"realistic": int(n[0]), "square": int(n[1])}
