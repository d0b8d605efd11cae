"""CPU restatement of CropAndPad (imgaug 0.4.0, keep_size=True) and of the two cv2.resize paths it resizes back with, for the
tests: INTER_CUBIC and INTER_AREA on uint8 images, written after OpenCV's resizeGeneric / resizeArea loops rather than after
the product's vectorised tables (augmentedautoencoder_b200/ae/augment.py), so the tests compare two restatements.

Pinned to the cv2 the tests import, with its IPP dispatch off (``cv2.ipp.setUseIPP(False)``): with IPP on, OpenCV hands
INTER_CUBIC to IPP, whose arithmetic differs (DESIGN.md section 2).  The vertical cubic sum is float32 in the order of
OpenCV's SIMD path (VResizeCubicVec_32s8u), which is what the library computes at every row width the pipeline uses; its
scalar fallback would compute (sum + 2^21) >> 22 in integers instead.

``augment_batch`` extends oracle.augment_oracle.augment_batch: the paste, then CropAndPad on the images whose ``crop_on``
fired, then the rest of the chain exactly as there."""
import numpy as np

from augmentedautoencoder_b200.ae import augment as A
from oracle import augment_oracle as AO

F = np.float32


def _cubic_coeffs(fx):
    """interpolateCubic (A = -0.75) in float32, then saturate_cast<short>(c * 2048)"""
    A_ = F(-0.75)
    x = F(fx)
    c0 = ((A_ * (x + F(1)) - F(5) * A_) * (x + F(1)) + F(8) * A_) * (x + F(1)) - F(4) * A_
    c1 = ((A_ + F(2)) * x - (A_ + F(3))) * x * x + F(1)
    c2 = ((A_ + F(2)) * (F(1) - x) - (A_ + F(3))) * (F(1) - x) * (F(1) - x) + F(1)
    c3 = F(1) - c0 - c1 - c2
    return [int(np.rint(F(c) * F(2048))) for c in (c0, c1, c2, c3)]


def _cubic_axis(dst, src):
    """per destination index: (sx, [4 int weights]) with sx the first of the four clamped source indices"""
    scale = 1.0 / (float(dst) / float(src))
    out = []
    for d in range(dst):
        fx = F((d + 0.5) * scale - 0.5)
        sx = int(np.floor(fx))
        out.append(([min(max(sx - 1 + k, 0), src - 1) for k in range(4)], _cubic_coeffs(fx - F(sx))))
    return out


def resize_cubic_u8(img, h, w):
    """cv2.resize(img, (w, h), interpolation=INTER_CUBIC) for uint8 [sh, sw, C]: integer horizontal pass, float32 vertical pass."""
    sh, sw, C = img.shape
    xs, ys = _cubic_axis(w, sw), _cubic_axis(h, sh)
    p = img.astype(np.int64)
    hrow = np.zeros((sh, w, C), np.int64)
    for d, (idx, wt) in enumerate(xs):
        hrow[:, d] = sum(p[:, idx[k]] * wt[k] for k in range(4))
    out = np.zeros((h, w, C), np.uint8)
    for d, (idx, wt) in enumerate(ys):
        b = [F(F(v) * F(1.0 / (2048 * 2048))) for v in wt]
        s = [hrow[idx[k]].astype(np.float32) for k in range(4)]
        v = s[0] * b[0] + (s[1] * b[1] + (s[2] * b[2] + s[3] * b[3]))
        out[d] = np.clip(np.rint(v), 0, 255).astype(np.uint8)
    return out


def _area_tab(ssize, dsize):
    """computeResizeAreaTab: [(dst index, src index, float32 weight)] in OpenCV's order"""
    scale = 1.0 / (float(dsize) / float(ssize))
    tab = []
    for dx in range(dsize):
        fsx1 = dx * scale
        fsx2 = fsx1 + scale
        cell = min(scale, ssize - fsx1)
        sx1, sx2 = int(np.ceil(fsx1)), int(np.floor(fsx2))
        sx2 = min(sx2, ssize - 1)
        sx1 = min(sx1, sx2)
        if sx1 - fsx1 > 1e-3:
            tab.append((dx, sx1 - 1, F((sx1 - fsx1) / cell)))
        for sx in range(sx1, sx2):
            tab.append((dx, sx, F(1.0 / cell)))
        if fsx2 - sx2 > 1e-3:
            tab.append((dx, sx2, F(min(min(fsx2 - sx2, 1.0), cell) / cell)))
    return tab


def resize_area_u8(img, h, w):
    """cv2.resize(img, (w, h), interpolation=INTER_AREA) for uint8 [sh, sw, C] with sh >= h, sw >= w and a non-integer ratio
    (ResizeArea_Invoker): per source row a float32 horizontal buffer, summed into the destination row in table order.  The
    integer-ratio fast path (ResizeAreaFast) is not restated: the Augmenter refuses a CropAndPad that could reach it."""
    sh, sw, C = img.shape
    xt, yt = _area_tab(sw, w), _area_tab(sh, h)
    s = img.astype(np.float32)
    bufs = np.zeros((sh, w, C), np.float32)            # the horizontal buffer of every source row (each row on its own)
    for dx, sx, a in xt:
        bufs[:, dx] = bufs[:, dx] + s[:, sx] * a
    out = np.zeros((h, w, C), np.uint8)
    acc = np.zeros((w, C), np.float32)
    prev = yt[0][0]
    for dy, sy, beta in yt:
        buf = bufs[sy]
        if dy != prev:
            out[prev] = np.clip(np.rint(acc), 0, 255).astype(np.uint8)
            acc = beta * buf
            prev = dy
        else:
            acc = acc + beta * buf
    out[prev] = np.clip(np.rint(acc), 0, 255).astype(np.uint8)
    return out


def crop_and_pad_u8(img, px, cval):
    """Crop (negative) and pad (positive, constant cval) the sides px = (top, right, bottom, left) of uint8 [H, W, C]."""
    top, right, bottom, left = (int(v) for v in px)
    H, W = img.shape[:2]
    out = img[max(-top, 0):H - max(-bottom, 0), max(-left, 0):W - max(-right, 0)]
    return np.pad(out, ((max(top, 0), max(bottom, 0)), (max(left, 0), max(right, 0)), (0, 0)), constant_values=int(cval))


def resize_back(img, h, w):
    """imresize_single_image at keep_size: a copy at the same size, else cubic or area by ``augment.crop_pad_rule``."""
    sh, sw = img.shape[:2]
    if (sh, sw) == (h, w):
        return img.copy()
    return resize_cubic_u8(img, h, w) if A.crop_pad_rule(sh, sw, h, w) == "cubic" else resize_area_u8(img, h, w)


def augment_batch(x, mask, bg, params, sigma, low=(6, 6)):
    """oracle.augment_oracle.augment_batch with CropAndPad first whenever the params carry it."""
    if "crop_on" not in params:
        return AO.augment_batch(x, mask, bg, params, sigma, low=low)
    B, H, W, C = x.shape
    pasted = np.where(mask[..., None], bg, x)
    for b in np.nonzero(params["crop_on"])[0]:
        pasted[b] = resize_back(crop_and_pad_u8(pasted[b], params["crop_px"][b], params["crop_cval"][b]), H, W)
    return AO.augment_batch(pasted, np.zeros(mask.shape, bool), pasted, params, sigma, low=low)
