"""CropAndPad in the training input pipeline, host side: the cv2.resize restatements are pinned to the installed OpenCV (its own
arithmetic, IPP dispatch off), the product's resampling tables agree with them, and the cfg is parsed, checked and sampled as
imgaug 0.4.0's CropAndPad (augment.py's named rules, UNVERIFIED).  No GPU needed."""
import hashlib

import numpy as np
import pytest

from augmentedautoencoder_b200.ae import augment as A
from tests import crop_pad_oracle as CP
from tests.test_augment_cpu import TEMPLATE_CODE

cv2 = pytest.importorskip("cv2")

CROP_LINE = "    Sometimes(0.5, CropAndPad(percent=(-0.05, 0.1))),\n"
CROP_CODE = TEMPLATE_CODE.replace("Sequential([\n", "Sequential([\n" + CROP_LINE)
GEOMETRIES = {"template": (128, 128, 3), "gray": (128, 128, 1), "px64": (64, 64, 3), "rect": (64, 128, 3)}


@pytest.fixture(autouse=True)
def _opencv_without_ipp():
    was = cv2.ipp.useIPP()
    cv2.ipp.setUseIPP(False)
    yield
    cv2.ipp.setUseIPP(was)


def _cv2_resize(img, h, w, kind):
    out = cv2.resize(img, (w, h), interpolation=cv2.INTER_CUBIC if kind == "cubic" else cv2.INTER_AREA)
    return out.reshape(h, w, img.shape[2])


def _reachable(shape):
    aug = A.Augmenter("Sequential([CropAndPad(percent=(-0.05, 0.1))])", shape)
    return aug, [(sh, sw) for sh in aug.crop["sizes"]["y"] for sw in aug.crop["sizes"]["x"]]


def _images(rng, sh, sw, c):
    return (rng.randint(0, 256, (sh, sw, c), dtype=np.uint8), (rng.rand(sh, sw, c) < 0.5).astype(np.uint8) * 255)


def test_template_range_reaches_116_to_154_pixels():
    aug, pairs = _reachable((128, 128, 3))
    assert list(aug.crop["sizes"]["y"]) == list(range(116, 155)) == list(aug.crop["sizes"]["x"])
    assert len(pairs) == 39 * 39


@pytest.mark.parametrize("geometry", sorted(GEOMETRIES))
def test_resize_restatements_are_bit_exact_with_opencv(geometry):
    """Every reachable (source h, source w) pair of the geometry (the template's at C = 3 and C = 1; a stride through the
    pairs elsewhere keeps the run short), on random images and on 0 / 255 images."""
    H, W, C = GEOMETRIES[geometry]
    _, pairs = _reachable((H, W, C))
    rng = np.random.RandomState(sorted(GEOMETRIES).index(geometry))
    step = 1 if geometry in ("template", "gray") else 3
    for sh, sw in pairs[::step]:
        if (sh, sw) == (H, W):
            continue
        kind = A.crop_pad_rule(sh, sw, H, W)
        fn = CP.resize_cubic_u8 if kind == "cubic" else CP.resize_area_u8
        for img in _images(rng, sh, sw, C):
            assert np.array_equal(fn(img, H, W), _cv2_resize(img, H, W, kind)), (sh, sw, kind)


def test_cubic_restatement_also_matches_opencv_where_area_would_be_chosen():
    rng = np.random.RandomState(1)
    for sh, sw in ((140, 150), (128, 154), (131, 129)):
        for img in _images(rng, sh, sw, 3):
            assert np.array_equal(CP.resize_cubic_u8(img, 128, 128), _cv2_resize(img, 128, 128, "cubic"))


def test_ipp_cubic_differs_by_at_most_one():
    """What OpenCV computes with its default IPP dispatch, for the record (DESIGN.md section 2): +-1 on a few per cent of values."""
    rng = np.random.RandomState(2)
    img = rng.randint(0, 256, (120, 140, 3), dtype=np.uint8)
    cv2.ipp.setUseIPP(True)
    ipp = _cv2_resize(img, 128, 128, "cubic").astype(int)
    cv2.ipp.setUseIPP(False)
    d = np.abs(ipp - CP.resize_cubic_u8(img, 128, 128).astype(int))
    assert d.max() <= 1
    print("IPP cubic: %.2f %% of values differ by 1" % (100.0 * (d != 0).mean()))


@pytest.mark.parametrize("geometry", sorted(GEOMETRIES))
def test_product_tables_equal_the_restatement(geometry):
    """The per-axis blocks the kernel reads, applied on the host, give the restatement's image."""
    H, W, C = GEOMETRIES[geometry]
    aug, pairs = _reachable((H, W, C))
    rng = np.random.RandomState(4)
    for sh, sw in pairs[::37]:
        kind = A.crop_pad_rule(sh, sw, H, W)
        img = rng.randint(0, 256, (sh, sw, C), dtype=np.uint8)
        iy, wy = (A.cubic_taps if kind == "cubic" else A.area_taps)(H, sh)
        ix, wx = (A.cubic_taps if kind == "cubic" else A.area_taps)(W, sw)
        s = img.astype(np.float32)
        if kind == "cubic":
            hs = sum(img[:, ix[:, j]].astype(np.int64) * wx[None, :, j, None] for j in range(4)).astype(np.float32)
            b = (wy.astype(np.float32) * np.float32(1.0 / 2 ** 22))[:, :, None, None]
            t = [hs[iy[:, k]] * b[:, k] for k in range(4)]
            v = t[0] + (t[1] + (t[2] + t[3]))
        else:
            buf = np.zeros((sh, W, C), np.float32)
            for j in range(4):
                buf = buf + s[:, ix[:, j]] * wx[None, :, j, None]
            v = np.zeros((H, W, C), np.float32)
            for k in range(4):
                v = v + wy[:, k, None, None] * buf[iy[:, k]]
        got = np.clip(np.rint(v), 0, 255).astype(np.uint8)
        assert np.array_equal(got, CP.resize_back(img, H, W)), (sh, sw, kind)
        blk = aug.crop["table"][aug.crop["offsets"][("y", kind, sh)]:][:8 * H].reshape(H, 8)
        assert np.array_equal(blk[:, :4], iy) and np.array_equal(blk[:, 4:], wy.view(np.int32) if kind == "area" else wy)


def test_crop_and_pad_then_resize_equals_the_cv2_composition():
    rng = np.random.RandomState(5)
    img = rng.randint(0, 256, (128, 128, 3), dtype=np.uint8)
    cases = [(-6, -6, -6, -6), (13, 13, 13, 13), (-6, 13, 4, -2), (5, -3, -5, 3), (-4, 0, 4, 0), (0, 7, 0, -7), (0, 0, 0, 0)]
    for px in cases:
        top, right, bottom, left = px
        crop = img[max(-top, 0):128 - max(-bottom, 0), max(-left, 0):128 - max(-right, 0)]
        padded = cv2.copyMakeBorder(crop, max(top, 0), max(bottom, 0), max(left, 0), max(right, 0), cv2.BORDER_CONSTANT, value=(17, 17, 17))
        assert np.array_equal(CP.crop_and_pad_u8(img, px, 17), padded)
        sh, sw = padded.shape[:2]
        if (sh, sw) == (128, 128):                                         # pure shifts and no-ops: a copy
            want = padded
        else:
            want = _cv2_resize(padded, 128, 128, A.crop_pad_rule(sh, sw, 128, 128))
        assert np.array_equal(CP.resize_back(padded, 128, 128), want), px


def test_template_with_the_line_uncommented_parses_and_orders():
    ops = A.parse_code(CROP_CODE)
    assert [op.kind for _, op in ops] == ["CropAndPad", "Affine", "CoarseDropout", "GaussianBlur", "Add", "Invert", "Multiply",
                                          "Multiply", "ContrastNormalization"]
    aug = A.Augmenter(CROP_CODE, seed=0)
    assert aug.crop["percent"] and (aug.crop["lo"], aug.crop["hi"]) == (-0.05, 0.1) and aug.crop["independent"]
    with pytest.raises(NotImplementedError, match="order"):
        A.Augmenter("Sequential([Sometimes(0.5, Affine(scale=(1.0, 1.2))), Sometimes(0.5, CropAndPad(percent=(-0.05, 0.1)))])")


@pytest.mark.parametrize("args,name", [
    ("percent=(-0.05, 0.1), pad_mode='edge'", "pad_mode"),
    ("percent=(-0.05, 0.1), keep_size=False", "keep_size"),
    ("percent=((-0.05, 0.1), 0, 0, 0)", "percent"),
    ("px=((0, 4), 0, 0, 0)", "px"),
    ("percent=(-0.05, 0.1), pad_cval=[0, 128, 255]", "pad_cval"),
    ("percent=(-0.05, 0.1), pad_cval=300", "pad_cval"),
    ("percent=(-0.05, 0.1), interpolation='linear'", "interpolation"),
    ("px=(-2, 3), percent=0.1", "px="),
    ("px=(64, 64)", "integer ratio"),
])
def test_unsupported_arguments_raise_and_are_named(args, name):
    with pytest.raises(NotImplementedError, match=name):
        A.Augmenter("Sequential([CropAndPad(%s)])" % args)


def test_sampled_draws_follow_the_cfg():
    aug = A.Augmenter(CROP_CODE, seed=11)
    B = 4000
    state = aug.rng.get_state()
    P = aug.sample(B)
    assert abs(P["crop_on"].mean() - 0.5) < 0.03 and P["crop_px"].shape == (B, 4) and P["crop_px"].dtype == np.int32
    # the same stream by hand: the Sometimes draw, then four uniform draws per image (top, right, bottom, left)
    r = np.random.RandomState(0)
    r.set_state(state)
    on = r.rand(B) < 0.5
    pct = r.uniform(-0.05, 0.1, (B, 4))
    assert np.array_equal(on, P["crop_on"])
    want = np.round(np.float32(128) * pct).astype(np.int32)
    assert np.array_equal(P["crop_px"], want)
    assert P["crop_px"].min() == -6 and P["crop_px"].max() == 13 and not P["crop_cval"].any()
    counts = np.bincount((P["crop_px"] + 6).ravel(), minlength=20)
    assert counts[0] > 0 and counts[19] > 0 and abs(counts[6] / counts[10] - 1) < 0.15           # -6 and 13 at the ends: half cells
    # exact .5 cases round half to even: 0.05 * 10 = 0.5 -> 0, 0.15 * 10 = 1.5 -> 2, -0.25 * 10 = -2.5 -> -2
    assert list(A.crop_pad_pixels(10, np.array([0.05, 0.15, -0.25]), True)) == [0, 2, -2]
    assert list(A.crop_pad_pixels(128, np.array([0.00390625, -0.01171875]), True)) == [0, -2]       # 0.5 and -1.5 exactly


def test_px_ranges_pad_cval_ranges_and_shared_draws():
    aug = A.Augmenter("Sequential([Sometimes(0.7, CropAndPad(px=(-3, 5), pad_cval=(10, 20), sample_independently=False))])",
                      (64, 64, 3), seed=2)
    P = aug.sample(3000)
    px = P["crop_px"]
    assert px.min() == -3 and px.max() == 5 and set(np.unique(px)) == set(range(-3, 6))
    assert (px == px[:, :1]).all()                                          # one draw for all four sides
    assert P["crop_cval"].min() == 10 and P["crop_cval"].max() == 20
    assert abs(P["crop_on"].mean() - 0.7) < 0.03


def test_crops_leave_at_least_one_pixel():
    start, end = A.crop_pad_limit_crops(10, np.array([6, 9, 0, 3]), np.array([6, 4, 12, 3]))
    assert list(10 - start - end) == [1, 1, 1, 4]
    assert (start >= 0).all() and (end >= 0).all()


def test_pack_crop_table_and_flag():
    aug = A.Augmenter(CROP_CODE, seed=3)
    P = aug.sample(64)
    P["crop_on"][:4] = True
    P["crop_px"][:4] = [(-4, 0, 4, 0), (13, 13, 13, 13), (-6, -6, -6, -6), (-6, 13, 4, -2)]
    geom, lut = aug.pack(P)
    t = aug.pack_crop(P)
    assert t.shape == (64, 8) and t.dtype == np.int32
    assert np.array_equal((geom[:, 0] & A.FLAG_CROP) != 0, P["crop_on"])
    assert list(t[0, :6]) == [2, 128, 128, -4, 0, 0]                       # pure shift: area at ratio 1, i.e. a copy
    assert list(t[1, :3]) == [2, 154, 154] and list(t[2, :3]) == [1, 116, 116]     # pad: area; crop: cubic
    assert list(t[3, :5]) == [1, 126, 139, -6, -2]
    assert not t[~P["crop_on"]].any()
    off = aug.crop["offsets"]
    assert t[3, 6] == off[("y", "cubic", 126)] and t[3, 7] == off[("x", "cubic", 139)]


PARENT_DIGESTS = {0: ("d16f128a03b5cadce6a631fb2c495854", "2b79a9e3609a77b0b246ec8375292a00"),
                  7: ("4e07af0e657d77d69f0f9cc8d6448a0f", "de1dda9d96e5fd4f26b589040c50f928"),
                  123: ("9887d6eafc32f40fff4968a3b9826b96", "712adf2696c86a074964830ec25d7b8e")}


@pytest.mark.parametrize("seed", sorted(PARENT_DIGESTS))
def test_chain_without_the_op_samples_and_packs_as_before(seed):
    """sha256 of sample() and pack() for the template chain at batch 64, as computed before CropAndPad existed."""
    np.random.seed(seed + 1)
    aug = A.Augmenter(TEMPLATE_CODE, seed=seed)
    P = aug.sample(64)
    h = hashlib.sha256()
    for k in sorted(P):
        h.update(k.encode())
        h.update(np.ascontiguousarray(P[k]).tobytes())
    geom, lut = aug.pack(P)
    h2 = hashlib.sha256(geom.tobytes() + lut.tobytes())
    assert (h.hexdigest()[:32], h2.hexdigest()[:32]) == PARENT_DIGESTS[seed]
    assert aug.crop is None and aug.pack_crop(P) is None


def test_restated_chain_applies_the_op_first():
    rng = np.random.RandomState(6)
    aug = A.Augmenter(CROP_CODE, seed=4)
    P = aug.sample(6)
    P["crop_on"][:] = True
    P["affine_on"][:] = False
    x = rng.randint(0, 256, (6, 128, 128, 3), dtype=np.uint8)
    bg = rng.randint(0, 256, (6, 128, 128, 3), dtype=np.uint8)
    mask = rng.rand(6, 128, 128) < 0.3
    got = CP.augment_batch(x, mask, bg, P, aug.sigma, low=aug.low)
    from oracle import augment_oracle as AO
    pasted = np.where(mask[..., None], bg, x)
    for b in range(6):
        pasted[b] = CP.resize_back(CP.crop_and_pad_u8(pasted[b], P["crop_px"][b], 0), 128, 128)
    want = AO.augment_batch(pasted, np.zeros_like(mask), pasted, P, aug.sigma, low=aug.low)
    assert np.array_equal(got, want)
