"""The CPU restatement of the training input pipeline pinned to OpenCV at the cfg geometries beyond the template: 64 x 64 x 3
(``px64``), 128 x 128 x 1 (``gray``) and 64 x 128 x 3 (``rect``) -- the shapes tests/test_gpu_q_input_geometry.py runs the device
kernels at.  tests/test_augment_cpu.py pins the same functions at 128 x 128 x 3 only; cv2 runs separate code for one channel and
for scales below 1, where source coordinates go negative.  No GPU needed."""
import numpy as np
import pytest

from augmentedautoencoder_b200.ae import augment as A
from oracle import augment_oracle as AO

cv2 = pytest.importorskip("cv2")

SHAPES = {"px64": (64, 64, 3), "gray": (128, 128, 1), "rect": (64, 128, 3)}
# a general matrix per shape (shear, rotation, translation in both signs), with the source partly outside the image
GENERAL = {"px64": [[0.8, 0.3, -6.2], [-0.2, 1.25, 9.7]], "gray": [[1.1, -0.35, 30.5], [0.4, 0.7, -12.25]],
           "rect": [[0.65, 0.15, 20.3], [-0.1, 1.4, -13.9]]}
# (rows, cols) of every CoarseDropout / square-occlusion grid the device tests use, with the crop it is upsampled to
GRIDS = [((4, 4), (64, 64)), ((4, 6), (64, 128)), ((6, 6), (128, 128)), ((8, 8), (128, 128)), ((3, 3), (64, 64)), ((4, 8), (64, 128))]


def _img(seed, shape):
    return np.random.RandomState(seed).randint(0, 256, shape, dtype=np.uint8)


def _cv2_hwc(out, c):
    """cv2 returns [h, w] for a one-channel image: put the channel axis back"""
    return out[..., None] if c == 1 and out.ndim == 2 else out


@pytest.mark.parametrize("geom", sorted(SHAPES))
def test_warp_affine_restatement_is_bit_exact_with_opencv(geom):
    h, w, c = SHAPES[geom]
    img = _img(0, (h, w, c))
    mats = [AO.scale_matrix(s, h, w) for s in np.linspace(0.5, 1.5, 41)] + [np.array(GENERAL[geom], np.float64)]
    for M in mats:
        ref = _cv2_hwc(cv2.warpAffine(img, M, (w, h), flags=cv2.INTER_LINEAR, borderMode=cv2.BORDER_CONSTANT, borderValue=0), c)
        got = AO.warp_affine_u8(img, M)
        assert got.shape == ref.shape == (h, w, c)
        assert np.array_equal(got, ref), (geom, M.tolist(), int((got != ref).sum()))
        # the product's packed tables are the restatement's, row tables H long and column tables W long
        for g_, w_ in zip(A.affine_tables(M, h, w), AO.affine_fixed_point(M, h, w)):
            assert np.array_equal(g_.astype(np.int64), w_)
    # below scale 1 the border is reached: the zero fill is part of what was compared
    small = AO.warp_affine_u8(np.full((h, w, c), 255, np.uint8), AO.scale_matrix(0.5, h, w))
    assert small[0, 0].max() == 0 and small[h // 2, w // 2].min() == 255


@pytest.mark.parametrize("geom", sorted(SHAPES))
def test_gaussian_blur_restatement_is_bit_exact_with_opencv(geom):
    h, w, c = SHAPES[geom]
    img = _img(1, (h, w, c))
    for sigma in (0.01, 0.3, 1.0, 1.49):
        assert AO.blur_ksize(sigma) == 5
        ref = _cv2_hwc(cv2.GaussianBlur(img, (5, 5), sigmaX=sigma, sigmaY=sigma, borderType=cv2.BORDER_REFLECT_101), c)
        got = AO.gaussian_blur5_u8(img, sigma)
        assert np.array_equal(got, ref), (geom, sigma, int((got != ref).sum()))
        assert np.array_equal(A.gaussian_taps_q8(sigma), AO.gaussian_kernel5_q8(sigma))
    assert AO.gaussian_kernel5_q8(0.01).tolist() == [0, 0, 256, 0, 0]           # a tiny sigma is the identity, flag on or off
    assert np.array_equal(AO.gaussian_blur5_u8(img, 0.01), img)


@pytest.mark.parametrize("grid,crop", GRIDS, ids=["%dx%d@%dx%d" % (g + s) for g, s in GRIDS])
def test_nearest_upsampling_maps_match_opencv(grid, crop):
    (lh, lw), (h, w) = grid, crop
    low = np.arange(lh * lw, dtype=np.uint8).reshape(lh, lw)
    ref = cv2.resize(low, (w, h), interpolation=cv2.INTER_NEAREST)              # dsize is (width, height)
    rmap, cmap = AO.nearest_index_map(h, lh), AO.nearest_index_map(w, lw)
    assert np.array_equal(low[rmap][:, cmap], ref)
    assert np.array_equal(A.nearest_cells(h, lh), rmap) and np.array_equal(A.nearest_cells(w, lw), cmap)
    assert set(ref.ravel().tolist()) == set(range(lh * lw))                    # every cell reaches the crop


def test_dropout_grids_of_the_device_tests():
    """The grids the device tests rely on come out of Augmenter / Occlusion as stated: 8 x 8 (all 64 keep bits) at 128 with
    size_percent 0.0625, 4 x 6 at 64 x 128 and 4 x 4 at 64 with the template's 0.05, and a 3 x 3 square-occlusion grid at 64."""
    code = lambda sp: "Sequential([Sometimes(0.5, CoarseDropout(p=0.2, size_percent=%r))])" % sp      # noqa: E731
    assert A.Augmenter(code(0.0625), (128, 128, 1)).low == (8, 8)
    assert A.Augmenter(code(0.05), (64, 128, 3)).low == (4, 6)
    assert A.Augmenter(code(0.05), (64, 64, 3)).low == (4, 4)
    assert A.Occlusion((64, 64), 0.25, 0.25).low == (3, 3)
    aug = A.Augmenter("Sequential([Sometimes(1.0, CoarseDropout(p=0.5, size_percent=0.0625))])", (128, 128, 1), seed=0)
    P = aug.sample(4)
    P["drop_keep"][0] = 0
    P["drop_keep"][0, 7, 7] = 1                                                # cell 63 alone: the top bit of the high word
    geom, _ = aug.pack(P)
    assert geom[0, 1] == 0 and np.uint32(geom[0, 2]) == np.uint32(1 << 31)
    for b in range(1, 4):
        keep = int(np.uint32(geom[b, 1])) | (int(np.uint32(geom[b, 2])) << 32)
        bits = np.array([(keep >> i) & 1 for i in range(64)], np.uint8).reshape(8, 8)
        assert np.array_equal(bits, P["drop_keep"][b])


def test_occlusion_bank_at_64_matches_opencv(tmp_path):
    bits = np.random.RandomState(2).rand(4, 224, 224) < 0.35
    path = tmp_path / "masks.bin"
    np.packbits(bits.reshape(-1)).tofile(path)
    # dataset.py:411-416: the bits as float32 224 x 224 masks, cv2.resize NEAREST to the crop
    ref = np.unpackbits(np.fromfile(path, np.uint8)).astype(np.float32).reshape(-1, 224, 224)
    want = np.array([cv2.resize(m, (64, 64), interpolation=cv2.INTER_NEAREST) for m in ref]).astype(bool)
    got = A.load_occlusion_bank(str(path), (64, 64))
    assert got.dtype == np.uint32 and got.shape == (4, 64, 2)                  # two 32-bit words per row
    unpacked = np.unpackbits(got.view(np.uint8), axis=-1, bitorder="little").reshape(-1, 64, 64).astype(bool)
    assert np.array_equal(unpacked, want)
