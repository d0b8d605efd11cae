"""CPU tests of the detection crops (no GPU needed):

* the numpy restatement of aae_extract_square_patches (oracle/crop_oracle.py) against cv2.resize(INTER_LINEAR) on the
  black-bordered square, for every square side 1..1024 at several output sizes, with OpenCV's IPP dispatch on and off;
* square_patch_boxes, the host half of the device crops, against the reference's scalar float64 expressions on detector
  boxes and pad factors where float32 arithmetic gives other integers;
* the refusal of a square smaller than its box."""
import cv2
import numpy as np
import pytest

from augmentedautoencoder_b200.m3_interface.ae_pose_estimator import AePoseEstimator, square_patch_boxes
from oracle import crop_oracle as CO

FRAMES = [(W, H) for W in (640, 641, 1280, 1920) for H in (480, 479, 720, 1080)]
PAD_FACTORS = [1.0, 1.1, 1.15, 1.2, 1.25, 1.3, 1.4, 1.5, 1.8, 1.9, 2.0]


def random_pad_factors():
    return [float(v) for v in np.random.RandomState(17).uniform(1.0, 2.0, 8)]


@pytest.fixture
def ipp_state():
    was = cv2.ipp.useIPP()
    yield
    cv2.ipp.setUseIPP(was)


# ---- resize arithmetic ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("out", [64, 96, 128, 256])
def test_restated_kernel_matches_cv2_resize_at_every_square_side(out, ipp_state):
    """Every square side 1..1024 (which includes out, out +- 1 and 2 * out, where cv2 hands INTER_LINEAR to its INTER_AREA
    code), with a random box pasted centred into it: some squares are filled, most have black borders on two sides."""
    rng = np.random.RandomState(out)
    scene = rng.randint(0, 256, (1100, 1100, 3), dtype=np.uint8)
    bad = []
    for side in range(1, 1025):
        longest = side if side % 3 == 0 else rng.randint((side + 1) // 2, side + 1)
        other = rng.randint(1, longest + 1)
        w, h = (longest, other) if side % 2 else (other, longest)
        x, y = rng.randint(0, 1100 - w + 1), rng.randint(0, 1100 - h + 1)
        square = np.zeros((side, side, 3), np.uint8)
        square[(side - h) // 2:(side - h) // 2 + h, (side - w) // 2:(side - w) // 2 + w] = scene[y:y + h, x:x + w]
        got = CO.square_patch(scene, (x, y, w, h, side), out)
        for ipp in (True, False):
            cv2.ipp.setUseIPP(ipp)
            want = cv2.resize(square, (out, out), interpolation=cv2.INTER_LINEAR)
            if not np.array_equal(got, want):
                bad.append((side, ipp, (x, y, w, h), int((got != want).sum())))
    assert not bad, bad[:10]


def test_restated_kernel_on_saturated_and_constant_squares():
    """All-255 and 0 / 255 checkerboard boxes: the extremes of the 11-bit sums and shifts."""
    for pattern in ("white", "checker"):
        scene = np.full((300, 300, 3), 255, np.uint8)
        if pattern == "checker":
            scene[(np.add.outer(np.arange(300), np.arange(300)) % 2) == 1] = 0
        for side in (1, 2, 3, 63, 64, 65, 127, 128, 129, 200, 256, 257, 299):
            for out in (64, 128):
                square = scene[:side, :side]
                want = cv2.resize(square, (out, out), interpolation=cv2.INTER_LINEAR)
                assert np.array_equal(CO.square_patch(scene, (0, 0, side, side, side), out), want), (pattern, side, out)


def test_restated_kernel_pads_past_the_frame_edge_with_black():
    """A box past the right or bottom edge reads black there: the reference's crop of the frame padded with black."""
    rng = np.random.RandomState(4)
    scene = rng.randint(0, 256, (480, 640, 3), dtype=np.uint8)
    padded = np.zeros((800, 900, 3), np.uint8)
    padded[:480, :640] = scene
    est = AePoseEstimator.__new__(AePoseEstimator)
    for box in ([600, 100, 80, 50], [100, 450, 60, 90], [620, 470, 100, 100], [639, 479, 5, 3]):
        for pf in (1.0, 1.3):
            want = est.extract_square_patch(padded, box, pf, resize=(64, 64), interpolation=cv2.INTER_LINEAR, black_borders=True)
            got = CO.square_patch(scene, square_patch_boxes(box, pf)[0], 64)
            assert np.array_equal(got, want), (box, pf)


# ---- host box arithmetic ----------------------------------------------------------------------------------------------------
def check_table(boxes, pad_factor):
    """square_patch_boxes against the reference's scalar expressions, box by box; returns how many boxes the float32 route
    would have given other integers."""
    table = square_patch_boxes(boxes, pad_factor)
    assert table.dtype == np.int32 and table.shape == (len(boxes), 5) and table.flags.c_contiguous
    want = np.array([CO.reference_box_ints(b, pad_factor) for b in boxes])
    mism = np.flatnonzero((table != want).any(axis=1))
    assert len(mism) == 0, (pad_factor, [(boxes[i], table[i].tolist(), want[i].tolist()) for i in mism[:5]])
    old = np.array([CO.float32_box_ints(b, pad_factor) for b in boxes])
    return int((old != want).any(axis=1).sum())


@pytest.mark.parametrize("W,H", FRAMES)
def test_box_table_on_whole_pixel_detector_boxes(W, H):
    rng = np.random.RandomState(W * 7 + H)
    boxes = CO.whole_pixel_boxes(W, H, 3000, rng)
    moved = {pf: check_table(boxes, pf) for pf in PAD_FACTORS + random_pad_factors()}
    assert all(v > 0 for v in moved.values()), moved          # the set keeps reaching values float32 rounds across an integer


@pytest.mark.parametrize("W,H", FRAMES)
def test_box_table_on_two_decimal_detector_boxes(W, H):
    rng = np.random.RandomState(W * 11 + H)
    boxes = CO.two_decimal_boxes(W, H, 3000, rng)
    moved = {pf: check_table(boxes, pf) for pf in PAD_FACTORS + random_pad_factors()}
    assert sum(moved.values()) > 0, moved      # on some frames only the pad factors that float32 moves reach an edge


def test_box_table_at_every_longest_side_and_pad_factor():
    """Whole-number boxes of every longest side 1..1500 (w = longest, h = longest and both): the square's side is a float64
    product with the Python float pad factor.  float32(1.3) < 1.3 < float64(1.3) makes a 50 px box a 65 px square, not 64."""
    boxes = [[3, 4, s, max(1, s // 2)] for s in range(1, 1501)] + [[5, 6, max(1, s // 3), s] for s in range(1, 1501)]
    boxes += [[7, 8, s, s] for s in range(1, 1501)]
    moved = {pf: check_table(boxes, pf) for pf in PAD_FACTORS + random_pad_factors()}
    assert moved[1.0] == moved[1.2] == moved[2.0] == 0
    assert all(moved[pf] > 0 for pf in (1.15, 1.3, 1.4, 1.8, 1.9)), moved
    assert square_patch_boxes([100, 100, 50, 40], 1.3)[0].tolist() == [100, 100, 50, 40, 65]
    box = CO.detector_box(1 / 640, 0.0, 23 / 640, 10 / 480, 640, 480)           # pixels 1 to 23: w = 21.999999999999996
    assert square_patch_boxes(box, 1.2)[0, 2] == 21 and CO.float32_box_ints(box, 1.2)[2] == 22


def test_box_table_truncates_toward_zero_like_the_reference():
    boxes = [[0.999, 1.999, 2.5, 0.7], [10.0, 20.0, 0.3, 0.2], [0.0, 0.0, 0.0, 0.0], [3.0, 4.0, 1.0, 1.0]]
    for pf in PAD_FACTORS:
        check_table(boxes, pf)
    assert square_patch_boxes(boxes, 1.2).tolist() == [[0, 1, 2, 0, 2], [10, 20, 0, 0, 0], [0, 0, 0, 0, 0], [3, 4, 1, 1, 1]]


def test_mirror_and_restatement_match_the_reference_at_the_edges(golden_dir):
    """Crops the reference's own extract_square_patch and process() made (tests/golden/make_crop_edges_golden.py): the host
    mirror and the restated kernel on the table of square_patch_boxes give them bit for bit; the float32 route does not."""
    import os
    g = np.load(os.path.join(golden_dir, "crops_edges.npz"))
    H, W = (int(v) for v in g["frame_hw"])
    scene = CO.smooth_scene(H, W)
    assert CO.scene_crc(scene) == int(g["scene_sum"][1]) and int(scene.astype(np.int64).sum()) == int(g["scene_sum"][0])
    est = AePoseEstimator.__new__(AePoseEstimator)
    out = int(g["out_size"])
    for pf, key in ((1.2, "crops_pf12"), (1.3, "crops_pf13")):
        boxes = g["boxes_xywh"]
        mirror = np.stack([est.extract_square_patch(scene, b, pf, resize=(out, out), interpolation=cv2.INTER_LINEAR,
                                                    black_borders=True) for b in boxes])
        assert np.array_equal(mirror, g[key]), pf
        assert np.array_equal(CO.square_patches(scene, square_patch_boxes(boxes, pf), out), g[key]), pf
        old = CO.square_patches(scene, [CO.float32_box_ints(b, pf) for b in boxes], out)
        assert sum(not np.array_equal(a, b) for a, b in zip(old, g[key])) > len(boxes) // 2, pf


# ---- refusals ---------------------------------------------------------------------------------------------------------------
def test_a_square_smaller_than_its_box_is_refused():
    """PAD_FACTOR < 1: the reference pastes at negative indices; the host refuses, naming the pad factor and the box."""
    with pytest.raises(ValueError, match=r"pad factor 0\.9 .*\[100\.5, 20\.0, 50\.0, 40\.0\]"):
        square_patch_boxes([[10, 10, 0, 0], [100.5, 20.0, 50.0, 40.0]], 0.9)
    with pytest.raises(ValueError, match="pad factor 0.5"):
        square_patch_boxes([3, 4, 1, 1], 0.5)
    est = AePoseEstimator.__new__(AePoseEstimator)
    with pytest.raises(ValueError, match="pad factor 0.99"):
        est.extract_square_patch(np.zeros((50, 50, 3), np.uint8), [1, 1, 20, 10], 0.99, resize=(64, 64),
                                 interpolation=cv2.INTER_LINEAR, black_borders=True)
    with pytest.raises(ValueError, match="pad factor 0.99"):
        square_patch_boxes([3, 4, 10, 10], 0.99)
    assert square_patch_boxes([3, 4, 0, 0], 0.5)[0].tolist() == [3, 4, 0, 0, 0]     # an empty box: an empty square, black
