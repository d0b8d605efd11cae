"""GPU tests of the detection crops (aae_extract_square_patches through AePoseEstimator.extract_square_patches_device) and of
AePoseEstimator.process built on them:

* the device crops bit for bit against the host mirror extract_square_patch (cv2) on whole-pixel and two-decimal detector
  boxes, where the float64 box sides and squares differ from float32 ones, at eleven pad factors and a few random ones;
* squares of side out, out +- 1 and 2, 3 and 4 times out; boxes of one pixel and less; boxes that end on, or run past, the
  frame's right and bottom edges; boxes that truncate to an empty one; a pad factor below 1;
* the device crops against crops the reference's own extract_square_patch and process() made (tests/golden/crops_edges.npz);
* process() end to end with two classes at PAD_FACTOR 1.2 and 1.3, one of them past the encoder's max_batch."""
import os

import cv2
import numpy as np
import pytest
import torch

from augmentedautoencoder_b200.m3_interface.ae_pose_estimator import AePoseEstimator, square_patch_boxes
from oracle import aae_oracle as O
from oracle import crop_oracle as CO
from tests.test_crops_cpu import PAD_FACTORS, random_pad_factors
from tests.test_gpu_c_plugin import M3_CFG, TRAIN_CFG, make_workspace

pytestmark = pytest.mark.gpu

EST = AePoseEstimator.__new__(AePoseEstimator)     # the crop methods need no workspace


def mirror(scene, box, pf, out):
    return EST.extract_square_patch(scene, box, pf, resize=(out, out), interpolation=cv2.INTER_LINEAR, black_borders=True)


def device(frame_dev, boxes, pf, out):
    return EST.extract_square_patches_device(frame_dev, boxes, pf, (out, out)).cpu().numpy()


def compare(got, scene, boxes, pf, out, what):
    """Device crops against the mirror, box by box.  A box that truncates to a 0 px square (a 1 px detector box whose
    float64 sides fall just below 1), which cv2.resize refuses, must come out black."""
    bad = []
    for b, g in zip(boxes, got):
        empty = square_patch_boxes(b, pf)[0, 4] == 0
        want = np.zeros_like(g) if empty else mirror(scene, b, pf, out)
        if not np.array_equal(g, want):
            bad.append((list(b), square_patch_boxes(b, pf)[0].tolist(), int((g != want).sum())))
    assert not bad, (what, pf, out, len(bad), len(boxes), bad[:4])


# ---- detector box sets ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("W,H", [(640, 480), (641, 479), (1280, 720), (1920, 1080)])
def test_device_crops_match_the_mirror_on_detector_boxes(W, H):
    """2000 boxes per launch: 1500 whole-pixel detector boxes and 500 two-decimal ones.  Per pad factor, how many of them
    the float32 route gave other integers is asserted positive, so each launch reaches the edge this test is about."""
    rng = np.random.RandomState(W + H)
    scene = rng.randint(0, 256, (H, W, 3), dtype=np.uint8)
    frame = torch.from_numpy(scene).cuda()
    boxes = CO.whole_pixel_boxes(W, H, 1500, rng, max_side=400) + CO.two_decimal_boxes(W, H, 500, rng, max_rel=0.25)
    for pf in PAD_FACTORS + random_pad_factors()[:3]:
        moved = sum(CO.float32_box_ints(b, pf) != CO.reference_box_ints(b, pf) for b in boxes)
        assert moved > 0, pf
        for out in (64, 128):
            compare(device(frame, boxes, pf, out), scene, boxes, pf, out, (W, H))


def test_device_crops_at_square_sides_around_the_output_size():
    """Squares of side out, out +- 1, 2 out (cv2's INTER_AREA hand-off), 3 out and 4 out, each reached at pad factor 1.0 by
    a filled square and at 1.3 / 1.37 by a padded one."""
    rng = np.random.RandomState(5)
    scene = rng.randint(0, 256, (1080, 1280, 3), dtype=np.uint8)
    frame = torch.from_numpy(scene).cuda()
    for out in (64, 128):
        sides = [out - 1, out, out + 1, 2 * out - 1, 2 * out, 2 * out + 1, 3 * out, 4 * out]
        cases = {1.0: [[17, 9, s, s] for s in sides] + [[30, 40, s, max(1, s // 2)] for s in sides]}
        for pf in (1.3, 1.37):
            cases[pf] = [[50, 20, m, max(1, m * 2 // 3)] for s in sides for m in range(1, s + 1) if int(m * pf) == s]
            assert len(cases[pf]) >= len(sides) // 2, (pf, out)
        for pf, boxes in cases.items():
            got = device(frame, boxes, pf, out)
            assert [int(square_patch_boxes(b, pf)[0, 4]) in sides for b in boxes] == [True] * len(boxes)
            compare(got, scene, boxes, pf, out, "sides")


def test_device_crops_of_tiny_empty_and_edge_boxes():
    rng = np.random.RandomState(6)
    H, W = 480, 640
    scene = rng.randint(0, 256, (H, W, 3), dtype=np.uint8)
    frame = torch.from_numpy(scene).cuda()
    one = [[0, 0, 1, 1], [639, 479, 1, 1], [320.4, 200.9, 1.0, 1.5], [10.2, 10.7, 1.3, 1.9], [5, 6, 1, 30], [7, 8, 40, 1]]
    under = [[100.5, 100.5, 0.5, 3.2], [200.0, 100.0, 4.0, 0.99], [300.2, 50.1, 0.999999, 12.0]]    # w or h truncates to 0
    on_edge = [[600, 100, 40, 50], [100, 430, 60, 50], [560, 400, 80, 80], [0, 0, 640, 480], [639, 0, 1, 480],
               CO.detector_box(600 / W, 100 / H, 640 / W, 150 / H, W, H), CO.detector_box(3 / W, 401 / H, 77 / W, 480 / H, W, H),
               CO.detector_box(0.0, 0.0, 1.0, 1.0, W, H), CO.detector_box(0.71, 0.8, 1.0, 1.0, W, H)]
    for pf in (1.0, 1.2, 1.3):
        for out in (64, 128):
            for what, boxes in (("1 px", one), ("under 1 px", under), ("on the edge", on_edge)):
                compare(device(frame, boxes, pf, out), scene, boxes, pf, out, what)
            got = device(frame, under, pf, out)
            assert not got.any()                                          # the reference's crop of an empty box is black
    # w and h both truncate to 0: a 0 px square, which cv2.resize refuses; the device writes a black crop
    empty = [[50.0, 60.0, 0.9, 0.4], [10, 10, 0, 0]]
    with pytest.raises(cv2.error):
        mirror(scene, empty[0], 1.2, 64)
    got = EST.extract_square_patches_device(frame, empty + [[100, 100, 30, 20]], 1.2, (64, 64)).cpu().numpy()
    assert not got[:2].any() and got[2].any()


def test_device_crops_past_the_right_and_bottom_edge_are_padded_with_black():
    """The reference refuses a box past the frame (its paste raises); the device crops it from the frame padded with black
    on the right and bottom, which the mirror shows on such a padded frame."""
    rng = np.random.RandomState(8)
    H, W = 480, 640
    scene = rng.randint(0, 256, (H, W, 3), dtype=np.uint8)
    padded = np.zeros((H + 400, W + 400, 3), np.uint8)
    padded[:H, :W] = scene
    frame = torch.from_numpy(scene).cuda()
    boxes = [[600, 100, 80, 50], [100, 450, 60, 90], [620, 470, 100, 100], [639, 479, 5, 3], [0, 0, 700, 500],
             CO.detector_box(0.9, 0.2, 1.02, 0.5, W, H), CO.detector_box(0.3, 0.95, 0.4, 1.004, W, H),
             CO.detector_box(0.97, 0.97, 1.1, 1.15, W, H)]
    with pytest.raises(ValueError):
        mirror(scene, boxes[0], 1.2, 64)
    for pf in (1.0, 1.2, 1.3):
        for out in (64, 128):
            compare(device(frame, boxes, pf, out), padded, boxes, pf, out, "past the edge")


def test_a_pad_factor_below_one_is_refused_before_the_launch():
    frame = torch.zeros((48, 64, 3), dtype=torch.uint8, device="cuda")
    for pf in (0.99, 0.5):
        with pytest.raises(ValueError, match="pad factor %s" % pf):
            EST.extract_square_patches_device(frame, [[1, 2, 3, 4], [5, 6, 10, 8]], pf, (64, 64))


# ---- the reference's own crops ----------------------------------------------------------------------------------------------
def test_device_crops_match_the_reference_at_the_edges(golden_dir):
    """Crops the reference's extract_square_patch and process() made of whole-pixel detections whose float64 sides fall
    just below an integer, of 1 px boxes, of boxes ending on the frame's edges, at PAD_FACTOR 1.2 and 1.3."""
    g = np.load(os.path.join(golden_dir, "crops_edges.npz"))
    H, W = (int(v) for v in g["frame_hw"])
    scene = CO.smooth_scene(H, W)
    assert CO.scene_crc(scene) == int(g["scene_sum"][1])
    frame = torch.from_numpy(scene).cuda()
    out = int(g["out_size"])
    for pf, key in ((1.2, "crops_pf12"), (1.3, "crops_pf13")):
        got = device(frame, g["boxes_xywh"], pf, out)
        bad = [i for i in range(len(got)) if not np.array_equal(got[i], g[key][i])]
        assert not bad, (pf, len(bad), g["pixel_boxes"][bad[:5]].tolist())
    # process(): each class's detections in one launch at its pad factor, in the order the reference fed them
    pads = {int(c): float(p) for c, p in g["class_pad_factors"]}
    rel, cls = g["rel_boxes"], g["det_classes"]
    fed = np.empty_like(g["process_crops_u8"])
    for c, pf in pads.items():
        sel = np.flatnonzero(cls == c)
        fed[sel] = device(frame, [CO.detector_box(*rel[i], W, H) for i in sel], pf, out)
    assert np.array_equal(fed, g["process_crops_u8"])


# ---- process() end to end ---------------------------------------------------------------------------------------------------
def test_process_end_to_end_on_whole_pixel_detections(tmp_path, monkeypatch):
    """Two classes at PAD_FACTOR 1.2 (40 detections) and 1.3 (300, past max_batch 256), whole-pixel detections, one of an
    unknown class and one at a negative coordinate.  Every pose must equal, bit for bit, the one built from host crops of
    the mirror -> Codebook.nearest_rotation (the same batch split) -> the oracle's pose lift; and each index must be the
    float64 oracle's wherever that oracle's top two cosines are more than MARGIN apart."""
    from augmentedautoencoder_b200.ae.dataset import Dataset
    from augmentedautoencoder_b200.m3_interface.m3_interfaces import BoundingBox
    MARGIN = 1e-4
    ws = tmp_path / "ws"
    monkeypatch.setenv("AE_WORKSPACE_PATH", str(ws))
    ds = Dataset(None, min_n_views=162, num_cyclo=36, radius=700)
    objs = make_workspace(ws, {"obj_a": (1, TRAIN_CFG), "obj_b": (2, TRAIN_CFG.replace("PAD_FACTOR: 1.2", "PAD_FACTOR: 1.3"))},
                          ds.embedding_size)
    cfg_path = tmp_path / "m3.cfg"
    cfg_path.write_text(M3_CFG)
    from augmentedautoencoder_b200.m3_interface.ae_pose_estimator import AePoseEstimator as Est
    est = Est(str(cfg_path))
    assert est.pad_factors == {1: 1.2, 5: 1.3} and est.all_codebooks[5].max_batch == 256
    H, W = 480, 640
    scene = cv2.resize(O.make_crops_u8(78, 1, hw=128)[0], (W, H), interpolation=cv2.INTER_CUBIC)
    K = np.array([[572.4114, 0, 325.2611], [0, 573.57043, 242.04899], [0, 0, 1]])
    rng = np.random.RandomState(12)
    dets = []
    for cls, count in ((1, 40), (5, 300)):
        for _ in range(count):
            w, h = rng.randint(20, 300), rng.randint(20, 300)
            x0, y0 = rng.randint(0, W - w + 1), rng.randint(0, H - h + 1)
            dets.append(BoundingBox(x0 / W, y0 / H, (x0 + w) / W, (y0 + h) / H, {cls: 0.9, 7: 0.05}))
    order = rng.permutation(len(dets))
    dets = [dets[i] for i in order]
    dets.insert(17, BoundingBox(0.1, 0.1, 0.3, 0.3, {7: 0.9, 1: 0.1}))            # unknown class: skipped
    dets.insert(60, BoundingBox(-3 / W, 0.2, 0.2, 0.4, {5: 0.9}))                # negative coordinate: skipped
    poses = est.process(dets, scene, K, mm=True)
    kept = [d for d in dets if max(d.classes, key=d.classes.get) in (1, 5) and d.xmin >= 0]
    assert len(poses) == len(kept) == 340 and [p.name for p in poses] == [max(d.classes, key=d.classes.get) for d in kept]
    k_train = np.array([1075.65, 0, 360, 0, 1073.90, 270, 0, 0, 1]).reshape(3, 3)
    checked = 0
    for cls, name in ((1, "obj_a"), (5, "obj_b")):
        p, E, bbs = objs[name]
        pf = est.pad_factors[cls]
        js = [j for j, d in enumerate(kept) if max(d.classes, key=d.classes.get) == cls]
        boxes = [CO.detector_box(kept[j].xmin, kept[j].ymin, kept[j].xmax, kept[j].ymax, W, H) for j in js]
        assert sum(CO.float32_box_ints(b, pf) != CO.reference_box_ints(b, pf) for b in boxes) > len(boxes) // 10, cls
        crops = np.stack([mirror(scene, b, pf, 128) for b in boxes])
        idcs = est.all_codebooks[cls].nearest_rotation(est._sessions[cls], crops, return_idcs=True)
        for j, b, idc in zip(js, boxes, idcs):
            R, t = O.auto_pose6d_lift(np.array([idc]), ds.viewsphere_for_embedding, bbs, b, K, k_train, 700.0)
            want = np.eye(4)
            want[:3, :3], want[:3, 3] = R.squeeze(), t.squeeze()
            assert np.array_equal(poses[j].trafo, want), (cls, j, b)
        idc64, cos64 = O.nearest_rotation_idcs(crops, p, E, dtype=torch.float64, return_cos=True, device="cuda")
        top2 = np.sort(cos64, axis=1)[:, -2:]
        sure = top2[:, 1] - top2[:, 0] > MARGIN
        assert np.array_equal(idcs[sure], idc64[sure]), (cls, np.flatnonzero(idcs[sure] != idc64[sure]))
        checked += int(sure.sum())
    print("process(): %d of %d indices checked against the float64 oracle (top-2 gap > %g)" % (checked, len(kept), MARGIN))
    assert checked >= len(kept) // 2
