#!/usr/bin/env python
"""Generate tests/golden/crops_edges.npz by running the REFERENCE's own crop code on edge detections.

Run in the build container only (needs /root/reference; the GPU box has no copy), after make_golden.py's stubs:

    python tests/golden/make_crop_edges_golden.py

Recorded, on the smooth 640 x 480 scene ``oracle.crop_oracle.smooth_scene`` builds from integers (its checksum is
stored):

* ``AePoseEstimator.extract_square_patch(..., INTER_LINEAR, black_borders=True)`` at 64 x 64 for every edge box at pad
  factors 1.2 and 1.3 (auto_pose/m3_interface/ae_pose_estimator.py:106-131);
* the crops ``AePoseEstimator.process`` feeds the session for the same detections as whole-pixel ``BoundingBox``es of two
  classes, one with PAD_FACTOR 1.2 and one with 1.3 (ae_pose_estimator.py:133-170), captured by the fake session.

The edge boxes are whole-pixel detector boxes (pixel x0 to pixel x1, normalised by the frame and multiplied back, as
process() does): ones whose float64 sides fall just below an integer, which float32 would round up, 1-pixel boxes (some of
which truncate to a width or height of 0: a black crop), boxes that end on the right or bottom edge, and boxes whose longest
side float32(1.3) would make a smaller square.
"""
import contextlib
import io
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(1, os.path.dirname(os.path.dirname(HERE)))
import make_golden as G  # noqa: E402  (sets sys.dont_write_bytecode; the stubs and the fake session)
from oracle import crop_oracle as CO  # noqa: E402
from oracle.crop_oracle import scene_crc as crc  # noqa: E402

W, H = 640, 480
PADS = {1: 1.2, 2: 1.3}                 # class -> PAD_FACTOR


def edge_pixel_boxes():
    """(x0, y0, x1, y1) whole-pixel boxes at the edges the device crops used to miss."""
    def moved(c0, c1, N):         # the float64 side lies just below an integer, which float32 rounds it to
        side = (c1 / N - c0 / N) * N
        return int(side) != int(np.float32(side))
    rng = np.random.RandomState(23)
    out = []
    while len(out) < 20:          # width or height float32 rounds up to the next integer
        x0, y0 = rng.randint(0, 500), rng.randint(0, 360)
        x1, y1 = x0 + rng.randint(20, 140), y0 + rng.randint(20, 120)
        if moved(x0, x1, W) or moved(y0, y1, H):
            out.append((x0, y0, x1, y1))
    one = [a for a in range(0, 600, 7) if moved(a, a + 1, W)][:3]
    out += [(a, 100, a + 1, 110) for a in one]                            # 1 px wide, truncates to 0: a black crop
    ones = [(a, b, a + 1, b + 1) for a, b in ((200, 200), (0, 0), (639, 479), (7, 3), (320, 240), (1, 1))]
    out += [q for q in ones if not moved(q[0], q[2], W) and not moved(q[1], q[3], H)]     # 1 px boxes (cv2 refuses a 0 px square)
    out += [(600, 300, 640, 350), (100, 430, 180, 480), (560, 400, 640, 480), (0, 0, 640, 480)]   # ending on the edges
    for m in (50, 60, 70, 100):                                           # float32(1.3) makes a smaller square
        if int(float(m) * float(np.float32(1.3))) != int(m * 1.3):
            out.append((150, 120, 150 + m, 120 + m * 3 // 4))
    return out


def main():
    m3i = G.install_stubs()
    from auto_pose.ae.codebook import Codebook
    from auto_pose.ae.dataset import Dataset
    from auto_pose.m3_interface.ae_pose_estimator import AePoseEstimator
    import cv2

    cfg, kw = G.template_dataset_kw()
    kw.update(noof_training_imgs="1", noof_bg_imgs="1", background_images_glob="/nonexistent/*.jpg", min_n_views="162",
              num_cyclo="12")
    ds = Dataset("/tmp/unused", **kw)

    class Enc:
        latent_space_size = 128
        x = object()
        z = object()

    cb = Codebook(Enc(), ds, True)
    n = ds.embedding_size
    cb.embed_obj_bbs_values = np.tile(np.array([[300, 200, 100, 120]], np.int32), (n, 1))
    sess = G.FakeSession()
    fed = []

    def answer(feed):
        fed.append(np.asarray(feed[Enc.x], dtype=np.float32))
        return np.zeros((1, n), np.float32)

    sess.table[id(cb.cos_similarity)] = answer
    est = AePoseEstimator.__new__(AePoseEstimator)
    est._camPose, est._upright, est._topk = False, False, 1
    est.class_2_encoder = {1: "grp/a", 2: "grp/b"}
    est.all_codebooks = {1: cb, 2: cb}
    est.all_train_args = {1: cfg, 2: cfg}
    est.pad_factors = dict(PADS)
    est.patch_sizes = {1: (64, 64), 2: (64, 64)}
    est.sess = sess

    img = CO.smooth_scene(H, W)
    px = edge_pixel_boxes()
    rel = np.array([(x0 / W, y0 / H, x1 / W, y1 / H) for x0, y0, x1, y1 in px])
    boxes = np.array([CO.detector_box(*r, W, H) for r in rel])
    crops = {pf: np.stack([est.extract_square_patch(img, b, pf, resize=(64, 64), interpolation=cv2.INTER_LINEAR,
                                                    black_borders=True) for b in boxes]) for pf in PADS.values()}
    classes = np.array([1 + (i % 2) for i in range(len(px))])
    dets = [m3i.BoundingBox(xmin=r[0], ymin=r[1], xmax=r[2], ymax=r[3], classes={int(c): 0.9}) for r, c in zip(rel, classes)]
    with contextlib.redirect_stdout(io.StringIO()):
        poses = est.process(dets, img, np.array([[572.4114, 0, 325.2611], [0, 573.57043, 242.04899], [0, 0, 1]]), mm=False)
    assert len(poses) == len(dets) == len(fed)
    fed = np.concatenate(fed)
    fed_u8 = np.rint(fed * 255.0).astype(np.uint8)
    assert np.array_equal((fed_u8 / 255.).astype(np.float32), fed)
    n_black = int(sum(not c.any() for c in crops[1.2]))
    n_moved = {pf: int(sum(CO.float32_box_ints(b, pf) != CO.reference_box_ints(b, pf) for b in boxes)) for pf in PADS.values()}
    np.savez_compressed(f"{HERE}/crops_edges.npz", scene_sum=np.array([int(img.astype(np.int64).sum()), crc(img)]), frame_hw=np.array([H, W]), pixel_boxes=np.array(px),
                        rel_boxes=rel, boxes_xywh=boxes, crops_pf12=crops[1.2], crops_pf13=crops[1.3],
                        det_classes=classes, class_pad_factors=np.array([[c, p] for c, p in PADS.items()]),
                        process_crops_u8=fed_u8, out_size=np.array(64))
    print("crops_edges.npz: %d boxes, %d black crops, float32 route moves %s; %d B" % (
        len(px), n_black, n_moved, os.path.getsize(f"{HERE}/crops_edges.npz")))


if __name__ == "__main__":
    main()
