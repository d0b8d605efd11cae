"""GPU tests of the drop-in surface: row-sharded codebook (shards emulated on one GPU through the real CUDA entry points),
AePoseEstimator.process end to end on a throw-away workspace, update_embedding."""
import os

import numpy as np
import pytest
import torch

from oracle import aae_oracle as O
from tests.test_gpu_a_parity import _codebook, _enc, sess  # noqa: F401

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("precision", [0, 1])
def test_row_sharded_match_is_bit_identical_to_unsharded(sess, precision):
    """config 5 geometry scaled down: N = 8 shards; the global best sits on each shard in turn, and one query's best row is
    duplicated across shards (the lower global index must win)."""
    from augmentedautoencoder_b200.parallel import ShardedCodebook, shard_bounds
    n, W = 36 * 512, 8
    E = O.make_codebook(21, n=n)
    E[36 * 400 + 3] = E[36 * 10 + 3]
    spans = [shard_bounds(n, W, r, 36) for r in range(W)]
    shards = [ShardedCodebook(E[lo:hi], num_cyclo=36, max_batch=64, precision=precision, row_range=(lo, hi), n_rows_total=n) for lo, hi in spans]
    rows = np.array([lo + 7 for lo, hi in spans] + [36 * 400 + 3, 35, n - 1])
    z = torch.from_numpy((E[rows] * 1.7).astype(np.float32)).cuda()
    k = 4
    def gather(kk, upright):
        """What the NCCL all-gather of the per-rank [2, B, k] exchange buffers produces: [W, 2, B, k]."""
        packed = torch.empty((W, 2, z.shape[0], kk), dtype=torch.int32, device=z.device)
        for r, sh in enumerate(shards):
            sh._local_match(z, kk, upright, packed[r, 0].view(torch.float32), packed[r, 1])
        return packed
    s, i = shards[0]._merge(gather(k, False))
    p = O.make_encoder_params(42)
    cb = _codebook(_enc(0, 64, p), E, max_batch=64, precision=precision)
    s_ref, i_ref = cb.match_device(z, k=1)
    assert np.array_equal(i.cpu().numpy()[:, 0], i_ref.cpu().numpy()[:, 0])
    assert np.array_equal(s.cpu().numpy()[:, 0], s_ref.cpu().numpy()[:, 0])
    want = rows.copy()
    want[W] = 36 * 10 + 3      # duplicate across shards
    want[W + 1] = 0            # cyclo end-point duplicate inside shard 0
    want[W + 2] = n - 36       # last row duplicates row n-36
    assert np.array_equal(i.cpu().numpy()[:, 0], want)
    cos = O.cos_similarity(z.cpu().numpy(), E)
    sk, ik = cb.match_device(z, k=k)          # sharded top-k lists merged == unsharded top-k, bit for bit, in both arithmetic modes
    assert np.array_equal(i.cpu().numpy(), ik.cpu().numpy()) and np.array_equal(s.cpu().numpy(), sk.cpu().numpy())
    for b in range(len(rows)):
        assert np.max(np.abs(s.cpu().numpy()[b] - cos[b, i.cpu().numpy()[b]])) < 2e-6
    _, iu = shards[0]._merge(gather(1, True))
    assert np.array_equal(iu.cpu().numpy()[:, 0], O.select_indices(cos, upright=True, num_cyclo=36))


TRAIN_CFG = """[Paths]
MODEL_PATH: /nonexistent.ply
BACKGROUND_IMAGES_GLOB: /nonexistent/*.jpg
[Dataset]
MODEL: reconst
H: 128
W: 128
C: 3
RADIUS: 700
RENDER_DIMS: (720, 540)
K: [1075.65, 0, 720/2, 0, 1073.90, 540/2, 0, 0, 1]
VERTEX_SCALE: 1
ANTIALIASING: 1
PAD_FACTOR: 1.2
CLIP_NEAR: 10
CLIP_FAR: 10000
NOOF_TRAINING_IMGS: 10
NOOF_BG_IMGS: 10
[Augmentation]
REALISTIC_OCCLUSION: False
[Embedding]
EMBED_BB: True
MIN_N_VIEWS: 162
NUM_CYCLO: 36
[Network]
BATCH_NORMALIZATION: False
AUXILIARY_MASK: False
VARIATIONAL: 0
LOSS: L2
BOOTSTRAP_RATIO: 4
NORM_REGULARIZE: 0
LATENT_SPACE_SIZE: 128
NUM_FILTER: [128, 256, 512, 512]
STRIDES: [2, 2, 2, 2]
KERNEL_SIZE_ENCODER: 5
KERNEL_SIZE_DECODER: 5
[Training]
OPTIMIZER: Adam
NUM_ITER: 30000
BATCH_SIZE: 64
LEARNING_RATE: 2e-4
SAVE_INTERVAL: 10000
[Queue]
NUM_THREADS: 10
QUEUE_SIZE: 50
"""

M3_CFG = """[methods]
object_pose_estimator = auto_pose
[auto_pose]
gpu_memory_fraction = 0.5
color_format = bgr
color_data_type = np.float32
depth_data_type = np.float32
class_2_encoder = {1:'grp/obj_a', 5:'grp/obj_b'}
camPose = False
upright = False
topk = 1
pose_visualization = False
"""


def make_workspace(ws, objects, n):
    """A throw-away AE_WORKSPACE_PATH with one experiment per object under group grp: its train cfg and a checkpoint of
    random encoder weights, an n-row codebook and rendered boxes.  objects: {name: (seed, train cfg text)}.  Returns
    {name: (encoder params, codebook, boxes)}."""
    objs = {}
    for name, (seed, cfg) in objects.items():
        d = ws / "experiments" / "grp" / name
        (d / "checkpoints").mkdir(parents=True)
        (d / (name + ".cfg")).write_text(cfg)
        p = O.make_encoder_params(40 + seed, bias_scale=0.02)
        E = O.make_codebook(60 + seed, n=n)
        rng = np.random.RandomState(seed)
        bbs = np.stack([rng.randint(200, 400, n), rng.randint(100, 300, n), rng.randint(60, 200, n), rng.randint(60, 200, n)], 1).astype(np.int32)
        ckpt = {name + "/" + k: v for k, v in p.items()}
        ckpt[name + "/embedding_normalized"] = E
        ckpt[name + "/embed_obj_bbs_var"] = bbs
        np.savez(d / "checkpoints" / "chkpt-30000.npz", **ckpt)
        objs[name] = (p, E, bbs)
    return objs


def test_pose_estimator_process_end_to_end(tmp_path, monkeypatch):
    """Two object classes, five detections (one of an unknown class), one frame: every detection must get exactly the pose
    the reference algorithm yields (crop -> encoder -> codebook NN -> pose lift), restated with the CPU oracle."""
    import cv2
    from augmentedautoencoder_b200.ae import factory
    from augmentedautoencoder_b200.ae.dataset import Dataset
    from augmentedautoencoder_b200.m3_interface.ae_pose_estimator import AePoseEstimator
    from augmentedautoencoder_b200.m3_interface.m3_interfaces import BoundingBox
    ws = tmp_path / "ws"
    monkeypatch.setenv("AE_WORKSPACE_PATH", str(ws))
    ds = Dataset(None, min_n_views=162, num_cyclo=36, radius=700)
    n = ds.embedding_size
    objs = make_workspace(ws, {"obj_a": (1, TRAIN_CFG), "obj_b": (2, TRAIN_CFG)}, n)
    cfg_path = tmp_path / "m3.cfg"
    cfg_path.write_text(M3_CFG)
    est = AePoseEstimator(str(cfg_path))
    assert est.query_process_requirements() == ['color_img', 'camK', 'bboxes'] and est.class_2_encoder == {1: 'grp/obj_a', 5: 'grp/obj_b'}
    assert set(est.all_codebooks) == {1, 5} and est.pad_factors[1] == 1.2 and est.patch_sizes[5] == (128, 128)
    scene = O.make_crops_u8(77, 1, hw=128)[0]
    scene = cv2.resize(scene, (640, 480), interpolation=cv2.INTER_CUBIC)
    K = np.array([[572.4114, 0, 325.2611], [0, 573.57043, 242.04899], [0, 0, 1]])
    dets = [BoundingBox(0.2, 0.25, 0.45, 0.6, {1: 0.9, 5: 0.1}), BoundingBox(0.5, 0.1, 0.9, 0.5, {7: 0.9}),
            BoundingBox(0.6, 0.5, 0.95, 0.9, {5: 0.8}), BoundingBox(0.05, 0.05, 0.3, 0.4, {5: 0.7, 1: 0.2}), BoundingBox(0.4, 0.4, 0.7, 0.8, {1: 1.0})]
    poses = est.process(dets, scene, K, mm=True)
    assert [p_.name for p_ in poses] == [1, 5, 5, 1]
    k_train = np.array([1075.65, 0, 360, 0, 1073.90, 270, 0, 0, 1]).reshape(3, 3)
    j = 0
    for det in dets:
        cls = max(det.classes, key=det.classes.get)
        if cls not in (1, 5):
            continue
        p, E, bbs = objs["obj_a" if cls == 1 else "obj_b"]
        box = [det.xmin * 640, det.ymin * 480, (det.xmax - det.xmin) * 640, (det.ymax - det.ymin) * 480]
        crop = est.extract_square_patch(scene, box, 1.2, resize=(128, 128), interpolation=cv2.INTER_LINEAR, black_borders=True)
        idc = O.nearest_rotation_idcs(crop, p, E)
        R, t = O.auto_pose6d_lift(idc, ds.viewsphere_for_embedding, bbs, box, K, k_train, 700.0)
        H = np.eye(4)
        H[:3, :3], H[:3, 3] = R.squeeze(), t.squeeze()
        assert np.array_equal(poses[j].trafo, H), (j, cls)
        j += 1
    poses_m = est.process(dets[:1], scene, K, mm=False)
    assert np.allclose(poses_m[0].trafo[:3, 3] * 1000.0, poses[0].trafo[:3, 3])


def test_update_embedding_builds_a_normalised_codebook(sess):
    from augmentedautoencoder_b200.ae.codebook import Codebook
    from augmentedautoencoder_b200.ae.dataset import Dataset
    ds = Dataset(None, min_n_views=12, num_cyclo=4, radius=700)
    p = O.make_encoder_params(42)
    enc = _enc(0, 16, p)
    cb = Codebook(enc, ds, True, max_batch=16)
    n = ds.embedding_size
    crops = O.make_crops_u8(5, n)
    bbs = np.arange(n * 4).reshape(n, 4)
    cb.update_embedding_from_crops(sess, crops, bbs, batch_size=16)
    E = sess.run(cb.embedding_normalized)
    z = O.encoder_forward(O.preprocess(crops), p)
    want = (z.astype(np.float64) / np.linalg.norm(z.astype(np.float64), axis=1, keepdims=True)).astype(np.float32)
    assert E.shape == (n, 128) and np.max(np.abs(E - want)) < 2e-6
    assert np.array_equal(sess.run(cb.embed_obj_bbs_var), bbs)
    idc = cb.nearest_rotation(sess, crops[:5], return_idcs=True)   # every view must find itself
    assert np.array_equal(idc, np.arange(5))
    with pytest.raises(NotImplementedError):
        cb.update_embedding(sess, 16)                               # rendering needs a user-supplied renderer


def test_async_streaming_call_matches_blocking_call(sess):
    p = O.make_encoder_params(42)
    E = O.make_codebook(7, n=36 * 300)
    enc = _enc(1, 64, p)
    cb = _codebook(enc, E, max_batch=64, precision=1)
    batches = [torch.from_numpy(O.make_crops_u8(100 + i, 64)).pin_memory() for i in range(4)]
    want = [cb.nearest_rotation(sess, b, return_idcs=True) for b in batches]
    pend = [cb.nearest_rotation_async(sess, b) for b in batches]      # all four in flight
    got = [h.result() for h in pend]
    for w, g_ in zip(want, got):
        assert g_.dtype == np.int64 and np.array_equal(w, g_)
    assert np.array_equal(cb.nearest_rotation_async(sess, batches[0].numpy()).result(), want[0])   # pageable numpy input works too


def test_device_crops_are_bit_exact_with_opencv(sess, golden_dir):
    """aae_extract_square_patches against (a) the crops the REFERENCE's extract_square_patch produced (golden) and (b) cv2 on
    random boxes of many sizes, including up- and down-scaling and boxes touching the frame border."""
    import cv2
    from augmentedautoencoder_b200.m3_interface.ae_pose_estimator import AePoseEstimator
    c = np.load(os.path.join(golden_dir, "crops_process.npz"))
    scene = np.random.RandomState(int(c["scene_seed"])).randint(0, 256, size=tuple(c["scene_shape"]), dtype=np.uint8)
    est = AePoseEstimator.__new__(AePoseEstimator)
    frame = torch.from_numpy(scene).cuda()
    got = est.extract_square_patches_device(frame, c["boxes"], 1.2, (128, 128)).cpu().numpy()
    assert np.array_equal(got, c["crops_black_borders_linear"])
    rng = np.random.RandomState(3)
    boxes = []
    for _ in range(200):
        w, h = rng.randint(8, 400), rng.randint(8, 400)
        x, y = rng.randint(0, 640 - min(w, 639)), rng.randint(0, 480 - min(h, 479))
        w, h = min(w, 640 - x), min(h, 480 - y)
        boxes.append([x + rng.rand() * 0.9, y + rng.rand() * 0.9, w + rng.rand() * 0.9, h + rng.rand() * 0.9])
    boxes += [[0, 0, 640, 480], [0, 0, 1, 1], [639, 479, 1, 1], [100, 100, 128, 128], [10, 20, 256, 256]]
    for pf in (1.2, 1.0, 1.37):
        got = est.extract_square_patches_device(frame, boxes, pf, (128, 128)).cpu().numpy()
        for b, g_ in zip(boxes, got):
            want = est.extract_square_patch(scene, b, pf, resize=(128, 128), interpolation=cv2.INTER_LINEAR, black_borders=True)
            assert np.array_equal(g_, want), (b, pf, int((g_ != want).sum()))
