"""GPU tests of the single-pass fp16 inference precision (AAE_PREC_TC_FP16): every operand rounded once to fp16, one
hi*hi product per K step.  The bounds come from the rounding model (include/aae_b200.h, DESIGN.md section 3), not from
measurement: each product carries relative error <= 2^-10 + 2^-22, so a layer output may deviate by 2^-9 * sum|a*w| (twice
that, room for the fp32 accumulation) + 2^-10 * |y| (hi-only storage of the output) + an fp16-subnormal term.  How often the
fp16 and split paths pick different rows is printed, not asserted."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import aae_oracle as O
from tests.test_gpu_a_parity import _codebook, _enc, sess  # noqa: F401

pytestmark = pytest.mark.gpu

FP16 = 2
SPLIT = 1
PROD = 2.0 ** -9           # bound on sum|a*w| relative error (twice the single-product bound)
STORE = 2.0 ** -10         # hi-only storage of a layer output
# fp16 subnormals: spacing 2^-24, so a stored value carries absolute error <= 2^-25 / scale
SUB_ACT = 2.0 ** -25 / 16.0        # activations are stored as 16 * x
SUB_W = 2.0 ** -25 / 256.0         # weights as 256 * w


def _conv_bound_check(a, w, b, y16, what):
    """a: layer input [B,H,W,C] as the fp16 path read it, w HWIO, y16 the fp16 path's post-ReLU output."""
    a64, w64, b64 = (torch.from_numpy(np.ascontiguousarray(t)).double() for t in (a, w, b))
    with torch.no_grad():
        y64 = O.conv2d_same(a64, w64, b64, 2, "relu").numpy()
        S = O.conv2d_same(a64.abs(), w64.abs(), torch.zeros_like(b64), 2, None).numpy()
    K = w.shape[0] * w.shape[1] * w.shape[2]
    eps_sub = SUB_ACT * np.abs(w).reshape(K, -1).sum(0) + SUB_W * K * np.abs(a).max() + SUB_ACT
    err = np.abs(y16.astype(np.float64) - y64)
    bound = PROD * S + STORE * np.abs(y64) + eps_sub
    worst = float(np.max(err / bound))
    print("%s: max |y16 - y64| = %.3e, worst error / bound = %.3f" % (what, err.max(), worst))
    assert worst <= 1.0, what


def _dense_bound_check(flat, W, b, z16):
    a64, W64 = flat.astype(np.float64), W.astype(np.float64)
    y64 = a64 @ W64 + b.astype(np.float64)
    S = np.abs(a64) @ np.abs(W64)
    eps_sub = SUB_ACT * np.abs(W64).sum(0) + SUB_W * W.shape[0] * np.abs(a64).max()
    err = np.abs(z16.astype(np.float64) - y64)
    bound = PROD * S + STORE * np.abs(y64) + eps_sub
    print("dense: max |z16 - z64| = %.3e, worst error / bound = %.3f" % (err.max(), float(np.max(err / bound))))
    assert np.all(err <= bound)


@pytest.mark.parametrize("feed", ["uint8", "float"])
def test_fp16_layers_meet_the_rounding_bound(sess, feed):
    p = O.make_encoder_params(42, bias_scale=0.05)
    enc = _enc(FP16, 4, p)
    xu8 = O.make_crops_u8(1234, 4)
    x = xu8 if feed == "uint8" else O.preprocess(xu8)
    z = sess.run(enc.z, {enc.x: x})
    a = O.preprocess(xu8).astype(np.float64) if feed == "uint8" else x     # u8 feed: the kernel reads the byte itself, a = byte / 255
    for layer in range(4):
        name = "conv2d" if layer == 0 else "conv2d_%d" % layer
        y16 = enc.activation_device(layer, sess.device).cpu().numpy()
        _conv_bound_check(a, p[name + "/kernel"], p[name + "/bias"], y16, "%s feed, conv %d" % (feed, layer + 1))
        a = y16
    flat = sess.run(enc.encoder_out, {enc.x: x})
    assert np.array_equal(flat, a.reshape(a.shape[0], -1))
    _dense_bound_check(flat, p["dense/kernel"], p["dense/bias"], z)
    # and the split path's latent, for the record (not asserted)
    enc1 = _enc(SPLIT, 4, p)
    z1 = sess.run(enc1.z, {enc1.x: x})
    print("%s feed: max |z_fp16 - z_split| / max |z_split| = %.3e" % (feed, np.abs(z - z1).max() / np.abs(z1).max()))


def _check_match(z, E, s, i, k, upright=False, num_cyclo=36):
    """The score, index and ordering bounds of the fp16 match, against float64 cosines of the latent the match was given."""
    cos64 = O.cos_similarity(z.astype(np.float64), E.astype(np.float64))
    cand = np.arange(E.shape[0])
    if upright:
        cand = cand[cand % num_cyclo == 0]
        assert np.all(i % num_cyclo == 0)
    best = -np.sort(-cos64[:, cand], axis=1)[:, :k]
    for b in range(z.shape[0]):
        got = cos64[b, i[b]]
        assert np.max(np.abs(s[b] - got)) <= PROD, (b, s[b], got)
        assert np.all(got >= best[b] - 2 * PROD), (b, got, best[b])
        assert np.all(np.diff(s[b]) <= 0) and len(set(i[b].tolist())) == k, (b, s[b], i[b])
    return cos64


def _agreement(tag, i16, i1, s16, s1):
    d = np.nonzero(i16[:, 0] != i1[:, 0])[0]
    print("%s: top-1 differs from split for %d of %d queries; max |score_fp16 - score_split| = %.3e"
          % (tag, len(d), i16.shape[0], float(np.max(np.abs(s16[:, 0] - s1[:, 0])))))


@pytest.mark.parametrize("n_rows,batch", [(64 * 5 + 17, 100), (64 * 300, 256), (36 * 700, 5), (92232, 129), (92232, 1)])
def test_fp16_match_meets_the_rounding_bound(sess, n_rows, batch):
    num_cyclo = 36 if n_rows % 36 == 0 else 1
    E = O.make_codebook(5, n=n_rows, num_cyclo=num_cyclo, duplicate_cyclo_endpoints=(num_cyclo == 36))
    p = O.make_encoder_params(42)
    cb = _codebook(_enc(FP16, 256, p), E, num_cyclo=num_cyclo, max_batch=256, precision=FP16)
    cb1 = _codebook(_enc(SPLIT, 256, p), E, num_cyclo=num_cyclo, max_batch=256, precision=SPLIT)
    rng = np.random.RandomState(n_rows + batch)
    z = (rng.standard_normal((batch, 128)) * rng.uniform(0.05, 50, (batch, 1))).astype(np.float32)
    if num_cyclo == 36:
        z[0] = E[36 * 3] * 2.0                 # a query that IS a duplicated row: rows 108 and 143 tie exactly
    zd = torch.from_numpy(z).cuda()
    for k in (1, 3, 8):
        s, i = (t.cpu().numpy() for t in cb.match_device(zd, k=k))
        _check_match(z, E, s, i, k)
        if num_cyclo == 36:
            assert i[0, 0] == 108 and (k == 1 or (i[0, 1] == 143 and s[0, 0] == s[0, 1]))
        s2, i2 = (t.cpu().numpy() for t in cb.match_device(zd, k=k))      # the last CTA re-arms the scratch
        assert np.array_equal(s2, s) and np.array_equal(i2, i)
        if k == 1:
            s1, i1 = (t.cpu().numpy() for t in cb1.match_device(zd, k=1))
            _agreement("match %d rows, batch %d" % (n_rows, batch), i, i1, s, s1)
    if num_cyclo == 36:
        for k in (1, 4):
            su, iu = (t.cpu().numpy() for t in cb.match_device(zd, k=k, upright=True))
            _check_match(z, E, su, iu, k, upright=True)
            assert iu[0, 0] == 108


@pytest.mark.parametrize("batch", [1, 2, 63, 127, 129, 255, 300])
def test_fp16_ragged_batches_end_to_end(sess, batch):
    """Small-batch split-K, partial tiles and host chunking above max_batch: the score and index bounds hold against the
    fp16 path's own latent."""
    p = O.make_encoder_params(42, bias_scale=0.03)
    E = O.make_codebook(9, n=36 * 700 + 5, num_cyclo=1, duplicate_cyclo_endpoints=False)
    crops = O.make_crops_u8(77 + batch, batch)
    res = {}
    for prec in (SPLIT, FP16):
        enc = _enc(prec, 256, p)
        cb = _codebook(enc, E, num_cyclo=1, max_batch=256, precision=prec)
        z = sess.run(enc.z, {enc.x: crops})
        s, i = cb.nearest_idx_device(torch.from_numpy(crops).cuda())
        res[prec] = (z, s.cpu().numpy(), i.cpu().numpy())
    z16, s16, i16 = res[FP16]
    assert z16.shape == (batch, 128) and np.all(np.isfinite(z16))
    _check_match(z16, E, s16, i16, 1)
    _agreement("ragged batch %d" % batch, i16, res[SPLIT][2], s16, res[SPLIT][1])


@pytest.mark.parametrize("k", [1, 4])
def test_fp16_row_sharded_match_is_bit_identical_to_unsharded(sess, k):
    from augmentedautoencoder_b200 import _lib
    lib = _lib.lib()
    n, B = 36 * 700, 64
    E = O.make_codebook(13, n=n)
    z = torch.from_numpy((np.random.RandomState(3).standard_normal((B, 128)) * 3).astype(np.float32)).cuda()
    z[1] = torch.from_numpy(E[36 * 10 + 3] * 0.5).cuda()            # a row of the first shard
    z[2] = torch.from_numpy(E[n - 36] * 4.0).cuda()                 # a row of the second shard
    cut = 36 * 333
    handles = []
    try:
        for lo, hi in ((0, cut), (cut, n), (0, n)):
            h = C.c_void_p()
            part = np.ascontiguousarray(E[lo:hi])
            _lib.check(lib.aae_codebook_create(0, _lib.ptr(part), hi - lo, 128, 36, lo, B, FP16, C.byref(h)), "codebook create")
            handles.append(h)
        packed = torch.empty((2, 2, B, k), dtype=torch.float32, device="cuda")     # [shard][scores | indices][B][k]
        for sh in range(2):
            idx_view = packed[sh, 1].view(torch.int32)
            _lib.check(lib.aae_codebook_match(handles[sh], _lib.ptr(z), B, k, 0, _lib.ptr(packed[sh, 0]), _lib.ptr(idx_view), None), "match")
        s, i = torch.empty((B, k), device="cuda"), torch.empty((B, k), dtype=torch.int32, device="cuda")
        _lib.check(lib.aae_topk_merge_packed(_lib.ptr(packed), 2, B, k, _lib.ptr(s), _lib.ptr(i), None), "merge")
        s0, i0 = torch.empty((B, k), device="cuda"), torch.empty((B, k), dtype=torch.int32, device="cuda")
        _lib.check(lib.aae_codebook_match(handles[2], _lib.ptr(z), B, k, 0, _lib.ptr(s0), _lib.ptr(i0), None), "match")
        torch.cuda.synchronize()
        assert torch.equal(i, i0) and torch.equal(s, s0)
        assert int(i[1, 0]) == 36 * 10 + 3 and int(i[2, 0]) == n - 36
    finally:
        for h in handles:
            lib.aae_codebook_destroy(h)


def test_fp16_range_guard_reports_overflow(sess):
    """The same static scales as the split mode: out-of-range weights and activations fail loudly, naming the layer."""
    from augmentedautoencoder_b200._lib import AaeError
    p = O.make_encoder_params(42, bias_scale=0.05)
    crops = O.make_crops_u8(5, 3)
    bad_w = dict(p)
    bad_w["conv2d_2/kernel"] = p["conv2d_2/kernel"].copy()
    bad_w["conv2d_2/kernel"][1, 2, 3, 4] = 300.0
    enc = _enc(FP16, 4, bad_w)
    with pytest.raises(AaeError, match=r"AAE_PREC_TC_FP16.*weight.*layer\(s\) 2"):
        sess.run(enc.z, {enc.x: crops})
    for name, layer in (("conv2d/bias", 0), ("conv2d_1/bias", 1)):
        bad_a = dict(p)
        bad_a[name] = p[name].copy()
        bad_a[name][7] = 5000.0
        enc = _enc(FP16, 4, bad_a)
        for feed in (crops, O.preprocess(crops)):
            with pytest.raises(AaeError, match=r"activation.*layer\(s\) %d" % layer):
                sess.run(enc.z, {enc.x: feed})
        cb = _codebook(enc, O.make_codebook(3, n=36 * 20), max_batch=4, precision=FP16)
        with pytest.raises(AaeError, match="activation"):
            cb.nearest_rotation(sess, crops, return_idcs=True)
        with pytest.raises(AaeError, match="activation"):
            cb.nearest_rotation_async(sess, torch.from_numpy(crops)).result()
        enc.load_weights(p)
        assert np.all(np.isfinite(sess.run(enc.z, {enc.x: crops})))


def test_fp16_refusals_leave_the_process_healthy(sess):
    from augmentedautoencoder_b200 import _lib
    from augmentedautoencoder_b200.ae.ae import AE
    from augmentedautoencoder_b200.ae.ae_factory import TrainOp
    from augmentedautoencoder_b200.ae.decoder import Decoder
    from augmentedautoencoder_b200.ae.encoder import Encoder
    from augmentedautoencoder_b200.ae.session import placeholder
    lib = _lib.lib()

    def cfg(prec):
        return _lib.make_cfg(128, 128, 3, list(O.NUM_FILTER), list(O.STRIDES), 5, 128, 4, prec)
    # the decoder is refused at fp16 with AAE_ERR_UNSUPPORTED
    h = C.c_void_p()
    assert lib.aae_decoder_create(0, C.byref(cfg(FP16)), C.byref(h)) == -3 and not h.value
    assert b"inference-only" in lib.aae_last_error_string()
    # precision 3 is not an aae_precision
    for create in (lib.aae_encoder_create, lib.aae_decoder_create):
        assert create(0, C.byref(cfg(3)), C.byref(h)) == -1 and not h.value
        assert b"precision" in lib.aae_last_error_string()
    E = O.make_codebook(1, n=100, num_cyclo=1, duplicate_cyclo_endpoints=False)
    assert lib.aae_codebook_create(0, _lib.ptr(E), 100, 128, 1, 0, 8, 3, C.byref(h)) == -1 and not h.value
    # the trainer refuses an fp16 encoder, here with a split decoder
    eh, dh = C.c_void_p(), C.c_void_p()
    _lib.check(lib.aae_encoder_create(0, C.byref(cfg(FP16)), C.byref(eh)), "encoder create")
    _lib.check(lib.aae_decoder_create(0, C.byref(cfg(SPLIT)), C.byref(dh)), "decoder create")
    try:
        th = C.c_void_p()
        assert lib.aae_trainer_create(eh, dh, 4, 2e-4, 0.9, 0.999, 1e-8, C.byref(th)) == -3 and not th.value
        assert b"inference-only" in lib.aae_last_error_string()
    finally:
        lib.aae_encoder_destroy(eh)
        lib.aae_decoder_destroy(dh)
    # TrainOp raises instead of switching the caller's precision
    x, y = placeholder(np.float32, [None, 128, 128, 3]), placeholder(np.float32, [None, 128, 128, 3])
    enc = Encoder(x, 128, list(O.NUM_FILTER), 5, list(O.STRIDES), False, is_training=True, max_batch=4, precision=FP16)
    dec = Decoder(y, enc.z, list(reversed(O.NUM_FILTER)), 5, list(reversed(O.STRIDES)), "L2", 4, False, False, is_training=True, max_batch=4,
                  precision=SPLIT)
    top = TrainOp(AE(enc, dec, 0, 0), 2e-4)
    with pytest.raises(_lib.AaeError, match="inference-only"):
        top.trainer(sess.device)
    assert enc.precision == FP16 and dec.precision == SPLIT
    # nothing sticky: a split-mode match still runs in this process
    cb = _codebook(_enc(SPLIT, 8, O.make_encoder_params(42)), O.make_codebook(3, n=36 * 20), max_batch=8, precision=SPLIT)
    s, i = cb.match_device(torch.randn(5, 128, device="cuda"))
    torch.cuda.synchronize()
    assert np.all(np.isfinite(s.cpu().numpy()))


def test_fp16_pose_estimator_and_async_calls(tmp_path, monkeypatch, sess):
    """AePoseEstimator(precision=PREC_TC_FP16).process and Codebook.nearest_rotation_async: poses equal the split path's
    wherever the chosen rows agree; where they differ the index bound holds."""
    import cv2
    from augmentedautoencoder_b200.ae.dataset import Dataset
    from augmentedautoencoder_b200.m3_interface.ae_pose_estimator import AePoseEstimator
    from augmentedautoencoder_b200.m3_interface.m3_interfaces import BoundingBox
    from tests.test_gpu_c_plugin import M3_CFG, TRAIN_CFG
    ws = tmp_path / "ws"
    monkeypatch.setenv("AE_WORKSPACE_PATH", str(ws))
    n = Dataset(None, min_n_views=162, num_cyclo=36, radius=700).embedding_size
    for name, seed in (("obj_a", 1), ("obj_b", 2)):
        d = ws / "experiments" / "grp" / name
        (d / "checkpoints").mkdir(parents=True)
        (d / (name + ".cfg")).write_text(TRAIN_CFG)
        rng = np.random.RandomState(seed)
        ckpt = {name + "/" + k: v for k, v in O.make_encoder_params(40 + seed, bias_scale=0.02).items()}
        ckpt[name + "/embedding_normalized"] = O.make_codebook(60 + seed, n=n)
        ckpt[name + "/embed_obj_bbs_var"] = np.stack([rng.randint(200, 400, n), rng.randint(100, 300, n), rng.randint(60, 200, n),
                                                      rng.randint(60, 200, n)], 1).astype(np.int32)
        np.savez(d / "checkpoints" / "chkpt-30000.npz", **ckpt)
    cfg_path = tmp_path / "m3.cfg"
    cfg_path.write_text(M3_CFG)
    est = {prec: AePoseEstimator(str(cfg_path), precision=prec) for prec in (SPLIT, FP16)}
    assert all(cb.precision == FP16 and cb._encoder.precision == FP16 for cb in est[FP16].all_codebooks.values())
    scene = cv2.resize(O.make_crops_u8(77, 1, hw=128)[0], (640, 480), interpolation=cv2.INTER_CUBIC)
    K = np.array([[572.4114, 0, 325.2611], [0, 573.57043, 242.04899], [0, 0, 1]])
    dets = [BoundingBox(0.2, 0.25, 0.45, 0.6, {1: 0.9, 5: 0.1}), BoundingBox(0.6, 0.5, 0.95, 0.9, {5: 0.8}),
            BoundingBox(0.05, 0.05, 0.3, 0.4, {5: 0.7, 1: 0.2}), BoundingBox(0.4, 0.4, 0.7, 0.8, {1: 1.0})]
    poses = {prec: e.process(dets, scene, K, mm=True) for prec, e in est.items()}
    assert [p_.name for p_ in poses[FP16]] == [p_.name for p_ in poses[SPLIT]] == [1, 5, 5, 1]
    crops = []
    for j, det in enumerate(dets):
        cls = max(det.classes, key=det.classes.get)
        box = [det.xmin * 640, det.ymin * 480, (det.xmax - det.xmin) * 640, (det.ymax - det.ymin) * 480]
        crop = est[FP16].extract_square_patch(scene, box, 1.2, resize=(128, 128), interpolation=cv2.INTER_LINEAR, black_borders=True)
        crops.append(crop)
        idx = {prec: int(est[prec].all_codebooks[cls].nearest_rotation(est[prec].sess, crop, return_idcs=True)[0]) for prec in (SPLIT, FP16)}
        if idx[SPLIT] == idx[FP16]:
            assert np.array_equal(poses[FP16][j].trafo, poses[SPLIT][j].trafo), j
        else:
            cb = est[FP16].all_codebooks[cls]
            z16 = cb._encoder.encode_device(torch.from_numpy(crop[None]).cuda()).cpu().numpy()
            E = cb.embedding_normalized.value()
            cos = O.cos_similarity(z16.astype(np.float64), E.astype(np.float64))[0]
            assert cos[idx[FP16]] >= cos.max() - 2 * PROD
        print("pose estimator detection %d: split row %d, fp16 row %d" % (j, idx[SPLIT], idx[FP16]))
    # the streaming call gives the blocking call's rows at fp16
    cb = est[FP16].all_codebooks[1]
    batch = torch.from_numpy(np.stack(crops)).pin_memory()
    want = cb.nearest_rotation(est[FP16].sess, batch, return_idcs=True)
    got = cb.nearest_rotation_async(est[FP16].sess, batch).result()
    assert np.array_equal(want, got)
