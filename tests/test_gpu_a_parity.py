"""GPU parity tests: the CUDA path (through the ctypes -> C ABI boundary) against the CPU oracle on the same seeded
inputs.  Tolerances: indices bit-exact; cosine scores |d| <= 1e-5 (BASELINE.json north_star)."""

import numpy as np
import pytest
import torch

from oracle import aae_oracle as O

pytestmark = pytest.mark.gpu

COS_TOL = 1e-5


@pytest.fixture(scope="module")
def sess():
    from augmentedautoencoder_b200 import build_ext
    build_ext.build()
    from augmentedautoencoder_b200.ae.session import Session
    torch.cuda.set_device(0)
    return Session(device=0)


def _enc(precision, max_batch, params, num_filters=O.NUM_FILTER, strides=O.STRIDES, hw=128, latent=128):
    from augmentedautoencoder_b200.ae.encoder import Encoder
    from augmentedautoencoder_b200.ae.session import placeholder
    x = placeholder(np.float32, [None, hw, hw, 3])
    e = Encoder(x, latent, list(num_filters), 5, list(strides), False, precision=precision, max_batch=max_batch)
    e.load_weights(params)
    return e


def _codebook(enc, E, num_cyclo=36, max_batch=None, precision=None):
    from augmentedautoencoder_b200.ae.codebook import Codebook

    class DS:  # the Codebook only needs these two members of Dataset
        embedding_size = E.shape[0]
        _kw = {"num_cyclo": str(num_cyclo)}
        viewsphere_for_embedding = np.zeros((E.shape[0], 3, 3))
    cb = Codebook(enc, DS(), True, max_batch=max_batch, precision=precision)
    cb.embedding_normalized.assign(E)
    return cb


# --------------------------------------------------------------------------------------- encoder
@pytest.mark.parametrize("hw,filters,strides,batch", [(32, (8, 16), (2, 2), 3), (16, (4, 8, 8), (2, 2, 1), 5)])
def test_small_encoder_matches_oracle(sess, hw, filters, strides, batch):
    p = O.make_encoder_params(3, num_filters=filters, in_hw=hw, strides=strides, latent=16, bias_scale=0.1)
    enc = _enc(0, 8, p, filters, strides, hw, 16)
    xu8 = O.make_crops_u8(4, batch, hw=hw)
    z = sess.run(enc.z, {enc.x: xu8})
    z64 = O.encoder_forward(O.preprocess(xu8), p, strides=strides, dtype=torch.float64)
    assert z.shape == (batch, 16)
    assert np.max(np.abs(z - z64)) < 2e-6 * max(1.0, np.abs(z64).max())
    zf = sess.run(enc.z, {enc.x: O.preprocess(xu8)})  # float feed must agree bit-for-bit with the fused u8/255 path
    assert np.array_equal(z, zf)


def test_full_encoder_layers_and_latent_match_oracle(sess):
    p = O.make_encoder_params(42, bias_scale=0.05)
    enc = _enc(0, 4, p)
    xu8 = O.make_crops_u8(1234, 4)
    z = sess.run(enc.z, {enc.x: xu8})
    outs64 = O.encoder_layers(O.preprocess(xu8), p, dtype=torch.float64)
    for layer in range(4):
        a = enc.activation_device(layer, sess.device).cpu().numpy()
        ref = outs64[layer].numpy()
        assert a.shape == ref.shape
        assert np.max(np.abs(a - ref)) < 1e-5 * max(1.0, np.abs(ref).max()), "layer %d" % layer
    flat = sess.run(enc.encoder_out, {enc.x: xu8})
    assert np.max(np.abs(flat - outs64[4].numpy())) < 1e-5
    z64 = outs64[5].numpy()
    z32 = O.encoder_forward(O.preprocess(xu8), p)
    err_gpu, err_cpu32 = np.max(np.abs(z - z64)), np.max(np.abs(z32 - z64))
    assert err_gpu < 5e-6 * np.abs(z64).max() + 1e-6, (err_gpu, err_cpu32)


def test_asymmetric_same_padding_known_answer(sess):
    # one-hot kernel tap (0,0) reads pixel (2*o - 1): TF 'SAME' pads 1 before / 2 after for k=5, s=2 (F4)
    p = O.make_encoder_params(1, num_filters=(4,), in_hw=16, strides=(2,), latent=4)
    p["conv2d/kernel"][:] = 0
    p["conv2d/kernel"][0, 0, 0, 0] = 1.0
    enc = _enc(0, 2, p, (4,), (2,), 16, 4)
    x = np.zeros((1, 16, 16, 3), np.float32)
    x[0, 1, 1, 0] = 1.0
    sess.run(enc.z, {enc.x: x})
    a = enc.activation_device(0, sess.device).cpu().numpy()
    assert a[0, 1, 1, 0] == 1.0 and a.sum() == 1.0


# --------------------------------------------------------------------------------------- codebook
def test_l2_normalize_matches_oracle(sess):
    from augmentedautoencoder_b200 import _lib
    z = np.random.RandomState(0).randn(37, 128).astype(np.float32)
    z[5] = 0
    zd = torch.from_numpy(z).cuda()
    out = torch.empty_like(zd)
    _lib.check(_lib.lib().aae_l2_normalize(_lib.ptr(zd), 37, 128, _lib.ptr(out), None))
    assert np.max(np.abs(out.cpu().numpy() - O.l2_normalize(z))) < 2e-7
    assert np.all(out[5].cpu().numpy() == 0)


@pytest.mark.parametrize("precision", [0, 1])
def test_match_full_codebook_argmax_bit_exact_10k_queries(sess, precision):
    """10 000 synthetic queries against the 92 232-row codebook (with the duplicate cyclo end-point rows real codebooks
    have): index bit-exact vs the fp32 oracle wherever the fp64 top-2 gap exceeds fp32 resolution, scores within 1e-5.
    precision 0 = fp32 CUDA-core kernel, 1 = the tensor-core kernel bench.py times (codebook.py:63-68 semantics for both)."""
    E = O.make_codebook(7)
    p = O.make_encoder_params(42)
    enc = _enc(precision, 256, p)
    cb = _codebook(enc, E, max_batch=256, precision=precision)
    rng = np.random.RandomState(99)
    n_q = 10000
    z = (rng.standard_normal((n_q, 128)) * rng.uniform(0.1, 30, (n_q, 1))).astype(np.float32)
    zd = torch.from_numpy(z).cuda()
    scores, idx = cb.match_device(zd)
    scores, idx = scores.cpu().numpy()[:, 0], idx.cpu().numpy()[:, 0]
    mism, max_err = 0, 0.0
    E64 = E.astype(np.float64)
    for a in range(0, n_q, 1000):
        cos32 = O.cos_similarity(z[a:a + 1000], E)
        want = np.argmax(cos32, axis=1)
        got = idx[a:a + 1000]
        max_err = max(max_err, np.max(np.abs(scores[a:a + 1000] - cos32[np.arange(len(got)), got])))
        bad = np.nonzero(want != got)[0]
        for b in bad:  # legitimate only if fp64 says the two candidates are closer than fp32 can resolve
            c64 = O.l2_normalize(z[a + b:a + b + 1].astype(np.float64)) @ E64[[want[b], got[b]]].T
            assert abs(c64[0, 0] - c64[0, 1]) < 2e-7, ("argmax mismatch beyond fp32 resolution", a + b, want[b], got[b], c64)
            mism += 1
    assert max_err <= COS_TOL, max_err
    assert mism <= 3, mism
    print("10k queries, precision %d: %d near-tie index differences (fp64 gap < 2e-7), max |dcos| = %.2e" % (precision, mism, max_err))


@pytest.mark.parametrize("precision", [0, 1])
def test_duplicate_rows_resolve_to_lowest_index_and_upright(sess, precision):
    E = O.make_codebook(7, n=36 * 200)
    p = O.make_encoder_params(42)
    enc = _enc(precision, 64, p)
    cb = _codebook(enc, E, max_batch=64, precision=precision)
    # queries that ARE codebook rows: rows v*36+35 duplicate v*36+0 -> the answer must be v*36 (np.argmax semantics, F7/F8)
    rows = np.array([35, 36 * 7 + 35, 36 * 150, 36 * 199 + 35, 17, 36 * 3 + 1])
    z = (E[rows] * 3.7).astype(np.float32)
    s, i = cb.match_device(torch.from_numpy(z).cuda())
    want = np.where(rows % 36 == 35, rows - 35, rows)
    assert np.array_equal(i.cpu().numpy()[:, 0], want)
    assert np.allclose(s.cpu().numpy()[:, 0], 1.0, atol=2e-6)
    cos = O.cos_similarity(z, E)
    assert np.array_equal(want, np.argmax(cos, axis=1))
    # upright: arg-max over every 36th row only (codebook.py:66)
    su, iu = cb.match_device(torch.from_numpy(z).cuda(), upright=True)
    want_u = O.select_indices(cos, upright=True, num_cyclo=36)
    assert np.array_equal(iu.cpu().numpy()[:, 0], want_u)
    # top-k: scores descending, ties by ascending index; same set + scores as the oracle's argpartition/argsort
    sk, ik = cb.match_device(torch.from_numpy(z[:1]).cuda(), k=8)
    sk, ik = sk.cpu().numpy()[0], ik.cpu().numpy()[0]
    ref = O.select_indices(cos[:1], top_n=8)
    assert set(ik.tolist()) == set(ref.tolist()) or np.allclose(np.sort(cos[0, ik]), np.sort(cos[0, ref]), atol=1e-7)
    assert np.all(np.diff(sk) <= 0) and ik[0] == 0 and ik[1] == 35
    assert np.max(np.abs(sk - cos[0, ik])) < COS_TOL


def test_cosine_matrix_fetch_matches_oracle(sess):
    E = O.make_codebook(11, n=5000)
    p = O.make_encoder_params(5, num_filters=(8, 16), in_hw=32, strides=(2, 2), latent=128)
    enc = _enc(0, 16, p, (8, 16), (2, 2), 32, 128)
    cb = _codebook(enc, E, max_batch=16)
    xu8 = O.make_crops_u8(8, 9, hw=32)
    cos = sess.run(cb.cos_similarity, {enc.x: xu8})
    z = O.encoder_forward(O.preprocess(xu8), p, strides=(2, 2))
    ref = O.cos_similarity(z, E)
    assert cos.shape == (9, 5000)
    assert np.max(np.abs(cos - ref)) < COS_TOL
    idc = sess.run(cb.nearest_neighbor_idx, {enc.x: xu8})
    assert idc.dtype == np.int64 and np.array_equal(idc, np.argmax(ref, axis=1))
    zq = cb.test_embedding(sess, xu8)
    assert np.max(np.abs(zq - O.l2_normalize(z))) < 1e-6


def test_topk_merge_equals_unsharded(sess):
    from augmentedautoencoder_b200 import _lib
    rng = np.random.RandomState(3)
    S, B, k = 8, 33, 4
    scores = rng.randn(S, B, k).astype(np.float32)
    scores[:, 0, :] = 1.0  # all equal -> lowest global indices win
    scores = -np.sort(-scores, axis=2)
    idx = np.stack([np.sort(rng.choice(1000, size=(B, k), replace=False), axis=1) + s * 1000 for s in range(S)]).astype(np.int32)
    so, io = torch.empty((B, k), device="cuda"), torch.empty((B, k), dtype=torch.int32, device="cuda")
    sd, idd = torch.from_numpy(scores).cuda(), torch.from_numpy(idx).cuda()  # keep the device tensors alive across the call
    _lib.check(_lib.lib().aae_topk_merge(_lib.ptr(sd), _lib.ptr(idd), S, B, k, _lib.ptr(so), _lib.ptr(io), None))
    torch.cuda.synchronize()
    so, io = so.cpu().numpy(), io.cpu().numpy()
    for b in range(B):
        pairs = sorted(((-scores[s, b, j], idx[s, b, j]) for s in range(S) for j in range(k)))[:k]
        assert [p[1] for p in pairs] == io[b].tolist()
        assert np.allclose([-p[0] for p in pairs], so[b])


# --------------------------------------------------------------------------------------- end to end
@pytest.mark.parametrize("precision", [0, 1])
def test_end_to_end_256_crops_index_parity(sess, precision):
    """config 2 of BASELINE.json: 256 uint8 crops -> encoder -> fused match on the 92 232-row codebook."""
    p = O.make_encoder_params(42)
    E = O.make_codebook(7)
    enc = _enc(precision, 256, p)
    cb = _codebook(enc, E, max_batch=256, precision=precision)
    crops = O.make_crops_u8(1234, 256)
    got = cb.nearest_rotation(sess, crops, return_idcs=True)
    with torch.cuda.device(0):
        s_dev, _ = cb.nearest_idx_device(torch.from_numpy(crops).cuda())
    want, cos = O.nearest_rotation_idcs(crops, p, E, return_cos=True)
    bad = np.nonzero(got != want)[0]
    if len(bad):
        z64 = O.encoder_forward(O.preprocess(crops[bad]), p, dtype=torch.float64)
        c64 = O.l2_normalize(z64) @ E.astype(np.float64).T
        for j, b in enumerate(bad):
            assert abs(c64[j, got[b]] - c64[j, want[b]]) < 2e-6, ("index mismatch beyond fp32 resolution", b)
    assert len(bad) <= 1
    assert np.max(np.abs(s_dev.cpu().numpy()[:, 0] - cos[np.arange(256), got])) <= COS_TOL


# --------------------------------------------------------------------------------------- decoder / loss / training
def _small_ae(max_batch=4, hw=16, filters=(4, 8), latent=8):
    from augmentedautoencoder_b200.ae.ae import AE
    from augmentedautoencoder_b200.ae.decoder import Decoder
    from augmentedautoencoder_b200.ae.encoder import Encoder
    from augmentedautoencoder_b200.ae.ae_factory import TrainOp
    from augmentedautoencoder_b200.ae.session import placeholder
    strides = (2,) * len(filters)
    x = placeholder(np.float32, [None, hw, hw, 3])
    y = placeholder(np.float32, [None, hw, hw, 3])
    enc = Encoder(x, latent, list(filters), 5, list(strides), False, is_training=True, max_batch=max_batch, precision=0)
    dec = Decoder(y, enc.z, list(reversed(filters)), 5, list(reversed(strides)), "L2", 4, False, False, is_training=True,
                  max_batch=max_batch, n_encoder_convs=len(filters))
    ep = O.make_encoder_params(5, num_filters=filters, in_hw=hw, strides=strides, latent=latent, bias_scale=0.1)
    dp = O.make_decoder_params(6, num_filters=filters, out_hw=hw, strides=strides, latent=latent, bias_scale=0.1, n_encoder_convs=len(filters))
    enc.load_weights(ep)
    dec.load_weights(dp)
    ae = AE(enc, dec, 0, 0)
    return x, y, enc, dec, ae, TrainOp(ae, 2e-4), ep, dp


@pytest.mark.parametrize("hw,filters,latent,batch", [(16, (4, 8), 8, 3), (32, (16, 32, 32), 16, 4)])
def test_decoder_loss_and_gradients_match_oracle(sess, hw, filters, latent, batch):
    x, y, enc, dec, ae, top, ep, dp = _small_ae(4, hw, filters, latent)
    xb = np.random.RandomState(3).rand(batch, hw, hw, 3).astype(np.float32)
    yb = np.random.RandomState(4).rand(batch, hw, hw, 3).astype(np.float32)
    rec, loss = sess.run([dec.x, ae.loss], {x: xb, y: yb})
    loss64, rec64, g64 = O.ae_forward_loss(xb, yb, ep, dp, dtype=torch.float64, with_grads=True)
    assert rec.shape == rec64.shape and np.max(np.abs(rec - rec64)) < 2e-6
    assert abs(float(loss) - loss64) < 1e-6
    l = top.step_device(torch.from_numpy(xb).cuda(), torch.from_numpy(yb).cuda(), update=False)
    assert abs(float(l) - loss64) < 1e-6
    grads = top.gradients(sess.device)
    for name, g in g64.items():
        scale = max(np.abs(g).max(), 1e-8)
        assert np.max(np.abs(grads[name] - g)) < 2e-4 * scale + 1e-9, name


def test_bootstrap_loss_tie_handling_and_gradient(sess):
    from augmentedautoencoder_b200.ae.decoder import Decoder
    B, n = 3, 16 * 16 * 3
    rng = np.random.RandomState(0)
    xb = rng.rand(B, n).astype(np.float32)
    yb = rng.rand(B, n).astype(np.float32)
    xb[1] = rng.randint(0, 128, n).astype(np.float32) / 256.0  # exactly representable, so that ...
    yb[1] = xb[1] + 0.25  # ... every squared error is identical: ties everywhere -> the first k elements are selected
    loss, grad = Decoder.loss_device(torch.from_numpy(xb).cuda(), torch.from_numpy(yb).cuda(), 4, with_grad=True)
    k = n // 4
    l2 = (yb - xb) ** 2
    want = np.sort(l2, axis=1)[:, -k:].mean()
    assert abs(float(loss) - want) < 1e-6
    g = grad.cpu().numpy()
    assert np.all((g != 0).sum(axis=1) == k)
    assert np.all(g[1, :k] != 0) and np.all(g[1, k:] == 0)  # stable top_k: lower index wins
    t = torch.from_numpy(xb).double().requires_grad_(True)
    O.bootstrapped_l2(t, torch.from_numpy(yb).double()).backward()
    sel = g[0] != 0
    assert np.allclose(g[0][sel], t.grad.numpy()[0][sel], atol=1e-7)


def test_train_step_applies_tf_adam(sess):
    x, y, enc, dec, ae, top, ep, dp = _small_ae(4)
    xb = np.random.RandomState(3).rand(4, 16, 16, 3).astype(np.float32)
    yb = np.random.RandomState(4).rand(4, 16, 16, 3).astype(np.float32)
    params = {**ep, **dp}
    m = {k: np.zeros_like(v) for k, v in params.items()}
    v = {k: np.zeros_like(v_) for k, v_ in params.items()}
    for step in range(1, 4):
        loss = sess.run(top, {x: xb, y: yb})
        e_ = {k: params[k] for k in ep}
        d_ = {k: params[k] for k in dp}
        loss_ref, _, g = O.ae_forward_loss(xb, yb, e_, d_, with_grads=True)
        assert abs(float(loss) - loss_ref) < 2e-6
        for k in params:
            params[k], m[k], v[k] = O.tf_adam_step(params[k], g[k], m[k], v[k], step)
    got = {**enc.get_weights(short_names=True), **dec.get_weights(short_names=True)}
    for k in params:
        assert np.max(np.abs(got[k] - params[k])) < 5e-6, k
    assert int(sess.run(ae.global_step)) == 3


def test_full_size_training_forward_backward(sess):
    """config 3 geometry (128x128, [128,256,512,512]) at batch 2: loss and a sample of gradients vs the fp32 oracle."""
    from augmentedautoencoder_b200.ae.ae import AE
    from augmentedautoencoder_b200.ae.ae_factory import TrainOp
    from augmentedautoencoder_b200.ae.decoder import Decoder
    from augmentedautoencoder_b200.ae.encoder import Encoder
    from augmentedautoencoder_b200.ae.session import placeholder
    x = placeholder(np.float32, [None, 128, 128, 3])
    y = placeholder(np.float32, [None, 128, 128, 3])
    enc = Encoder(x, 128, list(O.NUM_FILTER), 5, list(O.STRIDES), False, is_training=True, max_batch=2, precision=0)
    dec = Decoder(y, enc.z, list(reversed(O.NUM_FILTER)), 5, list(reversed(O.STRIDES)), "L2", 4, False, False, is_training=True, max_batch=2,
                  precision=0)
    ep, dp = O.make_encoder_params(42, bias_scale=0.02), O.make_decoder_params(43, bias_scale=0.02)
    enc.load_weights(ep)
    dec.load_weights(dp)
    top = TrainOp(AE(enc, dec, 0, 0), 2e-4)
    # A ReLU unit whose pre-activation is within fp32 rounding of zero can fall on either side in ANY fp32 implementation,
    # which changes gradients discretely; with ~2M units per crop that happens for most random inputs.  Pick the first
    # seeded input whose smallest |pre-activation| (float64) is clear of fp32 rounding, then compare strictly.
    for seed in range(3, 80):
        xb = np.random.RandomState(seed).rand(1, 128, 128, 3).astype(np.float32)
        if O.relu_margin(xb, ep, dp) > 8e-8:   # fp32 rounding of a pre-activation here is ~1e-8
            break
    else:
        pytest.skip("no well-conditioned input among the candidate seeds")
    yb = np.random.RandomState(4).rand(1, 128, 128, 3).astype(np.float32)
    loss = top.step_device(torch.from_numpy(xb).cuda(), torch.from_numpy(yb).cuda(), update=False)
    loss_ref, _, g32 = O.ae_forward_loss(xb, yb, ep, dp, with_grads=True)
    loss64, _, g64 = O.ae_forward_loss(xb, yb, ep, dp, dtype=torch.float64, with_grads=True)
    assert abs(float(loss) - loss64) < 1e-6
    grads = top.gradients(sess.device)
    worst = 0.0
    for name, gr in g64.items():
        scale = max(np.abs(gr).max(), 1e-12)
        err_ours = np.max(np.abs(grads[name] - gr)) / scale
        err_cpu32 = np.max(np.abs(g32[name] - gr)) / scale
        worst = max(worst, err_ours)
        assert err_ours < max(5 * err_cpu32, 2e-5), (name, seed, err_ours, err_cpu32)
    print("full-size gradients: seed %d, worst relative error vs float64 %.2e" % (seed, worst))
