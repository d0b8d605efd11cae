"""GPU parity tests of the tensor-core path (AAE_PREC_TC_SPLIT: wgmma + TMA, split-fp16 operands) against the
float64 oracle, layer by layer and end to end.  Same tolerances as the fp32 SIMT path: this path must be fp32-grade."""
import numpy as np
import pytest
import torch

from oracle import aae_oracle as O
from tests.test_gpu_a_parity import COS_TOL, _codebook, _enc, sess  # noqa: F401

pytestmark = pytest.mark.gpu


def test_tc_match_small_codebook_exact_fields(sess):
    """Tiny case first (one tile, B < 128): isolates descriptor / swizzle errors from pipeline errors."""
    E = O.make_codebook(3, n=64, num_cyclo=1, duplicate_cyclo_endpoints=False)
    p = O.make_encoder_params(42)
    enc = _enc(0, 8, p)
    cb = _codebook(enc, E, num_cyclo=1, max_batch=8, precision=1)
    z = np.random.RandomState(1).standard_normal((5, 128)).astype(np.float32)
    s, i = cb.match_device(torch.from_numpy(z).cuda())
    torch.cuda.synchronize()
    cos = O.cos_similarity(z.astype(np.float64), E.astype(np.float64))
    assert np.array_equal(i.cpu().numpy()[:, 0], np.argmax(cos, axis=1)), (i.cpu().numpy()[:, 0], np.argmax(cos, axis=1), s.cpu().numpy()[:, 0], cos.max(axis=1))
    assert np.max(np.abs(s.cpu().numpy()[:, 0] - cos.max(axis=1))) < 2e-6


@pytest.mark.parametrize("n_rows,batch", [(64 * 5 + 17, 100), (64 * 300, 256), (92232, 129)])
def test_tc_match_matches_oracle(sess, n_rows, batch):
    E = O.make_codebook(5, n=n_rows, num_cyclo=36 if n_rows % 36 == 0 else 1, duplicate_cyclo_endpoints=(n_rows % 36 == 0))
    p = O.make_encoder_params(42)
    enc = _enc(0, 256, p)
    cb = _codebook(enc, E, num_cyclo=36 if n_rows % 36 == 0 else 1, max_batch=256, precision=1)
    rng = np.random.RandomState(n_rows)
    z = (rng.standard_normal((batch, 128)) * rng.uniform(0.05, 50, (batch, 1))).astype(np.float32)
    s, i = cb.match_device(torch.from_numpy(z).cuda())
    s, i = s.cpu().numpy()[:, 0], i.cpu().numpy()[:, 0]
    cos64 = O.cos_similarity(z.astype(np.float64), E.astype(np.float64))
    want = np.argmax(cos64, axis=1)
    err = np.max(np.abs(s - cos64[np.arange(batch), i]))
    assert err < 2e-6, err
    for b in np.nonzero(want != i)[0]:
        assert abs(cos64[b, want[b]] - cos64[b, i[b]]) < 2e-7, (b, want[b], i[b])
    # twice in a row: the last CTA re-arms the scratch, the second launch must give the same answer
    s2, i2 = cb.match_device(torch.from_numpy(z).cuda())
    assert np.array_equal(i2.cpu().numpy()[:, 0], i) and np.array_equal(s2.cpu().numpy()[:, 0], s)


@pytest.mark.parametrize("n_rows,batch,k", [(36 * 700, 5, 8), (92232, 130, 8), (92232, 1, 3), (36 * 40, 64, 8)])
def test_tc_topk_and_upright_match_oracle(sess, n_rows, batch, k):
    """Codebook.nearest_rotation(top_n > 1) and upright=True on the tensor-core kernel (codebook.py:64-71): per-lane sorted
    lists in registers + last-CTA merge; upright = the same kernel on a tensor map with a row stride of num_cyclo rows."""
    E = O.make_codebook(5, n=n_rows)                      # with the duplicated cyclo end-point rows -> exact ties
    p = O.make_encoder_params(42)
    cb = _codebook(_enc(0, 256, p), E, max_batch=256, precision=1)
    rng = np.random.RandomState(n_rows + batch)
    z = (rng.standard_normal((batch, 128)) * rng.uniform(0.05, 50, (batch, 1))).astype(np.float32)
    z[0] = E[36 * 3] * 2.0                                # a query that IS a (duplicated) row: rows 108 and 143 tie at 1.0
    cos64 = O.cos_similarity(z.astype(np.float64), E.astype(np.float64))
    sk, ik = cb.match_device(torch.from_numpy(z).cuda(), k=k)
    sk, ik = sk.cpu().numpy(), ik.cpu().numpy()
    assert sk.shape == (batch, k) and ik.shape == (batch, k)
    assert ik[0, 0] == 36 * 3 and ik[0, 1] == 36 * 3 + 35          # equal scores: lowest index first
    for b in range(batch):
        want = np.lexsort((np.arange(n_rows), -cos64[b]))[:k]      # score descending, ties to the lowest index
        assert np.max(np.abs(sk[b] - cos64[b, ik[b]])) < 2e-6
        assert np.all(np.diff(sk[b]) <= 0) and len(set(ik[b].tolist())) == k
        for j in np.nonzero(want != ik[b])[0]:                     # a swap is legitimate only between fp32-indistinguishable scores
            assert abs(cos64[b, want[j]] - cos64[b, ik[b, j]]) < 2e-7, (b, j, want, ik[b])
    # k = 1 agrees with the head of the list, and twice in a row gives the same answer (scratch re-armed)
    s1, i1 = cb.match_device(torch.from_numpy(z).cuda(), k=1)
    assert np.array_equal(i1.cpu().numpy()[:, 0], ik[:, 0]) and np.array_equal(s1.cpu().numpy()[:, 0], sk[:, 0])
    sk2, ik2 = cb.match_device(torch.from_numpy(z).cuda(), k=k)
    assert np.array_equal(ik2.cpu().numpy(), ik) and np.array_equal(sk2.cpu().numpy(), sk)
    # upright (codebook.py:66): every 36th row only
    su, iu = cb.match_device(torch.from_numpy(z).cuda(), upright=True)
    su, iu = su.cpu().numpy()[:, 0], iu.cpu().numpy()[:, 0]
    want_u = O.select_indices(cos64, upright=True, num_cyclo=36)
    assert np.all(iu % 36 == 0) and np.max(np.abs(su - cos64[np.arange(batch), iu])) < 2e-6
    for b in np.nonzero(want_u != iu)[0]:
        assert abs(cos64[b, want_u[b]] - cos64[b, iu[b]]) < 2e-7
    suk, iuk = cb.match_device(torch.from_numpy(z).cuda(), k=min(k, 4), upright=True)
    assert np.array_equal(iuk.cpu().numpy()[:, 0], iu) and np.all(iuk.cpu().numpy() % 36 == 0)
    # and the exact-order fp32 path gives the same indices
    cb0 = _codebook(_enc(0, 256, p), E, max_batch=256, precision=0)
    s0, i0 = cb0.match_device(torch.from_numpy(z).cuda(), k=k)
    d = np.nonzero(i0.cpu().numpy() != ik)
    for b, j in zip(*d):
        assert abs(cos64[b, i0.cpu().numpy()[b, j]] - cos64[b, ik[b, j]]) < 2e-7


def test_tc_encoder_layers_and_latent_match_oracle(sess):
    p = O.make_encoder_params(42, bias_scale=0.05)
    enc = _enc(1, 4, p)
    xu8 = O.make_crops_u8(1234, 4)
    z = sess.run(enc.z, {enc.x: xu8})
    outs64 = O.encoder_layers(O.preprocess(xu8), p, dtype=torch.float64)
    errs = []
    for layer in range(4):
        a = enc.activation_device(layer, sess.device).cpu().numpy()
        ref = outs64[layer].numpy()
        assert a.shape == ref.shape
        errs.append(np.max(np.abs(a - ref)) / max(1.0, np.abs(ref).max()))
    z64 = outs64[5].numpy()
    errs.append(np.max(np.abs(z - z64)) / np.abs(z64).max())
    print("tc encoder relative errors per layer + latent:", ["%.2e" % e for e in errs])
    assert all(e < 1e-5 for e in errs), errs


@pytest.mark.parametrize("batch", [1, 2, 63, 127, 129, 255, 300])
def test_tc_path_agrees_with_fp32_path_for_ragged_batches(sess, batch):
    """Tile-boundary cases: batches that do not fill a 128-pixel tile / a CTA pair / a 128-query block, and a batch larger
    than max_batch (chunked by the host wrapper).  The tensor-core path must give the fp32 path's indices and scores."""
    p = O.make_encoder_params(42, bias_scale=0.03)
    E = O.make_codebook(9, n=36 * 700 + 5, num_cyclo=1, duplicate_cyclo_endpoints=False)
    crops = O.make_crops_u8(77 + batch, batch)
    res = []
    for prec in (0, 1):
        enc = _enc(prec, 256, p)
        cb = _codebook(enc, E, num_cyclo=1, max_batch=256, precision=prec)
        z = sess.run(enc.z, {enc.x: crops})
        s, i = cb.nearest_idx_device(torch.from_numpy(crops).cuda())
        res.append((z, s.cpu().numpy()[:, 0], i.cpu().numpy()[:, 0]))
    (z0, s0, i0), (z1, s1, i1) = res
    assert z1.shape == (batch, 128)
    assert np.max(np.abs(z0 - z1)) < 2e-5 * np.abs(z0).max()
    assert np.max(np.abs(s0 - s1)) < COS_TOL
    bad = np.nonzero(i0 != i1)[0]
    cos = O.cos_similarity(z0[bad].astype(np.float64), E.astype(np.float64)) if len(bad) else None
    for j, b in enumerate(bad):
        assert abs(cos[j, i0[b]] - cos[j, i1[b]]) < 2e-6, (b, i0[b], i1[b])


def test_c_abi_rejects_bad_calls_without_crashing(sess):
    import ctypes as C
    from augmentedautoencoder_b200 import _lib
    lib = _lib.lib()
    p = O.make_encoder_params(42)
    enc = _enc(1, 8, p)
    h = enc.handle(sess.device)
    x = torch.zeros((16, 128, 128, 3), dtype=torch.uint8, device="cuda")
    z = torch.zeros((16, 128), device="cuda")
    assert lib.aae_encoder_forward_u8(h, _lib.ptr(x), 16, _lib.ptr(z), None) == -1          # batch > max_batch
    assert b"max_batch" in lib.aae_last_error_string()
    assert lib.aae_encoder_forward_u8(h, None, 4, _lib.ptr(z), None) == -1
    assert lib.aae_encoder_forward_u8(h, _lib.ptr(x), 0, _lib.ptr(z), None) == -1
    assert lib.aae_encoder_forward_u8(h, x.data_ptr() + 1, 4, _lib.ptr(z), None) == -1             # crops not 16-byte aligned
    assert b"align" in lib.aae_last_error_string()
    xf = torch.zeros((5, 128, 128, 3), device="cuda")
    assert lib.aae_encoder_forward_f32(h, xf.data_ptr() + 4, 4, _lib.ptr(z), None) == -1
    assert b"align" in lib.aae_last_error_string()
    cbh = C.c_void_p()
    E = O.make_codebook(1, n=100, num_cyclo=1, duplicate_cyclo_endpoints=False)
    assert lib.aae_codebook_create(0, _lib.ptr(E), 100, 96, 1, 0, 8, 1, C.byref(cbh)) != 0     # TC match is built for latent 128
    assert b"latent" in lib.aae_last_error_string() and not cbh.value
    assert lib.aae_codebook_create(0, _lib.ptr(E), 100, 128, 1, 0, 8, 1, C.byref(cbh)) == 0
    s = torch.zeros((4, 1), device="cuda")
    i = torch.zeros((4, 1), dtype=torch.int32, device="cuda")
    assert lib.aae_codebook_match(cbh, _lib.ptr(z), 4, 101, 0, _lib.ptr(s), _lib.ptr(i), None) == -1   # k > rows
    assert lib.aae_codebook_match(cbh, _lib.ptr(z), 9, 1, 0, _lib.ptr(s), _lib.ptr(i), None) == -1     # batch > max_batch
    assert lib.aae_codebook_destroy(cbh) == 0
    assert lib.aae_encoder_forward_u8(h, _lib.ptr(x), 4, _lib.ptr(z), None) == 0                          # handle still healthy
    torch.cuda.synchronize()


@pytest.mark.parametrize("batch", [1, 3, 64])
def test_tc_decoder_forward_matches_oracle(sess, batch):
    """Decoder.x on the tensor cores (sub-pixel GEMMs, split-fp16) against the float64 oracle and the fp32 SIMT path."""
    from augmentedautoencoder_b200.ae.decoder import Decoder
    from augmentedautoencoder_b200.ae.session import placeholder
    dp = O.make_decoder_params(43, bias_scale=0.05)
    z = (np.random.RandomState(batch).standard_normal((batch, 128)) * 2.0).astype(np.float32)
    outs = []
    for prec in (0, 1):
        zin = placeholder(np.float32, [None, 128])
        dec = Decoder(placeholder(np.float32, [None, 128, 128, 3]), zin, list(reversed(O.NUM_FILTER)), 5, list(reversed(O.STRIDES)), "L2", 4,
                      False, False, max_batch=64, precision=prec)
        dec.load_weights(dp)
        outs.append(dec.decode_device(torch.from_numpy(z).cuda()).cpu().numpy())
    tp = {k: torch.from_numpy(v).double() for k, v in dp.items()}
    with torch.no_grad():
        ref = O.decoder_layers(torch.from_numpy(z).double(), tp)[-1].numpy()
    assert outs[1].shape == ref.shape == (batch, 128, 128, 3)
    e_simt, e_tc = np.max(np.abs(outs[0] - ref)), np.max(np.abs(outs[1] - ref))
    print("decoder forward max abs error vs float64: simt %.2e  tc %.2e" % (e_simt, e_tc))
    assert e_simt < 2e-6 and e_tc < 5e-6
    # the tensor-core output layer takes at most 3 channels; the fp32 path runs a 4-channel decoder
    from augmentedautoencoder_b200._lib import AaeError
    for prec in (1, 0):
        dec4 = Decoder(placeholder(np.float32, [None, 128, 128, 4]), placeholder(np.float32, [None, 128]), list(reversed(O.NUM_FILTER)), 5,
                       list(reversed(O.STRIDES)), "L2", 4, False, False, max_batch=64, precision=prec)
        dec4.load_weights(O.make_decoder_params(43, out_ch=4, bias_scale=0.05))
        if prec == 1:
            with pytest.raises(AaeError, match="at most 3"):
                dec4.decode_device(torch.from_numpy(z).cuda())
        else:
            x4 = dec4.decode_device(torch.from_numpy(z).cuda()).cpu().numpy()
            assert x4.shape == (batch, 128, 128, 4) and np.all((x4 >= 0) & (x4 <= 1))


def _train_pair(prec, B):
    from augmentedautoencoder_b200.ae.ae import AE
    from augmentedautoencoder_b200.ae.ae_factory import TrainOp
    from augmentedautoencoder_b200.ae.decoder import Decoder
    from augmentedautoencoder_b200.ae.encoder import Encoder
    from augmentedautoencoder_b200.ae.session import placeholder
    x = placeholder(np.float32, [None, 128, 128, 3])
    y = placeholder(np.float32, [None, 128, 128, 3])
    enc = Encoder(x, 128, list(O.NUM_FILTER), 5, list(O.STRIDES), False, is_training=True, max_batch=B, precision=prec)
    dec = Decoder(y, enc.z, list(reversed(O.NUM_FILTER)), 5, list(reversed(O.STRIDES)), "L2", 4, False, False, is_training=True, max_batch=B,
                  precision=prec)
    ep, dp = O.make_encoder_params(42, bias_scale=0.02), O.make_decoder_params(43, bias_scale=0.02)
    enc.load_weights(ep)
    dec.load_weights(dp)
    return enc, dec, TrainOp(AE(enc, dec, 0, 0), 2e-4), ep, dp


def test_tc_training_gradients_match_float64_oracle(sess):
    """Tensor-core trainer (wgmma forward, dgrad and wgrad GEMMs): loss and all 20 gradients of one forward/backward vs the
    float64 oracle.  Compared in relative L2 norm: a ReLU unit whose pre-activation is within the split-fp16 rounding of zero
    may fall on either side (as in any finite-precision implementation), which perturbs a few entries discretely."""
    enc, dec, top, ep, dp = _train_pair(1, 2)
    xb = np.random.RandomState(8).rand(1, 128, 128, 3).astype(np.float32)
    yb = np.random.RandomState(4).rand(1, 128, 128, 3).astype(np.float32)
    loss = top.step_device(torch.from_numpy(xb).cuda(), torch.from_numpy(yb).cuda(), update=False)
    loss64, _, g64 = O.ae_forward_loss(xb, yb, ep, dp, dtype=torch.float64, with_grads=True)
    assert abs(float(loss) - loss64) < 2e-6 * max(1.0, abs(loss64))
    grads = top.gradients(sess.device)
    worst = 0.0
    for name, gr in g64.items():
        rel = np.linalg.norm(grads[name].astype(np.float64) - gr) / max(np.linalg.norm(gr), 1e-30)
        worst = max(worst, rel)
        assert rel < 3e-4, (name, rel)
    print("tensor-core trainer: worst relative L2 gradient error vs float64 %.2e" % worst)


def test_tc_training_steps_track_the_fp32_trainer(sess):
    """Five Adam steps at batch 3 (ragged against the 128-row tiles): the loss trajectory of the tensor-core trainer follows
    the fp32 CUDA-core trainer, and the loss goes down."""
    xb = torch.from_numpy(np.random.RandomState(11).rand(3, 128, 128, 3).astype(np.float32)).cuda()
    yb = torch.from_numpy(np.random.RandomState(12).rand(3, 128, 128, 3).astype(np.float32)).cuda()
    traj = {}
    for prec in (0, 1):
        enc, dec, top, _, _ = _train_pair(prec, 4)
        traj[prec] = [float(top.step_device(xb, yb, update=True)) for _ in range(5)]
        del enc, dec, top
    assert traj[1][-1] < traj[1][0]
    assert np.max(np.abs(np.array(traj[0]) - np.array(traj[1]))) < 2e-4, traj


def test_inference_after_a_training_step_uses_the_updated_weights(sess):
    """Adam updates the fp32 master weights in place; the tensor-core plans keep packed (hi, lo) copies.  In-process inference
    after training (Codebook.update_embedding, decoder.x: ae_embed.py:84-91 run after ae_train.py) must use the step-N
    weights that get_weights() / the checkpoint hold -- i.e. equal a fresh handle loaded from get_weights()."""
    _check_inference_after_training(sess, 1)


def test_inference_after_a_training_step_uses_the_updated_weights_fp32(sess):
    """The same at the fp32 precision, whose decoder keeps merged sub-pixel weights derived from the masters."""
    _check_inference_after_training(sess, 0)


def _check_inference_after_training(sess, prec):
    from augmentedautoencoder_b200 import _lib
    from augmentedautoencoder_b200.ae.decoder import Decoder
    from augmentedautoencoder_b200.ae.encoder import Encoder
    from augmentedautoencoder_b200.ae.session import placeholder
    enc, dec, top, ep, dp = _train_pair(prec, 4)

    def fresh_pair():                                   # new handles loaded from what get_weights() returns now
        e = Encoder(placeholder(np.float32, [None, 128, 128, 3]), 128, list(O.NUM_FILTER), 5, list(O.STRIDES), False, max_batch=4, precision=prec)
        d = Decoder(placeholder(np.float32, [None, 128, 128, 3]), e.z, list(reversed(O.NUM_FILTER)), 5, list(reversed(O.STRIDES)), "L2", 4,
                    False, False, max_batch=4, precision=prec)
        e.load_weights(enc.get_weights())
        d.load_weights(dec.get_weights())
        return e, d
    xb = torch.from_numpy(np.random.RandomState(11).rand(3, 128, 128, 3).astype(np.float32)).cuda()
    yb = torch.from_numpy(np.random.RandomState(12).rand(3, 128, 128, 3).astype(np.float32)).cuda()
    z_before = enc.encode_device(xb).clone()
    for _ in range(2):
        top.step_device(xb, yb, update=True)
    z_after = enc.encode_device(xb).clone()
    rec_after = dec.decode_device(z_after).clone()
    assert float((z_after - z_before).abs().max()) > 1e-4           # the step did move the weights
    enc2, dec2 = fresh_pair()
    z_fresh = enc2.encode_device(xb)
    assert torch.equal(z_after, z_fresh), float((z_after - z_fresh).abs().max())
    assert torch.equal(rec_after, dec2.decode_device(z_fresh))
    # ... and training continues from the same state after the inference calls (the trainer's operands follow too)
    l3 = float(top.step_device(xb, yb, update=True))
    enc3, dec3, top3, _, _ = _train_pair(prec, 4)
    ref = [float(top3.step_device(xb, yb, update=True)) for _ in range(3)]
    assert abs(l3 - ref[2]) < 1e-6, (l3, ref)
    # set_weights of a single layer right after an Adam step packs that layer only: every other layer's derived copy is
    # still one step behind and must be rebuilt by the next forward
    lib = _lib.lib()
    for set_weights, mod, layer, name in ((lib.aae_encoder_set_weights, enc, 1, "conv2d_1"), (lib.aae_decoder_set_weights, dec, 2, "conv2d_5")):
        w = mod.get_weights(short_names=True)
        k, b = np.ascontiguousarray(w[name + "/kernel"] * 0.5), np.ascontiguousarray(w[name + "/bias"] * 0.5)
        _lib.check(set_weights(mod.handle(sess.device), layer, _lib.ptr(k), _lib.ptr(b), None), "set_weights")
    z_set = enc.encode_device(xb).clone()
    rec_set = dec.decode_device(z_set).clone()
    enc4, dec4 = fresh_pair()
    assert torch.equal(z_set, enc4.encode_device(xb))
    assert torch.equal(rec_set, dec4.decode_device(z_set))


def test_range_guard_reports_overflow_instead_of_garbage(sess):
    """The split-fp16 arithmetic needs |activation| < 4094 and |weight| < 255.9 (DESIGN.md section 3).  A model outside that range
    must fail loudly -- AAE_ERR_UNSUPPORTED naming the layer -- never return inf / garbage with status 0; the fp32 path takes
    the same model without complaint."""
    from augmentedautoencoder_b200._lib import AaeError
    from augmentedautoencoder_b200.ae.decoder import Decoder
    from augmentedautoencoder_b200.ae.session import placeholder
    p = O.make_encoder_params(42, bias_scale=0.05)
    crops = O.make_crops_u8(5, 3)
    # (1) a weight the fp16 operands cannot hold is refused when the weights reach the device
    bad_w = dict(p)
    bad_w["conv2d_2/kernel"] = p["conv2d_2/kernel"].copy()
    bad_w["conv2d_2/kernel"][1, 2, 3, 4] = 300.0
    enc = _enc(1, 4, bad_w)
    with pytest.raises(AaeError, match=r"weight.*layer\(s\) 2"):
        sess.run(enc.z, {enc.x: crops})
    # (2) activations: a large bias pushes conv1's (bit 0, tensor-core conv1 kernel) / conv2's (bit 1, GEMM epilogue) output past 4094
    for name, layer in (("conv2d/bias", 0), ("conv2d_1/bias", 1)):
        bad_a = dict(p)
        bad_a[name] = p[name].copy()
        bad_a[name][7] = 5000.0
        enc = _enc(1, 4, bad_a)
        for feed in (crops, O.preprocess(crops)):                      # uint8 and float feeds
            with pytest.raises(AaeError, match=r"activation.*layer\(s\) %d" % layer):
                sess.run(enc.z, {enc.x: feed})
        E = O.make_codebook(3, n=36 * 20)
        cb = _codebook(enc, E, max_batch=4, precision=1)
        with pytest.raises(AaeError, match="activation"):
            cb.nearest_rotation(sess, crops, return_idcs=True)
        with pytest.raises(AaeError, match="activation"):              # streaming call: reported by .result(), no pipeline sync otherwise
            cb.nearest_rotation_async(sess, torch.from_numpy(crops)).result()
        enc.load_weights(p)                                            # the guard was cleared by the report: good weights run clean
        z = sess.run(enc.z, {enc.x: crops})
        assert np.all(np.isfinite(z))
        # the exact fp32 path has no such limit
        enc0 = _enc(0, 4, bad_a)
        assert np.all(np.isfinite(sess.run(enc0.z, {enc0.x: crops})))
    # (3) decoder
    dp = O.make_decoder_params(43, bias_scale=0.05)
    bad_d = dict(dp)
    bad_d["dense_1/bias"] = dp["dense_1/bias"].copy()
    bad_d["dense_1/bias"][11] = 5000.0
    zin = placeholder(np.float32, [None, 128])
    dec = Decoder(placeholder(np.float32, [None, 128, 128, 3]), zin, list(reversed(O.NUM_FILTER)), 5, list(reversed(O.STRIDES)), "L2", 4,
                  False, False, max_batch=4, precision=1)
    dec.load_weights(bad_d)
    zz = np.random.RandomState(0).standard_normal((2, 128)).astype(np.float32)
    with pytest.raises(AaeError, match=r"activation.*layer\(s\) 0"):
        sess.run(dec.x, {zin: zz})
    with pytest.raises(AaeError, match="latent"):
        sess.run(dec.x, {zin: zz * 1e4})
    dec.load_weights(dp)
    assert np.all(np.isfinite(sess.run(dec.x, {zin: zz})))


def test_training_resumes_from_a_checkpoint_with_the_optimizer_state(sess, tmp_path):
    """tf.train.Saver stores the Adam slots and beta powers beside the weights (ae_train.py:82,111-115), so a resumed run continues
    exactly; a weights-only restore restarts the optimizer (zero moments, bias correction from t = 1)."""
    from augmentedautoencoder_b200.ae import factory
    from augmentedautoencoder_b200.ae.tf_checkpoint import read_tf_checkpoint
    xb = torch.from_numpy(np.random.RandomState(11).rand(3, 128, 128, 3).astype(np.float32)).cuda()
    yb = torch.from_numpy(np.random.RandomState(12).rand(3, 128, 128, 3).astype(np.float32)).cuda()
    enc, dec, top, _, _ = _train_pair(1, 4)
    for _ in range(2):
        top.step_device(xb, yb)
    saver = factory.Saver([enc, dec], global_step=top._ae.global_step, train_op=top)
    path = saver.save_tf(sess, str(tmp_path / "checkpoints" / "chkpt"), global_step=2)
    stored = read_tf_checkpoint(path)
    assert "conv2d_1/kernel/Adam" in stored and "conv2d_1/kernel/Adam_1" in stored and "dense_1/bias/Adam" in stored
    assert abs(float(stored["beta1_power"]) - 0.9 ** 3) < 1e-7 and abs(float(stored["beta2_power"]) - 0.999 ** 3) < 1e-7
    assert np.abs(stored["conv2d_1/kernel/Adam"]).max() > 0 and stored["conv2d_1/kernel/Adam_1"].min() >= 0
    l3 = float(top.step_device(xb, yb))
    w3 = enc.get_weights()["conv2d_2/kernel"]
    # full restore: same third step
    enc2, dec2, top2, _, _ = _train_pair(1, 4)
    factory.Saver([enc2, dec2], global_step=top2._ae.global_step, train_op=top2).restore(sess, path)
    assert int(top2._ae.global_step.value()) == 2
    l3b = float(top2.step_device(xb, yb))
    assert abs(l3 - l3b) < 1e-6 * max(1.0, abs(l3)), (l3, l3b)
    assert np.max(np.abs(enc2.get_weights()["conv2d_2/kernel"] - w3)) < 1e-7
    assert int(top2._ae.global_step.value()) == 3
    # weights-only restore: the loss of the next step is the same (same weights) but the update is not (fresh optimizer)
    enc3, dec3, top3, _, _ = _train_pair(1, 4)
    factory.Saver([enc3, dec3]).restore(sess, path)
    l3c = float(top3.step_device(xb, yb))
    assert abs(l3 - l3c) < 1e-6 * max(1.0, abs(l3))
    assert np.max(np.abs(enc3.get_weights()["conv2d_2/kernel"] - w3)) > 1e-6
