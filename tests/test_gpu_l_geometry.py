"""GPU tests of the network geometries a cfg reaches beyond the template (LATENT_SPACE_SIZE, NUM_FILTER, STRIDES, H / W / C,
KERNEL_SIZE_*, AUXILIARY_MASK), one table row per geometry (tests/geometry_table.py), against the float64 oracle evaluated on the
GPU.

Each row pins where the encoder, the codebook match, the decoder and the training step land with the automatic precision, and then
checks whichever path that is: the encoder layer by layer at batch 1, a ragged batch and max_batch; the end-to-end match at
latents other than 128; the decoder forward with and without the mask head; the loss and every gradient on weights with a
quarter of every ReLU layer's units dead; the split trainer's Adam trajectory and weights against the fp32 trainer's; after a
demotion to the fp32 trainer, handles that compute what fresh fp32 handles compute; and the single-pass fp16 trainer on two
tensor-core-trainable rows against its rounding-model bound.

Branches only these rows reach: the fp32 conv1 writing conv2's (hi, lo) space-to-depth input (conv1_64, px64, gray), layers
with a 4-pixel-wide output and their per-tap boxes (five_layer, px64, and the decoder's first layers there), N tiles narrower
than 128 on a conv (cout64) and on the dense layer (latent32/64/96), a zero-filled last N tile (wide_last, Cout 480), other dense
flat sizes and split counts, the tensor-core conv1 at 64 rows with BB = 4 (rect), the decoder at h0 = 4 and 32, a 1-channel
output conv and the mask head on every decoder, the fp32 match at latent 32/64/256, and every automatic fallback.

Crop sizes that are not powers of two (px112, px80, px96, px127, h127, px100) reach odd maps (7 x 7, 5 x 5, 25 x 25), TF's
symmetric (2, 2) SAME padding of odd inputs, images that straddle 128-row tiles, and the fp32 kernels the tensor cores leave
them: the generic conv1 weight gradient, stride-2 dgrad on odd maps in both orderings (PARITY_BATCH), decoders whose first map
is 5, 6 or 7 pixels wide, and the fp32 conv1 with pad (2, 2) (pad_t = 2 and pad_l = 1 at 127 x 128) writing the split
encoder's conv2 input.  The decoder refuses a crop that is not a multiple of 2^L."""
import gc

import numpy as np
import pytest
import torch

from oracle import aae_oracle as O
from oracle import mask_oracle as MO
from tests.geometry_table import (FP16, FP32, LANDING, MAXB, PARITY_BATCH, PARITY_ROWS, RAGGED, ROWS, SPLIT, T, dec_weights, decoder,
                                  encoder, output_conv, params, row, tc_conv1)
from tests.test_gpu_a_parity import COS_TOL, _codebook, sess  # noqa: F401
from tests.test_gpu_d_fp16 import _conv_bound_check, _dense_bound_check
from tests.test_gpu_e_fp16_train import U, _apply, _check_grads, _cond

pytestmark = pytest.mark.gpu

REL_TRAIN = 3e-4
IDS = list(ROWS)


def _free():
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


class _Peak:
    """Peak device memory a test adds: the library's handles (their own cudaMalloc allocations, which torch's allocator statistics do
    not see) and torch's tensors.  Taken as the drop of the device's free memory below its value at the start of the test, with
    torch's cache emptied, sampled after every handle build and step; so it assumes no other process allocates on the device
    meanwhile.  torch's own peak is reported beside it."""

    def __init__(self, tag):
        _free()
        torch.cuda.reset_peak_memory_stats()
        self.tag, self.free0, self.peak = tag, torch.cuda.mem_get_info()[0], 0

    def sample(self):
        torch.cuda.synchronize()
        self.peak = max(self.peak, self.free0 - torch.cuda.mem_get_info()[0])

    def report(self):
        print("%s: peak device memory added %.2f GB (torch tensors alone %.2f GB)"
              % (self.tag, self.peak / 2 ** 30, torch.cuda.max_memory_allocated() / 2 ** 30))


def _relu_layers(r):
    return ["conv2d" if i == 0 else "conv2d_%d" % i for i in range(r["L"])] + ["dense_1"] + \
        ["conv2d_%d" % (r["L"] + j) for j in range(r["L"] - 1)]


def _masked(r, ep, dp, head, seed=7):
    """Weights whose ReLU masks are not all ones, with a clear margin: every kernel scaled down (x 0.003; the output conv and the
    mask head x 0.05) so that the biases decide every sign, and every bias drawn from [1, 2], negated for a quarter of the units of
    each ReLU layer (those are dead).  tests/test_gpu_j_train_batch's masked set for any geometry."""
    rng = np.random.RandomState(seed)
    relu = set(_relu_layers(r))
    out = []
    for p in (ep, dp):
        q = {}
        for name, v in p.items():
            layer = name.rsplit("/", 1)[0]
            if name.endswith("kernel"):
                q[name] = (v * (0.05 if layer == output_conv(r) else 0.003)).astype(np.float32)
            else:
                b = rng.uniform(1.0, 2.0, v.shape)
                q[name] = (np.where(rng.rand(*b.shape) < 0.25, -b, b) if layer in relu else b).astype(np.float32)
        out.append(q)
    if head is not None:
        head = ((head[0] * 0.05).astype(np.float32), rng.uniform(1.0, 2.0, head[1].shape).astype(np.float32))
    return out[0], out[1], head


def _g(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to("cuda", torch.float64)


def _dead_shares(r, x, ep, dp):
    """{ReLU layer: share of its units (over the batch) with a negative float64 pre-activation}"""
    P = {k: _g(v) for k, v in {**ep, **dp}.items()}
    shares = {}
    with torch.no_grad():
        h = _g(x)
        for i, s in enumerate(r["strides"]):
            name = "conv2d" if i == 0 else "conv2d_%d" % i
            pre = O.conv2d_same(h, P[name + "/kernel"], P[name + "/bias"], s, None)
            shares[name], h = float((pre < 0).double().mean()), torch.relu(pre)
        z = h.reshape(h.shape[0], -1) @ P["dense/kernel"] + P["dense/bias"]
        pre = z @ P["dense_1/kernel"] + P["dense_1/bias"]
        d0 = r["h"] // int(np.prod(r["strides"]))
        shares["dense_1"], h = float((pre < 0).double().mean()), torch.relu(pre).reshape(-1, d0, d0, r["nf"][-1])
        for j in range(r["L"] - 1):
            name = "conv2d_%d" % (r["L"] + j)
            h = O.resize_nearest_2x(h, (2 * h.shape[1], 2 * h.shape[2]))
            pre = O.conv2d_same(h, P[name + "/kernel"], P[name + "/bias"], 1, None)
            shares[name], h = float((pre < 0).double().mean()), torch.relu(pre)
    return shares


def _check_relu_paths(r, x, ep, dp):
    """the masked weights leave dead units in every ReLU layer, and every pre-activation is clear of zero"""
    margin = O.relu_margin(x, ep, dp, device="cuda", strides=r["strides"])   # the mask head ends in a sigmoid: no ReLU of its own
    shares = _dead_shares(r, x, ep, dp)
    assert margin > 0.1, (r["id"], margin)
    assert all(0.1 < s < 0.5 for s in shares.values()), (r["id"], shares)
    return margin, shares


def _pair(r, ep, dp, head, precision=None, gemm=None, bootstrap=4):
    from augmentedautoencoder_b200.ae.ae import AE
    from augmentedautoencoder_b200.ae.ae_factory import TrainOp
    enc = encoder(r, precision, is_training=True)
    dec = decoder(r, enc, precision, bootstrap)
    enc.load_weights(ep)
    dec.load_weights(dec_weights(r, dp, head))
    return enc, dec, TrainOp(AE(enc, dec, 0, 0), 2e-4, precision=gemm)


def _enc64(x, ep, strides):
    """float64 encoder on the GPU: [conv activations..., z] as numpy"""
    outs = []
    with torch.no_grad():
        h = _g(x)
        for i, s in enumerate(strides):
            name = "conv2d" if i == 0 else "conv2d_%d" % i
            h = O.conv2d_same(h, _g(ep[name + "/kernel"]), _g(ep[name + "/bias"]), s, "relu")
            outs.append(h.cpu().numpy())
        outs.append((h.reshape(h.shape[0], -1) @ _g(ep["dense/kernel"]) + _g(ep["dense/bias"])).cpu().numpy())
    return outs


def _crops(r, B, seed):
    return O.make_crops_u8(seed, B, hw=r["h"], ch=r["c"], w=r["w"])


def _needs_decoder(rid):
    if LANDING[rid][2] is None:
        pytest.skip("%s: no decoder exists for this geometry on any precision (square crops and stride-2 stages only)" % rid)


# ------------------------------------------------------------------------------------------------------------ landing
@pytest.mark.parametrize("rid", IDS)
def test_where_each_module_lands(sess, rid):
    """The automatic precision of every module, against the literal table; explicit precisions are never replaced: a refused
    explicit precision raises AaeError naming the reason."""
    from augmentedautoencoder_b200 import _lib
    r = row(rid)
    ep, dp, head = params(r)
    peak = _Peak(rid + " landing")
    E = O.make_codebook(3, n=36 * 20, j=r["latent"])
    enc = encoder(r)
    enc.load_weights(ep)
    enc.handle(sess.device)
    cb = _codebook(enc, E, max_batch=MAXB)
    cb.handle(sess.device)
    got = [enc.precision, cb.precision]
    dec = decoder(r, encoder(r))
    try:
        dec.handle(sess.device)
        got.append(dec.precision)
    except _lib.AaeError as e:
        assert dec.precision == FP32, e                   # the automatic fallback ran and the fp32 decoder refused too
        got.append(None)
    peak.sample()
    enc.close(); cb.close(); dec.close()
    if got[2] is None:
        got.append(None)
    else:
        enc, dec, top = _pair(r, ep, dp, head)
        top.trainer(sess.device)
        assert enc.precision == dec.precision, (enc.precision, dec.precision)
        got.append(enc.precision)
        peak.sample()
        top.close(); enc.close(); dec.close()
    try:
        e16 = encoder(r, precision=FP16)
        e16.load_weights(ep)
        e16.handle(sess.device)
        got.append(True)
        assert e16.precision == FP16
        e16.close()
    except _lib.AaeError as e:
        assert "FP16" in str(e) or "unsupported" in str(e), e
        got.append(False)
    print("%s: encoder %s, match %s, decoder %s, trainer %s, fp16 encoder %s" % (rid, *got))
    peak.report()
    assert tuple(got) == LANDING[rid], (rid, got)
    # an explicit precision is never replaced
    for prec in (SPLIT, FP16):
        if LANDING[rid][0] == SPLIT and (prec == SPLIT or LANDING[rid][4]):
            continue
        e = encoder(r, precision=prec)
        with pytest.raises(_lib.AaeError, match="unsupported|needs|expected|FP16"):
            e.handle(sess.device)
        assert e.precision == prec
    if LANDING[rid][2] == FP32:
        d = decoder(r, encoder(r), precision=SPLIT)
        with pytest.raises(_lib.AaeError, match="decoder"):
            d.handle(sess.device)
        assert d.precision == SPLIT
    _free()


# ------------------------------------------------------------------------------------------------------------ encoder
@pytest.mark.parametrize("rid", IDS)
def test_encoder_layers_and_latent_match_float64(sess, rid):
    """Every conv activation (1e-5 relative to max(1, max |a|)) and z (2e-5 of max |z|) at batch 1, a ragged batch and max_batch; the
    float feed equals the uint8 feed bit for bit where conv1 is the fp32 kernel; the fp16 encoder meets its rounding bound where
    it is accepted."""
    r = row(rid)
    ep, _, _ = params(r)
    peak = _Peak(rid + " encoder")
    enc = encoder(r)
    enc.load_weights(ep)
    worst = np.zeros(r["L"] + 1)
    for B in (1, RAGGED, MAXB):
        xu8 = _crops(r, B, 100 + B)
        z = enc.encode_device(torch.from_numpy(xu8).cuda()).cpu().numpy()
        peak.sample()
        outs = _enc64(O.preprocess(xu8), ep, r["strides"])
        for l in range(r["L"]):
            a = enc.activation_device(l, sess.device).cpu().numpy()
            assert a.shape == outs[l].shape, (rid, l, a.shape, outs[l].shape)
            worst[l] = max(worst[l], np.max(np.abs(a - outs[l])) / max(1.0, np.abs(outs[l]).max()))
        assert z.shape == (B, r["latent"])
        worst[-1] = max(worst[-1], np.max(np.abs(z - outs[-1])) / np.abs(outs[-1]).max())
        if not tc_conv1(r):
            zf = enc.encode_device(torch.from_numpy(O.preprocess(xu8)).cuda()).cpu().numpy()
            assert np.array_equal(z, zf), rid
    print("%s encoder (precision %d): worst relative error per layer + z %s" % (rid, enc.precision, ["%.1e" % e for e in worst]))
    assert np.all(worst[:-1] < 1e-5) and worst[-1] < 2e-5, (rid, worst)
    enc.close()
    if LANDING[rid][4]:
        e16 = encoder(r, precision=FP16)
        e16.load_weights(ep)
        xu8 = _crops(r, RAGGED, 7)
        z16 = e16.encode_device(torch.from_numpy(xu8).cuda()).cpu().numpy()
        peak.sample()
        acts = [O.preprocess(xu8)] + [e16.activation_device(l, sess.device).cpu().numpy() for l in range(r["L"])]
        for l in range(r["L"]):
            name = "conv2d" if l == 0 else "conv2d_%d" % l
            _conv_bound_check(acts[l], ep[name + "/kernel"], ep[name + "/bias"], acts[l + 1], "%s fp16 %s" % (rid, name))
        _dense_bound_check(acts[-1].reshape(RAGGED, -1), ep["dense/kernel"], ep["dense/bias"], z16)
        e16.close()
    peak.report()
    _free()


# ------------------------------------------------------------------------------------------------------------ codebook
@pytest.mark.parametrize("rid", ["latent32", "latent64", "latent256", "px127", "px100"])
def test_codebook_match_at_other_latents(sess, rid):
    """nearest_idx_device end to end (encoder + the fp32 match the automatic precision picks at latent != 128; at 127 px the split
    encoder with its fp32 conv1 and the tensor-core match, at 100 px the fp32 encoder and match), k = 8 and upright: scores
    within 1e-5 of the float64 cosine of the returned row, and an index other than float64's argmax only where float64 puts the
    two within 2e-6."""
    r = row(rid)
    ep, _, _ = params(r)
    E = O.make_codebook(5, n=36 * 300, j=r["latent"])
    enc = encoder(r)
    enc.load_weights(ep)
    cb = _codebook(enc, E, max_batch=MAXB)
    xu8 = _crops(r, RAGGED, 21)
    cos64 = O.cos_similarity(_enc64(O.preprocess(xu8), ep, r["strides"])[-1], E.astype(np.float64))
    x = torch.from_numpy(xu8).cuda()
    worst = 0.0
    for k, upright in ((1, False), (8, False), (1, True)):
        s, i = cb.nearest_idx_device(x, k=k, upright=upright)
        s, i = s.cpu().numpy(), i.cpu().numpy()
        assert s.shape == (RAGGED, k)
        c = cos64[:, ::36] if upright else cos64
        for b in range(RAGGED):
            got = i[b] // 36 if upright else i[b]
            if upright:
                assert np.all(i[b] % 36 == 0)
            worst = max(worst, float(np.max(np.abs(s[b] - c[b, got]))))
            want = np.lexsort((np.arange(c.shape[1]), -c[b]))[:k]
            for j in np.nonzero(want != got)[0]:
                assert abs(c[b, want[j]] - c[b, got[j]]) < 2e-6, (rid, b, j, want, got)
            assert np.all(np.diff(s[b]) <= 0)
    print("%s match (precision %d): worst |score - cos64| %.1e" % (rid, cb.precision, worst))
    assert cb.precision == LANDING[rid][1]
    assert worst < COS_TOL, worst
    cb.close()
    enc.close()
    _free()


# ------------------------------------------------------------------------------------------------------------ decoder
@pytest.mark.parametrize("rid", IDS)
def test_decoder_forward_matches_float64(sess, rid):
    """x, without and with the mask head (and the head's output), at batch 1 and a ragged batch: 5e-6 absolute on the tensor cores,
    2e-6 on the fp32 kernels.  The head does not move the decoder to another precision."""
    _needs_decoder(rid)
    tol = 5e-6 if LANDING[rid][2] == SPLIT else 2e-6
    for mask in (False, True):
        r = row(rid, mask=mask)
        ep, dp, head = params(r)
        dec = decoder(r, encoder(r))
        dec.load_weights(dec_weights(r, dp, head))
        P = {k: _g(v) for k, v in dp.items()}
        worst_x, worst_m = 0.0, 0.0
        for B in (1, RAGGED):
            z = np.random.RandomState(B).standard_normal((B, r["latent"])).astype(np.float32)
            zt = torch.from_numpy(z).cuda()
            with torch.no_grad():
                if head is None:
                    x64 = O.decoder_layers(_g(z), P, out_hw=r["h"], strides=r["strides"], n_encoder_convs=r["L"])[-1].cpu().numpy()
                    x = dec.decode_device(zt).cpu().numpy()
                else:
                    x64, m64 = (t.cpu().numpy() for t in MO.decoder_with_mask(_g(z), P, _g(head[0]), _g(head[1]), r["h"], r["strides"], r["L"]))
                    x, m = (t.cpu().numpy() for t in dec.decode_device(zt, with_mask=True))
                    assert m.shape == m64.shape, (m.shape, m64.shape)
                    worst_m = max(worst_m, float(np.max(np.abs(m - m64))))
            assert x.shape == x64.shape, (x.shape, x64.shape)
            worst_x = max(worst_x, float(np.max(np.abs(x - x64))))
        print("%s decoder%s (precision %d): worst |x - x64| %.1e%s (bound %.0e)"
              % (rid, " + mask head" if mask else "", dec.precision, worst_x, ", |xmask - m64| %.1e" % worst_m if mask else "", tol))
        assert dec.precision == LANDING[rid][2], (rid, mask, dec.precision)
        assert worst_x < tol and worst_m < tol, (rid, mask, worst_x, worst_m)
        dec.close()
        _free()


@pytest.mark.parametrize("rid,L", [("px100", 4), ("px127", 4), ("px112", 5)])
def test_decoder_refuses_a_crop_that_is_not_a_multiple_of_2_to_the_L(sess, rid, L):
    """Every stage doubles its map, so H = 100 would give 6 -> ... -> 96 and H = 127 (or 112 with five convs) 7 -> ... -> 112: the
    handle is refused when it is created, on every precision, naming H and 2^L; the automatic precision ends on fp32 and raises."""
    from augmentedautoencoder_b200 import _lib
    r = row(rid) if L == 4 else row(rid, nf=(128, 256, 512, 512, 512), strides=(2,) * 5, L=5)
    msg = r"H = %d is not a multiple of 2\^L = %d" % (r["h"], 2 ** L)
    for prec in (FP32, SPLIT, None):
        d = decoder(r, encoder(r), precision=prec)
        with pytest.raises(_lib.AaeError, match=msg):
            d.handle(sess.device)
        assert d.precision == (FP32 if prec is None else prec)
        d.close()


# ------------------------------------------------------------------------------------------------------------ training
def _reference(r, x, y, ep, dp, head, bootstrap=4):
    if head is None:
        loss, _, g = O.ae_forward_loss(x, y, ep, dp, dtype=torch.float64, with_grads=True, device="cuda", strides=r["strides"],
                                       bootstrap_ratio=bootstrap)
    else:
        loss, _, _, g = MO.mask_forward_loss(x, y, ep, dp, head, dtype=torch.float64, with_grads=True, device="cuda",
                                             bootstrap_ratio=bootstrap)
    return loss, g


def _rel(a, b):
    return float(np.linalg.norm(a.astype(np.float64) - b) / max(np.linalg.norm(b), 1e-300))


@pytest.mark.parametrize("rid", IDS)
def test_training_step_matches_float64(sess, rid):
    """The loss and every gradient at batch 1 and a ragged batch (and PARITY_BATCH on PARITY_ROWS, where one step takes both
    orderings of the fp32 trainer's stride-2 dgrad), on whichever trainer the row settles on, within 3e-4 relative L2,
    on weights that leave a quarter of every ReLU layer dead with every pre-activation clear of zero.  Where the split trainer
    runs, five Adam steps follow the fp32 trainer: losses within 5e-5, and each variable's five-step update within 0.1 relative L2
    of the fp32 trainer's (Adam's normalised step turns the 3e-5 gradient differences of components near zero into differences
    of up to 2 lr, so an update differs by a few percent although its gradients agree; a wrong gradient moves it by order 1).
    After a demotion both handles are fp32 and compute what fresh handles loaded from get_weights() compute."""
    _needs_decoder(rid)
    r = row(rid)
    ep, dp, head = _masked(r, *params(r))
    peak = _Peak(rid + " training")
    enc, dec, top = _pair(r, ep, dp, head)
    worst = 0.0
    for B in (1, RAGGED) + ((PARITY_BATCH,) if rid in PARITY_ROWS else ()):
        x = np.random.RandomState(8).rand(B, r["h"], r["w"], r["c"]).astype(np.float32)
        y = np.random.RandomState(4).rand(B, r["h"], r["w"], r["c"]).astype(np.float32)
        margin, shares = _check_relu_paths(r, x, ep, dp)
        loss64, g64 = _reference(r, x, y, ep, dp, head)
        enc.load_weights(ep)
        dec.load_weights(dec_weights(r, dp, head))
        loss = float(top.step_device(torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda(), update=False))
        grads = top.gradients(sess.device)
        peak.sample()
        assert abs(loss - loss64) <= 2e-6 * abs(loss64), (rid, B, loss, loss64)
        assert sorted(grads) == sorted(g64)
        for name, g in g64.items():
            rel = _rel(grads[name], g)
            assert rel <= REL_TRAIN, (rid, B, name, rel)
            worst = max(worst, rel)
    assert (enc.precision, dec.precision) == (LANDING[rid][3],) * 2
    print("%s trainer (precision %d): ReLU margin %.2f, dead shares %.2f..%.2f, worst relative L2 gradient error %.1e"
          % (rid, enc.precision, margin, min(shares.values()), max(shares.values()), worst))
    xt = torch.from_numpy(np.random.RandomState(11).rand(RAGGED, r["h"], r["w"], r["c"]).astype(np.float32)).cuda()
    yt = torch.from_numpy(np.random.RandomState(12).rand(RAGGED, r["h"], r["w"], r["c"]).astype(np.float32)).cuda()
    if enc.precision == SPLIT:
        w0 = {**ep, **dec_weights(r, dp, head)}
        enc.load_weights(ep)
        dec.load_weights(dec_weights(r, dp, head))
        split = [float(top.step_device(xt, yt)) for _ in range(5)]
        ws = {**enc.get_weights(short_names=True), **dec.get_weights(short_names=True)}
        top.close(); enc.close(); dec.close()
        enc, dec, top = _pair(r, ep, dp, head, precision=FP32)
        ref = [float(top.step_device(xt, yt)) for _ in range(5)]
        wr = {**enc.get_weights(short_names=True), **dec.get_weights(short_names=True)}
        upd = {n: _rel(ws[n] - w0[n], (wr[n] - w0[n]).astype(np.float64)) for n in w0}
        dl = float(np.max(np.abs(np.array(split) - np.array(ref))))
        print("%s Adam, five steps: largest loss difference %.1e, largest relative L2 difference of a weight update %.1e (%s)"
              % (rid, dl, max(upd.values()), max(upd, key=upd.get)))
        assert dl < 5e-5, (split, ref)
        assert max(upd.values()) < 0.1, upd
    else:
        top.step_device(xt, yt)
        z = enc.encode_device(xt).cpu().numpy()
        rec = dec.decode_device(torch.from_numpy(z).cuda()).cpu().numpy()
        e0 = encoder(r, precision=FP32)
        e0.load_weights(enc.get_weights())
        d0 = decoder(r, e0, precision=FP32)
        d0.load_weights(dec.get_weights())
        assert np.array_equal(z, e0.encode_device(xt).cpu().numpy()), rid
        assert np.array_equal(rec, d0.decode_device(torch.from_numpy(z).cuda()).cpu().numpy()), rid
        e0.close(); d0.close()
    peak.sample()
    peak.report()
    top.close(); enc.close(); dec.close()
    _free()


# ------------------------------------------------------------------------------------------------------------ fp16 trainer
def _fp16_layers(r):
    """forward order and kind (tests/test_gpu_e_fp16_train.LAYERS for any depth)"""
    L = r["L"]
    return ([("conv2d" if i == 0 else "conv2d_%d" % i, "enc") for i in range(L)] + [("dense", "dense"), ("dense_1", "dense1")] +
            [("conv2d_%d" % (L + j), "dec") for j in range(L - 1)] + [(output_conv(r), "out")])


def _analyse(r, x, y, ep, dp):
    """tests/test_gpu_e_fp16_train._analyse for the row's layers and bottleneck size, without bootstrapping"""
    layers, d0 = _fp16_layers(r), r["h"] // int(np.prod(r["strides"]))
    P = {k: _g(v) for k, v in {**ep, **dp}.items()}
    a = _g(x)
    ins, masks, fwd_rel, relu_need = [], [], 0.0, 0.0
    for name, kind in layers:
        w, b = P[name + "/kernel"], P[name + "/bias"]
        ins.append(a)
        pre = _apply(kind, a, w, b)
        fwd_rel += U * _cond(_apply(kind, a.abs(), w.abs(), torch.zeros_like(b)), pre)
        if kind == "out":
            break
        if kind == "dense":
            a = pre
            masks.append(None)
            continue
        relu_need = max(relu_need, fwd_rel * float(pre.abs().max()))
        m = (pre > 0).double()
        if kind == "dense1":
            pre, m = (t.reshape(-1, d0, d0, t.shape[1] // (d0 * d0)) for t in (pre, m))
        masks.append(m)
        a = pre * m
    rec = torch.sigmoid(pre)
    sig = rec * (1 - rec)
    B = rec.shape[0]
    yd = _g(y)
    k = yd[0].numel()
    d_rec = sig * fwd_rel * float(pre.abs().max())
    seed = (2.0 / (B * k)) * (rec - yd) * sig
    d_seed = (2.0 / (B * k)) * (sig + (rec - yd).abs()) * d_rec
    loss_bound = float((2 * (rec - yd).abs() * d_rec + d_rec ** 2).sum() / (B * k))
    return dict(P=P, ins=ins, masks=masks, seed=seed, seed_rel=_cond(d_seed, seed), fwd_rel=fwd_rel, loss_bound=loss_bound,
                relu_need=relu_need, layers=layers)


def _grad_bounds(A):
    """tests/test_gpu_e_fp16_train._grad_bounds over the row's layers"""
    layers = A["layers"]
    out, g, bwd_rel = {}, A["seed"], 0.0
    for i in reversed(range(len(layers))):
        name, kind = layers[i]
        ops = (A["ins"][i], A["P"][name + "/kernel"], A["P"][name + "/bias"])
        val = [t.detach().clone().requires_grad_(True) for t in ops]
        mag = [t.abs().detach().clone().requires_grad_(True) for t in ops]
        yv = _apply(kind, *val)
        yv.backward(g.reshape(yv.shape))
        _apply(kind, *mag).backward(g.abs().reshape(yv.shape))
        base = A["fwd_rel"] + A["seed_rel"] + bwd_rel
        out[name + "/kernel"] = 2 * (base + U * _cond(mag[1].grad, val[1].grad))
        out[name + "/bias"] = 2 * (base + U * _cond(mag[2].grad, val[2].grad))
        if i > 0:
            bwd_rel += U * _cond(mag[0].grad, val[0].grad)
            g = val[0].grad if A["masks"][i - 1] is None else val[0].grad * A["masks"][i - 1].reshape(val[0].grad.shape)
    return out


@pytest.mark.parametrize("rid", ["narrow", "latent256"])
def test_fp16_trainer_meets_the_rounding_bound(sess, rid):
    """The single-pass fp16 trainer (TrainOp(precision=PREC_TC_FP16) on split handles: hi-only encoder and decoder plans of its own)
    at batch 1 and a ragged batch, on the masked weights: the loss within twice its rounding-model bound and every gradient within
    its bound (tests/test_gpu_e_fp16_train's model, generalised to the row's layers).  No bootstrapping: the model has no term for a
    discrete top-k choice."""
    r = row(rid)
    ep, dp, head = _masked(r, *params(r))
    peak = _Peak(rid + " fp16 trainer")
    enc, dec, top = _pair(r, ep, dp, head, precision=SPLIT, gemm=FP16, bootstrap=1)
    for B in (1, RAGGED):
        x = np.random.RandomState(8).rand(B, r["h"], r["w"], r["c"]).astype(np.float32)
        y = np.random.RandomState(4).rand(B, r["h"], r["w"], r["c"]).astype(np.float32)
        _check_relu_paths(r, x, ep, dp)
        A = _analyse(r, x, y, ep, dp)
        margin = O.relu_margin(x, ep, dp, device="cuda", strides=r["strides"])
        assert margin > 2 * A["relu_need"], (rid, B, margin, A["relu_need"])
        bounds = _grad_bounds(A)
        loss64, g64 = _reference(r, x, y, ep, dp, head, bootstrap=1)
        loss = float(top.step_device(torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda(), update=False))
        grads = top.gradients(sess.device)
        peak.sample()
        assert (enc.precision, dec.precision) == (SPLIT, SPLIT)
        tag = "%s fp16 trainer, B=%d" % (rid, B)
        print("%s: |loss - loss64| = %.2e, bound %.2e; gradient bounds %.1e .. %.1e"
              % (tag, abs(loss - loss64), 2 * A["loss_bound"], min(bounds.values()), max(bounds.values())))
        assert abs(loss - loss64) <= 2 * A["loss_bound"], (tag, loss, loss64)
        assert sorted(grads) == sorted(g64)
        _check_grads(grads, g64, bounds, tag)
        del A
    peak.report()
    top.close(); enc.close(); dec.close()
    _free()


# ------------------------------------------------------------------------------------------------------------ loss limit
def test_bootstrapped_l2_at_its_shared_memory_limit(sess):
    """aae_bootstrap_l2_loss at exactly AAE_BOOTSTRAP_MAX_NUMEL = 51 200 values per sample (the whole dynamic shared-memory row
    buffer), ratio 4, with squared errors on a few hundred exact levels so that every cut splits a tie: the selected set equals a
    stable float64 top-k (lowest index first among ties) element for element, and the loss and the gradient on that set match.
    One value more is refused before anything is launched."""
    from augmentedautoencoder_b200 import _lib
    from augmentedautoencoder_b200.ae.decoder import Decoder
    B, numel, ratio = 6, 51200, 4
    k = numel // ratio
    rng = np.random.RandomState(22)
    q = rng.randint(1, 301, (B, numel))                    # |x - t| = q 2^-10 and its square are exact in fp32
    t = np.full((B, numel), 0.5)
    x = t + np.where(rng.rand(B, numel) < 0.5, -1.0, 1.0) * q * 2.0 ** -10
    shape = (B, 160, 160, 2)
    loss, grad = Decoder.loss_device(torch.from_numpy(x.astype(np.float32).reshape(shape)).cuda(),
                                     torch.from_numpy(t.astype(np.float32).reshape(shape)).cuda(), ratio, with_grad=True)
    grad = grad.reshape(B, numel).cpu().numpy()
    l2 = (x - t) ** 2
    order = np.argsort(-l2, axis=1, kind="stable")[:, :k]
    want = np.zeros((B, numel), bool)
    np.put_along_axis(want, order, True, axis=1)
    thr = np.take_along_axis(l2, order[:, -1:], axis=1)
    at_thr = l2 == thr
    assert np.all(np.sum(at_thr & want, axis=1) > 0) and np.all(np.sum(at_thr & ~want, axis=1) > 0)   # every cut splits a tie
    bad_rows = np.nonzero(np.any((grad != 0) != want, axis=1))[0]
    assert not len(bad_rows), ("selection differs in rows", bad_rows)
    loss64 = float(np.take_along_axis(l2, order, axis=1).mean())
    assert abs(float(loss) - loss64) < 1e-6, (float(loss), loss64)
    g64 = 2.0 * (x - t) / (B * k)
    assert np.allclose(grad[want], g64[want], rtol=1e-6, atol=0.0)
    over = torch.zeros((1, numel + 1), device="cuda")
    with pytest.raises(_lib.AaeError, match="51200"):
        Decoder.loss_device(over, over, ratio)


@pytest.mark.parametrize("precision", [None, FP32])
def test_trainer_refuses_a_crop_above_the_loss_limit(sess, precision):
    """A 144 x 144 x 3 crop (62 208 values) is more than the bootstrapped L2 loss holds per sample: the encoder and decoder are
    created (on fp32: 72 and 9 are no powers of two), and the trainer is refused when it is created, naming the limit, instead of
    failing at its first step."""
    from augmentedautoencoder_b200 import _lib
    from augmentedautoencoder_b200.ae.ae import AE
    from augmentedautoencoder_b200.ae.ae_factory import TrainOp
    r = dict(T, h=144, w=144, L=len(T["nf"]), id="px144")
    enc = encoder(r, precision, is_training=True)
    dec = decoder(r, enc, precision)
    top = TrainOp(AE(enc, dec, 0, 0), 2e-4)
    with pytest.raises(_lib.AaeError, match="144 x 144 x 3 crop is 62208 values.*AAE_BOOTSTRAP_MAX_NUMEL = 51200"):
        top.trainer(sess.device)
    assert (enc.precision, dec.precision) == (FP32, FP32)
    top.close(); enc.close(); dec.close()
    _free()
