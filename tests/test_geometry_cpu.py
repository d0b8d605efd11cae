"""CPU tests of the geometries tests/geometry_table.py lists: the Python modules declare the variables the oracle builds for each
row, and the oracle's forward for those shapes (more than four convs, H != W, one channel, kernel 3, a stride-1 conv) equals a
direct loop implementation (no GPU: no device handle is created)."""
import numpy as np
import pytest
import torch

from oracle import aae_oracle as O
from oracle import mask_oracle as MO
from tests.geometry_table import ROWS, dec_weights, decoder, encoder, params, row


def _shapes(mod):
    return {n: tuple(s) for kn, ks, bn, bs in mod._var_shapes for n, s in ((kn, ks), (bn, bs))}


@pytest.mark.parametrize("rid", list(ROWS))
def test_module_variables_equal_the_oracle_params(rid):
    """Names and shapes of every Encoder and Decoder variable equal the oracle's make_*_params for the row (with the mask head
    under the decoder's own numbering)."""
    r = row(rid)
    ep, dp, head = params(r)
    enc = encoder(r)
    assert _shapes(enc) == {n: v.shape for n, v in ep.items()}
    assert enc.variable_names == list(_shapes(enc))
    dec = decoder(r, enc)
    assert _shapes(dec) == {n: v.shape for n, v in dec_weights(r, dp, head).items()}
    enc.load_weights(ep)                                      # host-side only: the shapes are checked against the declaration
    dec.load_weights(dec_weights(r, dp, head))


def test_oracle_defaults_are_unchanged():
    """The width arguments default to square crops, drawing the same values as before"""
    a, b = O.make_encoder_params(42), O.make_encoder_params(42, in_w=O.W)
    assert a.keys() == b.keys() and all(np.array_equal(a[k], b[k]) for k in a)
    assert np.array_equal(O.make_crops_u8(3, 2), O.make_crops_u8(3, 2, w=O.W))
    assert O.make_crops_u8(3, 2, hw=16, w=32).shape == (2, 16, 32, 3)


def _loop_encoder(x, p, strides):
    h = x.astype(np.float64)
    for i, s in enumerate(strides):
        name = "conv2d" if i == 0 else "conv2d_%d" % i
        h = np.maximum(O.conv2d_same_loops(h, p[name + "/kernel"], p[name + "/bias"], s), 0.0)
    return h, h.reshape(h.shape[0], -1) @ p["dense/kernel"].astype(np.float64) + p["dense/bias"].astype(np.float64)


def _loop_decoder(z, p, hw, L):
    st = [2] * L
    d0 = hw // int(np.prod(st))
    h = np.maximum(z @ p["dense_1/kernel"].astype(np.float64) + p["dense_1/bias"].astype(np.float64), 0.0)
    h = h.reshape(z.shape[0], d0, d0, -1)
    for j in range(L):
        k = L + j
        h = np.repeat(np.repeat(h, 2, axis=1), 2, axis=2)     # nearest x2
        y = O.conv2d_same_loops(h, p["conv2d_%d/kernel" % k], p["conv2d_%d/bias" % k], 1)
        h = np.maximum(y, 0.0) if j + 1 < L else 1.0 / (1.0 + np.exp(-y))
    return h


# small stand-ins of the GPU table's shapes: (in h, in w, channels, filters, strides, kernel)
SMALL = {
    "five_layer": (32, 32, 3, (4, 4, 8, 8, 8), (2,) * 5, 5),
    "rect": (16, 32, 3, (4, 8), (2, 2), 5),
    "gray": (16, 16, 1, (4, 8), (2, 2), 5),
    "k3": (16, 16, 3, (4, 8), (2, 2), 3),
    "stride1": (16, 16, 3, (4, 4, 8), (2, 1, 2), 5),
}


@pytest.mark.parametrize("case", list(SMALL))
def test_oracle_encoder_equals_loop_conv(case):
    h, w, c, nf, strides, k = SMALL[case]
    p = O.make_encoder_params(3, num_filters=nf, ksize=k, latent=8, in_ch=c, in_hw=h, strides=strides, bias_scale=0.1, in_w=w)
    x = O.preprocess(O.make_crops_u8(4, 2, hw=h, ch=c, w=w))
    outs = O.encoder_layers(x, p, strides=strides, dtype=torch.float64)
    last, z = _loop_encoder(x, p, strides)
    assert outs[len(strides) - 1].shape == last.shape
    assert np.max(np.abs(outs[len(strides) - 1].numpy() - last)) < 1e-12
    assert np.max(np.abs(outs[-1].numpy() - z)) < 1e-12


@pytest.mark.parametrize("case", ["five_layer", "gray"])
def test_oracle_training_forward_equals_loop_conv(case):
    """ae_forward_loss and relu_margin with an explicit strides argument (five convs, which the template's STRIDES cannot
    describe): the reconstruction equals a loop forward and the loss its bootstrapped L2; relu_margin walks the same layers."""
    h, w, c, nf, strides, k = SMALL[case]
    L = len(nf)
    ep = O.make_encoder_params(3, num_filters=nf, ksize=k, latent=8, in_ch=c, in_hw=h, strides=strides, bias_scale=0.1)
    dp = O.make_decoder_params(4, num_filters=nf, ksize=k, latent=8, out_ch=c, out_hw=h, strides=strides, bias_scale=0.1,
                               n_encoder_convs=L)
    x = np.random.RandomState(1).rand(2, h, w, c).astype(np.float32)
    y = np.random.RandomState(2).rand(2, h, w, c).astype(np.float32)
    # (torch's CPU float64 conv backward refuses the 1-channel output conv's kernel layout: gradients for the 5-conv case only)
    grads = case != "gray"
    loss, rec, g = O.ae_forward_loss(x, y, ep, dp, dtype=torch.float64, with_grads=grads, strides=strides)
    _, z = _loop_encoder(x, ep, strides)
    rec_loop = _loop_decoder(z, dp, h, L)
    assert rec.shape == rec_loop.shape and np.max(np.abs(rec - rec_loop)) < 1e-12
    l2 = ((y.astype(np.float64) - rec_loop) ** 2).reshape(2, -1)
    kk = l2.shape[1] // O.BOOTSTRAP_RATIO
    assert abs(loss - np.sort(l2, axis=1)[:, -kk:].mean()) < 1e-12
    assert not grads or sorted(g) == sorted({**ep, **dp})
    assert O.relu_margin(x, ep, dp, strides=strides) > 0.0


def test_mask_oracle_matches_loop_conv_at_one_channel():
    """the gray + AUXILIARY_MASK row's reference: the mask head's output equals a loop conv over the decoder's last hidden layer"""
    h, nf, L = 16, (4, 8), 2
    dp = O.make_decoder_params(4, num_filters=nf, latent=8, out_ch=1, out_hw=h, strides=(2, 2), bias_scale=0.1, n_encoder_convs=L)
    hk, hb = MO.make_mask_head(5, nf[0], 5, 0.1)
    z = np.random.RandomState(3).standard_normal((2, 8))
    P = {n: torch.from_numpy(v).double() for n, v in dp.items()}
    x, m = MO.decoder_with_mask(torch.from_numpy(z), P, torch.from_numpy(hk).double(), torch.from_numpy(hb).double(), h, (2, 2), L)
    assert np.max(np.abs(x.numpy() - _loop_decoder(z, dp, h, L))) < 1e-12
    # the hidden activation entering the output conv, and the head on it
    d0 = h // 4
    a = np.maximum(z @ dp["dense_1/kernel"].astype(np.float64) + dp["dense_1/bias"], 0.0).reshape(2, d0, d0, -1)
    a = np.maximum(O.conv2d_same_loops(np.repeat(np.repeat(a, 2, 1), 2, 2), dp["conv2d_2/kernel"], dp["conv2d_2/bias"], 1), 0.0)
    want = 1.0 / (1.0 + np.exp(-O.conv2d_same_loops(np.repeat(np.repeat(a, 2, 1), 2, 2), hk, hb, 1)))
    assert m.shape == (2, h, h, 1) and np.max(np.abs(m.numpy() - want)) < 1e-12
