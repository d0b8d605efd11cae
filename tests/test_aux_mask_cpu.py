"""CPU tests of AUXILIARY_MASK: TF variable names with and without the mask head, the mask target at its threshold, the oracle's
loss and gradient, and the checkpoint round trip of the head's variables (no GPU: no device handle is created)."""
import numpy as np
import pytest
import torch

from oracle import aae_oracle as O
from oracle import mask_oracle as MO


def _graph(aux_mask, variational=False, seed=43):
    from augmentedautoencoder_b200.ae.decoder import Decoder
    from augmentedautoencoder_b200.ae.encoder import Encoder
    from augmentedautoencoder_b200.ae.session import placeholder
    x, y = placeholder(np.float32, [None, 128, 128, 3]), placeholder(np.float32, [None, 128, 128, 3])
    enc = Encoder(x, 128, list(O.NUM_FILTER), 5, list(O.STRIDES), False, is_training=True, max_batch=2)
    dec = Decoder(y, enc.sampled_z if variational else enc.z, list(reversed(O.NUM_FILTER)), 5, list(reversed(O.STRIDES)), "L2", 4,
                  aux_mask, False, is_training=True, max_batch=2, seed=seed)
    return enc, dec


def _shapes(dec):
    return {n: s for kn, ks, bn, bs in dec._var_shapes for n, s in ((kn, ks), (bn, bs))}


@pytest.mark.parametrize("variational", [False, True])
def test_names_follow_tf_layer_numbering(variational):
    """With the head, TF numbers it conv2d_7 and the output conv conv2d_8 (the head is created first); dense names are unchanged,
    with or without the sigma head.  Without it, every name and shape is as before."""
    dense = "dense_2" if variational else "dense_1"
    _, plain = _graph(False, variational)
    _, masked = _graph(True, variational)
    want_plain = [dense + "/kernel", dense + "/bias"] + ["conv2d_%d/%s" % (k, p) for k in (4, 5, 6, 7) for p in ("kernel", "bias")]
    assert plain.variable_names == want_plain
    assert masked.variable_names == want_plain[:-2] + ["conv2d_8/kernel", "conv2d_8/bias", "conv2d_7/kernel", "conv2d_7/bias"]
    s = _shapes(masked)
    assert s["conv2d_7/kernel"] == (5, 5, 128, 1) and s["conv2d_7/bias"] == (1,)
    assert s["conv2d_8/kernel"] == (5, 5, 128, 3) and s["conv2d_8/bias"] == (3,)
    assert not hasattr(plain, "_xmask") and masked._xmask.get_shape().as_list() == [None, 128, 128, 1]


def test_switch_off_keeps_the_random_stream_and_on_appends_the_head():
    """The head's initial kernel is drawn after every other variable: the other variables keep the values a decoder without the head
    draws from the same seed.  The head's bias starts at zero."""
    _, plain = _graph(False)
    _, masked = _graph(True)
    a, b = plain.get_weights(), masked.get_weights()
    for name in plain.variable_names:
        renamed = name.replace("conv2d_7/", "conv2d_8/")
        assert np.array_equal(a[name], b[renamed]), name
    assert np.all(b["conv2d_7/bias"] == 0) and np.abs(b["conv2d_7/kernel"]).max() > 0


def test_mask_target_at_the_threshold():
    """m = float(sum over channels > 0.0001) in float32, channels summed in order: a sum equal to float32(0.0001) is background, the
    next float32 above it is object, and the channel order of the fp32 sum is the one that decides."""
    t = np.float32(0.0001)
    up = np.nextafter(t, np.float32(1))
    y = np.zeros((1, 2, 3, 3), np.float32)
    y[0, 0, 0] = (t, 0, 0)
    y[0, 0, 1] = (up, 0, 0)
    y[0, 0, 2] = (0, 0, up)
    y[0, 1, 0] = (t / 2, t / 2, 0)                 # exactly 0.0001 in float32: background
    a, b = np.float32(6e-5), np.float32(4e-5)      # a + b rounds to the float32 0.0001 or to a neighbour: follow fp32 in order
    y[0, 1, 1] = (a, b, 0)
    y[0, 1, 2] = (1.0, 0, 0)
    m = MO.mask_target(y)
    assert m.shape == (1, 2, 3, 1) and m.dtype == np.float32
    s = np.float32(np.float32(a + b) + np.float32(0))
    assert list(m[0, :, :, 0].ravel()) == [0, 1, 1, 0, float(s > t), 1]
    assert float(np.float32(t / 2) + np.float32(t / 2)) == float(t)


def test_oracle_mask_loss_and_gradient():
    """The oracle's closed-form gradient 2 (xmask - m) / (B H W) equals autograd of tf.losses.mean_squared_error(m, xmask) in float64,
    and the loss is their mean squared difference."""
    rng = np.random.RandomState(0)
    y = rng.rand(2, 8, 8, 3).astype(np.float32)
    y[rng.rand(2, 8, 8) < 0.5] = 0
    xm = rng.rand(2, 8, 8, 1)
    xt = torch.from_numpy(xm).requires_grad_(True)
    loss = MO.mask_loss(xt, torch.from_numpy(MO.mask_target(y)).double())
    loss.backward()
    l2, g = MO.mask_loss_grad(xm, y)
    assert abs(float(loss.detach()) - l2) < 1e-15 and np.allclose(xt.grad.numpy(), g, rtol=0, atol=1e-17)
    assert abs(l2 - np.mean((xm - MO.mask_target(y)) ** 2)) < 1e-15


def test_oracle_head_is_a_conv_over_the_output_conv_input():
    """decoder_with_mask's x is aae_oracle.decoder_layers' output, and a head equal to one channel of the output conv reproduces that
    channel of x: the two read the same input."""
    dp = O.make_decoder_params(3, num_filters=(4, 8), out_hw=16, strides=(2, 2), latent=8, bias_scale=0.1, n_encoder_convs=2)
    tp = {k: torch.from_numpy(v).double() for k, v in dp.items()}
    z = torch.from_numpy(np.random.RandomState(1).standard_normal((2, 8)))
    hk, hb = tp["conv2d_3/kernel"][..., 1:2], tp["conv2d_3/bias"][1:2]
    x, xm = MO.decoder_with_mask(z, tp, hk, hb, 16, (2, 2), 2)
    ref = O.decoder_layers(z, tp, out_hw=16, strides=(2, 2), n_encoder_convs=2)[-1]
    assert torch.equal(x, ref) and torch.allclose(xm[..., 0], x[..., 1], rtol=0, atol=1e-15)


def test_tf_bundle_round_trip_carries_the_head_and_its_slots(tmp_path):
    """The head's kernel and bias and their optimizer slots under TF names survive a TF tensor-bundle write / read, and a strict
    Saver.restore from it loads the head into a decoder with the switch on."""
    from augmentedautoencoder_b200.ae import ae_factory as F
    from augmentedautoencoder_b200.ae.tf_checkpoint import read_tf_checkpoint, write_tf_checkpoint
    _, src = _graph(True, seed=5)
    w = src.get_weights()
    rng = np.random.RandomState(2)
    w["conv2d_7/bias"] = np.full(1, 0.25, np.float32)
    for name in ("conv2d_7/kernel", "conv2d_7/bias", "conv2d_8/kernel", "conv2d_8/bias"):
        for slot in ("Adam", "Adam_1"):
            w[name + "/" + slot] = rng.rand(*w[name].shape).astype(np.float32)
    prefix = str(tmp_path / "chkpt-7")
    write_tf_checkpoint(prefix, w)
    back = read_tf_checkpoint(prefix)
    assert sorted(back) == sorted(w) and all(np.array_equal(back[k], w[k]) for k in w)
    assert back["conv2d_7/kernel/Adam"].shape == (5, 5, 128, 1)
    _, dst = _graph(True, seed=9)
    F.Saver([dst]).restore(None, prefix)
    got = dst.get_weights()
    assert all(np.array_equal(got[k], w[k]) for k in dst.variable_names)
    _, plain = _graph(False)
    with pytest.raises(ValueError, match="conv2d_7/kernel"):      # a decoder without the head reads conv2d_7 as its output conv
        F.Saver([plain]).restore(None, prefix)
