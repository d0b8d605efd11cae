"""CPU tests of the geometries tests/geometry_table.py lists: the Python modules declare the variables the oracle builds for each
row, and the oracle's forward for those shapes (more than four convs, H != W, one channel, kernel 3, a stride-1 conv) equals a
direct loop implementation (no GPU: no device handle is created)."""
import numpy as np
import pytest
import torch

from oracle import aae_oracle as O
from oracle import mask_oracle as MO
from tests.geometry_table import ROWS, T, dec_weights, decoder, encoder, params, row


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


# the rows that were in the table before crop sizes other than powers of two
POW2_ROWS = [rid for rid in ROWS if rid not in ("px112", "px80", "px96", "px127", "h127", "px100")]


@pytest.mark.parametrize("rid", ["template"] + POW2_ROWS)
def test_encoder_params_at_power_of_two_sizes_are_unchanged(rid):
    """make_encoder_params takes TF SAME's ceil(in / stride) per map; at the template and every power-of-two row that equals the
    floor it took before, so the dense kernel keeps its shape and every draw its value"""
    r = dict(T, L=len(T["nf"]), id=rid) if rid == "template" else row(rid)
    h, w = r["h"], r["w"]
    for s in r["strides"]:
        assert -(-h // s) == h // s and -(-w // s) == w // s, (rid, h, w, s)
        h, w = h // s, w // s
    ep, _, _ = params(r)
    assert ep["dense/kernel"].shape == (h * w * r["nf"][-1], r["latent"])


@pytest.mark.parametrize("rid,maps", [("px112", (56, 28, 14, 7)), ("px80", (40, 20, 10, 5)), ("px96", (48, 24, 12, 6)),
                                      ("px127", (64, 32, 16, 8)), ("h127", (64, 32, 16, 8)), ("px100", (50, 25, 13, 7))])
def test_encoder_params_take_the_ceiling_of_each_map(rid, maps):
    """the dense kernel of the rows whose maps SAME padding rounds up: ceil(in / 2) per conv, 8 x 8 at 127 (the floor gave 7 x 7);
    the oracle's forward on a crop of the row's size produces those maps and feeds that kernel (127 x 128 has the same maps in
    both directions)"""
    r = row(rid)
    ep, _, _ = params(r)
    assert ep["dense/kernel"].shape == (maps[-1] * maps[-1] * r["nf"][-1], r["latent"])
    x = O.preprocess(O.make_crops_u8(5, 1, hw=r["h"], ch=r["c"], w=r["w"]))
    outs = O.encoder_layers(x, ep, strides=r["strides"], dtype=torch.float64)
    assert [tuple(o.shape[1:3]) for o in outs[:r["L"]]] == [(m, m) for m in maps], rid
    assert outs[-1].shape == (1, r["latent"])


def _old_crops_u8(seed, batch, hw, ch, w):
    """make_crops_u8 as it was while every crop size was a multiple of its cell count"""
    rng = np.random.RandomState(seed)
    cells, cells_w = max(hw // 16, 1), max(w // 16, 1)
    coarse = rng.randint(0, 256, size=(batch, cells, cells_w, ch)).astype(np.int32)
    img = np.repeat(np.repeat(coarse, hw // cells, axis=1), w // cells_w, axis=2)
    img = img + rng.randint(-40, 41, size=(batch, hw, w, ch))
    return np.clip(img, 0, 255).astype(np.uint8)


@pytest.mark.parametrize("hw,w,ch", [(128, 128, 3), (128, 128, 1), (64, 64, 3), (64, 128, 3), (32, 32, 3), (16, 32, 3),
                                     (16, 16, 3), (16, 16, 1)])
def test_crops_at_sizes_in_use_are_unchanged(hw, w, ch):
    """make_crops_u8 draws the same bytes as before at every size the suite used before odd sizes"""
    assert np.array_equal(O.make_crops_u8(9, 3, hw=hw, ch=ch, w=w), _old_crops_u8(9, 3, hw, ch, w))


@pytest.mark.parametrize("hw,w", [(100, 100), (127, 127), (127, 128), (80, 80), (112, 112), (96, 96), (25, 25)])
def test_crops_at_any_size(hw, w):
    """at a size its cell count does not divide, each cell is ceil(size / cells) pixels and the last one is cut short: the coarse
    pattern is constant over each cell up to the +-40 noise"""
    x = O.make_crops_u8(9, 2, hw=hw, w=w)
    assert x.shape == (2, hw, w, 3) and x.dtype == np.uint8
    cells, cells_w = max(hw // 16, 1), max(w // 16, 1)
    ph, pw = -(-hw // cells), -(-w // cells_w)
    coarse = np.random.RandomState(9).randint(0, 256, size=(2, cells, cells_w, 3))
    want = np.repeat(np.repeat(coarse, ph, axis=1), pw, axis=2)[:, :hw, :w]
    d = x.astype(int) - want
    assert np.all((d >= -40) & (d <= 40) | (x == 0) | (x == 255))


# TF SAME padding of a k = 5, stride-2 conv, derived by hand from out = ceil(in / 2), total = max((out - 1) * 2 + 5 - in, 0),
# before = total // 2, after = total - before
SAME_K5_S2 = {128: (1, 2), 127: (2, 2), 112: (1, 2), 100: (1, 2), 25: (2, 2), 14: (1, 2), 13: (2, 2), 7: (2, 2)}


@pytest.mark.parametrize("size", list(SAME_K5_S2))
def test_same_padding_known_answers(size):
    """_same_pads, conv2d_same and conv2d_same_loops against the literal table.  The input's pixels are 1 + their flat index and
    output channel 5 dy + dx of the kernel is the one-hot tap (dy, dx), so each output is one known input pixel or 0; the height
    takes the row's size and the width another row's, so that a swapped pad_t / pad_l shows."""
    sizes = list(SAME_K5_S2)
    ih, iw = size, sizes[(sizes.index(size) + 1) % len(sizes)]
    (pt, pb), (pl, pr) = SAME_K5_S2[ih], SAME_K5_S2[iw]
    assert O._same_pads(ih, 5, 2) == (pt, pb) and O._same_pads(iw, 5, 2) == (pl, pr)
    oh, ow = (ih + pt + pb - 5) // 2 + 1, (iw + pl + pr - 5) // 2 + 1
    assert (oh, ow) == (-(-ih // 2), -(-iw // 2))
    x = (1.0 + np.arange(ih * iw, dtype=np.float64)).reshape(1, ih, iw, 1)
    k = np.zeros((5, 5, 1, 25))
    for t in range(25):
        k[t // 5, t % 5, 0, t] = 1.0
    want = np.zeros((1, oh, ow, 25))
    for t in range(25):
        dy, dx = divmod(t, 5)
        for r in range(oh):
            iy = 2 * r + dy - pt
            for c in range(ow):
                ix = 2 * c + dx - pl
                if 0 <= iy < ih and 0 <= ix < iw:
                    want[0, r, c, t] = x[0, iy, ix, 0]
    # the bottom / right pad is what the last output row / column reads past the image
    assert np.all(want[0, -1, :, 5 * (5 - pb):] == 0) and np.any(want[0, -1, :, :5 * (5 - pb)] != 0)
    assert np.all(want[0, :, -1, [5 * dy + dx for dy in range(5) for dx in range(5 - pr, 5)]] == 0)
    got = O.conv2d_same(torch.from_numpy(x), torch.from_numpy(k), torch.zeros(25, dtype=torch.float64), 2, None).numpy()
    assert np.array_equal(got, want), size
    assert np.array_equal(O.conv2d_same_loops(x, k, np.zeros(25), 2), want), size


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
    # odd sizes: TF's symmetric (2, 2) padding of odd inputs, and (1, 2) / (2, 2) on the two axes of one conv
    "13x16": (13, 16, 3, (4, 8), (2, 2), 5),
    "15x15": (15, 15, 3, (4, 8, 8), (2, 2, 2), 5),
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
