"""Halo edges of the tensor-core conv GEMMs, whose taps of one column offset share one A box of BH + 2 rows (row oh0 - 1 and
row oh0 + BH come from TMA's zero fill at the image border).  Crops that are zero except for their first or last two rows or
columns, with zero biases, put all of the signal next to a border: a wrong row offset into the box, a box at the wrong column
or a missing zero fill moves or adds signal where the float64 oracle has none.  Same bounds as test_gpu_b_tc.
(A training step on such crops is ill-conditioned -- the uniform interiors make ReLU decisions flip together -- so the
dgrad GEMMs' halo boxes are checked by the gradient tests of test_gpu_b_tc and test_gpu_e_fp16_train.)"""
import numpy as np
import pytest
import torch

from oracle import aae_oracle as O
from tests.test_gpu_a_parity import _enc, sess  # noqa: F401

pytestmark = pytest.mark.gpu


def _edge_crops(seed):
    """Four uint8 crops: signal in the first two rows, the last two rows, the first two columns, the last two columns."""
    rng = np.random.RandomState(seed)
    x = np.zeros((4, 128, 128, 3), np.uint8)
    x[0, :2] = rng.randint(1, 256, (2, 128, 3))
    x[1, -2:] = rng.randint(1, 256, (2, 128, 3))
    x[2, :, :2] = rng.randint(1, 256, (128, 2, 3))
    x[3, :, -2:] = rng.randint(1, 256, (128, 2, 3))
    return x


@pytest.mark.parametrize("batch", [256, 37, 1])
def test_tc_encoder_layers_at_the_image_border(sess, batch):
    """256: full tiles; 37: a padded two-image tile in conv4; 1: the small-batch split-K forward."""
    p = O.make_encoder_params(42)
    enc = _enc(1, 256, p)
    pattern = _edge_crops(5)
    crops = pattern[np.arange(batch) % 4]
    z = sess.run(enc.z, {enc.x: crops})
    outs64 = O.encoder_layers(O.preprocess(pattern), p, dtype=torch.float64)
    errs = []
    for layer in range(4):
        a = enc.activation_device(layer, sess.device).cpu().numpy()
        ref = outs64[layer].numpy()[np.arange(batch) % 4]
        assert a.shape == ref.shape
        errs.append(np.max(np.abs(a - ref)) / max(1.0, np.abs(ref).max()))
    z64 = outs64[5].numpy()[np.arange(batch) % 4]
    errs.append(np.max(np.abs(z - z64)) / np.abs(z64).max())
    print("edge crops, batch %d: relative errors per layer + latent:" % batch, ["%.2e" % e for e in errs])
    # the latents of these nearly empty crops are small, so their bound is the ragged-batch test's 2e-5 of max |z|
    assert all(e < 1e-5 for e in errs[:4]) and errs[4] < 2e-5, errs


def test_tc_decoder_forward_at_a_ragged_batch(sess):
    """Decoder sub-pixel GEMMs (3 x 3 taps grouped by column offset) at 37 latents against the float64 oracle."""
    from augmentedautoencoder_b200.ae.decoder import Decoder
    from augmentedautoencoder_b200.ae.session import placeholder
    dp = O.make_decoder_params(43, bias_scale=0.05)
    z = (np.random.RandomState(37).standard_normal((37, 128)) * 2.0).astype(np.float32)
    dec = Decoder(placeholder(np.float32, [None, 128, 128, 3]), placeholder(np.float32, [None, 128]), list(reversed(O.NUM_FILTER)), 5,
                  list(reversed(O.STRIDES)), "L2", 4, False, False, max_batch=64, precision=1)
    dec.load_weights(dp)
    out = dec.decode_device(torch.from_numpy(z).cuda()).cpu().numpy()
    tp = {k: torch.from_numpy(v).double() for k, v in dp.items()}
    with torch.no_grad():
        ref = O.decoder_layers(torch.from_numpy(z).double(), tp)[-1].numpy()
    err = np.max(np.abs(out - ref))
    print("decoder forward at 37 latents: max abs error vs float64 %.2e" % err)
    assert err < 5e-6

