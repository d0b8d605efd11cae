"""The cfg geometries beyond the template that tests/test_gpu_l_geometry.py runs and tests/test_geometry_cpu.py checks on the host:
one row per geometry, where each module lands with the automatic precision, the oracle's parameters for the row, and builders of
the Python modules (which create no device handle until one is asked for)."""
import numpy as np

from oracle import aae_oracle as O
from oracle import mask_oracle as MO

FP32, SPLIT, FP16 = 0, 1, 2
MAXB, RAGGED = 40, 13
T = dict(h=128, w=128, c=3, nf=(128, 256, 512, 512), strides=(2, 2, 2, 2), k=5, latent=128, mask=False)

# id: cfg change from the template
ROWS = {
    "latent64": dict(latent=64),
    "latent32": dict(latent=32),
    "latent96": dict(latent=96),
    "latent256": dict(latent=256),
    "narrow": dict(nf=(128, 128, 256, 256)),
    "cout64": dict(nf=(128, 64, 128, 256)),
    "two_layer": dict(nf=(128, 256), strides=(2, 2)),
    "conv1_64": dict(nf=(64, 128, 256, 256)),
    "five_layer": dict(nf=(128, 256, 512, 512, 512), strides=(2,) * 5),
    "px64": dict(h=64, w=64),
    "gray": dict(c=1),
    "gray_mask": dict(c=1, mask=True),
    "wide_last": dict(nf=(128, 256, 512, 480)),
    "rect": dict(h=64),
    "refused_stride": dict(strides=(2, 2, 1, 2)),
    "refused_k3": dict(k=3),
    # crop sizes that are not powers of two: odd maps, TF's symmetric (2, 2) SAME padding of odd inputs, images that straddle
    # 128-row tiles
    "px112": dict(h=112, w=112),                          # maps 56/28/14/7
    "px80": dict(h=80, w=80),                             # 40/20/10/5
    "px96": dict(h=96, w=96),                             # 48/24/12/6
    "px127": dict(h=127, w=127),                          # 64/32/16/8, conv1 padded (2, 2)
    "h127": dict(h=127),                                  # 127 x 128: conv1 padded (2, 2) in height, (1, 2) in width
    "px100": dict(h=100, w=100),                          # 50/25/13/7, pads (1, 2), (1, 2), (2, 2), (2, 2)
}

# Where each module settles with the automatic precision: (encoder, codebook match, decoder, encoder and decoder once the
# training step exists, explicit TC_FP16 encoder accepted).  None: no decoder or trainer exists for the geometry on any precision.
LANDING = {
    "latent64": (SPLIT, FP32, SPLIT, SPLIT, True),
    "latent32": (SPLIT, FP32, FP32, FP32, True),          # decoder: latent % 64; mixed handles -> the trainer demotes both
    "latent96": (SPLIT, FP32, FP32, FP32, True),
    "latent256": (SPLIT, FP32, SPLIT, SPLIT, True),
    "narrow": (SPLIT, SPLIT, SPLIT, SPLIT, True),
    "cout64": (SPLIT, SPLIT, SPLIT, FP32, True),          # conv3's Cin 64: the split trainer's units need Cin % 128
    "two_layer": (SPLIT, SPLIT, SPLIT, SPLIT, True),
    "conv1_64": (SPLIT, SPLIT, SPLIT, FP32, False),       # fp32 conv1: the split trainer refuses it
    "five_layer": (SPLIT, SPLIT, SPLIT, FP32, True),      # 4 x 4 decoder layers: the split trainer refuses them
    "px64": (SPLIT, SPLIT, SPLIT, FP32, False),
    "gray": (SPLIT, SPLIT, SPLIT, FP32, False),
    "gray_mask": (SPLIT, SPLIT, SPLIT, FP32, False),
    "wide_last": (SPLIT, SPLIT, FP32, FP32, True),        # decoder: Cin 480 % 64
    "rect": (SPLIT, SPLIT, None, None, True),             # the decoder takes square crops only
    "refused_stride": (FP32, FP32, None, None, False),    # the decoder takes stride-2 stages only
    "refused_k3": (FP32, FP32, FP32, FP32, False),
    "px112": (FP32, FP32, FP32, FP32, False),             # the tensor cores take power-of-two maps only
    "px80": (FP32, FP32, FP32, FP32, False),
    "px96": (FP32, FP32, FP32, FP32, False),
    "px127": (SPLIT, SPLIT, None, None, False),           # fp32 conv1; the decoder's x2 stages cannot build 127 from 8
    "h127": (SPLIT, SPLIT, None, None, False),            # fp32 conv1 (odd height); the decoder takes square crops only
    "px100": (FP32, FP32, None, None, False),             # 100 is not a multiple of 2^4
}

# rows whose training check also runs at this batch: the fp32 trainer orders a stride-2 dgrad parity-major only when
# (B * PH * PW / 4) % 128 == 0, which at B = 32 holds for 56 x 56, 28 x 28, 40 x 40, 20 x 20 and every px96 map but not for
# 14 x 14 or 10 x 10, so one step takes both orderings
PARITY_BATCH = 32
PARITY_ROWS = ("px112", "px80", "px96")


def row(rid, **change):
    r = dict(T)
    r.update(ROWS[rid])
    r.update(change)
    r["id"] = rid
    r["L"] = len(r["nf"])
    return r


def tc_conv1(r):
    return r["w"] == 128 and r["h"] % 2 == 0 and r["c"] == 3 and r["nf"][0] == 128 and r["k"] == 5 and r["strides"][0] == 2


def params(r, bias_scale=0.05):
    """(encoder params, decoder params without the head, mask head (kernel, bias) or None)"""
    ep = O.make_encoder_params(42, num_filters=r["nf"], ksize=r["k"], latent=r["latent"], in_ch=r["c"], in_hw=r["h"],
                               strides=r["strides"], bias_scale=bias_scale, in_w=r["w"])
    dp = O.make_decoder_params(43, num_filters=r["nf"], ksize=r["k"], latent=r["latent"], out_ch=r["c"], out_hw=r["h"],
                               strides=r["strides"], bias_scale=bias_scale, n_encoder_convs=r["L"])
    head = MO.make_mask_head(44, r["nf"][0], r["k"], bias_scale) if r["mask"] else None
    return ep, dp, head


def output_conv(r):
    """name of the decoder's output conv in the oracle's decoder params (the graph without the mask head)"""
    return "conv2d_%d" % (2 * r["L"] - 1)


def dec_weights(r, dp, head):
    """the decoder's variables under its own names: with the head, the output conv moves up one number (conv2d_7 -> conv2d_8 for
    four encoder convs) and the head takes its place"""
    if head is None:
        return dp
    k = 2 * r["L"] - 1
    w = {n: v for n, v in dp.items() if not n.startswith("conv2d_%d/" % k)}
    w["conv2d_%d/kernel" % (k + 1)], w["conv2d_%d/bias" % (k + 1)] = dp["conv2d_%d/kernel" % k], dp["conv2d_%d/bias" % k]
    w["conv2d_%d/kernel" % k], w["conv2d_%d/bias" % k] = head
    return w


def encoder(r, precision=None, is_training=False):
    from augmentedautoencoder_b200.ae.encoder import Encoder
    from augmentedautoencoder_b200.ae.session import placeholder
    x = placeholder(np.float32, [None, r["h"], r["w"], r["c"]])
    return Encoder(x, r["latent"], list(r["nf"]), r["k"], list(r["strides"]), False, is_training=is_training, precision=precision,
                   max_batch=MAXB)


def decoder(r, enc, precision=None, bootstrap=4):
    from augmentedautoencoder_b200.ae.decoder import Decoder
    from augmentedautoencoder_b200.ae.session import placeholder
    y = placeholder(np.float32, [None, r["h"], r["w"], r["c"]])
    return Decoder(y, enc.z, list(reversed(r["nf"])), r["k"], list(reversed(r["strides"])), "L2", bootstrap, r["mask"], False,
                   is_training=True, max_batch=MAXB, n_encoder_convs=r["L"], precision=precision)
