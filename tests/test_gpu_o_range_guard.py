"""GPU tests of the tensor-core range guard at its limits (include/aae_b200.h: aae_encoder_range_status; DESIGN.md section 3,
"Range guard").  Activations are stored as fp16 16 x and weights as fp16 256 x; the guard fires where that product is no longer
below 65520, the smallest magnitude that rounds to fp16 infinity.  So an activation of 4094.5 (x 16 = 65512) must be computed
like the float64 oracle computes it, with status 0, and one of 4095.5 (x 16 = 65528) must be reported, naming exactly the layer
that wrote it.  Both are exact in fp32, and the models below produce them exactly on every precision (fp16-exact operands,
products and sums).

Encoder cases: a "delta chain".  Conv1's channel 0 fires on a single white 5 x 5 patch in one image of a dark batch; every later
layer's channel 0 reads the previous channel 0 through one tap and nothing else, and the layer after the chosen one does not
read channel 0 at all, so one pixel of one image reaches the chosen magnitude in the chosen layer and everything else stays in
range.  (A value past the limit is stored as fp16 infinity; a later layer that read it with a nonzero weight would write
infinity too and be reported as well.  With zero weights the product is NaN, which the ReLU drops, so the report names the
overflowing layer alone.)  The patch sits in the first image near the top-left corner or in the last image near the bottom-right one (the
partial last M tile where M is not a multiple of 128).  Batch 3 runs every GEMM layer through the split-K finish kernel, batch 40
the layers with more than 66 tiles through the persistent epilogue (every GEMM layer of the template)."""
import ctypes as C
import gc

import numpy as np
import pytest
import torch

from oracle import aae_oracle as O
from tests.geometry_table import FP16, FP32, SPLIT, T, dec_weights, encoder, params, row, tc_conv1
from tests.test_gpu_a_parity import sess  # noqa: F401
from tests.test_gpu_d_fp16 import PROD, STORE, SUB_ACT, SUB_W

pytestmark = pytest.mark.gpu

OK_V, BAD_V = 4094.5, 4095.5
W_OK, W_BAD = 255.93359375, 255.9375               # x 256: 65519 (accepted), 65520 (refused)
C1_OK, C1_BAD = 254.9375, 254.9453125              # x 256 x 256/255 (the uint8 operand): 65519.0 and 65521.0
W1 = 15.9375                                       # conv1's channel-0 taps: x 256 and x 256 x 256/255 are both exact in fp16
ENC_ROWS = ("template", "five_layer", "conv1_64", "gray")
BATCHES = (3, 40)
ERR_BAD = -3
_peak = [0]


def _row(rid):
    return dict(T, id="template", L=len(T["nf"])) if rid == "template" else row(rid)


def _note_peak():
    torch.cuda.synchronize()
    _peak[0] = max(_peak[0], torch.cuda.max_memory_allocated())


def _lib():
    from augmentedautoencoder_b200 import _lib
    return _lib


def _last_error():
    return _lib().lib().aae_last_error_string().decode()


def _layers_named(msg, kind):
    """the layer list after '<kind> ... layer(s)' in a range-guard message, as a tuple of ints"""
    import re
    m = re.search(kind + r"[^;]*?layer\(s\)((?: \d+)+)", msg)
    return tuple(int(t) for t in m.group(1).split()) if m else ()


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


# ------------------------------------------------------------------------------------------------ the delta chain
def _sizes(r):
    """[(in_h, in_w, pad_t, pad_l, stride)] of every encoder conv (the oracle's TF-SAME padding)"""
    out, h, w = [], r["h"], r["w"]
    for s in r["strides"]:
        out.append((h, w, O._same_pads(h, r["k"], s)[0], O._same_pads(w, r["k"], s)[0], s))
        h, w = -(-h // s), -(-w // s)
    return out


def _chain(r, layer, value, last):
    """(weights, crops u8 [40, ...], image index, [(row, col) of the chain pixel per layer]): channel 0 of layer `layer` is `value`
    at one pixel of one image, every other value of the model is in range."""
    ep, _, _ = params(r)
    ep = {k: v.copy() for k, v in ep.items()}
    sz = _sizes(r)
    h0, w0, pt0, pl0, s0 = sz[0]
    o0 = ((h0 + s0 - 1) // s0 - 2, (w0 + s0 - 1) // s0 - 2) if last else (1, 1)
    rng = np.random.RandomState(5 + layer)
    x = rng.randint(0, 33, size=(max(BATCHES), r["h"], r["w"], r["c"])).astype(np.uint8)   # dark: no 5 x 5 window reaches conv1's threshold
    b = max(BATCHES) - 1 if last else 0
    i0, j0 = o0[0] * s0 - pt0, o0[1] * s0 - pl0
    x[b, i0:i0 + 5, j0:j0 + 5, :] = 255
    k1 = ep["conv2d/kernel"]
    k1[..., 0] = W1
    ep["conv2d/bias"][0] = (value if layer == 0 else 64.0) - W1 * k1[..., 0].size
    pos = [o0]
    for k in range(1, r["L"]):
        name = "conv2d_%d" % k
        kern, bias = ep[name + "/kernel"], ep[name + "/bias"]
        kern[:, :, 0, :] = 0.0
        ih, iw = pos[-1]
        h, w, pt, pl, s = sz[k]
        o = (min((ih + pt) // s, -(-h // s) - 1), min((iw + pl) // s, -(-w // s) - 1))
        pos.append(o)
        if k <= layer:
            kern[..., 0] = 0.0
            kern[ih + pt - o[0] * s, iw + pl - o[1] * s, 0, 0] = 1.0 if k < layer else 64.0
            bias[0] = 0.0 if k < layer else value - 4096.0
    oh, ow = sz[-1][0] // sz[-1][4], sz[-1][1] // sz[-1][4]
    dk = ep["dense/kernel"].reshape(oh, ow, r["nf"][-1], -1)
    dk[:, :, 0, :] = 0.0
    return ep, x, b, pos


def _g(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to("cuda", torch.float64)


def _oracle(r, x, ep):
    """float64 encoder on the GPU: ([conv activations], z) as cuda float64 tensors"""
    acts = []
    with torch.no_grad():
        h = _g(O.preprocess(x))
        for i, s in enumerate(r["strides"]):
            name = "conv2d" if i == 0 else "conv2d_%d" % i
            h = O.conv2d_same(h, _g(ep[name + "/kernel"]), _g(ep[name + "/bias"]), s, "relu")
            acts.append(h)
        z = h.reshape(h.shape[0], -1) @ _g(ep["dense/kernel"]) + _g(ep["dense/bias"])
    return acts, z


def _fp16_bound(a_in, w, b, s, y16):
    """worst |y16 - y64| / bound of one conv layer of the fp16 path (tests/test_gpu_d_fp16._conv_bound_check on the GPU)"""
    with torch.no_grad():
        a64, w64, b64 = a_in, _g(w), _g(b)
        y64 = O.conv2d_same(a64, w64, b64, s, "relu")
        S = O.conv2d_same(a64.abs(), w64.abs(), torch.zeros_like(b64), s, None)
        K = w.shape[0] * w.shape[1] * w.shape[2]
        eps_sub = SUB_ACT * w64.abs().reshape(K, -1).sum(0) + SUB_W * K * a64.abs().max() + SUB_ACT
        bound = PROD * S + STORE * y64.abs() + eps_sub
        return float(((y16 - y64).abs() / bound).max())


def _splitk_everywhere(r, B):
    """the encoder's split-K rule (tc_encoder_forward): tiles * 2 <= 132 for every GEMM conv after conv1"""
    sz = _sizes(r)
    tiles = []
    for k in range(1, r["L"]):
        h, w, _, _, s = sz[k]
        tiles.append(-(-B * (h // s) * (w // s) // 128) * -(-r["nf"][k] // 128))
    return [t * 2 <= 132 for t in tiles]


# ------------------------------------------------------------------------------------------------ encoder activations
CASES = [(rid, l) for rid in ENC_ROWS for l in range(_row(rid)["L"])]


@pytest.mark.parametrize("rid,layer", CASES, ids=["%s-conv%d" % c for c in CASES])
def test_encoder_activation_at_the_limit(sess, rid, layer):
    """One pixel at 4094.5 in layer `layer`: status OK, the layer's activation and z equal the float64 oracle (split: the fp32-grade
    bar of tests/test_gpu_l_geometry; fp16: the section-3 rounding bound).  At 4095.5: the C ABI and Session.run name exactly that
    layer, and the report clears the word."""
    lib = _lib().lib()
    AaeError = _lib().AaeError
    r = _row(rid)
    assert _splitk_everywhere(r, 3) == [True] * (r["L"] - 1)
    print("%s: GEMM convs on the split-K finish kernel at batch 40: %s" % (rid, _splitk_everywhere(r, 40)))
    precs = (SPLIT, FP16) if tc_conv1(r) else (SPLIT,)
    worst = {}
    for prec in precs:
        enc = encoder(r, precision=prec)
        for last in (False, True):
            for value in (OK_V, BAD_V):
                ep, x, b, pos = _chain(r, layer, value, last)
                enc.load_weights(ep)
                h = enc.handle(sess.device)
                for B in BATCHES:
                    xb = x[:B] if not last else x[max(BATCHES) - B:]
                    ref = None
                    if value == OK_V:
                        acts64, z64 = _oracle(r, xb, ep)
                        a = acts64[layer]
                        ib = B - 1 if last else 0
                        assert float(a[ib, pos[layer][0], pos[layer][1], 0]) == value, "the chain misses its pixel"
                        a[ib, pos[layer][0], pos[layer][1], 0] = 0.0
                        assert float(a.max()) < 4000.0
                        a[ib, pos[layer][0], pos[layer][1], 0] = value
                        ref = (acts64, z64)
                    for feed in ("uint8", "float"):
                        xd = torch.from_numpy(xb if feed == "uint8" else O.preprocess(xb)).cuda()
                        z = enc.encode_device(xd)
                        _note_peak()
                        st = lib.aae_encoder_range_status(h, _stream())
                        tag = "%s prec %d conv%d %s B=%d %s feed" % (rid, prec, layer + 1, "last image" if last else "first image", B, feed)
                        if value == BAD_V:
                            msg = _last_error()
                            assert st == ERR_BAD, tag
                            assert _layers_named(msg, "activation") == (layer,) and "weight" not in msg and "latent" not in msg, (tag, msg)
                            assert lib.aae_encoder_range_status(h, _stream()) == 0, tag           # the report cleared the word
                            continue
                        assert st == 0, (tag, _last_error())
                        acts64, z64 = ref
                        y = enc.activation_device(layer, sess.device).double()
                        if prec == SPLIT:
                            e = float((y - acts64[layer]).abs().max()) / max(1.0, float(acts64[layer].abs().max()))
                            ez = float((z.double() - z64).abs().max() / z64.abs().max())
                            assert e < 1e-5 and ez < 2e-5, (tag, e, ez)
                        else:
                            a_in = _g(O.preprocess(xb)) if layer == 0 else enc.activation_device(layer - 1, sess.device).double()
                            name = "conv2d" if layer == 0 else "conv2d_%d" % layer
                            e = _fp16_bound(a_in, ep[name + "/kernel"], ep[name + "/bias"], r["strides"][layer], y)
                            assert e <= 1.0, (tag, e)
                            ez = float((z.double() - z64).abs().max() / z64.abs().max())
                            assert ez < 2e-2, (tag, ez)
                        worst[prec] = max(worst.get(prec, 0.0), e)
                # Session.run reports the same, and names the same layer
                xs = x[:3] if not last else x[max(BATCHES) - 3:]
                if value == BAD_V:
                    with pytest.raises(AaeError) as ei:
                        sess.run(enc.z, {enc.x: xs})
                    assert _layers_named(str(ei.value), "activation") == (layer,), str(ei.value)
                else:
                    assert np.all(np.isfinite(sess.run(enc.z, {enc.x: xs})))
        enc.close()
    print("%s conv%d at %.1f: worst error %s (split: relative to max(1, max|a|); fp16: error / bound)"
          % (rid, layer + 1, OK_V, {p: "%.2e" % e for p, e in worst.items()}))


def test_fp32_handles_take_the_same_models(sess):
    """The fp32 path has no such limit: the 4095.5 models of every row run with status OK and equal the float64 oracle."""
    worst = 0.0
    for rid in ENC_ROWS:
        r = _row(rid)
        enc = encoder(r, precision=FP32)
        for layer in range(r["L"]):
            ep, x, _, _ = _chain(r, layer, BAD_V, True)
            enc.load_weights(ep)
            z = enc.encode_device(torch.from_numpy(x[-3:]).cuda())
            assert _lib().lib().aae_encoder_range_status(enc.handle(sess.device), _stream()) == 0
            acts64, z64 = _oracle(r, x[-3:], ep)
            y = enc.activation_device(layer, sess.device).double()
            e = float((y - acts64[layer]).abs().max()) / float(acts64[layer].abs().max())
            ez = float((z.double() - z64).abs().max() / z64.abs().max())
            assert e < 1e-5 and ez < 2e-5, (rid, layer, e, ez)
            worst = max(worst, e)
        enc.close()
    print("fp32 handles at %.1f: worst relative error %.2e" % (BAD_V, worst))


# ------------------------------------------------------------------------------------------------ weights
def _expect_refused(enc_or_dec, h, layer, fwd):
    """every forward of a handle with refused weights fails, naming the layer, until the layer is set again"""
    st = fwd()
    assert st == ERR_BAD, st
    msg = _last_error()
    assert "refused" in msg and _layers_named(msg, "refused the weights") == (layer,), msg


def _enc_weight_cases(r):
    """(layer, variable, index, accepted value, refused value) for every packed encoder layer"""
    out = [(0, "conv2d/kernel", (2, 3, 1, 5), C1_OK, C1_BAD)] if tc_conv1(r) else []
    for k in range(1, r["L"]):
        out.append((k, "conv2d_%d/kernel" % k, (1, 2, 3, 4), W_OK, W_BAD))
    out.append((r["L"], "dense/kernel", (7, 3), W_OK, W_BAD))
    return out


@pytest.mark.parametrize("rid", ["template", "conv1_64"])
def test_encoder_weights_at_the_limit(sess, rid):
    """Largest accepted and smallest refused weight of every packed layer (tensor-core conv1: 254.94, its uint8 operand is
    packed at 256 x 256/255; the fp32 conv1 has no limit).  The accepted one gives oracle-grade z; after a refusal every forward
    fails through the C ABI and Session.run until a clean set_weights of that layer, and set_weights leaves a pending activation
    overflow to aae_encoder_range_status."""
    lib = _lib().lib()
    AaeError = _lib().AaeError
    r = _row(rid)
    ep0, _, _ = params(r)
    x = O.make_crops_u8(9, 3, hw=r["h"], ch=r["c"], w=r["w"]) // 8                   # dark crops: the big weights stay in range
    xd = torch.from_numpy(x).cuda()
    z_out = torch.empty((3, r["latent"]), device="cuda")
    enc = encoder(r, precision=SPLIT)
    enc.load_weights(ep0)
    h = enc.handle(sess.device)
    for layer, name, idx, ok, bad in _enc_weight_cases(r) + ([] if tc_conv1(r) else [(0, "conv2d/kernel", (2, 2, 0, 3), 1000.0, None)]):
        kern = ep0[name].copy()
        kern[idx] = ok
        assert lib.aae_encoder_set_weights(h, layer, _lib().ptr(kern), None, _stream()) == 0, (name, _last_error())
        z = enc.encode_device(xd)
        assert lib.aae_encoder_range_status(h, _stream()) == 0, (name, _last_error())
        ep = dict(ep0)
        ep[name] = kern
        _, z64 = _oracle(r, x, ep)
        ez = float((z.double() - z64).abs().max() / z64.abs().max())
        assert ez < 2e-5, (name, ok, ez)
        if bad is None:
            continue
        kern[idx] = bad
        assert lib.aae_encoder_set_weights(h, layer, _lib().ptr(kern), None, _stream()) == ERR_BAD, name
        msg = _last_error()
        assert _layers_named(msg, "weight") == (layer,) and "activation" not in msg, msg
        for fwd in (lib.aae_encoder_forward_u8, lib.aae_encoder_forward_f32):
            _expect_refused(enc, h, layer, lambda: fwd(h, _lib().ptr(xd), 3, _lib().ptr(z_out), _stream()))
        with pytest.raises(AaeError, match="refused"):
            sess.run(enc.z, {enc.x: x})
        assert lib.aae_encoder_set_weights(h, layer, _lib().ptr(ep0[name]), None, _stream()) == 0   # clean: the handle runs again
        enc.encode_device(xd)
        assert lib.aae_encoder_range_status(h, _stream()) == 0
    # set_weights reports weights only: an activation overflow of an earlier forward stays for the range check
    ep, xc, _, _ = _chain(r, 1, BAD_V, False)
    enc.load_weights(ep)
    enc.encode_device(torch.from_numpy(xc[:3]).cuda())
    assert lib.aae_encoder_set_weights(h, 1, _lib().ptr(ep["conv2d_1/kernel"]), None, _stream()) == 0, _last_error()
    assert lib.aae_encoder_range_status(h, _stream()) == ERR_BAD and _layers_named(_last_error(), "activation") == (1,)
    _note_peak()
    enc.close()


# ------------------------------------------------------------------------------------------------ decoder
def _decoder(r, mask, precision=SPLIT):
    from augmentedautoencoder_b200.ae.decoder import Decoder
    from augmentedautoencoder_b200.ae.session import placeholder
    zin = placeholder(np.float32, [None, r["latent"]])
    dec = Decoder(placeholder(np.float32, [None, r["h"], r["w"], r["c"]]), zin, list(reversed(r["nf"])), r["k"],
                  list(reversed(r["strides"])), "L2", 4, mask, False, max_batch=40, n_encoder_convs=r["L"], precision=precision)
    return dec, zin


def _dec64(r, z, dp):
    P = {k: _g(v) for k, v in dp.items()}
    with torch.no_grad():
        return O.decoder_layers(_g(z), P, out_hw=r["h"], strides=r["strides"], n_encoder_convs=r["L"])


def _dec_model(r, layer, value):
    """decoder params and z with unit 0 of layer `layer` (0 = dense_1, 1.. = hidden convs, channel 0 everywhere) at `value`
    exactly; nothing reads it (see the module docstring)"""
    _, dp, _ = params(r)
    dp = {k: v.copy() for k, v in dp.items()}
    z = (np.random.RandomState(3).standard_normal((40, r["latent"])) * 0.1).astype(np.float32)
    names = ["dense_1"] + ["conv2d_%d" % (r["L"] + j) for j in range(r["L"])]
    if layer == 0:
        dp["dense_1/kernel"][:, 0] = 0.0
        dp["dense_1/bias"][0] = value
    else:
        dp[names[layer] + "/kernel"][..., 0] = 0.0
        dp[names[layer] + "/bias"][0] = value
    nxt = dp[names[layer + 1] + "/kernel"]
    if layer == 0:
        d0 = r["h"] // int(np.prod(r["strides"]))
        nxt[:, :, 0, :] = 0.0                                       # dense_1 unit 0 is channel 0 of pixel (0, 0) of the first map
        assert d0 >= 1
    else:
        nxt[:, :, 0, :] = 0.0
    return dp, z


@pytest.mark.parametrize("rid,mask", [("template", False), ("template", True), ("narrow", False)])
def test_decoder_at_the_limit(sess, rid, mask):
    """The latent (bit 15), dense_1 (layer 0) and every hidden conv at 4094.5 (status OK, x equals the float64 oracle) and at
    4095.5 (exactly that layer named); then the largest accepted and smallest refused merged weight of the convs: four taps of
    63.984375 (each below 64) sum to 255.9375 in one sub-pixel weight and are refused, naming the layer; the mask head is
    packed with the output conv and its refusal names the output conv's layer, num_layers.  After a refusal every forward fails
    until a clean set_weights."""
    lib = _lib().lib()
    AaeError = _lib().AaeError
    r = _row(rid)
    if mask:
        r = dict(r, mask=True)
    dec, zin = _decoder(r, mask)
    _, dp0, head = params(r)
    h = None
    worst = 0.0
    L = r["L"]
    for layer in range(L):
        for value in (OK_V, BAD_V):
            dp, z = _dec_model(r, layer, value)
            dec.load_weights(dec_weights(r, dp, head))
            h = dec.handle(sess.device)
            for B in (3, 40):
                zd = torch.from_numpy(z[:B]).cuda()
                x = dec.decode_device(zd)
                st = lib.aae_decoder_range_status(h, _stream())
                if value == BAD_V:
                    assert st == ERR_BAD and _layers_named(_last_error(), "activation") == (layer,), _last_error()
                    continue
                assert st == 0, _last_error()
                if mask:
                    continue                                          # x is the same with and without the head: checked below
                x64 = _dec64(r, z[:B], dp)[-1]
                e = float((x.double() - x64).abs().max())
                assert e < 5e-6, (rid, layer, B, e)
                worst = max(worst, e)
            with pytest.raises(AaeError) if value == BAD_V else _nothing():
                sess.run(dec.x, {zin: z[:3]})
    # the latent
    dec.load_weights(dec_weights(r, dp0, head))
    for value in (OK_V, BAD_V):
        z = (np.random.RandomState(4).standard_normal((3, r["latent"])) * 0.1).astype(np.float32)
        z[2, 5] = value
        dec.decode_device(torch.from_numpy(z).cuda())
        st = lib.aae_decoder_range_status(h, _stream())
        if value == OK_V:
            assert st == 0, _last_error()
        else:
            assert st == ERR_BAD and "latent" in _last_error() and "activation" not in _last_error(), _last_error()
    # weights: dense_1 single value; convs: four taps that merge into one sub-pixel weight
    zd = torch.from_numpy((np.random.RandomState(6).standard_normal((3, r["latent"])) * 0.01).astype(np.float32)).cuda()
    names = ["dense_1"] + ["conv2d_%d" % (L + j) for j in range(L)]
    layers = list(range(L + 1)) + ([L + 1] if mask else [])
    for layer in layers:
        wname = (names[layer] if layer <= L else None)
        if layer == L + 1:
            kern0 = head[0]
        else:
            key = wname + "/kernel" if not (mask and layer == L) else "conv2d_%d/kernel" % (2 * L)
            kern0 = dec_weights(r, dp0, head)[key]
        packed = min(layer, L)
        for per_tap, refused in ((W_OK / 4, False), (W_BAD / 4, True)):
            kern = kern0.copy()
            if layer == 0:
                kern[5, 9] = per_tap * 4
            else:
                kern[0:2, 0:2, 1, 0] = per_tap
            st = lib.aae_decoder_set_weights(h, layer, _lib().ptr(kern), None, _stream())
            if not refused:
                assert st == 0, (layer, _last_error())
                x = dec.decode_device(zd)
                assert lib.aae_decoder_range_status(h, _stream()) == 0, _last_error()
                w = dec_weights(r, dp0, head).copy()
                if layer == L + 1:
                    pass
                else:
                    w[key if layer else "dense_1/kernel"] = kern
                    if not mask:
                        outs = _dec64(r, zd.cpu().numpy(), w)
                        # fp32-grade relative to the size of the four big products: sum |a w| <= 4 * 64 * max |input|
                        a_in = zd.double().abs().max() if layer == 0 else outs[layer - 1].abs().max()
                        tol = 5e-6 * max(1.0, 4 * per_tap * float(a_in))
                        assert float((x.double() - outs[-1]).abs().max()) < tol, (layer, tol)
                continue
            assert st == ERR_BAD, layer
            msg = _last_error()
            assert _layers_named(msg, "weight") == (packed,), msg
            _expect_refused(dec, h, packed, lambda: lib.aae_decoder_forward(h, _lib().ptr(zd), 3, _lib().ptr(x), _stream()))
            with pytest.raises(AaeError, match="refused"):
                sess.run(dec.x, {zin: zd.cpu().numpy()})
            assert lib.aae_decoder_set_weights(h, layer, _lib().ptr(kern0), None, _stream()) == 0, _last_error()
            dec.decode_device(zd)
            assert lib.aae_decoder_range_status(h, _stream()) == 0, _last_error()
    _note_peak()
    dec.close()
    print("decoder %s%s at %.1f: worst |x - x64| %.2e" % (rid, " + mask head" if mask else "", OK_V, worst))


class _nothing:
    def __enter__(self):
        return self

    def __exit__(self, *a):
        return False


# ------------------------------------------------------------------------------------------------ trainers
@pytest.mark.parametrize("gemm", [None, FP16], ids=["split", "single_pass"])
def test_trainer_reports_activations_and_weights_at_the_limit(sess, gemm):
    """During step_device an activation of 4095.5 in encoder conv3 and in the decoder's first hidden conv is reported by the owning
    handle's check, naming the layer; the same pair at 4094.5 steps clean.  A weight that an Adam step carries across
    255.9375 is reported by the next check, and every later step and sess.run(train_op) fails until the layer is set again."""
    from augmentedautoencoder_b200.ae.ae import AE
    from augmentedautoencoder_b200.ae.ae_factory import TrainOp
    from tests.geometry_table import decoder as mk_decoder
    lib = _lib().lib()
    AaeError = _lib().AaeError
    r = dict(_row("template"), id="template")
    for value in (OK_V, BAD_V):
        ep, x, _, _ = _chain(r, 2, value, True)
        dp, _ = _dec_model(r, 1, value)
        enc = encoder(r, precision=SPLIT, is_training=True)
        dec = mk_decoder(r, enc, precision=SPLIT)
        enc.load_weights(ep)
        dec.load_weights(dp)
        top = TrainOp(AE(enc, dec, 0, 0), 2e-4, precision=gemm)
        xb = torch.from_numpy(O.preprocess(x[-3:])).cuda()
        top.step_device(xb, xb, update=False)
        _note_peak()
        for mod, layer in ((enc, 2), (dec, 1)):
            if value == OK_V:
                mod.check_range(sess.device)
            else:
                with pytest.raises(AaeError) as ei:
                    mod.check_range(sess.device)
                assert _layers_named(str(ei.value), "activation") == (layer,), str(ei.value)
        top.close(); enc.close(); dec.close()
    # a weight carried across the limit by an update: a dense weight of +-255 whose gradient points away from zero (the dense layer
    # has no ReLU, so either sign occurs), and an Adam step of learning rate 2.  Adam's first step moves every weight by about the
    # learning rate whatever the size of its gradient, so that weight ends near +-257 and every other weight stays far below the
    # limit; a gradient-descent step large enough for a weight with a small gradient would carry many others across as well.
    ep, dp, _ = params(r)
    L = r["L"]
    enc = encoder(r, precision=SPLIT, is_training=True)
    dec = mk_decoder(r, enc, precision=SPLIT)
    enc.load_weights(ep)
    dec.load_weights(dp)
    xb = torch.from_numpy(np.random.RandomState(11).rand(3, 128, 128, 3).astype(np.float32)).cuda()
    top = TrainOp(AE(enc, dec, 0, 0), 2.0, precision=gemm)
    th = top.trainer(sess.device)
    loss = torch.zeros(1, device="cuda")
    g = np.empty_like(ep["dense/kernel"])
    found = None
    for j in range(32):
        i = (37 * j + 5) % g.shape[0]
        for w0 in (255.0, -255.0):
            k = ep["dense/kernel"].copy()
            k[i, j] = w0
            enc.load_weights(dict(ep, **{"dense/kernel": k}))
            assert lib.aae_trainer_forward_backward(th, _lib().ptr(xb), _lib().ptr(xb), 3, _lib().ptr(loss), _stream()) == 0, _last_error()
            assert lib.aae_trainer_get_grads(th, 0, L, _lib().ptr(g), None, _stream()) == 0, _last_error()
            if float(g[i, j]) * w0 < -1e-5:                           # |g| >> Adam's epsilon: the step moves it by ~2
                found = (w0, float(g[i, j]))
                break
        if found:
            break
    assert found, "no dense weight whose gradient points away from zero"
    top.step_device(xb, xb)                                           # +-255 -> +-257 in the fp32 master
    enc.encode_device(xb)                                             # packs the moved weight: the guard records it
    with pytest.raises(AaeError) as ei:
        enc.check_range(sess.device)
    assert _layers_named(str(ei.value), "weight") == (L,), str(ei.value)
    with pytest.raises(AaeError, match="refused"):
        top.step_device(xb, xb)
    with pytest.raises(AaeError, match="refused"):
        enc.encode_device(xb)
    _note_peak()
    top.close(); enc.close(); dec.close()


def test_zz_peak_device_memory(sess):
    gc.collect()
    print("peak torch device memory of this file: %.2f GB" % (_peak[0] / 2 ** 30))
