"""The stream contract of include/aae_b200.h on a caller's non-blocking stream (the source half is tests/test_stream_lint_cpu.py).

Every other GPU test runs on the current stream of a fresh process, the legacy default stream, which serialises against itself
whatever the library does.  A torch.cuda.Stream is created cudaStreamNonBlocking: it does not wait for the legacy stream, so a
launch, fill or copy the library issues anywhere but on the caller's stream races the caller's work there.  Two helpers make that
visible without relying on timing:

  run_on_side_stream      the inputs reach the device on the side stream BEHIND a bounded delay (one spinning thread), while the
                          buffers the library is given hold poison until then; anything issued on another stream runs during the
                          delay, reads poison or is overwritten, and the result differs from the default-stream run bit for bit.
  returns_before_the_device
                          an event behind the delay is still pending when an asynchronous call returns (no host-side wait), and an
                          event behind a delay on the legacy stream is still pending when the side stream has drained (the call
                          neither waited for nor queued behind the legacy stream).

The delay runs once per case and nothing is retried."""
import ctypes as C
import gc

import numpy as np
import pytest
import torch

from augmentedautoencoder_b200 import _lib
from augmentedautoencoder_b200.ae import augment as A
from augmentedautoencoder_b200.m3_interface.ae_pose_estimator import square_patch_boxes
from oracle import aae_oracle as O
from tests.test_augment_cpu import TEMPLATE_CODE
from tests.test_gpu_a_parity import _codebook, _enc, sess  # noqa: F401

pytestmark = pytest.mark.gpu

FP32, SPLIT, FP16 = 0, 1, 2
PRECISIONS = [FP32, SPLIT, FP16]
DELAY_MS = 40.0


# ------------------------------------------------------------------------------------------------ helpers
@pytest.fixture(scope="module")
def delay(sess):
    """delay(ms) enqueues about `ms` milliseconds of one spinning thread on the current stream (torch.cuda._sleep; cycles per
    millisecond from one event-timed call)."""
    torch.cuda._sleep(1000)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    torch.cuda._sleep(20_000_000)
    b.record()
    b.synchronize()
    per_ms = 20_000_000 / a.elapsed_time(b)

    def enqueue(ms=DELAY_MS):
        torch.cuda._sleep(int(per_ms * ms))
    return enqueue


@pytest.fixture(autouse=True)
def _quiet_device():
    """every case starts and ends with an idle device, and frees what it built"""
    torch.cuda.synchronize()
    yield
    torch.cuda.synchronize()
    gc.collect()
    torch.cuda.empty_cache()


def S():
    """the current stream as the void* of the C ABI"""
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def ok(status, what="aae call"):
    _lib.check(status, what)


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def poisoned(shape, dtype):
    """0xFF bytes: NaN as float32, -1 as int32, 255 as uint8; written on the current stream"""
    t = torch.empty(tuple(shape), dtype=dtype, device="cuda")
    t.view(torch.uint8).fill_(0xFF)
    return t


def other(t):
    """the same rows in another order: a valid input (every table row stays whole) that gives another result per position"""
    return t.flip(0).contiguous()


def tup(x):
    return tuple(x) if isinstance(x, (tuple, list)) else (x,)


def same(got, want, what):
    assert len(got) == len(want)
    for i, (g, w) in enumerate(zip(got, want)):
        g, w = np.atleast_1d(np.ascontiguousarray(g)), np.atleast_1d(np.ascontiguousarray(w))
        assert g.shape == w.shape and g.dtype == w.dtype, (what, i)
        assert np.array_equal(g.view(np.uint8), w.view(np.uint8)), \
            "%s: output %d differs in %d of %d elements (first at %s)" % (what, i, int(np.count_nonzero(g != w)), g.size, np.argwhere(g != w)[:1].tolist())


def run_on_side_stream(fn, inputs, delay, what):
    """fn(*device tensors) -> device tensor(s), launched on the current stream.  Asserts that a run on a new non-blocking stream,
    whose inputs arrive on that stream behind the delay, gives the bits of the default-stream run.  Returns those (numpy)."""
    want = [o.cpu().numpy() for o in tup(fn(*inputs))]
    again = [o.cpu().numpy() for o in tup(fn(*inputs))]
    same(again, want, what + " (two default-stream runs)")
    fn(*[other(t) for t in inputs])                    # the handle's workspace now holds another call's values
    staged = [poisoned(t.shape, t.dtype) for t in inputs]
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        delay()
        for d, t in zip(staged, inputs):
            d.copy_(t, non_blocking=True)
        outs = tup(fn(*staged))
        host = [torch.empty(o.shape, dtype=o.dtype, pin_memory=True).copy_(o, non_blocking=True) for o in outs]
    s.synchronize()                                    # the side stream only
    same([h.numpy() for h in host], want, what + " (side stream)")
    torch.cuda.synchronize()
    return want


def returns_before_the_device(call, delay, synchronises=False, leaves_legacy_alone=True, ms=DELAY_MS):
    """`call()` launches on the current stream.  synchronises=False: it returns while the device is still inside a delay queued
    ahead of it on the side stream.  synchronises=True (documented to wait for its stream): it does not.  Either way it neither
    waits for nor queues behind the legacy stream."""
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        call()                                         # scratch that appears on first use is behind us
    torch.cuda.synchronize()
    ev = torch.cuda.Event()
    with torch.cuda.stream(s):
        delay(ms)
        ev.record()
        call()
        done_on_return = ev.query()
    s.synchronize()
    assert done_on_return == synchronises, "the call %s for its stream" % ("did not wait" if synchronises else "waited")
    if not leaves_legacy_alone:
        return
    legacy = torch.cuda.Event()
    delay(ms)                                          # current stream here: the legacy default stream
    legacy.record()
    with torch.cuda.stream(s):
        call()
    s.synchronize()
    legacy_done = legacy.query()
    torch.cuda.synchronize()
    assert not legacy_done, "the call waited for, or queued work behind, the legacy default stream"


# ------------------------------------------------------------------------------------------------ handles
EP = O.make_encoder_params(42, bias_scale=0.05)
DP = O.make_decoder_params(43, bias_scale=0.05)
N_ROWS = 36 * 300


def encoder(prec, max_batch=130, params=EP, sigma=False):
    e = _enc(prec, max_batch, params)
    if sigma:
        e.q_sigma                                      # registers the head (zero kernel: sigma = ln 2) ...
        rng = np.random.RandomState(5)
        e.load_weights({"dense_1/kernel": (0.01 * rng.standard_normal((e._flat, 128))).astype(np.float32),
                        "dense_1/bias": np.full(128, 0.3, np.float32)}, strict=False)       # ... and gives it values
    return e


def decoder(prec, mask=False, max_batch=8):
    from augmentedautoencoder_b200.ae.decoder import Decoder
    from augmentedautoencoder_b200.ae.session import placeholder
    from tests.test_gpu_k_aux_mask import _head, _named
    d = Decoder(placeholder(np.float32, [None, 128, 128, 3]), placeholder(np.float32, [None, 128]), list(reversed(O.NUM_FILTER)), 5,
                list(reversed(O.STRIDES)), "L2", 4, mask, False, max_batch=max_batch, precision=prec)
    d.load_weights(_named(DP, _head(scale=0.05)) if mask else DP)
    return d


def crops(seed, batch, hw=128):
    return dev(O.make_crops_u8(seed, batch, hw=hw))


def latents(seed, batch):
    return dev((np.random.RandomState(seed).standard_normal((batch, 128)) * 2.0).astype(np.float32))


# ------------------------------------------------------------------------------------------------ encoder
@pytest.mark.parametrize("batch", [3, 130])            # 3: split-K forward and its finish kernel; 130: two match blocks
@pytest.mark.parametrize("prec", PRECISIONS)
def test_encoder_forward_match_and_activation(sess, delay, prec, batch):
    """forward_u8 and forward_f32, the fused match behind them, the sigma head and aae_encoder_activation of the same forward, all
    enqueued on the side stream without a synchronise in between."""
    enc = encoder(prec, sigma=True)
    cb = _codebook(enc, O.make_codebook(7, n=N_ROWS), max_batch=130, precision=prec)
    lib, nl = _lib.lib(), len(O.NUM_FILTER)

    def fn(x):
        h, hc, B = enc.handle(0), cb.handle(0), x.shape[0]
        z, sig = poisoned((B, 128), torch.float32), poisoned((B, 128), torch.float32)
        sc, ix = poisoned((B, 1), torch.float32), poisoned((B, 1), torch.int32)
        fwd = lib.aae_encoder_forward_u8 if x.dtype == torch.uint8 else lib.aae_encoder_forward_f32
        ok(fwd(h, _lib.ptr(x), B, _lib.ptr(z), S()), "forward")
        ok(lib.aae_codebook_match(hc, _lib.ptr(z), B, 1, 0, _lib.ptr(sc), _lib.ptr(ix), S()), "match")
        ok(lib.aae_encoder_sigma_forward(h, B, _lib.ptr(sig), S()), "sigma forward")
        flat = enc.activation_device(nl - 1, torch.device("cuda", 0))      # takes no stream: must still see the forward above
        return z, sig, sc, ix, flat

    xu = crops(1234, batch)
    zu = run_on_side_stream(fn, [xu], delay, "u8 forward, precision %d, batch %d" % (prec, batch))[0]
    zf = run_on_side_stream(fn, [xu.to(torch.float32) / 255.0], delay, "f32 forward, precision %d, batch %d" % (prec, batch))[0]
    assert np.isfinite(zu).all() and np.abs(zu).max() > 1e-3 and np.abs(zu - zf).max() < 1e-2


def test_encoder_px64_fp32_conv1_feeds_a_split_conv2(sess, delay):
    from tests import geometry_table as G
    r = G.row("px64")
    enc = G.encoder(r, precision=SPLIT)
    enc.load_weights(G.params(r)[0])

    def fn(x):
        return enc.encode_device(x, out=poisoned((x.shape[0], r["latent"]), torch.float32))
    for batch in (3, G.MAXB):
        run_on_side_stream(fn, [crops(7, batch, hw=64)], delay, "px64, batch %d" % batch)


@pytest.mark.parametrize("prec", PRECISIONS)
def test_encoder_forward_is_asynchronous_and_range_status_is_not(sess, delay, prec):
    enc = encoder(prec, max_batch=8)
    h, lib = enc.handle(0), _lib.lib()
    x, z = crops(3, 8), torch.empty((8, 128), device="cuda")
    returns_before_the_device(lambda: ok(lib.aae_encoder_forward_u8(h, _lib.ptr(x), 8, _lib.ptr(z), S())), delay)
    returns_before_the_device(lambda: ok(lib.aae_encoder_range_status(h, S())), delay, synchronises=prec != FP32)
    if prec != FP32:
        # the tensor-core form unpacks on the legacy stream behind a device-wide wait (it takes no stream argument)
        returns_before_the_device(lambda: enc.activation_device(1, torch.device("cuda", 0)), delay, synchronises=True, leaves_legacy_alone=False)


# ------------------------------------------------------------------------------------------------ match
@pytest.mark.parametrize("prec,k,upright", [(SPLIT, 1, False), (SPLIT, 8, False), (SPLIT, 1, True), (SPLIT, 8, True), (SPLIT, 12, False),
                                            (FP16, 1, False), (FP16, 8, False), (FP32, 1, False), (FP32, 4, True)])
def test_match_twice_back_to_back(sess, delay, prec, k, upright):
    """k = 1 re-arms its atomicMax scratch and k = 8 its last-CTA counter for the next call: two calls back to back on the side
    stream, the second on other queries.  k = 12 on a split handle takes the fp32 kernels."""
    enc = encoder(prec, max_batch=8)
    cb = _codebook(enc, O.make_codebook(7, n=N_ROWS), max_batch=130, precision=prec)
    lib = _lib.lib()

    def fn(z1, z2):
        h, outs = cb.handle(0), []
        for z in (z1, z2):
            sc, ix = poisoned((z.shape[0], k), torch.float32), poisoned((z.shape[0], k), torch.int32)
            ok(lib.aae_codebook_match(h, _lib.ptr(z), z.shape[0], k, int(upright), _lib.ptr(sc), _lib.ptr(ix), S()), "match")
            outs += [sc, ix]
        return outs
    sc1, ix1, sc2, ix2 = run_on_side_stream(fn, [latents(1, 130), latents(2, 37)], delay, "match precision %d k %d upright %d" % (prec, k, upright))
    assert (ix1 >= 0).all() and (ix1 < N_ROWS).all() and (np.diff(sc1, axis=1) <= 0).all() and not np.array_equal(ix1[:37], ix2)
    if upright:
        assert (ix1 % 36 == 0).all()


def test_cosine_normalize_and_merges(sess, delay):
    enc = encoder(FP32, max_batch=8)
    cb = _codebook(enc, O.make_codebook(7, n=5000), max_batch=16, precision=FP32)
    lib = _lib.lib()

    def cosine(z):
        B = z.shape[0]
        zq, cos = poisoned((B, 128), torch.float32), poisoned((B, 5000), torch.float32)
        ok(lib.aae_l2_normalize(_lib.ptr(z), B, 128, _lib.ptr(zq), S()))
        ok(lib.aae_codebook_cosine(cb.handle(0), _lib.ptr(z), B, _lib.ptr(cos), S()))
        return zq, cos
    run_on_side_stream(cosine, [latents(3, 9)], delay, "cosine")

    rng = np.random.RandomState(3)
    n, B, k = 8, 33, 4
    scores = -np.sort(-rng.randn(n, B, k).astype(np.float32), axis=2)
    idx = np.stack([np.sort(rng.choice(1000, size=(B, k), replace=False), axis=1) + s * 1000 for s in range(n)]).astype(np.int32)
    packed = np.concatenate([scores.view(np.int32)[:, None], idx[:, None]], axis=1)        # [n][2][B][k]

    def merges(sd, idd, pk):
        so, io = poisoned((B, k), torch.float32), poisoned((B, k), torch.int32)
        sp, ip = poisoned((B, k), torch.float32), poisoned((B, k), torch.int32)
        ok(lib.aae_topk_merge(_lib.ptr(sd), _lib.ptr(idd), n, B, k, _lib.ptr(so), _lib.ptr(io), S()))
        ok(lib.aae_topk_merge_packed(_lib.ptr(pk), n, B, k, _lib.ptr(sp), _lib.ptr(ip), S()))
        return so, io, sp, ip
    so, io, sp, ip = run_on_side_stream(merges, [dev(scores), dev(idx), dev(packed)], delay, "top-k merges")
    assert np.array_equal(so, sp) and np.array_equal(io, ip)


# ------------------------------------------------------------------------------------------------ decoder and losses
@pytest.mark.parametrize("prec", [FP32, SPLIT])
def test_decoder_forward_mask_and_losses(sess, delay, prec):
    plain, masked = decoder(prec), decoder(prec, mask=True)
    lib = _lib.lib()

    def fn(z, y):
        B = z.shape[0]
        x0, x1, m = (poisoned((B, 128, 128, 3), torch.float32), poisoned((B, 128, 128, 3), torch.float32), poisoned((B, 128, 128), torch.float32))
        loss, g, gm = poisoned((1,), torch.float32), poisoned((B, 128 * 128 * 3), torch.float32), poisoned((B, 128 * 128), torch.float32)
        ok(lib.aae_decoder_forward(plain.handle(0), _lib.ptr(z), B, _lib.ptr(x0), S()))
        ok(lib.aae_decoder_forward_mask(masked.handle(0), _lib.ptr(z), B, _lib.ptr(x1), _lib.ptr(m), S()))
        ok(lib.aae_bootstrap_l2_loss(_lib.ptr(x1), _lib.ptr(y), B, 128 * 128 * 3, 4, _lib.ptr(loss), _lib.ptr(g), S()))
        ok(lib.aae_mask_loss(_lib.ptr(m), _lib.ptr(y), B, 128 * 128, 3, _lib.ptr(loss), _lib.ptr(gm), S()))
        return x0, x1, m, loss, g, gm
    from tests.test_gpu_k_aux_mask import _target
    x0, x1, m, loss, g, gm = run_on_side_stream(fn, [latents(7, 5), dev(_target(4, 5))], delay, "decoder precision %d" % prec)
    assert np.array_equal(x0, x1) and 0 < loss[0] < 1 and 0 < np.count_nonzero(g) <= 5 * 128 * 128 * 3 // 4 and m.std() > 1e-4

    z, y = latents(7, 5), dev(_target(4, 5))
    x, msk, l = torch.empty((5, 128, 128, 3), device="cuda"), torch.empty((5, 128, 128), device="cuda"), torch.zeros(1, device="cuda")
    returns_before_the_device(lambda: ok(lib.aae_decoder_forward_mask(masked.handle(0), _lib.ptr(z), 5, _lib.ptr(x), _lib.ptr(msk), S())), delay)
    # both losses take their per-sample scratch from the stream's memory pool (cudaMallocAsync)
    returns_before_the_device(lambda: ok(lib.aae_bootstrap_l2_loss(_lib.ptr(x), _lib.ptr(y), 5, 128 * 128 * 3, 4, _lib.ptr(l), None, S())), delay)
    returns_before_the_device(lambda: ok(lib.aae_mask_loss(_lib.ptr(msk), _lib.ptr(y), 5, 128 * 128, 3, _lib.ptr(l), None, S())), delay)


def test_uint8_targets_of_the_loss_wrappers(sess, delay):
    from augmentedautoencoder_b200.ae.decoder import Decoder

    def fn(x, y8):
        loss, g = Decoder.loss_device(x, y8, 4, with_grad=True)
        return loss.reshape(1), g
    x = dev(np.random.RandomState(0).rand(3, 16, 16, 3).astype(np.float32))
    run_on_side_stream(fn, [x, dev(np.random.RandomState(1).randint(0, 256, (3, 16, 16, 3), dtype=np.uint8))], delay, "uint8 target")


# ------------------------------------------------------------------------------------------------ training
SWITCHES = dict(variational=0.1, norm=0.5)
_OPEN = []


@pytest.fixture(autouse=True)
def _close_trainers():
    yield
    while _OPEN:
        top, enc, dec = _OPEN.pop()
        top.close()
        enc.close()
        dec.close()


def trainer(handles, gemm, switches, optimizer, B=2):
    """a template encoder / decoder / TrainOp; `switches`: VARIATIONAL, NORM_REGULARIZE and AUXILIARY_MASK on.  The fp32 trainer
    joins the mask head with an output conv of at most 3 channels, which the template's is."""
    from augmentedautoencoder_b200.ae.ae import AE
    from augmentedautoencoder_b200.ae.ae_factory import TrainOp
    from augmentedautoencoder_b200.ae.decoder import Decoder
    from augmentedautoencoder_b200.ae.encoder import Encoder
    from augmentedautoencoder_b200.ae.session import placeholder
    from tests.test_gpu_h_latent_terms import _head as sigma_head
    from tests.test_gpu_k_aux_mask import _head as mask_head
    from tests.test_gpu_m_all_switches import SIGMA, _dec_named
    x, y = placeholder(np.float32, [None, 128, 128, 3]), placeholder(np.float32, [None, 128, 128, 3])
    enc = Encoder(x, 128, list(O.NUM_FILTER), 5, list(O.STRIDES), False, is_training=True, max_batch=B, precision=handles)
    if switches:
        head = sigma_head(0.05)
        dec = Decoder(y, enc.sampled_z, list(reversed(O.NUM_FILTER)), 5, list(reversed(O.STRIDES)), "L2", 4, True, False, is_training=True,
                      max_batch=B, precision=handles)
        enc.load_weights({**EP, SIGMA + "/kernel": head[0], SIGMA + "/bias": head[1]})
        dec.load_weights(_dec_named(DP, mask_head(scale=0.05), True))
        ae = AE(enc, dec, SWITCHES["norm"], SWITCHES["variational"])
    else:
        dec = Decoder(y, enc.z, list(reversed(O.NUM_FILTER)), 5, list(reversed(O.STRIDES)), "L2", 4, False, False, is_training=True,
                      max_batch=B, precision=handles)
        enc.load_weights(EP)
        dec.load_weights(DP)
        ae = AE(enc, dec, 0, 0)
    top = TrainOp(ae, 2e-4, precision=gemm, optimizer=optimizer)
    _OPEN.append((top, enc, dec))
    return enc, dec, top


def two_steps(enc, dec, top, x, y):
    """forward_backward, then two updates, on the current stream with no synchronise between the launches; then everything the
    trainer holds, read on the same stream: the losses, every gradient of the second step, the masters and the slots."""
    l0 = top.step_device(x, y, update=False, eps=0.7).reshape(1).clone()
    l1 = top.step_device(x, y, update=True, eps=0.7).reshape(1).clone()
    l2 = top.step_device(x.flip(0), y.flip(0), update=True, eps=-0.3).reshape(1).clone()
    grads = top.gradients(torch.device("cuda", 0))     # the first host read: get_grads must itself be ordered behind the steps
    z = enc.encode_device(x)                           # inference right behind the update: the handle's plan re-packs on this stream
    rec = tup(dec.decode_device(z, with_mask=bool(dec._auxiliary_mask)))
    host = [t.cpu().numpy() for t in (l0, l1, l2, z) + rec]          # .cpu() waits for the current stream only
    slots = top.optimizer_variables()
    weights = {**enc.get_weights(), **dec.get_weights()}
    for d in (grads, slots, weights):
        host += [np.asarray(d[k]) for k in sorted(d)]
    return host


TRAINERS = [(FP32, None, False, "Adam"), (SPLIT, None, False, "Adam"), (SPLIT, FP16, False, "Adam"),
            (FP32, None, True, "GradientDescent"), (SPLIT, None, True, "Adagrad"), (SPLIT, FP16, True, "Adam")]


@pytest.mark.parametrize("handles,gemm,switches,optimizer", TRAINERS)
def test_training_steps_on_a_side_stream(sess, delay, handles, gemm, switches, optimizer):
    """Three identical trainers: two run the sequence on the default stream (they must agree bit for bit), the third on a side
    stream whose inputs arrive behind the delay.  The second update re-packs the tensor-core operands from the masters the first
    one changed, and the inference calls behind it re-pack the handles' own plans, all on the side stream."""
    from tests.test_gpu_k_aux_mask import _target
    x, y = dev(np.random.RandomState(8).rand(2, 128, 128, 3).astype(np.float32)), dev(_target(4, 2))
    what = "trainer handles %d gemm %s switches %s %s" % (handles, gemm, switches, optimizer)
    want = two_steps(*trainer(handles, gemm, switches, optimizer), x, y)
    again = two_steps(*trainer(handles, gemm, switches, optimizer), x, y)
    same(again, want, what + " (two default-stream runs)")
    assert all(np.isfinite(w).all() for w in want) and want[0][0] != want[2][0]
    enc, dec, top = trainer(handles, gemm, switches, optimizer)
    top.trainer(torch.device("cuda", 0))               # creation is not what this case is about
    xs, ys = poisoned(x.shape, x.dtype), poisoned(y.shape, y.dtype)
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        delay()
        xs.copy_(x, non_blocking=True)
        ys.copy_(y, non_blocking=True)
        got = two_steps(enc, dec, top, xs, ys)
    same(got, want, what + " (side stream)")


@pytest.mark.parametrize("handles,gemm", [(FP32, None), (SPLIT, None), (SPLIT, FP16)])
def test_training_step_is_asynchronous_and_its_readers_are_not(sess, delay, handles, gemm):
    enc, dec, top = trainer(handles, gemm, True, "Adam")
    from tests.test_gpu_k_aux_mask import _target
    x, y = dev(np.random.RandomState(8).rand(2, 128, 128, 3).astype(np.float32)), dev(_target(4, 2))
    h, lib, loss = top.trainer(torch.device("cuda", 0)), _lib.lib(), torch.empty(1, device="cuda")
    ok(lib.aae_trainer_profile(h, 1, None, 0))         # phase events are recorded on the launching stream
    ms = 400.0 if handles == FP32 else 100.0           # the fp32 CUDA-core step must fit inside the legacy stream's delay
    returns_before_the_device(lambda: ok(lib.aae_train_step(h, _lib.ptr(x), _lib.ptr(y), 2, _lib.ptr(loss), S())), delay, ms=ms)
    returns_before_the_device(lambda: ok(lib.aae_trainer_forward_backward(h, _lib.ptr(x), _lib.ptr(y), 2, _lib.ptr(loss), S())), delay, ms=ms)
    phases = (C.c_float * 8)()
    if handles != FP32:
        assert lib.aae_trainer_profile(h, 0, phases, 8) == 7 and sum(phases) > 0
    g = np.empty((5, 5, 3, 128), np.float32)
    m, v = np.empty_like(g), np.empty_like(g)
    returns_before_the_device(lambda: ok(lib.aae_trainer_get_grads(h, 0, 0, _lib.ptr(g), None, S())), delay, synchronises=True)
    returns_before_the_device(lambda: ok(lib.aae_trainer_get_state(h, 0, 0, _lib.ptr(m), _lib.ptr(v), None, None, S())), delay, synchronises=True)
    returns_before_the_device(lambda: ok(lib.aae_trainer_set_state(h, 0, 0, _lib.ptr(m), _lib.ptr(v), None, None, S())), delay, synchronises=True)
    returns_before_the_device(lambda: ok(lib.aae_encoder_get_weights(enc.handle(0), 0, _lib.ptr(g), None, S())), delay, synchronises=True)
    returns_before_the_device(lambda: ok(lib.aae_encoder_set_weights(enc.handle(0), 0, _lib.ptr(g), None, S())), delay, synchronises=True)
    returns_before_the_device(lambda: ok(lib.aae_decoder_range_status(dec.handle(0), S())), delay, synchronises=handles != FP32)


# ------------------------------------------------------------------------------------------------ state copies
@pytest.mark.parametrize("prec", [FP32, SPLIT])
def test_set_weights_then_forward_on_the_side_stream(sess, delay, prec):
    """set_weights from a DEVICE pointer that is filled on the side stream behind the delay, then a forward there: the forward
    uses the new weights (the tensor-core pack is ordered behind the copy), and get_weights into a device buffer returns them."""
    enc = encoder(prec, max_batch=8)
    h, lib, nl = enc.handle(0), _lib.lib(), len(O.NUM_FILTER)
    new = O.make_encoder_params(77, bias_scale=0.05)
    wk, wb = dev(new["dense/kernel"]), dev(new["dense/bias"])

    def fn(x, k, b):
        z, back = poisoned((x.shape[0], 128), torch.float32), poisoned(k.shape, torch.float32)
        ok(lib.aae_encoder_set_weights(h, nl, _lib.ptr(k), _lib.ptr(b), S()))
        ok(lib.aae_encoder_forward_u8(h, _lib.ptr(x), x.shape[0], _lib.ptr(z), S()))
        ok(lib.aae_encoder_get_weights(h, nl, _lib.ptr(back), None, S()))
        return z, back
    z, back = run_on_side_stream(fn, [crops(5, 4), wk, wb], delay, "set_weights precision %d" % prec)
    assert np.array_equal(back, new["dense/kernel"])
    want = _enc(prec, 8, {**EP, "dense/kernel": new["dense/kernel"], "dense/bias": new["dense/bias"]}).encode_device(crops(5, 4)).cpu().numpy()
    assert np.array_equal(z, want)


# ------------------------------------------------------------------------------------------------ input pipeline
def test_augment_args_occlusion_args_and_crop_table_extraction(sess, delay, tmp_path):
    """aae_augment, aae_occlusion and aae_extract_square_patches, the last with its int32 (x, y, w, h, size) box table, on a
    caller's side stream."""
    from tests.test_gpu_g_occlusion import _bank, _objects
    from tests.test_gpu_z_augment import _inputs
    lib, B = _lib.lib(), 24
    x, mask, bg = _inputs(0, B)
    aug = A.Augmenter(TEMPLATE_CODE, seed=1)
    aug.sigma = 1.17
    P = aug.sample(B)
    for key in ("affine_on", "drop_on", "blur_on", "add_on", "invert_on", "mul1_on", "mul2_on", "contrast_on"):
        P[key][:4] = True
    geom, lut = aug.pack(P)
    k = aug._constants(torch.device("cuda", 0))
    taps = k["taps"]

    def augment(xd, md, bd, gd, ld):
        tmp, ou, of = poisoned(xd.shape, torch.uint8), poisoned(xd.shape, torch.uint8), poisoned(xd.shape, torch.float32)
        ok(lib.aae_augment(C.byref(_lib.AugmentArgs(
            batch=B, h=128, w=128, c=3, low_w=aug.low[1], x=xd, mask=md, bg=bd, geom=gd, lut=ld, bilinear_tab=k["tab"], row_cell=k["rows"],
            col_cell=k["cols"], blur_kernel_q8=taps, u8_to_float=k["to_float"], tmp=tmp, out_u8=ou, out_f32=of)), S()))
        return ou, of
    inputs = [dev(x), dev(mask.astype(np.uint8)), dev(bg), dev(geom.astype(np.int32)), dev(lut.astype(np.uint8))]
    want = aug.augment_device(inputs[0], inputs[1], inputs[2], params=P, want_u8=True)
    ou, of = run_on_side_stream(augment, inputs, delay, "augment")
    assert np.array_equal(ou, want[1].cpu().numpy()) and np.array_equal(of, want[0].cpu().numpy())

    rng = np.random.RandomState(0)
    _, words, _ = _bank(tmp_path, rng)
    masks = _objects(rng, B)
    occl = A.Occlusion((128, 128), 0.4, 0.2, seed=1)
    PO = occl.sample(B, len(words))
    st = occl._state(torch.device("cuda", 0))
    bank = dev(np.ascontiguousarray(words, np.uint32).view(np.int32))

    def occlude(md, cand, bk):
        out, fb = poisoned(md.shape, torch.uint8), torch.zeros(2, dtype=torch.int32, device="cuda")
        ok(lib.aae_occlusion(C.byref(_lib.OcclusionArgs(
            batch=B, h=128, w=128, realistic=1, max_occl=0.4, square=1, min_kept=1.0 - 0.2, mask=md, cand=cand, n_cand=occl.K,
            n_bank=len(words), bank=bk, row_cell=st["rows"], col_cell=st["cols"], low_h=occl.low[0], low_w=occl.low[1], mask_out=out,
            fallbacks=fb)), S()))
        return out, fb
    md = dev(masks.astype(np.uint8))
    want_o = occl.apply_device(md, words, params=PO).cpu().numpy()
    out, _ = run_on_side_stream(occlude, [md, dev(occl.pack(PO)), bank], delay, "occlusion")
    assert np.array_equal(out, want_o) and 0 < out.mean() < 1

    frame = dev(np.random.RandomState(2).randint(0, 256, (480, 640, 3), dtype=np.uint8))
    boxes = dev(square_patch_boxes([[100, 120, 80, 60], [-10, -20, 90, 120], [600, 440, 70, 70], [300, 200, 200, 150], [0, 0, 640, 480]], 1.2))

    def extract(fr, bx):
        out = poisoned((5, 128, 128, 3), torch.uint8)
        ok(lib.aae_extract_square_patches(_lib.ptr(fr), 480, 640, _lib.ptr(bx), 5, 128, _lib.ptr(out), S()))
        return out
    patches = run_on_side_stream(extract, [frame, boxes], delay, "extract_square_patches")[0]
    assert patches.std() > 10


# ------------------------------------------------------------------------------------------------ timers
@pytest.mark.parametrize("prec", [FP32, SPLIT])
def test_stage_timers_record_on_the_side_stream(sess, delay, prec):
    enc = encoder(prec, max_batch=8)
    cb = _codebook(enc, O.make_codebook(7, n=N_ROWS), max_batch=8, precision=prec)
    lib, ms = _lib.lib(), (C.c_float * 16)()

    def fn(x):
        return cb.nearest_idx_device(x)
    x = crops(9, 8)
    plain = [o.cpu().numpy() for o in fn(x)]
    ok(lib.aae_encoder_profile(enc.handle(0), 1, None, 0))
    ok(lib.aae_codebook_profile(cb.handle(0), 1, None, 0))
    timed = run_on_side_stream(fn, [x], delay, "timed forward + match precision %d" % prec)
    same(timed, plain, "timers change nothing")
    assert lib.aae_encoder_profile(enc.handle(0), 0, ms, 16) == len(O.NUM_FILTER) + 1 and min(ms[:5]) > 0
    assert lib.aae_codebook_profile(cb.handle(0), 0, ms, 16) == 1 and ms[0] > 0


# ------------------------------------------------------------------------------------------------ creation ordering
def _create_then_use(use, delay, on_side):
    """legacy stream busy -> build (the creators run inside `use`, on first use of the Python modules) -> use on a fresh side
    stream -> wait for that stream -> let the device drain -> use again.  Whatever creation left pending on the legacy stream
    lands after the first use (zeroing what set_weights and the first update wrote), so the second use would show it."""
    if not on_side:
        return use() + use()
    s = torch.cuda.Stream()
    delay()                                            # on the legacy default stream
    with torch.cuda.stream(s):
        first = use()
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        second = use()
    return first + second


@pytest.mark.parametrize("prec", PRECISIONS)
def test_new_encoder_codebook_and_sigma_head_are_complete_on_return(sess, delay, prec):
    x = crops(11, 3)

    def build():
        enc = encoder(prec, max_batch=8, sigma=True)
        cb = _codebook(enc, O.make_codebook(7, n=N_ROWS), max_batch=8, precision=prec)

        def use():
            z = enc.encode_device(x)                   # first call: aae_encoder_create, enable_sigma_head, set_weights, forward
            sig = enc._sigma_of_last_forward(torch.device("cuda", 0), 3)
            sc, ix = cb.match_device(z, k=1)           # first call: aae_codebook_create
            sc8, ix8 = cb.match_device(z, k=8)
            return [t.cpu().numpy() for t in (z, sig, sc, ix, sc8, ix8)]
        return use
    want = _create_then_use(build(), delay, on_side=False)
    got = _create_then_use(build(), delay, on_side=True)
    same(got, want, "encoder / codebook created under a busy legacy stream, precision %d" % prec)
    assert np.abs(want[0]).max() > 1e-3 and abs(want[1][0, 0] - np.log(2)) > 1e-3


@pytest.mark.parametrize("prec", [FP32, SPLIT])
def test_new_decoder_and_mask_head_are_complete_on_return(sess, delay, prec):
    z = latents(7, 3)

    def build():
        dec = decoder(prec, mask=True)
        return lambda: [t.cpu().numpy() for t in dec.decode_device(z, with_mask=True)]
    want = _create_then_use(build(), delay, on_side=False)
    got = _create_then_use(build(), delay, on_side=True)
    same(got, want, "decoder created under a busy legacy stream, precision %d" % prec)
    assert want[1].std() > 1e-4


@pytest.mark.parametrize("handles,gemm", [(FP32, None), (SPLIT, None), (SPLIT, FP16)])
@pytest.mark.parametrize("optimizer", ["Adam", "Adagrad", "GradientDescent"])
def test_new_trainer_is_complete_on_return(sess, delay, handles, gemm, optimizer):
    """two updates on a fresh side stream right after aae_trainer_create_opt, then (device drained) the gradients, slots and
    masters, and one more update."""
    from tests.test_gpu_k_aux_mask import _target
    x, y = dev(np.random.RandomState(8).rand(2, 128, 128, 3).astype(np.float32)), dev(_target(4, 2))

    def build():
        enc, dec, top = trainer(handles, gemm, True, optimizer)
        state = {"first": True}

        def use():
            if state.pop("first", False):
                return [top.step_device(x, y, eps=0.7).reshape(1).cpu().numpy(), top.step_device(x, y, eps=0.2).reshape(1).cpu().numpy()]
            grads, slots = top.gradients(torch.device("cuda", 0)), top.optimizer_variables()
            weights = {**enc.get_weights(), **dec.get_weights()}
            out = [np.asarray(d[k]) for d in (grads, slots, weights) for k in sorted(d)]
            return out + [top.step_device(x, y, eps=0.1).reshape(1).cpu().numpy()]
        return use
    want = _create_then_use(build(), delay, on_side=False)
    got = _create_then_use(build(), delay, on_side=True)
    same(got, want, "trainer created under a busy legacy stream (%d, %s, %s)" % (handles, gemm, optimizer))


# ------------------------------------------------------------------------------------------------ handles and streams
def test_two_encoders_and_codebooks_on_two_streams_at_once(sess):
    """The AePoseEstimator.process pattern at a size where the kernels overlap: two encoder + codebook pairs with different
    weights, batch 64 each, launched alternately on two streams without a synchronise.  No state is shared between handles."""
    pairs = []
    for seed in (42, 43):
        enc = _enc(SPLIT, 64, O.make_encoder_params(seed, bias_scale=0.05))
        pairs.append((enc, _codebook(enc, O.make_codebook(seed, n=N_ROWS), max_batch=64, precision=SPLIT)))
    xs = [[crops(100 + 10 * p + r, 64) for r in range(4)] for p in range(2)]
    serial = [[[t.cpu().numpy() for t in pairs[p][1].nearest_idx_device(xs[p][r], k=8)] for r in range(4)] for p in range(2)]
    torch.cuda.synchronize()
    streams, got = [torch.cuda.Stream(), torch.cuda.Stream()], [[None] * 4, [None] * 4]
    for r in range(4):
        for p in range(2):
            with torch.cuda.stream(streams[p]):
                got[p][r] = pairs[p][1].nearest_idx_device(xs[p][r], k=8)
    torch.cuda.synchronize()
    for p in range(2):
        for r in range(4):
            same([t.cpu().numpy() for t in got[p][r]], serial[p][r], "pair %d round %d" % (p, r))
    assert not np.array_equal(serial[0][0][1], serial[1][0][1])


def test_two_split_trainers_on_two_streams_at_once(sess):
    from tests.test_gpu_k_aux_mask import _target
    data = [(dev(np.random.RandomState(8 + p).rand(2, 128, 128, 3).astype(np.float32)), dev(_target(4 + p, 2))) for p in range(2)]
    serial = []
    for p in range(2):
        enc, dec, top = trainer(SPLIT, None, False, "Adam")
        losses = [top.step_device(*data[p]).reshape(1).clone() for _ in range(3)]
        serial.append([l.cpu().numpy() for l in losses] + [enc.get_weights()["conv2d_2/kernel"], dec.get_weights()["conv2d_5/kernel"]])
    built = [trainer(SPLIT, None, False, "Adam") for _ in range(2)]
    for enc, dec, top in built:
        top.trainer(torch.device("cuda", 0))
    torch.cuda.synchronize()
    streams, losses = [torch.cuda.Stream(), torch.cuda.Stream()], [[], []]
    for _ in range(3):
        for p in range(2):
            with torch.cuda.stream(streams[p]):
                losses[p].append(built[p][2].step_device(*data[p]).reshape(1).clone())
    torch.cuda.synchronize()
    for p in range(2):
        enc, dec, _ = built[p]
        got = [l.cpu().numpy() for l in losses[p]] + [enc.get_weights()["conv2d_2/kernel"], dec.get_weights()["conv2d_5/kernel"]]
        same(got, serial[p], "trainer %d" % p)


@pytest.mark.parametrize("prec", PRECISIONS)
def test_one_handle_handed_from_stream_to_stream_with_an_event(sess, delay, prec):
    """A handle owns one workspace: one stream at a time, any stream, and the caller orders the hand-over."""
    enc = encoder(prec, max_batch=8)
    cb = _codebook(enc, O.make_codebook(7, n=N_ROWS), max_batch=8, precision=prec)
    x1, x2 = crops(21, 8), crops(22, 5)
    want = [t.cpu().numpy() for x in (x1, x2) for t in cb.nearest_idx_device(x)]
    torch.cuda.synchronize()
    s1, s2, ev = torch.cuda.Stream(), torch.cuda.Stream(), torch.cuda.Event()
    with torch.cuda.stream(s1):
        delay()
        a = cb.nearest_idx_device(x1)
        ev.record()
    with torch.cuda.stream(s2):
        s2.wait_event(ev)
        b = cb.nearest_idx_device(x2)
    torch.cuda.synchronize()
    same([t.cpu().numpy() for t in a + b], want, "hand-over, precision %d" % prec)
