"""GPU tests of the training step at the production batch (BATCH_SIZE 64), at a ragged batch on the same trainers, and across batch
changes, against the float64 oracle evaluated on the GPU.

The strict gradient tests elsewhere run batch 1.  At batch 64 the trainers take other paths: the wgrad split-K count is set by the
tile count instead of the batch, the 8x8 dgrad GEMMs stop splitting K, every grid-stride elementwise loop runs several iterations
per thread, the fp32 trainer's split counts and dgrad parity order change with M = B * pixels, and the latent kernel's warps each
take several rows.  Batch 37 is odd (the 8x8 layers' last tile pairs an image with padding) and leaves rows 37..63 of every
max_batch-sized buffer stale.

Trainers: fp32 CUDA-core, split tensor-core, and single-pass fp16 GEMMs on split handles.  Bounds: relative L2 error 3e-4 per
gradient tensor for the fp32 and split trainers (the batch-1 tests' bound) and the rounding-model bound of tests/test_gpu_e for the
fp16 trainer, evaluated on the actual batch."""
import gc

import numpy as np
import pytest
import torch

from oracle import aae_oracle as O
from oracle import latent_oracle as LO
from tests.test_gpu_a_parity import sess  # noqa: F401
from tests.test_gpu_e_fp16_train import FP16, FP32, SPLIT, _analyse, _check_grads, _clear_margin_params, _grad_bounds, _pair
from tests.test_gpu_h_latent_terms import _build, _head

pytestmark = pytest.mark.gpu

B_MAX, B_RAGGED = 64, 37
# trainer: (GEMM precision, handle precision, bootstrap ratio).  The fp16 trainer's rounding model has no term for a discrete top-k
# choice, so it runs without bootstrapping, as in tests/test_gpu_e; the others run the production ratio 4.
KINDS = {"fp32": (None, FP32, 4), "split": (None, SPLIT, 4), "fp16": (FP16, SPLIT, 1)}
REL = 3e-4
PROBES = [0, 1, 36, 63]       # first image, second image of a 2-image tile, last image of a 37-batch, last image
RELU_LAYERS = ("conv2d_1", "conv2d_2", "conv2d_3", "dense_1", "conv2d_4", "conv2d_5", "conv2d_6")


def _masked_params():
    """ReLU masks that are not all ones, with a guaranteed margin.  conv1: kernel on a 2^-4 grid, biases odd multiples of 2^-5, so on
    binary inputs every pre-activation is exact in fp32, in split fp16 and in the fp16 trainer's 16 * pre (an odd multiple of 2^-1,
    below 1024) and at least 2^-5 from zero.  Half its channels have a bias within 0.5 of zero and switch per pixel; the other half a
    bias in [4, 8], which keeps the layer's rounding condition (and so the rounding-model margin below) small.  Every later ReLU layer
    has a quarter of its units dead (bias in [-2, -1]) and the rest on (bias in [1, 2]); its kernel is scaled down far enough that
    the bias decides the sign with a margin above the fp16 rounding model's need."""
    ep, dp = O.make_encoder_params(42), O.make_decoder_params(43)
    rng = np.random.RandomState(7)
    k1 = ep["conv2d/kernel"]
    ep["conv2d/kernel"] = (rng.randint(-1, 2, k1.shape) / 16.0).astype(np.float32)
    n = k1.shape[3]
    near = 2 * rng.randint(-8, 8, n) + 1              # odd, |b| <= 15/32
    far = 2 * rng.randint(64, 128, n) + 1             # odd, b in [129/32, 255/32]
    ep["conv2d/bias"] = (np.where(np.arange(n) % 2 == 0, near, far) / 32.0).astype(np.float32)
    for p in (ep, dp):
        for name in p:
            layer = name.rsplit("/", 1)[0]
            if layer == "conv2d":
                continue
            if name.endswith("kernel"):
                p[name] = (p[name] * (0.05 if layer == "conv2d_7" else 0.003)).astype(np.float32)
            else:
                b = rng.uniform(1.0, 2.0, p[name].shape)
                if layer in RELU_LAYERS:
                    b = np.where(rng.rand(*b.shape) < 0.25, -b, b)
                p[name] = b.astype(np.float32)
    return ep, dp


def _positive_params():
    """Non-negative kernels, each output unit's |w| summing to 1 over its fan-in, and biases in [0.2, 0.3] ([1, 1.5] and gain 0.5 at the
    output layer).  On a non-negative input every activation and, for a target below the reconstruction, every gradient is
    non-negative, so no GEMM cancels: each forward, dgrad and wgrad condition of the rounding model is at most 1, and the fp16
    trainer's batch-1 bound falls below 0.2 for every tensor (with random-sign weights it exceeds 1 for the encoder's)."""
    ep, dp = O.make_encoder_params(42), O.make_decoder_params(43)
    rng = np.random.RandomState(11)
    for p in (ep, dp):
        for name in p:
            out = name.startswith("conv2d_7/")
            if name.endswith("kernel"):
                k = np.abs(p[name]).astype(np.float64)
                p[name] = ((0.5 if out else 1.0) * k / k.reshape(-1, k.shape[-1]).sum(0)).astype(np.float32)
            else:
                p[name] = rng.uniform(*((1.0, 1.5) if out else (0.2, 0.3)), p[name].shape).astype(np.float32)
    return ep, dp


PARAMS = {"clear": _clear_margin_params, "masked": _masked_params}


def _inputs(pset):
    """[64, 128, 128, 3] float32 input and target; the masked set feeds binary images (exactly 0.0 or 1.0)"""
    x = np.random.RandomState(8).rand(B_MAX, 128, 128, 3)
    x = (x < 0.5) if pset == "masked" else x
    return x.astype(np.float32), np.random.RandomState(4).rand(B_MAX, 128, 128, 3).astype(np.float32)


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


@pytest.fixture(scope="module")
def data():
    """parameter sets and inputs, built once per module.  Handles that earlier modules left in reference cycles are collected first:
    the batch-64 trainers and the float64 reference need room on the device."""
    gc.collect()
    torch.cuda.empty_cache()
    free, total = torch.cuda.mem_get_info()
    print("device memory free at module start: %.1f of %.1f GB" % (free / 2 ** 30, total / 2 ** 30))
    d = {p: (*PARAMS[p](), *_inputs(p)) for p in PARAMS}
    d["positive"] = _positive_params()
    return d


@pytest.fixture(scope="module")
def refs(data):
    """float64 references on the GPU, shared by the three trainers: (params, B, bootstrap ratio, target) -> results"""
    cache = {}

    def get(pset, B, bootstrap, probe=None):
        key = (pset, B, bootstrap, probe)
        if key in cache:
            return cache[key]
        if bootstrap != 1 and probe is None:
            get(pset, B, 1)                           # the batch's ReLU margin is asserted with the fp16 bounds, for every trainer
        ep, dp, x, y = data[pset]
        x, y = x[:B], (y[:B] if probe is None else _probe_target(get, data, probe))
        torch.cuda.reset_peak_memory_stats()
        loss, rec, g = O.ae_forward_loss(x, y, ep, dp, dtype=torch.float64, bootstrap_ratio=bootstrap, with_grads=True, device="cuda")
        if B == B_MAX and probe is None:
            print("float64 reference, %s, B=%d, bootstrap %d: peak device memory %.2f GB"
                  % (pset, B, bootstrap, torch.cuda.max_memory_allocated() / 2 ** 30))
        r = dict(loss=loss, rec=rec, grads=g)
        if bootstrap == 1:                            # the fp16 trainer's bounds on this batch
            A = _analyse(x, y, ep, dp, 1)
            margin = O.relu_margin(x, ep, dp, device="cuda")
            assert margin > 2 * A["relu_need"], (pset, B, probe, margin, A["relu_need"])
            r.update(bounds=_grad_bounds(A), loss_bound=A["loss_bound"])
            del A
        cache[key] = r
        torch.cuda.empty_cache()
        return r

    yield get
    cache.clear()


def _probe_target(get, data, p):
    """the clear set's float64 reconstruction (rounded to fp32) as target of every image but p, which keeps its random target: the
    loss gradient of the batch is image p's.  (Not 1 - reconstruction: the clear set's reconstruction is nearly constant over the
    pixels, so that target would put thousands of squared errors within fp32 rounding of the top-k threshold, and which of them a
    trainer selects would be decided by rounding.)"""
    rec = get("clear", B_MAX, 1)["rec"]
    y = rec.astype(np.float32)
    y[p] = data["clear"][3][p]
    return y


def _free(enc, dec, top):
    torch.cuda.synchronize()
    top.close()
    enc.close()
    dec.close()


@pytest.fixture(scope="module", params=list(KINDS))
def trainer(request, data):
    """one trainer of each kind at max_batch 64, freed before the next is built"""
    gemm, handles, bootstrap = KINDS[request.param]
    ep, dp = data["clear"][:2]
    enc, dec, top = _pair(gemm, B_MAX, ep, dp, bootstrap, handles)
    yield request.param, enc, dec, top
    _free(enc, dec, top)
    torch.cuda.empty_cache()


def _step(sess, enc, dec, top, ep, dp, x, y):
    enc.load_weights(ep)
    dec.load_weights(dp)
    loss = float(top.step_device(_dev(x), _dev(y), update=False))
    return loss, top.gradients(sess.device)


def _check(kind, loss, grads, r, tag):
    tag = "%s trainer, %s" % (kind, tag)
    if kind == "fp16":
        bound, bounds = 2 * r["loss_bound"], r["bounds"]
        print("%s: gradient bounds %.2e .. %.2e, below 1 for %s" % (tag, min(bounds.values()), max(bounds.values()),
                                                                  sorted(k for k, v in bounds.items() if v < 1)))
    else:
        bound, bounds = 2e-6 * abs(r["loss"]), {k: REL for k in r["grads"]}
    print("%s: |loss - loss64| = %.3e, bound %.3e" % (tag, abs(loss - r["loss"]), bound))
    assert abs(loss - r["loss"]) <= bound, (tag, loss, r["loss"])
    assert sorted(grads) == sorted(r["grads"]) and len(grads) == 20
    _check_grads(grads, r["grads"], bounds, tag)


@pytest.mark.parametrize("B", [B_MAX, B_RAGGED])
@pytest.mark.parametrize("pset", ["clear", "masked"])
def test_loss_and_gradients_match_float64(sess, trainer, data, refs, pset, B):
    """The loss and all 20 gradients of one forward/backward at batch 64, and at batch 37 on the same max_batch-64 trainer.  With the
    masked set, conv1's activation (exact by construction) is also compared bit for bit with the float64 one."""
    kind, enc, dec, top = trainer
    ep, dp, x, y = data[pset]
    x, y = x[:B], y[:B]
    bootstrap = KINDS[kind][2]
    r = refs(pset, B, bootstrap)
    loss, grads = _step(sess, enc, dec, top, ep, dp, x, y)
    _check(kind, loss, grads, r, "%s, B=%d" % (pset, B))
    if pset == "masked" and kind != "fp16":           # the fp16 trainer runs private plans; the handles keep no activation
        k, b = (torch.from_numpy(ep["conv2d/" + n]).to("cuda", torch.float64) for n in ("kernel", "bias"))
        want = torch.relu(O.conv2d_same(_dev(x).double(), k, b, 2, None)).float()
        got = enc.activation_device(0, sess.device)
        assert got.shape == want.shape and torch.equal(got, want), float((got - want).abs().max())


@pytest.mark.parametrize("p", PROBES)
def test_each_image_position_counts_once(sess, trainer, data, refs, p):
    """Only image p is far from its target; every other image's target is its own float64 reconstruction.  An image's contribution
    dropped, moved to another position or counted twice gives a relative gradient error of order 1, far outside the fp32 and split
    trainers' bound.  The fp16 trainer's bound on such a batch exceeds 1 (the forward rounding of the 63 quiet images enters its loss
    gradient), so it runs the differential probe below instead."""
    kind, enc, dec, top = trainer
    if kind == "fp16":
        _fp16_position_probe(sess, enc, dec, top, data, p)
        return
    ep, dp, x, _ = data["clear"]
    bootstrap = KINDS[kind][2]
    r = refs("clear", B_MAX, bootstrap, p)
    y = _probe_target(refs, data, p)
    loss, grads = _step(sess, enc, dec, top, ep, dp, x, y)
    _check(kind, loss, grads, r, "loud image %d of 64" % p)


def _fp16_position_probe(sess, enc, dec, top, data, p):
    """The fp16 trainer's gradient of a batch whose image p has target 0, minus its gradient of the same batch with image p's target
    at its float64 reconstruction, times 64: image p's own gradient.  The other 63 images keep their reconstruction as target in both
    steps; their forward is the same bits in both, and their loss gradients differ only by the power-of-two G scale, so they cancel.
    The difference is compared with the float64 difference of image p alone at batch 1, under twice the batch-1 rounding-model bound:
    the errors of the two steps add, and the second step's loss-gradient perturbation (sigmoid' times the reconstruction's error) is
    part of the first's.  The positive parameter set keeps that bound below 0.25, so a dropped or duplicated contribution (error 1)
    fails.  Image p is the only bright one (the others are scaled by 0.1), so its contribution moved to another image's activations
    changes the conv1 gradient by most of its size."""
    ep, dp = data["positive"]
    u = data["clear"][2]                                   # uniform [0, 1) images
    x = (0.1 * u).astype(np.float32)
    x[p] = u[p]
    rec = O.ae_forward_loss(x, x, ep, dp, dtype=torch.float64, bootstrap_ratio=1, device="cuda")[1]
    y_quiet = rec.astype(np.float32)
    y_loud = y_quiet.copy()
    y_loud[p] = 0.0
    xp = x[p:p + 1]
    A = _analyse(xp, y_loud[p:p + 1], ep, dp, 1)
    margin = O.relu_margin(xp, ep, dp, device="cuda")
    assert margin > 2 * A["relu_need"], (p, margin, A["relu_need"])
    bounds = {k: 2 * v for k, v in _grad_bounds(A).items()}
    del A
    assert max(bounds.values()) < 0.5, bounds              # an error of order 1 cannot pass
    _, _, g_loud = O.ae_forward_loss(xp, y_loud[p:p + 1], ep, dp, dtype=torch.float64, bootstrap_ratio=1, with_grads=True,
                                     device="cuda")
    _, _, g_quiet = O.ae_forward_loss(xp, y_quiet[p:p + 1], ep, dp, dtype=torch.float64, bootstrap_ratio=1, with_grads=True,
                                      device="cuda")
    torch.cuda.empty_cache()
    want = {k: g_loud[k] - g_quiet[k] for k in g_loud}
    _, g1 = _step(sess, enc, dec, top, ep, dp, x, y_loud)
    _, g0 = _step(sess, enc, dec, top, ep, dp, x, y_quiet)
    got = {k: B_MAX * (g1[k].astype(np.float64) - g0[k]) for k in g1}
    print("fp16 trainer, image %d of 64 by difference: bounds %.3f .. %.3f" % (p, min(bounds.values()), max(bounds.values())))
    _check_grads(got, want, bounds, "fp16 trainer, image %d of 64 by difference" % p)


def test_history_and_max_batch_do_not_change_a_step(sess, trainer, data, refs):
    """A batch-37 step after a batch-64 step whose images 37..63 are far from their targets (large gradients in every buffer row
    that the batch-37 step does not own) is bit-identical, loss and gradients, to the same step on a fresh max_batch-64 trainer and
    on a trainer created with max_batch 37.  The trainers use no float atomics, so nothing but the stale rows could change a bit."""
    kind, enc, dec, top = trainer
    gemm, handles, bootstrap = KINDS[kind]
    ep, dp, x, y = data["clear"]
    rec = refs("clear", B_MAX, 1)["rec"]
    y_far = y.copy()
    y_far[B_RAGGED:] = (rec[B_RAGGED:] < 0.5).astype(np.float32)
    enc.load_weights(ep)
    dec.load_weights(dp)
    top.step_device(_dev(x), _dev(y_far), update=False)
    runs = [_step(sess, enc, dec, top, ep, dp, x[:B_RAGGED], y[:B_RAGGED])]
    for max_batch in (B_MAX, B_RAGGED):
        fresh = _pair(gemm, max_batch, ep, dp, bootstrap, handles)
        try:
            runs.append(_step(sess, *fresh, ep, dp, x[:B_RAGGED], y[:B_RAGGED]))
        finally:
            _free(*fresh)
    for what, (loss, grads) in zip(("fresh max_batch 64", "max_batch 37"), runs[1:]):
        assert loss == runs[0][0], (kind, what, loss, runs[0][0])
        diff = [k for k in grads if not np.array_equal(grads[k], runs[0][1][k])]
        assert not diff, (kind, what, diff)


@pytest.mark.parametrize("handles", [FP32, SPLIT])
def test_latent_terms_at_batch_64(sess, data, handles):
    """VARIATIONAL 0.1 and NORM_REGULARIZE 0.5 at batch 64 (each latent-kernel warp takes four rows): the total loss and all 22
    gradients against the float64 oracle, with the bounds of tests/test_gpu_h."""
    ep, dp, x, y = data["clear"]
    head = _head(0.05)
    enc, dec, top = _build(handles, None, B_MAX, ep, dp, head, 0.1, 0.5)
    eps = 0.7
    try:
        loss = float(top.step_device(_dev(x), _dev(y), update=False, eps=eps))
        grads = top.gradients(sess.device)
    finally:
        _free(enc, dec, top)
    loss64, terms, g64 = LO.vae_forward_loss(x, y, ep, dp, head=head, variational=0.1, norm_regularize=0.5, eps=eps,
                                             dtype=torch.float64, with_grads=True, device="cuda")
    # the decoder reads the sampled z: no ReLU unit of that forward may sit within rounding of zero (the split trainer keeps 22
    # significant bits of pre-activations of order one, so 1e-4 is far outside it)
    margin = O.relu_margin(x, ep, dp, device="cuda", latent=terms["sampled_z"])
    torch.cuda.empty_cache()
    assert margin > 1e-4, margin
    assert abs(loss - loss64) < 4e-6 * max(1.0, abs(loss64)), (loss, loss64)
    assert sorted(grads) == sorted(g64) and len(g64) == 22
    _check_grads(grads, g64, {k: REL for k in g64}, "latent terms, precision %d, B=64" % handles)


def test_bootstrapped_l2_ties_at_production_size(sess):
    """Decoder.loss_device at B = 64, 128x128x3 and ratio 4 (48 elements per thread of the tie ranking): squared errors on a few
    hundred exact levels, so that many elements tie at the threshold across thread ranges.  The selected set equals a stable float64
    top-k (lowest index first among ties, as tf.nn.top_k) element for element; the loss and the gradient on that set match."""
    from augmentedautoencoder_b200.ae.decoder import Decoder
    B, numel, ratio = B_MAX, 128 * 128 * 3, 4
    k = numel // ratio
    rng = np.random.RandomState(21)
    q = rng.randint(1, 301, (B, numel))                    # |x - t| = q 2^-10 and its square are exact in fp32
    t = np.full((B, numel), 0.5)
    x = t + np.where(rng.rand(B, numel) < 0.5, -1.0, 1.0) * q * 2.0 ** -10
    loss, grad = Decoder.loss_device(_dev(x.astype(np.float32).reshape(B, 128, 128, 3)),
                                     _dev(t.astype(np.float32).reshape(B, 128, 128, 3)), ratio, with_grad=True)
    grad = grad.reshape(B, numel).cpu().numpy()
    l2 = (x - t) ** 2
    order = np.argsort(-l2, axis=1, kind="stable")[:, :k]
    want = np.zeros((B, numel), bool)
    np.put_along_axis(want, order, True, axis=1)
    thr = np.take_along_axis(l2, order[:, -1:], axis=1)
    at_thr = l2 == thr
    assert np.all(np.sum(at_thr & want, axis=1) > 0) and np.all(np.sum(at_thr & ~want, axis=1) > 0)   # every cut splits a tie
    got = grad != 0
    bad_rows = np.nonzero(np.any(got != want, axis=1))[0]
    assert not len(bad_rows), ("selection differs in rows", bad_rows[:8])
    loss64 = float(np.take_along_axis(l2, order, axis=1).mean())
    assert abs(float(loss) - loss64) < 1e-6, (float(loss), loss64)
    g64 = 2.0 * (x - t) / (B * k)
    assert np.allclose(grad[want], g64[want], rtol=1e-6, atol=0.0)
