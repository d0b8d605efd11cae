"""Handle lifetimes: creating and destroying a handle gives all of its device memory back, and so does a creator that is refused
after it has allocated part of its object.

Every case creates and destroys its object ROUNDS times, after one warm-up round that loads the kernels the creator and the calls
in the round set up, and compares the device's free memory (cudaMemGetInfo) before and after the loop.  The lazily allocated
buffers are grown inside each round: the tensor-core encoder's split-K partials and activation view, the codebook's cosine rows
and the trainer's latent-term sums.  A refused aae_decoder_enable_mask_head leaves the decoder forwarding bit for bit as before.

No case provokes an out-of-memory error, because the device is shared: the out-of-memory paths of the creators free what they
allocated through the same owners as the refusals below."""
import ctypes as C

import numpy as np
import pytest
import torch

from augmentedautoencoder_b200 import _lib
from oracle import aae_oracle as O

pytestmark = pytest.mark.gpu

FP32, SPLIT, FP16 = _lib.PREC_FP32_SIMT, _lib.PREC_TC_SPLIT, _lib.PREC_TC_FP16
UNSUPPORTED = -3
ROUNDS = 10
# Free memory may differ by the driver's bookkeeping after a loop; a leaked plan or trainer costs far more (tens of MB per
# round).  On an H100 80GB HBM3 every case below came back within TOLERANCE (largest difference 0 bytes).
TOLERANCE = 2 << 20
N_ROWS = 72 * 36
OPTIMIZERS = {0: _lib.OPT_GRADIENT_DESCENT, 1: _lib.OPT_ADAGRAD, 2: _lib.OPT_RMSPROP}   # slots -> rule (non-zero slot fills)


def lib():
    return _lib.lib()


def cfg(precision, hw=128, c=3, max_batch=8):
    return _lib.make_cfg(hw, hw, c, O.NUM_FILTER, O.STRIDES, O.KSIZE, O.LATENT, max_batch, precision)


def create(fn, *args):
    h = C.c_void_p()
    _lib.check(fn(*args, C.byref(h)), fn.__name__)
    return h


def encoder(precision, sigma=False, **kw):
    h = create(lib().aae_encoder_create, 0, C.byref(cfg(precision, **kw)))
    if sigma:
        _lib.check(lib().aae_encoder_enable_sigma_head(h), "enable_sigma_head")
    return h


def decoder(precision, mask=False, **kw):
    h = create(lib().aae_decoder_create, 0, C.byref(cfg(precision, **kw)))
    if mask:
        _lib.check(lib().aae_decoder_enable_mask_head(h), "enable_mask_head")
    return h


def optimizer(slots):
    o = _lib.Optimizer()
    o.kind, o.learning_rate = OPTIMIZERS[slots], 1e-3
    o.hp[0], o.hp[1], o.hp[2] = 0.1, 0.9, 1e-7
    return o


def free_bytes():
    torch.cuda.synchronize()
    return torch.cuda.mem_get_info()[0]


def assert_gives_back(round_, record_property):
    """round_() creates, uses and destroys one object"""
    round_()
    before = free_bytes()
    for _ in range(ROUNDS):
        round_()
    lost = before - free_bytes()
    record_property("device_bytes_not_given_back", lost)
    assert lost <= TOLERANCE, ("device memory not given back", lost)


@pytest.fixture(scope="module")
def inputs():
    torch.cuda.set_device(0)
    g = torch.Generator().manual_seed(5)
    return {"crops": torch.randint(0, 256, (8, 128, 128, 3), dtype=torch.uint8, generator=g).cuda(),
            "z": torch.randn(8, O.LATENT, generator=g).cuda(),
            "scores": torch.empty(8, 9, device="cuda"), "idx": torch.empty(8, 9, dtype=torch.int32, device="cuda"),
            "E": O.make_codebook(7, n=N_ROWS, num_cyclo=36).astype(np.float32)}


@pytest.mark.parametrize("sigma", [False, True])
@pytest.mark.parametrize("precision", [FP32, SPLIT, FP16])
def test_encoder_gives_its_memory_back(inputs, precision, sigma, record_property):
    z = torch.empty(8, O.LATENT, device="cuda")

    def round_():
        h = encoder(precision, sigma)
        # batch 1 grows the tensor-core plan's split-K partials; the activation view grows its fp32 copy
        _lib.check(lib().aae_encoder_forward_u8(h, _lib.ptr(inputs["crops"]), 1, _lib.ptr(z), None), "forward")
        p, n = C.c_void_p(), C.c_int64()
        _lib.check(lib().aae_encoder_activation(h, 1, C.byref(p), C.byref(n)), "activation")
        _lib.check(lib().aae_encoder_destroy(h), "destroy")
    assert_gives_back(round_, record_property)


@pytest.mark.parametrize("precision", [FP32, SPLIT, FP16])
def test_codebook_gives_its_memory_back(inputs, precision, record_property):
    E = inputs["E"]

    def round_():
        h = create(lib().aae_codebook_create, 0, _lib.ptr(E), N_ROWS, O.LATENT, 36, 0, 8, precision)
        # k = 9 is past the fused tensor-core kernel on every precision: the cosine rows appear on first use
        _lib.check(lib().aae_codebook_match(h, _lib.ptr(inputs["z"]), 8, 9, 0, _lib.ptr(inputs["scores"]), _lib.ptr(inputs["idx"]), None),
                   "match")
        _lib.check(lib().aae_codebook_destroy(h), "destroy")
    assert_gives_back(round_, record_property)


@pytest.mark.parametrize("mask", [False, True])
@pytest.mark.parametrize("precision", [FP32, SPLIT])
def test_decoder_gives_its_memory_back(precision, mask, record_property):
    assert_gives_back(lambda: _lib.check(lib().aae_decoder_destroy(decoder(precision, mask)), "destroy"), record_property)


@pytest.mark.parametrize("slots", [0, 1, 2])
@pytest.mark.parametrize("heads", [False, True])
@pytest.mark.parametrize("gemm", [FP32, SPLIT, FP16])
def test_trainer_gives_its_memory_back(gemm, heads, slots, record_property):
    handles = FP32 if gemm == FP32 else SPLIT
    enc, dec = encoder(handles, sigma=heads), decoder(handles, mask=heads)
    o = optimizer(slots)

    def round_():
        h = create(lib().aae_trainer_create_opt, enc, dec, 4, C.byref(o), gemm)
        _lib.check(lib().aae_trainer_set_latent_terms(h, 0.0, 0.1), "latent terms")   # allocates the term sums
        _lib.check(lib().aae_trainer_destroy(h), "destroy")
    try:
        assert_gives_back(round_, record_property)
    finally:
        lib().aae_decoder_destroy(dec)
        lib().aae_encoder_destroy(enc)


def test_refused_tensor_core_decoder_gives_its_memory_back(record_property):
    """4 output channels: the plan is refused at its output layer, after the masters and the plan's other layers exist"""
    def round_():
        h = C.c_void_p()
        assert lib().aae_decoder_create(0, C.byref(cfg(SPLIT, c=4)), C.byref(h)) == UNSUPPORTED and not h.value
        assert b"at most 3" in lib().aae_last_error_string()
    assert_gives_back(round_, record_property)


def test_refused_fp32_trainer_gives_its_memory_back(record_property):
    """mask head over a sub-pixel output conv (4 channels): refused after the gradients and optimizer slots exist"""
    enc, dec = encoder(FP32, hw=64, c=4), decoder(FP32, mask=True, hw=64, c=4)
    o = optimizer(2)

    def round_():
        h = C.c_void_p()
        assert lib().aae_trainer_create_opt(enc, dec, 4, C.byref(o), FP32, C.byref(h)) == UNSUPPORTED and not h.value
        assert b"at most 3 channels" in lib().aae_last_error_string()
    try:
        assert_gives_back(round_, record_property)
    finally:
        lib().aae_decoder_destroy(dec)
        lib().aae_encoder_destroy(enc)


@pytest.mark.parametrize("precision", [FP32, SPLIT])
def test_refused_mask_head_leaves_the_decoder_as_it_was(inputs, precision):
    rng = np.random.RandomState(11)
    enc, dec = encoder(precision), decoder(precision)
    nf = list(reversed(O.NUM_FILTER)) + [3]
    h0 = 128 >> len(O.NUM_FILTER)
    shapes = [((O.LATENT, h0 * h0 * nf[0]), h0 * h0 * nf[0])] + [((5, 5, nf[l - 1], nf[l]), nf[l]) for l in range(1, len(nf))]
    for layer, (k, b) in enumerate(shapes):
        kernel = (rng.randn(*k) * 0.02).astype(np.float32)
        bias = (rng.randn(b) * 0.02).astype(np.float32)
        _lib.check(lib().aae_decoder_set_weights(dec, layer, _lib.ptr(kernel), _lib.ptr(bias), None), "set_weights")
    z = inputs["z"]

    def forward():
        x = torch.empty(8, 128, 128, 3, device="cuda")
        _lib.check(lib().aae_decoder_forward(dec, _lib.ptr(z), 8, _lib.ptr(x), None), "forward")
        torch.cuda.synchronize()
        return x
    try:
        x0 = forward()
        tr = create(lib().aae_trainer_create_opt, enc, dec, 4, C.byref(optimizer(2)), precision)
        assert lib().aae_decoder_enable_mask_head(dec) == UNSUPPORTED and b"trainer" in lib().aae_last_error_string()
        x1 = forward()
        mask = torch.empty(8, 128, 128, device="cuda")
        assert lib().aae_decoder_forward_mask(dec, _lib.ptr(z), 8, _lib.ptr(x1), _lib.ptr(mask), None) == UNSUPPORTED
        _lib.check(lib().aae_trainer_destroy(tr), "destroy trainer")
        assert torch.equal(x0, x1) and torch.equal(x0, forward())
        _lib.check(lib().aae_decoder_enable_mask_head(dec), "enable_mask_head once the trainer is gone")
    finally:
        lib().aae_decoder_destroy(dec)
        lib().aae_encoder_destroy(enc)
