"""GPU tests of AUXILIARY_MASK: the decoder's mask head (auto_pose/ae/decoder.py:68-75) and the mask loss (decoder.py:134-142) in
the decoder forward and in the fused training step of the fp32 CUDA-core, split tensor-core and single-pass fp16 trainers, against
the float64 oracle (oracle/mask_oracle.py)."""
import configparser
import gc

import numpy as np
import pytest
import torch

from oracle import aae_oracle as O
from oracle import mask_oracle as MO
from tests.test_gpu_a_parity import sess  # noqa: F401
from tests.test_gpu_e_fp16_train import _analyse, _clear_margin_params, _grad_bounds

pytestmark = pytest.mark.gpu

FP32, SPLIT, FP16 = 0, 1, 2
_OPEN = []      # (train op, encoder, decoder) built by a test: its trainers and handles are freed when the test ends


def _track(top, *modules):
    _OPEN.append((top, modules))
    return top


@pytest.fixture(autouse=True)
def _device_memory_free():
    """The tests build max_batch-64 handles and trainers with cudaMalloc: each test frees its own trainers (before the handles they
    run on) and handles, and torch's cached blocks (the float64 oracle's) are released around it."""
    gc.collect()
    torch.cuda.empty_cache()
    yield
    while _OPEN:
        top, modules = _OPEN.pop()
        if top is not None:
            top.close()
        for m in modules:
            m.close()
    gc.collect()
    torch.cuda.empty_cache()


OUT, HEAD = "conv2d_8", "conv2d_7"          # template network: the head is created before the output conv


def _head(seed=21, scale=1.0, bias=0.2):
    k, _ = MO.make_mask_head(seed, 128)
    return (scale * k).astype(np.float32), np.full(1, bias, np.float32)


def _named(dp, head):
    """decoder variables under the names of the graph with the head: the output conv moves from conv2d_7 to conv2d_8"""
    out = {("conv2d_8" + k[len("conv2d_7"):] if k.startswith("conv2d_7/") else k): v for k, v in dp.items()}
    out[HEAD + "/kernel"], out[HEAD + "/bias"] = head
    return out


def _target(seed, B):
    """random target with about 10 % background pixels (every channel 0), so m takes both values.  (With many more, the
    bootstrapped L2 selects background pixels almost only and the gradients of the weights-scaled-down test network are so
    ill-conditioned that torch's own float32 CPU evaluation is 2e-3 off float64 in dense_1.)"""
    rng = np.random.RandomState(seed)
    y = rng.rand(B, 128, 128, 3).astype(np.float32)
    y[rng.rand(B, 128, 128) < 0.1] = 0.0
    return y


def _decoder(prec, mask, B=64):
    from augmentedautoencoder_b200.ae.decoder import Decoder
    from augmentedautoencoder_b200.ae.session import placeholder
    zin = placeholder(np.float32, [None, 128])
    dec = Decoder(placeholder(np.float32, [None, 128, 128, 3]), zin, list(reversed(O.NUM_FILTER)), 5, list(reversed(O.STRIDES)), "L2", 4,
                  mask, False, max_batch=B, precision=prec)
    return zin, dec


def _build(handles, gemm, B, ep, dp, head, bootstrap=4):
    from augmentedautoencoder_b200.ae.ae import AE
    from augmentedautoencoder_b200.ae.ae_factory import TrainOp
    from augmentedautoencoder_b200.ae.decoder import Decoder
    from augmentedautoencoder_b200.ae.encoder import Encoder
    from augmentedautoencoder_b200.ae.session import placeholder
    x, y = placeholder(np.float32, [None, 128, 128, 3]), placeholder(np.float32, [None, 128, 128, 3])
    enc = Encoder(x, 128, list(O.NUM_FILTER), 5, list(O.STRIDES), False, is_training=True, max_batch=B, precision=handles)
    dec = Decoder(y, enc.z, list(reversed(O.NUM_FILTER)), 5, list(reversed(O.STRIDES)), "L2", bootstrap, True, False, is_training=True,
                  max_batch=B, precision=handles)
    enc.load_weights(ep)
    dec.load_weights(_named(dp, head))
    return enc, dec, _track(TrainOp(AE(enc, dec, 0, 0), 2e-4, precision=gemm), enc, dec)


def _rel(a, b):
    return float(np.linalg.norm(a.astype(np.float64) - b) / max(np.linalg.norm(b), 1e-300))


@pytest.mark.parametrize("prec", [FP32, SPLIT])
def test_forward_matches_oracle_and_leaves_x_unchanged(sess, prec):
    """x and the mask of one forward at batch 64 against the float64 oracle, at the decoder forward bounds of test_gpu_b_tc; x is
    bit-identical with and without the head, and a forward that does not ask for the mask launches what a decoder without the head
    launches."""
    from augmentedautoencoder_b200 import _lib
    lib = _lib.lib()
    dp = O.make_decoder_params(43, bias_scale=0.05)
    head = _head()
    z = torch.from_numpy((np.random.RandomState(7).standard_normal((64, 128)) * 2.0).astype(np.float32)).cuda()
    _, plain = _decoder(prec, False)
    plain.load_weights(dp)
    _, masked = _decoder(prec, True)
    masked.load_weights(_named(dp, head))
    _track(None, plain, masked)
    x0 = plain.decode_device(z)                   # first calls pack the weights
    x1 = masked.decode_device(z)
    counts = []
    for dec in (plain, masked):
        torch.cuda.synchronize()
        n0 = lib.aae_launch_count()
        dec.decode_device(z)
        counts.append(lib.aae_launch_count() - n0)
    x2, xm = masked.decode_device(z, with_mask=True)
    assert counts[0] == counts[1], counts
    assert torch.equal(x0, x1) and torch.equal(x0, x2)
    tp = {k: O._t(v, torch.float64, "cuda") for k, v in dp.items()}
    with torch.no_grad():
        ref, ref_m = MO.decoder_with_mask(z.double(), tp, O._t(head[0], torch.float64, "cuda"), O._t(head[1], torch.float64, "cuda"),
                                          128, O.STRIDES, 4)
    e_x, e_m = float((x2.double() - ref).abs().max()), float((xm.double() - ref_m).abs().max())
    print("precision %d: max abs error vs float64: x %.2e, mask %.2e" % (prec, e_x, e_m))
    assert xm.shape == (64, 128, 128, 1) and float(ref_m.std()) > 1e-2
    bound = 2e-6 if prec == FP32 else 5e-6
    assert e_x < bound and e_m < bound
    masked.check_range()


def _oracle(xb, yb, ep, dp, head, chunk=16):
    """float64 loss, mask and gradients of a batch, evaluated 16 samples at a time to bound the oracle's device memory: both loss
    terms are means over the samples (of the same number of terms each), so the batch's values are the chunks' weighted by size."""
    B, loss, xms, grads = xb.shape[0], 0.0, [], None
    for a in range(0, B, chunk):
        n = min(B, a + chunk) - a
        l, _, xm, g = MO.mask_forward_loss(xb[a:a + n], yb[a:a + n], ep, dp, head, dtype=torch.float64, with_grads=True, device="cuda")
        torch.cuda.empty_cache()
        loss += l * n / B
        xms.append(xm)
        grads = {k: v * (n / B) for k, v in g.items()} if grads is None else {k: grads[k] + v * (n / B) for k, v in g.items()}
    return loss, np.concatenate(xms), grads


def _check_step(sess, top, ep, dp, head, xb, yb):
    loss = float(top.step_device(torch.from_numpy(xb).cuda(), torch.from_numpy(yb).cuda(), update=False))
    loss64, xm64, g64 = _oracle(xb, yb, ep, dp, head)
    grads = top.gradients(sess.device)
    assert sorted(grads) == sorted(g64) and len(g64) == 22
    assert abs(loss - loss64) < 4e-6 * max(1.0, abs(loss64)), (loss, loss64)
    errs = {k: _rel(grads[k], g64[k]) for k in g64}
    bad = {k: e for k, e in errs.items() if not e < 3e-4}
    if bad:
        print("batch %d: relative L2 gradient errors %s" % (xb.shape[0], {k: "%.2e" % e for k, e in errs.items()}))
    assert not bad, bad
    m = MO.mask_target(yb)
    assert 0.05 < 1 - m.mean() < 0.2 and np.std(xm64) > 1e-3
    return abs(loss - loss64), max(errs.values()), errs[HEAD + "/kernel"], errs[HEAD + "/bias"]


@pytest.mark.parametrize("handles", [FP32, SPLIT])
def test_loss_and_gradients_match_float64_oracle(sess, handles):
    """The loss (bootstrapped L2 + mask loss) and all 22 gradients, the head's kernel and bias included, at batch 1, 64 and a ragged
    37 on one max_batch-64 trainer pair, against the float64 oracle: every tensor within 3e-4 relative L2.  Weights keep every ReLU
    unit far from zero, so any difference is rounding."""
    ep, dp = _clear_margin_params()
    head = _head(scale=0.05)
    enc, dec, top = _build(handles, None, 64, ep, dp, head)
    for B in (1, 64, 37):
        xb = np.random.RandomState(8 + B).rand(B, 128, 128, 3).astype(np.float32)
        yb = _target(4 + B, B)
        dl, worst, hk, hb = _check_step(sess, top, ep, dp, head, xb, yb)
        print("precision %d, batch %d: |loss - loss64| %.2e, worst relative L2 gradient error %.2e (head kernel %.2e, bias %.2e)"
              % (handles, B, dl, worst, hk, hb))
        torch.cuda.empty_cache()


def test_fp16_trainer_meets_the_rounding_bound(sess):
    """The single-pass trainer with the head, batch 1, no bootstrapping: every gradient within twice the rounding-model bound of
    test_gpu_e for the plain network (the joined output layer carries a second loss gradient through the same GEMMs), the head's
    within the output conv's bound; the loss within twice the plain bound plus the mask loss's share of the forward error."""
    ep, dp = _clear_margin_params()
    head = _head(scale=0.05)
    xb = np.random.RandomState(8).rand(1, 128, 128, 3).astype(np.float32)
    yb = _target(4, 1)
    A = _analyse(xb, yb, ep, dp, 1)
    assert O.relu_margin(xb, ep, dp) > 2 * A["relu_need"]
    plain = _grad_bounds(A)
    bounds = {k: 2 * v for k, v in plain.items() if not k.startswith("conv2d_7/")}
    for part in ("kernel", "bias"):
        bounds[OUT + "/" + part] = bounds[HEAD + "/" + part] = 2 * plain["conv2d_7/" + part]
    enc, dec, top = _build(SPLIT, FP16, 2, ep, dp, head, bootstrap=1)
    loss = float(top.step_device(torch.from_numpy(xb).cuda(), torch.from_numpy(yb).cuda(), update=False))
    loss64, _, xm64, g64 = MO.mask_forward_loss(xb, yb, ep, dp, head, dtype=torch.float64, bootstrap_ratio=1, with_grads=True, device="cuda")
    xm = xm64.astype(np.float64)
    d_xm = 0.25 * A["fwd_rel"] * float(np.abs(np.log(xm / (1 - xm))).max())
    mask_bound = float(np.mean(2 * np.abs(xm - MO.mask_target(yb)) * d_xm + d_xm ** 2))
    bound = 2 * (A["loss_bound"] + mask_bound)
    assert abs(loss - loss64) <= bound, (loss, loss64, bound)
    grads = top.gradients(sess.device)
    assert sorted(grads) == sorted(g64) == sorted(bounds)
    over = {k: (_rel(grads[k], g64[k]), bounds[k]) for k in g64 if not _rel(grads[k], g64[k]) <= bounds[k]}
    assert not over, over
    print("fp16 trainer with the mask head: |loss - loss64| %.2e (bound %.2e), largest share of a gradient bound %.3f"
          % (abs(loss - loss64), bound, max(_rel(grads[k], g64[k]) / bounds[k] for k in g64)))


def test_split_trainer_tracks_the_fp32_trainer(sess):
    """Five Adam steps at batch 3: the split trainer's loss trajectory follows the fp32 trainer's (the tolerance of the plain and
    latent-term tests), the loss falls, and the head's masters move."""
    ep, dp = O.make_encoder_params(42, bias_scale=0.02), O.make_decoder_params(43, bias_scale=0.02)
    head = _head()
    xb = torch.from_numpy(np.random.RandomState(11).rand(3, 128, 128, 3).astype(np.float32)).cuda()
    yb = torch.from_numpy(_target(12, 3)).cuda()
    traj = {}
    for prec in (FP32, SPLIT):
        enc, dec, top = _build(prec, None, 4, ep, dp, head)
        traj[prec] = [float(top.step_device(xb, yb, update=True)) for _ in range(5)]
        w = dec.get_weights()
        assert np.abs(w[HEAD + "/kernel"] - head[0]).max() > 1e-4 and np.abs(w[HEAD + "/bias"] - head[1]).max() > 1e-4
        del enc, dec, top
    print("loss trajectories: fp32 %s, split %s" % (traj[FP32], traj[SPLIT]))
    assert traj[FP32][-1] < traj[FP32][0]
    assert np.max(np.abs(np.array(traj[FP32]) - np.array(traj[SPLIT]))) < 2e-4, traj


def test_checkpoint_holds_the_head_and_resumes_bit_identically(sess, tmp_path):
    """Saver(..., train_op=...) writes the head (conv2d_7), the output conv (conv2d_8) and their Adam slots in .npz and TF-bundle form;
    a fresh pair restored from either continues bit-identically, and two identical steps give bit-identical losses."""
    from augmentedautoencoder_b200.ae import ae_factory as F
    from augmentedautoencoder_b200.ae.tf_checkpoint import read_tf_checkpoint
    ep, dp = O.make_encoder_params(42, bias_scale=0.02), O.make_decoder_params(43, bias_scale=0.02)
    xb = torch.from_numpy(np.random.RandomState(11).rand(3, 128, 128, 3).astype(np.float32)).cuda()
    yb = torch.from_numpy(_target(12, 3)).cuda()
    enc, dec, top = _build(SPLIT, None, 4, ep, dp, _head())
    a, b = float(top.step_device(xb, yb, update=False)), float(top.step_device(xb, yb, update=False))
    assert a == b
    for _ in range(2):
        top.step_device(xb, yb)
    saver = F.Saver([enc, dec], global_step=top._ae.global_step, train_op=top)
    paths = [saver.save(sess, str(tmp_path / "npz" / "chkpt"), global_step=2), saver.save_tf(sess, str(tmp_path / "tf" / "chkpt"), global_step=2)]
    want = [float(top.step_device(xb, yb)) for _ in range(2)]
    w_want = dec.get_weights()
    for path in paths:
        stored = dict(np.load(path)) if path.endswith(".npz") else read_tf_checkpoint(path)
        assert stored[HEAD + "/kernel"].shape == (5, 5, 128, 1) and stored[OUT + "/kernel"].shape == (5, 5, 128, 3)
        for k in (HEAD + "/kernel", HEAD + "/bias", OUT + "/kernel", OUT + "/bias"):
            assert k + "/Adam" in stored and k + "/Adam_1" in stored, k
        assert np.abs(stored[HEAD + "/kernel/Adam"]).max() > 0
        enc2, dec2, top2 = _build(SPLIT, None, 4, ep, dp, _head(seed=3))
        F.Saver([enc2, dec2], global_step=top2._ae.global_step, train_op=top2).restore(sess, path)
        got = [float(top2.step_device(xb, yb)) for _ in range(2)]
        assert got == want, (path, got, want)
        w_got = dec2.get_weights()
        assert all(np.array_equal(w_got[k], w_want[k]) for k in w_want), path


def _cfg():
    c = configparser.ConfigParser()
    c.read_dict({"Network": {"LATENT_SPACE_SIZE": "128", "NUM_FILTER": "[128, 256, 512, 512]", "KERNEL_SIZE_ENCODER": "5",
                             "KERNEL_SIZE_DECODER": "5", "STRIDES": "[2, 2, 2, 2]", "BATCH_NORMALIZATION": "False", "LOSS": "L2",
                             "BOOTSTRAP_RATIO": "4", "VARIATIONAL": "0", "AUXILIARY_MASK": "True", "NORM_REGULARIZE": "0"},
                 "Training": {"BATCH_SIZE": "2", "LEARNING_RATE": "2e-4", "OPTIMIZER": "Adam"}})
    return c


def test_session_fetches_and_the_train_op_match_the_oracle(sess):
    """A graph built by build_* from a cfg with AUXILIARY_MASK: Session.run of x, decoder._xmask and reconstr_loss against the
    oracle (uint8 target as the reference feeds it, divided by 255), and sess.run(train_op) returns the same loss."""
    from augmentedautoencoder_b200.ae import ae_factory as F
    from augmentedautoencoder_b200.ae import session as S
    args = _cfg()
    x, y = S.placeholder(np.float32, [None, 128, 128, 3]), S.placeholder(np.float32, [None, 128, 128, 3])
    enc = F.build_encoder(x, args, is_training=True)
    dec = F.build_decoder(y, enc, args, is_training=True)
    ae = F.build_ae(enc, dec, args)
    top = _track(F.build_train_op(ae, args), enc, dec)
    assert dec.variable_names[-4:] == ["conv2d_8/kernel", "conv2d_8/bias", "conv2d_7/kernel", "conv2d_7/bias"]
    ep, dp = O.make_encoder_params(42, bias_scale=0.02), O.make_decoder_params(43, bias_scale=0.02)
    head = _head()
    enc.load_weights(ep)
    dec.load_weights(_named(dp, head))
    xb = np.random.RandomState(8).rand(2, 128, 128, 3).astype(np.float32)
    yu8 = (_target(4, 2) * 255).astype(np.uint8)
    yb = yu8.astype(np.float32) / np.float32(255.0)
    rec, xm, rl = sess.run([dec.x, dec._xmask, dec.reconstr_loss], {x: xb, y: yu8})
    loss64, rec64, xm64, _ = MO.mask_forward_loss(xb, yb, ep, dp, head, dtype=torch.float64, device="cuda")
    assert xm.shape == (2, 128, 128, 1)
    assert np.max(np.abs(rec - rec64)) < 5e-6 and np.max(np.abs(xm - xm64)) < 5e-6
    assert abs(float(rl) - loss64) < 4e-6 * max(1.0, abs(loss64)), (rl, loss64)
    loss_t = float(sess.run(top, {x: xb, y: yb}))
    assert abs(loss_t - loss64) < 4e-6 * max(1.0, abs(loss64)), (loss_t, loss64)
    assert int(ae.global_step.value()) == 1


def test_refusals_leave_the_process_healthy(sess):
    """The head cannot be added under a live trainer; forward_mask and the head's layer without a head are refused; the handles keep
    working."""
    from augmentedautoencoder_b200 import _lib
    lib = _lib.lib()
    ep, dp = O.make_encoder_params(42, bias_scale=0.02), O.make_decoder_params(43, bias_scale=0.02)
    zin, dec = _decoder(SPLIT, False, B=4)
    _track(None, dec)
    dec.load_weights(dp)
    dh = dec.handle(sess.device)
    z = torch.zeros((2, 128), device="cuda")
    x, m = torch.empty((2, 128, 128, 3), device="cuda"), torch.empty((2, 128, 128, 1), device="cuda")
    assert lib.aae_decoder_forward_mask(dh, _lib.ptr(z), 2, _lib.ptr(x), _lib.ptr(m), None) == -3
    k = np.zeros((5, 5, 128, 1), np.float32)
    assert lib.aae_decoder_set_weights(dh, 5, _lib.ptr(k), None, None) == -1
    enc, dec2, top = _build(SPLIT, None, 2, ep, dp, _head())
    xb = torch.from_numpy(np.random.RandomState(8).rand(2, 128, 128, 3).astype(np.float32)).cuda()
    yb = torch.from_numpy(_target(4, 2)).cuda()
    first = top.step_device(xb, yb, update=False).item()
    from augmentedautoencoder_b200.ae.ae import AE
    from augmentedautoencoder_b200.ae.ae_factory import TrainOp
    _, dec3 = _decoder(SPLIT, False, B=2)
    dec3.load_weights(dp)
    top3 = _track(TrainOp(AE(enc, dec3, 0, 0), 2e-4), dec3)
    top3.trainer(sess.device)
    assert lib.aae_decoder_enable_mask_head(dec3.handle(sess.device)) == -3 and b"trainer" in lib.aae_last_error_string()
    top3.close()
    assert lib.aae_decoder_enable_mask_head(dec3.handle(sess.device)) == 0
    dec.decode_device(z)
    assert top.step_device(xb, yb, update=False).item() == first
    torch.cuda.synchronize()
