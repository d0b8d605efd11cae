"""GPU tests of the latent terms of the AE loss in the fused training step: VARIATIONAL (sigma head, sampled z, KL term) and
NORM_REGULARIZE (auto_pose/ae/encoder.py:70-100, ae.py:43-53, ae_factory.py:50-77), on the fp32 CUDA-core, split tensor-core and
single-pass fp16 trainers, against the float64 oracle."""
import configparser
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import aae_oracle as O
from oracle import latent_oracle as LO
from tests.test_gpu_a_parity import sess  # noqa: F401
from tests.test_gpu_e_fp16_train import _analyse, _clear_margin_params, _grad_bounds

pytestmark = pytest.mark.gpu

FP32, SPLIT, FP16 = 0, 1, 2
EPS = 0.7


def _head(scale, seed=9):
    rng = np.random.RandomState(seed)
    return (scale * O.glorot_uniform(rng, (32768, 128))).astype(np.float32), np.full(128, 0.5, np.float32)


def _named(dp, variational):
    """decoder variables under the variational graph's names (its dense layer is the scope's third: dense_2)"""
    return {("dense_2" + k[len("dense_1"):] if variational and k.startswith("dense_1/") else k): v for k, v in dp.items()}


def _build(handles, gemm, B, ep, dp, head, variational, norm, bootstrap=4):
    from augmentedautoencoder_b200.ae.ae import AE
    from augmentedautoencoder_b200.ae.ae_factory import TrainOp
    from augmentedautoencoder_b200.ae.decoder import Decoder
    from augmentedautoencoder_b200.ae.encoder import Encoder
    from augmentedautoencoder_b200.ae.session import placeholder
    x, y = placeholder(np.float32, [None, 128, 128, 3]), placeholder(np.float32, [None, 128, 128, 3])
    enc = Encoder(x, 128, list(O.NUM_FILTER), 5, list(O.STRIDES), False, is_training=True, max_batch=B, precision=handles)
    dec = Decoder(y, enc.sampled_z if variational else enc.z, list(reversed(O.NUM_FILTER)), 5, list(reversed(O.STRIDES)), "L2", bootstrap,
                  False, False, is_training=True, max_batch=B, precision=handles)
    enc.load_weights({**ep, "dense_1/kernel": head[0], "dense_1/bias": head[1]} if variational else ep)
    dec.load_weights(_named(dp, variational))
    return enc, dec, TrainOp(AE(enc, dec, norm, variational), 2e-4, precision=gemm)


def _rel(a, b):
    return float(np.linalg.norm(a.astype(np.float64) - b) / max(np.linalg.norm(b), 1e-300))


CASES = [(0.1, 0.0), (0.0, 0.5), (0.1, 0.5)]     # (VARIATIONAL, NORM_REGULARIZE): each term alone, then both


@pytest.mark.parametrize("variational,norm", CASES)
@pytest.mark.parametrize("handles,gemm", [(FP32, None), (SPLIT, None)])
def test_loss_and_gradients_match_float64_oracle(sess, handles, gemm, variational, norm):
    """One forward/backward with a non-zero sigma head and a fixed eps: the total loss and all 20 (22 with the head) gradients
    against the float64 oracle, in relative L2 norm as the plain step's parity tests.  The weights keep every ReLU unit far from
    zero (the sampled z moves the decoder's pre-activations, and with the plain test weights some land within split-fp16 rounding
    of zero), so any difference is rounding, not a unit on the other side of its ReLU."""
    ep, dp = _clear_margin_params()
    head = _head(0.05)
    enc, dec, top = _build(handles, gemm, 2, ep, dp, head, variational, norm)
    xb = np.random.RandomState(8).rand(1, 128, 128, 3).astype(np.float32)
    yb = np.random.RandomState(4).rand(1, 128, 128, 3).astype(np.float32)
    loss = float(top.step_device(torch.from_numpy(xb).cuda(), torch.from_numpy(yb).cuda(), update=False, eps=EPS))
    loss64, terms, g64 = LO.vae_forward_loss(xb, yb, ep, dp, head=head if variational else None, variational=variational,
                                             norm_regularize=norm, eps=EPS, dtype=torch.float64, with_grads=True)
    if variational:
        s = terms["q_sigma"]
        assert 0.1 < s.min() and s.max() < 20.0 and s.std() > 1e-2, (s.min(), s.max(), s.std())
    assert abs(loss - loss64) < 4e-6 * max(1.0, abs(loss64)), (loss, loss64)
    grads = top.gradients(sess.device)
    assert sorted(grads) == sorted(g64) and len(g64) == (22 if variational else 20)
    worst = max(_rel(grads[k], g64[k]) for k in g64)
    bad = {k: _rel(grads[k], g64[k]) for k in g64 if _rel(grads[k], g64[k]) >= 3e-4}
    assert not bad, bad
    print("precision %d, VARIATIONAL %g, NORM_REGULARIZE %g: |loss - loss64| %.2e, worst relative L2 gradient error %.2e"
          % (handles, variational, norm, abs(loss - loss64), worst))


@pytest.mark.parametrize("variational,norm", CASES)
def test_fp16_trainer_meets_the_rounding_bound(sess, variational, norm):
    """The single-pass trainer with the latent terms: every gradient within the rounding-model bound of the plain step on the same
    network (tests/test_gpu_e_fp16_train.py; the head and the latent terms add fp32 operations only), the head's within the bound of
    the encoder's dense layer, whose GEMM structure it shares.  The loss: the plain bound plus the forward rounding of z passed
    through the latent terms."""
    ep, dp = _clear_margin_params()
    head = _head(0.05)
    xb = np.random.RandomState(8).rand(1, 128, 128, 3).astype(np.float32)
    yb = np.random.RandomState(4).rand(1, 128, 128, 3).astype(np.float32)
    A = _analyse(xb, yb, ep, dp, 1)
    assert O.relu_margin(xb, ep, dp) > 2 * A["relu_need"]
    bounds = _grad_bounds(A)
    if variational:
        bounds = _named(bounds, True)
        bounds["dense_1/kernel"], bounds["dense_1/bias"] = bounds["dense/kernel"], bounds["dense/bias"]
    enc, dec, top = _build(SPLIT, FP16, 2, ep, dp, head, variational, norm, bootstrap=1)
    loss = float(top.step_device(torch.from_numpy(xb).cuda(), torch.from_numpy(yb).cuda(), update=False, eps=0.3))
    loss64, t, g64 = LO.vae_forward_loss(xb, yb, ep, dp, head=head if variational else None, variational=variational,
                                         norm_regularize=norm, eps=0.3, dtype=torch.float64, bootstrap_ratio=1, with_grads=True)
    z = t["z"]
    mag = norm * float(np.mean(np.linalg.norm(z, axis=1) + 1))
    if variational:
        s2 = t["q_sigma"] ** 2
        mag += variational * float(np.mean(0.5 * z * z + 0.5 * (s2 + 1 + np.abs(np.log(s2)))))
    bound = 2 * A["loss_bound"] + 4 * A["fwd_rel"] * mag
    assert abs(loss - loss64) <= bound, (loss, loss64, bound)
    grads = top.gradients(sess.device)
    assert sorted(grads) == sorted(g64)
    over = {k: (_rel(grads[k], g64[k]), bounds[k]) for k in g64 if not _rel(grads[k], g64[k]) <= bounds[k]}
    assert not over, over
    print("fp16 trainer, VARIATIONAL %g, NORM_REGULARIZE %g: largest share of the bound %.3f"
          % (variational, norm, max(_rel(grads[k], g64[k]) / bounds[k] for k in g64)))


@pytest.mark.parametrize("handles", [FP32, SPLIT])
def test_terms_off_change_nothing(sess, handles):
    """Both weights 0 -- never set, or set explicitly (also after a step with the terms on): the loss and the 20 gradients are
    bit-identical to the plain step and every step launches the same kernels."""
    from augmentedautoencoder_b200 import _lib
    lib = _lib.lib()
    ep, dp = O.make_encoder_params(42, bias_scale=0.02), O.make_decoder_params(43, bias_scale=0.02)
    xb = torch.from_numpy(np.random.RandomState(8).rand(2, 128, 128, 3).astype(np.float32)).cuda()
    yb = torch.from_numpy(np.random.RandomState(4).rand(2, 128, 128, 3).astype(np.float32)).cuda()
    runs = []
    for mode in ("never", "explicit", "after"):
        enc, dec, top = _build(handles, None, 2, ep, dp, None, 0.0, 0.0)
        h = top.trainer(sess.device)
        if mode != "never":
            _lib.check(lib.aae_trainer_set_latent_terms(h, 0.0, 0.5 if mode == "after" else 0.0), "set_latent_terms")
        top.step_device(xb, yb, update=False)              # the first step also packs / merges the weights
        if mode == "after":
            _lib.check(lib.aae_trainer_set_latent_terms(h, 0.0, 0.0), "set_latent_terms")
        torch.cuda.synchronize()
        n0 = lib.aae_launch_count()
        loss = top.step_device(xb, yb, update=False).item()
        runs.append((loss, lib.aae_launch_count() - n0, top.gradients(sess.device)))
    for loss, launches, grads in runs[1:]:
        assert loss == runs[0][0] and launches == runs[0][1], (loss, launches, runs[0][:2])
        assert len(grads) == 20 and all(np.array_equal(grads[k], runs[0][2][k]) for k in grads)


def test_split_trainer_tracks_the_fp32_trainer_with_both_terms(sess):
    """Five Adam steps at batch 3 with both terms on and the same eps: the split trainer's loss trajectory follows the fp32 trainer's
    (the tolerance of the plain step's test), and the head's masters move.  (With eps drawn per step the total loss is not monotone:
    each draw moves the decoder's input.)"""
    ep, dp = O.make_encoder_params(42, bias_scale=0.02), O.make_decoder_params(43, bias_scale=0.02)
    head = _head(0.5)
    xb = torch.from_numpy(np.random.RandomState(11).rand(3, 128, 128, 3).astype(np.float32)).cuda()
    yb = torch.from_numpy(np.random.RandomState(12).rand(3, 128, 128, 3).astype(np.float32)).cuda()
    traj = {}
    for prec in (FP32, SPLIT):
        enc, dec, top = _build(prec, None, 4, ep, dp, head, 0.1, 0.5)
        traj[prec] = [float(top.step_device(xb, yb, update=True, eps=0.1)) for _ in range(5)]
        w = enc.get_weights()
        assert np.abs(w["dense_1/kernel"] - head[0]).max() > 1e-4 and np.abs(w["dense_1/bias"] - head[1]).max() > 1e-4
        del enc, dec, top
    print("loss trajectories: fp32 %s, split %s" % (traj[FP32], traj[SPLIT]))
    assert np.max(np.abs(np.array(traj[FP32]) - np.array(traj[SPLIT]))) < 2e-4, traj


def test_checkpoint_holds_the_head_and_resumes_bit_identically(sess, tmp_path):
    """Saver(..., train_op=...) writes the head (dense_1), the decoder dense (dense_2) and their Adam slots in .npz and TF-bundle form;
    resuming with the same eps sequence continues bit-identically; an inference encoder (no head) restores from it strictly."""
    from augmentedautoencoder_b200.ae import ae_factory as F
    from augmentedautoencoder_b200.ae.encoder import Encoder
    from augmentedautoencoder_b200.ae.session import placeholder
    from augmentedautoencoder_b200.ae.tf_checkpoint import read_tf_checkpoint
    ep, dp = O.make_encoder_params(42, bias_scale=0.02), O.make_decoder_params(43, bias_scale=0.02)
    head = _head(0.5)
    xb = torch.from_numpy(np.random.RandomState(11).rand(3, 128, 128, 3).astype(np.float32)).cuda()
    yb = torch.from_numpy(np.random.RandomState(12).rand(3, 128, 128, 3).astype(np.float32)).cuda()
    eps = [0.4, -1.2, 0.9, 0.1]
    enc, dec, top = _build(SPLIT, None, 4, ep, dp, head, 0.1, 0.5)
    for e in eps[:2]:
        top.step_device(xb, yb, eps=e)
    saver = F.Saver([enc, dec], global_step=top._ae.global_step, train_op=top)
    paths = [saver.save(sess, str(tmp_path / "npz" / "chkpt"), global_step=2), saver.save_tf(sess, str(tmp_path / "tf" / "chkpt"), global_step=2)]
    want = [float(top.step_device(xb, yb, eps=e)) for e in eps[2:]]
    w_want = enc.get_weights()
    for path in paths:
        stored = dict(np.load(path)) if path.endswith(".npz") else read_tf_checkpoint(path)
        assert stored["dense_1/kernel"].shape == (32768, 128) and stored["dense_2/kernel"].shape == (128, 32768)
        for k in ("dense_1/kernel", "dense_1/bias", "dense_2/kernel", "dense_2/bias"):
            assert k + "/Adam" in stored and k + "/Adam_1" in stored, k
        assert np.abs(stored["dense_1/kernel/Adam"]).max() > 0
        enc2, dec2, top2 = _build(SPLIT, None, 4, ep, dp, _head(0.0), 0.1, 0.5)
        F.Saver([enc2, dec2], global_step=top2._ae.global_step, train_op=top2).restore(sess, path)
        got = [float(top2.step_device(xb, yb, eps=e)) for e in eps[2:]]
        assert got == want, (path, got, want)
        w_got = enc2.get_weights()
        assert all(np.array_equal(w_got[k], w_want[k]) for k in w_want), path
        inf = Encoder(placeholder(np.float32, [None, 128, 128, 3]), 128, list(O.NUM_FILTER), 5, list(O.STRIDES), False, max_batch=4)
        F.Saver([inf]).restore(sess, path)
        assert "dense_1/kernel" not in inf.variable_names
        assert np.array_equal(inf.get_weights()["dense/kernel"], stored["dense/kernel"])


def _cfg():
    c = configparser.ConfigParser()
    c.read_dict({"Network": {"LATENT_SPACE_SIZE": "128", "NUM_FILTER": "[128, 256, 512, 512]", "KERNEL_SIZE_ENCODER": "5",
                             "KERNEL_SIZE_DECODER": "5", "STRIDES": "[2, 2, 2, 2]", "BATCH_NORMALIZATION": "False", "LOSS": "L2",
                             "BOOTSTRAP_RATIO": "4", "VARIATIONAL": "0.1", "AUXILIARY_MASK": "False", "NORM_REGULARIZE": "0.5"},
                 "Training": {"BATCH_SIZE": "2", "LEARNING_RATE": "2e-4", "OPTIMIZER": "Adam"}})
    return c


def test_session_fetches_and_the_train_op_match_the_oracle(sess):
    """Session.run of q_sigma, sampled_z, kl_div_loss, reg_loss and ae.loss against the oracle; every fetch of one run sees the same
    eps, the next run draws another; sess.run(train_op) of a graph built by build_* from a cfg with VARIATIONAL 0.1 and
    NORM_REGULARIZE 0.5 returns the total loss."""
    from augmentedautoencoder_b200.ae import ae_factory as F
    from augmentedautoencoder_b200.ae import session as S
    args = _cfg()
    x, y = S.placeholder(np.float32, [None, 128, 128, 3]), S.placeholder(np.float32, [None, 128, 128, 3])
    enc = F.build_encoder(x, args, is_training=True)
    dec = F.build_decoder(y, enc, args, is_training=True)
    ae = F.build_ae(enc, dec, args)
    top = F.build_train_op(ae, args)
    ep, dp = O.make_encoder_params(42, bias_scale=0.02), O.make_decoder_params(43, bias_scale=0.02)
    head = _head(0.5)
    enc.load_weights({**ep, "dense_1/kernel": head[0], "dense_1/bias": head[1]})
    dec.load_weights(_named(dp, True))
    xb = np.random.RandomState(8).rand(2, 128, 128, 3).astype(np.float32)
    yb = np.random.RandomState(4).rand(2, 128, 128, 3).astype(np.float32)
    feed = {x: xb, y: yb}
    out = sess.run([enc.q_sigma, enc.sampled_z, enc.z, enc.kl_div_loss, enc.reg_loss, ae.loss], feed)
    s, sz, z, kl, reg, loss = out
    e = (sz.astype(np.float64) - z) / s
    eps = float(np.median(e))
    assert np.max(np.abs(e - eps)) < 1e-4 * max(1.0, abs(eps)), "one eps per run"
    loss64, t, _ = LO.vae_forward_loss(xb, yb, ep, dp, head=head, variational=0.1, norm_regularize=0.5, eps=float(np.float32(eps)),
                                       dtype=torch.float64)
    assert np.max(np.abs(s - t["q_sigma"])) < 1e-5 * np.abs(t["q_sigma"]).max()
    assert np.max(np.abs(z - t["z"])) < 1e-5 * np.abs(t["z"]).max()
    assert abs(float(kl) - t["kl"]) < 1e-5 * abs(t["kl"]) and abs(float(reg) - t["reg"]) < 1e-5 * max(abs(t["reg"]), 1e-3)
    assert abs(float(loss) - loss64) < 4e-6 * max(1.0, abs(loss64)), (loss, loss64)
    sz2 = sess.run(enc.sampled_z, feed)
    assert not np.array_equal(sz2, sz), "the next run draws another eps"
    # the train op: total loss with the first draw of its seeded stream
    eps0 = float(np.float32(np.random.RandomState(0).standard_normal()))
    loss_t = float(sess.run(top, feed))
    loss64, _, _ = LO.vae_forward_loss(xb, yb, ep, dp, head=head, variational=0.1, norm_regularize=0.5, eps=eps0, dtype=torch.float64)
    assert abs(loss_t - loss64) < 4e-6 * max(1.0, abs(loss64)), (loss_t, loss64)
    assert int(ae.global_step.value()) == 1


def test_refusals_leave_the_process_healthy(sess):
    """VARIATIONAL without a sigma head (AAE_ERR_UNSUPPORTED), a negative weight (AAE_ERR_INVALID_ARG), sigma_forward and the head's
    weights without a head: refused, and the trainer then runs its step as before."""
    from augmentedautoencoder_b200 import _lib
    lib = _lib.lib()
    ep, dp = O.make_encoder_params(42, bias_scale=0.02), O.make_decoder_params(43, bias_scale=0.02)
    xb = torch.from_numpy(np.random.RandomState(8).rand(2, 128, 128, 3).astype(np.float32)).cuda()
    yb = torch.from_numpy(np.random.RandomState(4).rand(2, 128, 128, 3).astype(np.float32)).cuda()
    enc, dec, top = _build(SPLIT, None, 2, ep, dp, None, 0.0, 0.0)
    first = top.step_device(xb, yb, update=False).item()
    h = top.trainer(sess.device)
    assert lib.aae_trainer_set_latent_terms(h, 0.1, 0.0) == -3 and b"sigma head" in lib.aae_last_error_string()
    assert lib.aae_trainer_set_latent_terms(h, 0.0, -0.5) == -1
    assert lib.aae_trainer_set_latent_terms(h, -0.1, 0.0) == -1
    eh = enc.handle(sess.device)
    out = torch.empty((2, 128), device="cuda")
    assert lib.aae_encoder_sigma_forward(eh, 2, _lib.ptr(out), None) == -3
    k = np.zeros((32768, 128), np.float32)
    assert lib.aae_encoder_set_weights(eh, 5, _lib.ptr(k), None, None) == -1
    assert top.step_device(xb, yb, update=False).item() == first
    # a head enabled after the trainer was created is not part of that trainer
    assert lib.aae_encoder_enable_sigma_head(eh) == 0
    assert lib.aae_trainer_set_latent_terms(h, 0.1, 0.0) == -3
    assert top.step_device(xb, yb, update=False).item() == first
    torch.cuda.synchronize()
