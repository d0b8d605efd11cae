"""GPU tests of the training step with every loss switch on at once: VARIATIONAL (sigma head, sampled z, KL term), NORM_REGULARIZE
and AUXILIARY_MASK (mask head, mask loss), under every OPTIMIZER.  The reference allows the combination: build_decoder feeds the
sampled z into a decoder with the mask head (auto_pose/ae/ae_factory.py:58), and AE.loss adds the latent terms to a reconstr_loss
that already holds the mask loss (ae.py:43-53, decoder.py:134-142).  Where the switches meet: the decoder reads the sampled z and
runs the mask head joined to the output conv; three kernels write one loss word (bootstrapped L2 =, mask loss +=, latent terms +=);
the gradient and slot tables hold both heads (24 tensors, one optimizer launch); checkpoint names move (dense_1 sigma head, dense_2
decoder dense, conv2d_7 mask head, conv2d_8 output conv).  Reference: oracle/latent_oracle.vae_forward_loss with mask_head."""
import configparser

import numpy as np
import pytest
import torch

from oracle import aae_oracle as O
from oracle import latent_oracle as LO
from oracle import mask_oracle as MO
from oracle import optimizer_oracle as OO
from tests.test_gpu_a_parity import sess  # noqa: F401
from tests.test_gpu_e_fp16_train import _analyse, _check_grads, _clear_margin_params, _grad_bounds
from tests.test_gpu_h_latent_terms import _head as _sigma_head
from tests.test_gpu_h_latent_terms import _named as _dense_named
from tests.test_gpu_i_optimizers import INITIAL, RULES, _check_state, _replay, _weights
from tests.test_gpu_k_aux_mask import _device_memory_free, _target, _track  # noqa: F401  (autouse fixture: frees handles)
from tests.test_gpu_k_aux_mask import _head as _mask_head
from tests.test_gpu_k_aux_mask import _named as _mask_named

pytestmark = pytest.mark.gpu

FP32, SPLIT, FP16 = 0, 1, 2
VAR, NORM, EPS = 0.1, 0.5, 0.7
ALL_RULES = ["Adam"] + list(RULES)
SIGMA, DEC_DENSE, MASK, OUT = "dense_1", "dense_2", "conv2d_7", "conv2d_8"      # template names with both heads
REL = 3e-4


def _dec_named(dp, mhead, sigma=True):
    """decoder variables under the names of the graph with the mask head and (sigma) the sigma head"""
    return _dense_named(_mask_named(dp, mhead), sigma)


def _build(handles, gemm, B, ep, dp, head, mhead, variational=VAR, norm=NORM, bootstrap=4, optimizer="Adam", sigma=True):
    """template pair with the mask head, and the sigma head when ``sigma`` (the decoder then reads the sampled z)"""
    from augmentedautoencoder_b200.ae.ae import AE
    from augmentedautoencoder_b200.ae.ae_factory import TrainOp
    from augmentedautoencoder_b200.ae.decoder import Decoder
    from augmentedautoencoder_b200.ae.encoder import Encoder
    from augmentedautoencoder_b200.ae.session import placeholder
    x, y = placeholder(np.float32, [None, 128, 128, 3]), placeholder(np.float32, [None, 128, 128, 3])
    enc = Encoder(x, 128, list(O.NUM_FILTER), 5, list(O.STRIDES), False, is_training=True, max_batch=B, precision=handles)
    dec = Decoder(y, enc.sampled_z if sigma else enc.z, list(reversed(O.NUM_FILTER)), 5, list(reversed(O.STRIDES)), "L2", bootstrap,
                  True, False, is_training=True, max_batch=B, precision=handles)
    enc.load_weights({**ep, SIGMA + "/kernel": head[0], SIGMA + "/bias": head[1]} if sigma else ep)
    dec.load_weights(_dec_named(dp, mhead, sigma))
    return enc, dec, _track(TrainOp(AE(enc, dec, norm, variational), 2e-4, precision=gemm, optimizer=optimizer), enc, dec)


def _small_params():
    """fp32-trainer geometry of tests/test_gpu_i (16x16, filters (4, 8), latent 8) with both heads: sigma head [128, 8], mask head
    [5, 5, 4, 1]; the 3-channel output conv admits the head on the fp32 trainer"""
    geo = dict(num_filters=(4, 8), strides=(2, 2), latent=8, bias_scale=0.1)
    ep = O.make_encoder_params(5, in_hw=16, **geo)
    dp = O.make_decoder_params(6, out_hw=16, n_encoder_convs=2, **geo)
    rng = np.random.RandomState(7)
    head = ((0.3 * rng.standard_normal((128, 8))).astype(np.float32), np.full(8, 0.5, np.float32))
    mhead = MO.make_mask_head(8, 4, bias_scale=0.2)
    return ep, dp, head, mhead


def _small_build(optimizer, ep, dp, head, mhead, max_batch=4):
    from augmentedautoencoder_b200.ae.ae import AE
    from augmentedautoencoder_b200.ae.ae_factory import TrainOp
    from augmentedautoencoder_b200.ae.decoder import Decoder
    from augmentedautoencoder_b200.ae.encoder import Encoder
    from augmentedautoencoder_b200.ae.session import placeholder
    x, y = placeholder(np.float32, [None, 16, 16, 3]), placeholder(np.float32, [None, 16, 16, 3])
    enc = Encoder(x, 8, [4, 8], 5, [2, 2], False, is_training=True, max_batch=max_batch, precision=FP32)
    dec = Decoder(y, enc.sampled_z, [8, 4], 5, [2, 2], "L2", 4, True, False, is_training=True, max_batch=max_batch,
                  n_encoder_convs=2, precision=FP32)
    enc.load_weights({**ep, "dense_1/kernel": head[0], "dense_1/bias": head[1]})
    d = {("dense_2" + k[7:] if k.startswith("dense_1/") else "conv2d_4" + k[8:] if k.startswith("conv2d_3/") else k): v
         for k, v in dp.items()}
    d["conv2d_3/kernel"], d["conv2d_3/bias"] = mhead
    dec.load_weights(d)
    return enc, dec, _track(TrainOp(AE(enc, dec, NORM, VAR), 2e-4, optimizer=optimizer), enc, dec)


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _rel(a, b):
    return float(np.linalg.norm(a.astype(np.float64) - b) / max(np.linalg.norm(b), 1e-300))


def _oracle(xb, yb, ep, dp, head, mhead, eps=EPS, chunk=16, bootstrap=4):
    """float64 loss, terms and 24 gradients of a batch, 16 samples at a time on the GPU: every loss term is a mean over the samples
    of equally many entries each (the KL term's over b and j, the norm term's over b), so the batch's values are the chunks'
    weighted by size.  terms: sampled_z and xmask concatenated over the chunks."""
    B, loss, grads, sz, xm = xb.shape[0], 0.0, None, [], []
    for a in range(0, B, chunk):
        n = min(B, a + chunk) - a
        l, t, g = LO.vae_forward_loss(xb[a:a + n], yb[a:a + n], ep, dp, head=head, mask_head=mhead, variational=VAR, norm_regularize=NORM,
                                      eps=eps, dtype=torch.float64, bootstrap_ratio=bootstrap, with_grads=True, device="cuda")
        torch.cuda.empty_cache()
        loss += l * n / B
        sz.append(t["sampled_z"])
        xm.append(t["xmask"])
        grads = {k: v * (n / B) for k, v in g.items()} if grads is None else {k: grads[k] + v * (n / B) for k, v in g.items()}
    return loss, {"sampled_z": np.concatenate(sz), "xmask": np.concatenate(xm)}, grads


# ---- a. loss and 24 gradients against float64 ----------------------------------------------------------------------------------
@pytest.mark.parametrize("handles", [FP32, SPLIT])
def test_loss_and_gradients_match_float64_oracle(sess, handles):
    """VARIATIONAL 0.1, NORM_REGULARIZE 0.5 and the mask head: the loss and all 24 gradients at batch 1, 64 and a ragged 37 on one
    max_batch-64 pair against the float64 oracle, at the bars of the single-switch tests (loss 4e-6 relative, every gradient 3e-4
    relative L2).  The decoder reads the sampled z, so the ReLU margin is asserted on that forward."""
    ep, dp = _clear_margin_params()
    head, mhead = _sigma_head(0.05), _mask_head(scale=0.05)
    enc, dec, top = _build(handles, None, 64, ep, dp, head, mhead)
    for B in (1, 64, 37):
        xb = np.random.RandomState(8 + B).rand(B, 128, 128, 3).astype(np.float32)
        yb = _target(4 + B, B)
        loss = float(top.step_device(_dev(xb), _dev(yb), update=False, eps=EPS))
        grads = top.gradients(sess.device)
        loss64, terms, g64 = _oracle(xb, yb, ep, dp, head, mhead)
        margin = O.relu_margin(xb, ep, dp, device="cuda", latent=terms["sampled_z"])
        torch.cuda.empty_cache()
        assert margin > 1e-4, margin
        assert 0.05 < 1 - MO.mask_target(yb).mean() < 0.2 and np.std(terms["xmask"]) > 1e-3
        assert sorted(grads) == sorted(g64) and len(g64) == 24
        assert {SIGMA + "/kernel", DEC_DENSE + "/kernel", MASK + "/kernel", OUT + "/kernel"} <= set(g64)
        tag = "precision %d, batch %d" % (handles, B)
        print("%s: |loss - loss64| %.2e (loss64 %.6f)" % (tag, abs(loss - loss64), loss64))
        assert abs(loss - loss64) < 4e-6 * max(1.0, abs(loss64)), (tag, loss, loss64)
        _check_grads(grads, g64, {k: REL for k in g64}, tag)


# ---- b. single-pass fp16 trainer ------------------------------------------------------------------------------------------------
def test_fp16_trainer_meets_the_composed_rounding_bound(sess):
    """The single-pass trainer with every switch on, batch 1, no bootstrapping.  Gradients: twice the plain step's rounding-model
    bound (tests/test_gpu_e), as with the mask head alone (tests/test_gpu_k: the joined output layer carries a second loss gradient
    through the same GEMMs); the mask head and the output conv get the output conv's bound, the sigma head the encoder dense layer's
    (its GEMMs have that layer's structure and add fp32 operations only, tests/test_gpu_h).  Loss: 2 (loss_bound + mask_bound) +
    4 fwd_rel mag, the mask test's bound plus the latent test's term for the forward rounding of z passed through the latent terms
    (mag = their magnitude).  The two parts bound disjoint terms of the sum (the reconstruction terms read the decoder's output, the
    latent terms read z), so they add with no further factor."""
    ep, dp = _clear_margin_params()
    head, mhead = _sigma_head(0.05), _mask_head(scale=0.05)
    xb = np.random.RandomState(8).rand(1, 128, 128, 3).astype(np.float32)
    yb = _target(4, 1)
    eps = 0.3
    A = _analyse(xb, yb, ep, dp, 1)
    loss64, t, g64 = LO.vae_forward_loss(xb, yb, ep, dp, head=head, mask_head=mhead, variational=VAR, norm_regularize=NORM, eps=eps,
                                         dtype=torch.float64, bootstrap_ratio=1, with_grads=True, device="cuda")
    assert O.relu_margin(xb, ep, dp) > 2 * A["relu_need"]
    assert O.relu_margin(xb, ep, dp, latent=t["sampled_z"]) > 2 * A["relu_need"]
    plain = _grad_bounds(A)
    bounds = {k: 2 * v for k, v in plain.items() if not k.startswith("conv2d_7/")}
    for part in ("kernel", "bias"):
        bounds[OUT + "/" + part] = bounds[MASK + "/" + part] = 2 * plain["conv2d_7/" + part]
    bounds = _dense_named(bounds, True)
    for part in ("kernel", "bias"):
        bounds[SIGMA + "/" + part] = 2 * plain["dense/" + part]
    enc, dec, top = _build(SPLIT, FP16, 2, ep, dp, head, mhead, bootstrap=1)
    loss = float(top.step_device(_dev(xb), _dev(yb), update=False, eps=eps))
    grads = top.gradients(sess.device)
    xm = t["xmask"].astype(np.float64)
    d_xm = 0.25 * A["fwd_rel"] * float(np.abs(np.log(xm / (1 - xm))).max())
    mask_bound = float(np.mean(2 * np.abs(xm - MO.mask_target(yb)) * d_xm + d_xm ** 2))
    z = t["z"]
    s2 = t["q_sigma"] ** 2
    mag = NORM * float(np.mean(np.linalg.norm(z, axis=1) + 1)) + VAR * float(np.mean(0.5 * z * z + 0.5 * (s2 + 1 + np.abs(np.log(s2)))))
    bound = 2 * (A["loss_bound"] + mask_bound) + 4 * A["fwd_rel"] * mag
    print("fp16 trainer, every switch: |loss - loss64| %.2e, bound %.2e (share %.3f); gradient bounds %.2e .. %.2e"
          % (abs(loss - loss64), bound, abs(loss - loss64) / bound, min(bounds.values()), max(bounds.values())))
    assert abs(loss - loss64) <= bound, (loss, loss64, bound)
    assert sorted(grads) == sorted(g64) == sorted(bounds) and len(g64) == 24
    _check_grads(grads, g64, bounds, "fp16 trainer, every switch")


# ---- c. VARIATIONAL off with both heads present ---------------------------------------------------------------------------------
@pytest.mark.parametrize("handles", [FP32, SPLIT])
def test_variational_off_with_both_heads_is_the_step_without_the_sigma_head(sess, handles):
    """Mask head on, sigma head enabled, VARIATIONAL 0, NORM_REGULARIZE 0.5: the loss and the 22 gradients that exist without the
    sigma head are bit-identical to those of a pair built without it (its decoder dense is dense_1 there, dense_2 here)."""
    ep, dp = O.make_encoder_params(42, bias_scale=0.02), O.make_decoder_params(43, bias_scale=0.02)
    head, mhead = _sigma_head(0.5), _mask_head()
    xb, yb = _dev(np.random.RandomState(11).rand(3, 128, 128, 3).astype(np.float32)), _dev(_target(12, 3))
    runs = []
    for sigma in (True, False):
        enc, dec, top = _build(handles, None, 4, ep, dp, head, mhead, variational=0.0, sigma=sigma)
        loss = float(top.step_device(xb, yb, update=False))
        runs.append((loss, top.gradients(sess.device)))
    (l1, g1), (l0, g0) = runs
    assert len(g1) == 24 and len(g0) == 22
    assert l1 == l0, (l1, l0)
    for k0 in g0:
        k1 = DEC_DENSE + k0[len("dense_1"):] if k0.startswith("dense_1/") else k0
        assert np.array_equal(g1[k1], g0[k0]), (k0, k1)


@pytest.mark.parametrize("name", ALL_RULES)
def test_variational_off_leaves_the_sigma_head_and_its_slots_alone(sess, name):
    """The same switches, one update under each rule: the sigma head's masters and slots keep their values (TF applies no update
    to a variable without a gradient), the mask head's masters move."""
    ep, dp = O.make_encoder_params(42, bias_scale=0.02), O.make_decoder_params(43, bias_scale=0.02)
    head, mhead = _sigma_head(0.5), _mask_head()
    xb, yb = _dev(np.random.RandomState(11).rand(2, 128, 128, 3).astype(np.float32)), _dev(_target(12, 2))
    enc, dec, top = _build(SPLIT, None, 2, ep, dp, head, mhead, variational=0.0, optimizer=name)
    top.trainer(sess.device)
    s0 = top.optimizer_variables()
    top.step_device(xb, yb)
    w, s1 = {**enc.get_weights(short_names=True), **dec.get_weights(short_names=True)}, top.optimizer_variables()
    initial = (0.0, 0.0) if name == "Adam" else INITIAL[name]
    for part, h0 in (("kernel", head[0]), ("bias", head[1])):
        assert np.array_equal(w[SIGMA + "/" + part], h0), part
        for slot, v0 in zip(top._slots, initial):
            k = SIGMA + "/" + part + "/" + slot
            assert np.array_equal(s1[k], s0[k]) and np.all(s1[k] == np.float32(v0)), k
    assert not np.array_equal(w[MASK + "/kernel"], mhead[0])
    if top._slots:
        assert not np.array_equal(s1[MASK + "/kernel/" + top._slots[0]], s0[MASK + "/kernel/" + top._slots[0]])


# ---- d. every OPTIMIZER with both heads -----------------------------------------------------------------------------------------
def _replay_any(sess, name, enc, dec, top, xb, yb, steps=3):
    """tests/test_gpu_i's replay for the seven rules of oracle/optimizer_oracle; Adam replayed the same way with OO.adam (the
    kernel's rounding of TF's ApplyAdam: two FMAs, lr_t rounded once) -- masters and both slots bit-exact after every step"""
    if name != "Adam":
        _replay(sess, name, enc, dec, top, xb, yb, steps)
        return
    lr, hp = top._opt.learning_rate, list(top._opt.hp)
    top.trainer(sess.device)
    w = _weights(enc, dec)
    w0 = dict(w)
    s = {k: (np.zeros_like(v), np.zeros_like(v)) for k, v in w.items()}
    for t in range(1, steps + 1):
        top.step_device(xb, yb)
        g = top.gradients(sess.device)
        lr_t = OO.adam_lr_t(lr, t, hp[0], hp[1])
        for k in w:
            w[k], s[k] = OO.adam(w[k], g[k], s[k], lr_t, hp)
        got_s = {k: v for k, v in top.optimizer_variables().items() if not k.endswith("_power")}
        got_w = _weights(enc, dec)
        bad = [k for k in w if not np.array_equal(got_w[k], w[k])]
        assert not bad, ("Adam step %d masters" % t, bad)
        want_s = {k + "/" + suf: a for k, arrs in s.items() for suf, a in zip(top._slots, arrs)}
        assert sorted(got_s) == sorted(want_s)
        bad = [k for k in want_s if not np.array_equal(got_s[k], want_s[k])]
        assert not bad, ("Adam step %d slots" % t, bad)
    assert all(not np.array_equal(w[k], w0[k]) for k in w if k.endswith("/kernel"))


def _batch(B, hw, seed=3):
    xb = np.random.RandomState(seed).rand(B, hw, hw, 3).astype(np.float32)
    return _dev(xb), _dev(_target(seed + 1, B) if hw == 128 else np.random.RandomState(seed + 1).rand(B, hw, hw, 3).astype(np.float32))


@pytest.mark.parametrize("name", ALL_RULES)
def test_fp32_trainer_replays_bit_exact(sess, name):
    ep, dp, head, mhead = _small_params()
    enc, dec, top = _small_build(name, ep, dp, head, mhead)
    assert len(_weights(enc, dec)) == 16
    _replay_any(sess, name, enc, dec, top, *_batch(4, 16))


@pytest.mark.parametrize("name", ALL_RULES)
def test_split_trainer_replays_bit_exact(sess, name):
    ep, dp = O.make_encoder_params(42, bias_scale=0.02), O.make_decoder_params(43, bias_scale=0.02)
    enc, dec, top = _build(SPLIT, None, 2, ep, dp, _sigma_head(0.5), _mask_head(), optimizer=name)
    assert len(_weights(enc, dec)) == 24
    _replay_any(sess, name, enc, dec, top, *_batch(2, 128))


@pytest.mark.parametrize("name", ["GradientDescent", "RMSProp"])
def test_single_pass_trainer_replays_bit_exact(sess, name):
    ep, dp = O.make_encoder_params(42, bias_scale=0.02), O.make_decoder_params(43, bias_scale=0.02)
    enc, dec, top = _build(SPLIT, FP16, 2, ep, dp, _sigma_head(0.5), _mask_head(), optimizer=name)
    _replay_any(sess, name, enc, dec, top, *_batch(2, 128))


def test_one_update_launch_for_24_tensors_under_every_rule(sess):
    """Every rule's step launches the same kernels, and the update of the 24 tensors is one launch (they fit one OptBatch): a step
    with the update launches exactly one kernel more than the forward/backward alone."""
    from augmentedautoencoder_b200 import _lib
    lib = _lib.lib()
    ep, dp = O.make_encoder_params(42, bias_scale=0.02), O.make_decoder_params(43, bias_scale=0.02)
    xb, yb = _batch(2, 128)
    counts = {}
    for name in ALL_RULES:
        enc, dec, top = _build(SPLIT, None, 2, ep, dp, _sigma_head(0.5), _mask_head(), optimizer=name)
        top.step_device(xb, yb, eps=0.2)
        n = []
        for update in (True, False):
            torch.cuda.synchronize()
            n0 = lib.aae_launch_count()
            top.step_device(xb, yb, update=update, eps=0.2)
            n.append(lib.aae_launch_count() - n0)
        counts[name] = tuple(n)
        top.close()
        enc.close()
        dec.close()
    print("launches per step (with update, without): %s" % counts)
    assert len(set(counts.values())) == 1, counts
    with_update, without = counts["Adam"]
    assert with_update == without + 1, counts


# ---- e. checkpoints -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["Adam", "Adagrad", "RMSProp", "Ftrl"])
def test_checkpoint_holds_both_heads_and_resumes_bit_identically(sess, tmp_path, name):
    """Saver(..., train_op=...) writes the 24 variables and the rule's slots of each under TF's names, in .npz and TF-bundle form; a
    fresh pair restored from either continues two steps with the same eps sequence bit-identically (losses and masters).  An
    inference encoder (no sigma head) restores strictly from the same files.  A decoder without the heads cannot: the file's
    dense_1 is the sigma head and its conv2d_7 the mask head, so the restore is refused naming the shape, as the reference's is,
    and the decoder keeps its values."""
    from augmentedautoencoder_b200.ae import ae_factory as F
    from augmentedautoencoder_b200.ae.decoder import Decoder
    from augmentedautoencoder_b200.ae.encoder import Encoder
    from augmentedautoencoder_b200.ae.session import placeholder
    from augmentedautoencoder_b200.ae.tf_checkpoint import read_tf_checkpoint
    ep, dp = O.make_encoder_params(42, bias_scale=0.02), O.make_decoder_params(43, bias_scale=0.02)
    xb, yb = _dev(np.random.RandomState(11).rand(3, 128, 128, 3).astype(np.float32)), _dev(_target(12, 3))
    eps = [0.4, -1.2, 0.9, 0.1]
    enc, dec, top = _build(SPLIT, None, 4, ep, dp, _sigma_head(0.5), _mask_head(), optimizer=name)
    for e in eps[:2]:
        top.step_device(xb, yb, eps=e)
    saver = F.Saver([enc, dec], global_step=top._ae.global_step, train_op=top)
    paths = [saver.save(sess, str(tmp_path / "npz" / "chkpt"), global_step=2), saver.save_tf(sess, str(tmp_path / "tf" / "chkpt"), global_step=2)]
    want = [float(top.step_device(xb, yb, eps=e)) for e in eps[2:]]
    w_want = _weights(enc, dec)
    names = sorted(w_want)
    assert len(names) == 24
    slots = F.OPTIMIZERS[name][2]
    for path in paths:
        stored = dict(np.load(path)) if path.endswith(".npz") else read_tf_checkpoint(path)
        assert set(names) <= set(stored)
        for k in names:
            for suf in slots:
                assert k + "/" + suf in stored and stored[k + "/" + suf].shape == stored[k].shape, (path, k, suf)
        assert stored[SIGMA + "/kernel"].shape == (32768, 128) and stored[DEC_DENSE + "/kernel"].shape == (128, 32768)
        assert stored[MASK + "/kernel"].shape == (5, 5, 128, 1) and stored[OUT + "/kernel"].shape == (5, 5, 128, 3)
        # both heads trained: their masters moved from the initial values (their slots travel under the names checked above; the
        # resume below is bit-identical only if the restored slots are the saved ones)
        assert not np.array_equal(stored[SIGMA + "/kernel"], _sigma_head(0.5)[0]) and not np.array_equal(stored[MASK + "/kernel"], _mask_head()[0])
        enc2, dec2, top2 = _build(SPLIT, None, 4, ep, dp, _sigma_head(0.0), _mask_head(seed=3), optimizer=name)
        F.Saver([enc2, dec2], global_step=top2._ae.global_step, train_op=top2).restore(sess, path)
        got = [float(top2.step_device(xb, yb, eps=e)) for e in eps[2:]]
        assert got == want, (path, got, want)
        w_got = _weights(enc2, dec2)
        assert all(np.array_equal(w_got[k], w_want[k]) for k in w_want), path
        top2.close()
        enc2.close()
        dec2.close()
        inf = Encoder(placeholder(np.float32, [None, 128, 128, 3]), 128, list(O.NUM_FILTER), 5, list(O.STRIDES), False, max_batch=4)
        F.Saver([inf]).restore(sess, path)
        assert SIGMA + "/kernel" not in inf.variable_names
        assert np.array_equal(inf.get_weights()["dense/kernel"], stored["dense/kernel"])
        inf_dec = Decoder(placeholder(np.float32, [None, 128, 128, 3]), inf.z, list(reversed(O.NUM_FILTER)), 5, list(reversed(O.STRIDES)),
                          "L2", 4, False, False, max_batch=4)
        before = inf_dec.get_weights()["dense_1/kernel"].copy()
        with pytest.raises(ValueError, match=r"dense_1/kernel: shape \(32768, 128\) != expected \(128, 32768\)"):
            F.Saver([inf_dec]).restore(sess, path)
        assert np.array_equal(inf_dec.get_weights()["dense_1/kernel"], before)
        inf.close()
        inf_dec.close()


# ---- f. the cfg path ------------------------------------------------------------------------------------------------------------
def _cfg():
    c = configparser.ConfigParser()
    c.read_dict({"Network": {"LATENT_SPACE_SIZE": "128", "NUM_FILTER": "[128, 256, 512, 512]", "KERNEL_SIZE_ENCODER": "5",
                             "KERNEL_SIZE_DECODER": "5", "STRIDES": "[2, 2, 2, 2]", "BATCH_NORMALIZATION": "False", "LOSS": "L2",
                             "BOOTSTRAP_RATIO": "4", "VARIATIONAL": str(VAR), "AUXILIARY_MASK": "True", "NORM_REGULARIZE": str(NORM)},
                 "Training": {"BATCH_SIZE": "2", "LEARNING_RATE": "2e-4", "OPTIMIZER": "RMSProp"}})
    return c


def test_cfg_graph_names_and_train_op(sess):
    """build_* from a cfg with VARIATIONAL 0.1, NORM_REGULARIZE 0.5, AUXILIARY_MASK and OPTIMIZER RMSProp: TF's names in the
    reference's creation order (conv2d .. conv2d_3, dense, the sigma head dense_1, the decoder dense dense_2, conv2d_4 .. conv2d_6,
    the mask head conv2d_7, the output conv conv2d_8; the decoder lists the mask head after the output conv, as every decoder with
    the head does), and sess.run(train_op) returns the oracle's loss with the first eps of its stream and advances the step."""
    from augmentedautoencoder_b200.ae import ae_factory as F
    from augmentedautoencoder_b200.ae import session as S
    args = _cfg()
    x, y = S.placeholder(np.float32, [None, 128, 128, 3]), S.placeholder(np.float32, [None, 128, 128, 3])
    enc = F.build_encoder(x, args, is_training=True)
    dec = F.build_decoder(y, enc, args, is_training=True)
    ae = F.build_ae(enc, dec, args)
    top = _track(F.build_train_op(ae, args), enc, dec)
    creation = ["conv2d", "conv2d_1", "conv2d_2", "conv2d_3", "dense", "dense_1", "dense_2", "conv2d_4", "conv2d_5", "conv2d_6",
                "conv2d_7", "conv2d_8"]
    want = [l + "/" + p for l in creation for p in ("kernel", "bias")]
    short = [n.split("/", 1)[1] if n.count("/") == 2 else n for n in enc.variable_names + dec.variable_names]
    assert short[:20] == want[:20] and short[20:] == want[22:] + want[20:22], short
    assert dec._latent_code is enc.sampled_z and dec._auxiliary_mask and top._slots == ("RMSProp", "RMSProp_1")
    ep, dp = O.make_encoder_params(42, bias_scale=0.02), O.make_decoder_params(43, bias_scale=0.02)
    head, mhead = _sigma_head(0.5), _mask_head()
    enc.load_weights({**ep, SIGMA + "/kernel": head[0], SIGMA + "/bias": head[1]})
    dec.load_weights(_dec_named(dp, mhead))
    xb = np.random.RandomState(8).rand(2, 128, 128, 3).astype(np.float32)
    yb = _target(4, 2)
    eps0 = float(np.float32(np.random.RandomState(0).standard_normal()))
    loss_t = float(sess.run(top, {x: xb, y: yb}))
    loss64, _, _ = LO.vae_forward_loss(xb, yb, ep, dp, head=head, mask_head=mhead, variational=VAR, norm_regularize=NORM, eps=eps0,
                                       dtype=torch.float64, device="cuda")
    print("cfg train_op: loss %.7f, float64 %.7f" % (loss_t, loss64))
    assert abs(loss_t - loss64) < 4e-6 * max(1.0, abs(loss64)), (loss_t, loss64)
    assert int(ae.global_step.value()) == 1


# ---- the loss composition, bit for bit ------------------------------------------------------------------------------------------
A_NORM = np.float32(1 + 1234 / 2048)        # 12 significant bits: a^2, sqrt, a - 1 and their batch means are exact in fp32
W_CANDIDATES = [0.5, 0.3, 0.7, 0.1, 0.9, 0.37, 0.61, 0.83, 1.7, 2.3]


@pytest.mark.parametrize("gemm,handles", [(None, FP32), (None, SPLIT), (FP16, SPLIT)])
def test_norm_term_joins_the_loss_with_two_roundings(sess, gemm, handles):
    """TF adds NORM_REGULARIZE as two ops, reg_loss * w and then loss + ...: two fp32 roundings.  With the encoder's dense kernel 0
    and its bias (a, 0, .., 0), a = 1 + 1234/2048, every z row is exactly that bias on every trainer, so reg_loss = a - 1 exactly
    at any batch size.  L0 is the loss of the same step with the terms off (the decoder reads z in both steps, so the bootstrapped
    L2 and the mask loss are the same bits).  The step's loss must be f32(L0 + f32(r w)), and the test first picks a w for which
    that differs from the single rounding f32(L0 + r w) of a fused multiply-add, so an FMA in the composition fails it."""
    from augmentedautoencoder_b200 import _lib
    lib = _lib.lib()
    ep, dp = _clear_margin_params()
    ep["dense/kernel"] = np.zeros_like(ep["dense/kernel"])
    ep["dense/bias"] = np.zeros_like(ep["dense/bias"])
    ep["dense/bias"][0] = A_NORM
    enc, dec, top = _build(handles, gemm, 4, ep, dp, _sigma_head(0.05), _mask_head(scale=0.05), variational=0.0, norm=0.0,
                           bootstrap=1 if gemm == FP16 else 4)
    h = top.trainer(sess.device)
    xb, yb = _dev(np.random.RandomState(8).rand(3, 128, 128, 3).astype(np.float32)), _dev(_target(4, 3))
    L0 = np.float32(top.step_device(xb, yb, update=False).item())
    r = np.float32(A_NORM - np.float32(1))
    two, one, w = None, None, None
    for c in W_CANDIDATES:
        c = np.float32(c)
        two, one = np.float32(L0 + np.float32(r * c)), OO.fma32(r, c, L0)
        if two != one:
            w = c
            break
    assert w is not None, ("no candidate weight separates one rounding from two for L0 = %r" % L0)
    _lib.check(lib.aae_trainer_set_latent_terms(h, 0.0, float(w)), "set_latent_terms")
    loss = np.float32(top.step_device(xb, yb, update=False).item())
    print("L0 %r, w %r: loss %r, two roundings %r, one rounding %r" % (float(L0), float(w), float(loss), float(two), float(one)))
    z = enc.encode_device(xb).cpu().numpy() if handles == FP32 else None
    if z is not None:
        assert np.all(z == ep["dense/bias"])
    assert loss == two, (float(loss), float(two), float(one))
