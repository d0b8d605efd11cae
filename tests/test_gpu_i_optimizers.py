"""GPU tests of the OPTIMIZER switch: every tf.train optimizer a cfg can build (auto_pose/ae/ae_factory.py:79-95) trains in the fused
step on the fp32, split and single-pass fp16 trainers.  Masters and slots are replayed bit for bit with the float32 oracle
(oracle/optimizer_oracle.py) over the trainer's own gradients; checkpoints carry the rule's slots under TF's names."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import aae_oracle as O
from oracle import optimizer_oracle as OO
from tests.test_gpu_a_parity import sess  # noqa: F401
from tests.test_gpu_h_latent_terms import _head, _named

pytestmark = pytest.mark.gpu

FP32, SPLIT, FP16 = 0, 1, 2
RULES = {"GradientDescent": OO.gradient_descent, "ProximalGradientDescent": OO.proximal_gradient_descent, "Adagrad": OO.adagrad,
         "ProximalAdagrad": OO.proximal_adagrad, "Adadelta": OO.adadelta, "RMSProp": OO.rmsprop, "Ftrl": OO.ftrl}
INITIAL = {"GradientDescent": (), "ProximalGradientDescent": (), "Adagrad": (0.1,), "ProximalAdagrad": (0.1,), "Adadelta": (0.0, 0.0),
           "RMSProp": (1.0, 0.0), "Ftrl": (0.1, 0.0)}          # slot values of a new trainer, in TF's creation order
WITH_SLOTS = [n for n in RULES if INITIAL[n]]


def _small_ae(optimizer, max_batch=4, hw=16, filters=(4, 8), latent=8, hp=None):
    """fp32 trainer at a small geometry; hp overrides aae_optimizer.hp entries {index: value} (aae_trainer_create_opt)."""
    from augmentedautoencoder_b200.ae.ae import AE
    from augmentedautoencoder_b200.ae.ae_factory import TrainOp
    from augmentedautoencoder_b200.ae.decoder import Decoder
    from augmentedautoencoder_b200.ae.encoder import Encoder
    from augmentedautoencoder_b200.ae.session import placeholder
    strides = (2,) * len(filters)
    x, y = placeholder(np.float32, [None, hw, hw, 3]), placeholder(np.float32, [None, hw, hw, 3])
    enc = Encoder(x, latent, list(filters), 5, list(strides), False, is_training=True, max_batch=max_batch, precision=FP32)
    dec = Decoder(y, enc.z, list(reversed(filters)), 5, list(reversed(strides)), "L2", 4, False, False, is_training=True,
                  max_batch=max_batch, n_encoder_convs=len(filters), precision=FP32)
    enc.load_weights(O.make_encoder_params(5, num_filters=filters, in_hw=hw, strides=strides, latent=latent, bias_scale=0.1))
    dec.load_weights(O.make_decoder_params(6, num_filters=filters, out_hw=hw, strides=strides, latent=latent, bias_scale=0.1,
                                           n_encoder_convs=len(filters)))
    top = TrainOp(AE(enc, dec, 0, 0), 2e-4, optimizer=optimizer)
    for i, v in (hp or {}).items():
        top._opt.hp[i] = v
    return enc, dec, top


def _full_ae(optimizer, handles, gemm, B=2):
    from augmentedautoencoder_b200.ae.ae import AE
    from augmentedautoencoder_b200.ae.ae_factory import TrainOp
    from augmentedautoencoder_b200.ae.decoder import Decoder
    from augmentedautoencoder_b200.ae.encoder import Encoder
    from augmentedautoencoder_b200.ae.session import placeholder
    x, y = placeholder(np.float32, [None, 128, 128, 3]), placeholder(np.float32, [None, 128, 128, 3])
    enc = Encoder(x, 128, list(O.NUM_FILTER), 5, list(O.STRIDES), False, is_training=True, max_batch=B, precision=handles)
    dec = Decoder(y, enc.z, list(reversed(O.NUM_FILTER)), 5, list(reversed(O.STRIDES)), "L2", 4, False, False, is_training=True,
                  max_batch=B, precision=handles)
    enc.load_weights(O.make_encoder_params(42, bias_scale=0.02))
    dec.load_weights(O.make_decoder_params(43, bias_scale=0.02))
    return enc, dec, TrainOp(AE(enc, dec, 0, 0), 2e-4, precision=gemm, optimizer=optimizer)


def _batch(B, hw, seed=3):
    xb = torch.from_numpy(np.random.RandomState(seed).rand(B, hw, hw, 3).astype(np.float32)).cuda()
    yb = torch.from_numpy(np.random.RandomState(seed + 1).rand(B, hw, hw, 3).astype(np.float32)).cuda()
    return xb, yb


def _weights(enc, dec):
    return {**enc.get_weights(), **dec.get_weights()}


def _initial_slots(name, w):
    return {k: tuple(np.full(v.shape, np.float32(s), np.float32) for s in INITIAL[name]) for k, v in w.items()}


def _check_state(top, enc, dec, w, s, name, where):
    got_w, got_s = _weights(enc, dec), top.optimizer_variables()
    assert sorted(got_w) == sorted(w)
    bad = [k for k in w if not np.array_equal(got_w[k], w[k])]
    assert not bad, (where, "masters", bad)
    want_s = {k + "/" + suf: a for k, arrs in s.items() for suf, a in zip(top._slots, arrs)}
    assert sorted(got_s) == sorted(want_s), (where, sorted(got_s)[:4], sorted(want_s)[:4])
    bad = [k for k in want_s if not np.array_equal(got_s[k], want_s[k])]
    assert not bad, (where, "slots", bad)


def _replay(sess, name, enc, dec, top, xb, yb, steps=3):
    """`steps` training steps, each replayed with the oracle over the trainer's gradients: masters and slots bit-exact."""
    rule = RULES[name]
    lr, hp = top._opt.learning_rate, list(top._opt.hp)
    top.trainer(sess.device)
    w = _weights(enc, dec)
    w0 = dict(w)
    s = _initial_slots(name, w)
    _check_state(top, enc, dec, w, s, name, "initial")
    for t in range(steps):
        top.step_device(xb, yb)
        g = top.gradients(sess.device)
        for k in w:
            w[k], s[k] = rule(w[k], g[k], s[k], lr, hp)
        _check_state(top, enc, dec, w, s, name, "step %d" % (t + 1))
    assert all(not np.array_equal(w[k], w0[k]) for k in w if k.endswith("/kernel"))


@pytest.mark.parametrize("name", list(RULES))
def test_fp32_trainer_replays_bit_exact(sess, name):
    enc, dec, top = _small_ae(name)
    _replay(sess, name, enc, dec, top, *_batch(4, 16))


@pytest.mark.parametrize("name", list(RULES))
def test_split_trainer_replays_bit_exact(sess, name):
    enc, dec, top = _full_ae(name, SPLIT, None)
    _replay(sess, name, enc, dec, top, *_batch(2, 128))


@pytest.mark.parametrize("name", ["GradientDescent", "RMSProp"])
def test_single_pass_trainer_replays_bit_exact(sess, name):
    enc, dec, top = _full_ae(name, SPLIT, FP16)
    _replay(sess, name, enc, dec, top, *_batch(2, 128))


@pytest.mark.parametrize("name,hp", [("RMSProp", {1: 0.9}), ("Adadelta", {0: 0.8, 1: 1e-6})])
def test_non_default_hyperparameters_replay_bit_exact(sess, name, hp):
    """RMSProp with momentum 0.9 and Adadelta with rho 0.8: terms TF's defaults zero out or keep fixed"""
    enc, dec, top = _small_ae(name, hp=hp)
    _replay(sess, name, enc, dec, top, *_batch(4, 16))


@pytest.mark.parametrize("geometry", ["small_fp32", "full_split"])
def test_adam_through_create_opt_equals_trainer_create(sess, geometry):
    """Three steps of two trainers over equal handles: aae_trainer_create vs aae_trainer_create_opt(AAE_OPT_ADAM) -- the same loss,
    masters and slots, bit for bit."""
    from augmentedautoencoder_b200 import _lib
    lib = _lib.lib()
    runs = []
    for via_opt in (False, True):
        enc, dec, top = _small_ae("Adam") if geometry == "small_fp32" else _full_ae("Adam", SPLIT, None)
        B, hw = (4, 16) if geometry == "small_fp32" else (2, 128)
        xb, yb = _batch(B, hw)
        eh, dh = enc.handle(sess.device), dec.handle(sess.device)
        h = C.c_void_p()
        if via_opt:
            opt = _lib.Optimizer(_lib.OPT_ADAM, 2e-4, (C.c_float * 4)(0.9, 0.999, 1e-8))
            _lib.check(lib.aae_trainer_create_opt(eh, dh, 4, C.byref(opt), enc.precision, C.byref(h)), "create_opt")
        else:
            _lib.check(lib.aae_trainer_create(eh, dh, 4, 2e-4, 0.9, 0.999, 1e-8, C.byref(h)), "create")
        loss = torch.empty((1,), dtype=torch.float32, device="cuda")
        losses = []
        for _ in range(3):
            _lib.check(lib.aae_train_step(h, _lib.ptr(xb), _lib.ptr(yb), B, _lib.ptr(loss), None), "train step")
            losses.append(loss.item())
        slots = []
        for which, mod in ((0, enc), (1, dec)):
            for i, (kn, ks, bn, bs) in enumerate(mod._var_shapes):
                arrs = [np.empty(ks, np.float32), np.empty(ks, np.float32), np.empty(bs, np.float32), np.empty(bs, np.float32)]
                _lib.check(lib.aae_trainer_get_state(h, which, i, *[_lib.ptr(a) for a in arrs], None), "get_state")
                slots += arrs
        runs.append((losses, _weights(enc, dec), slots))
        lib.aae_trainer_destroy(h)
    (la, wa, sa), (lb, wb, sb) = runs
    assert la == lb
    assert all(np.array_equal(wa[k], wb[k]) for k in wa)
    assert len(sa) == len(sb) and all(np.array_equal(a, b) for a, b in zip(sa, sb))
    assert np.abs(sa[0]).max() > 0


def test_launches_per_step_are_the_same_for_every_rule(sess):
    from augmentedautoencoder_b200 import _lib
    lib = _lib.lib()
    xb, yb = _batch(4, 16)
    counts = {}
    for name in ["Adam"] + list(RULES):
        enc, dec, top = _small_ae(name)
        top.step_device(xb, yb)
        torch.cuda.synchronize()
        n0 = lib.aae_launch_count()
        top.step_device(xb, yb)
        counts[name] = lib.aae_launch_count() - n0
    assert len(set(counts.values())) == 1, counts


@pytest.mark.parametrize("name", WITH_SLOTS)
def test_checkpoints_hold_the_rule_slots_and_resume_bit_identically(sess, tmp_path, name):
    """.npz and TF bundle: exactly the rule's slot names (no /Adam, no beta powers); a full restore makes the third step
    bit-identical; a weights-only restore restarts the slots at their initial values (one step replayed from them)."""
    from augmentedautoencoder_b200.ae import ae_factory as F
    from augmentedautoencoder_b200.ae.tf_checkpoint import read_tf_checkpoint
    xb, yb = _batch(4, 16)
    enc, dec, top = _small_ae(name)
    for _ in range(2):
        top.step_device(xb, yb)
    saver = F.Saver([enc, dec], global_step=top._ae.global_step, train_op=top)
    paths = [saver.save(sess, str(tmp_path / "npz" / "chkpt"), global_step=2), saver.save_tf(sess, str(tmp_path / "tf" / "chkpt"), global_step=2)]
    weights_only = F.Saver([enc, dec], global_step=top._ae.global_step).save(sess, str(tmp_path / "w" / "chkpt"), global_step=2)
    w_names = sorted(_weights(enc, dec))
    loss_want = float(top.step_device(xb, yb))
    w_want, s_want = _weights(enc, dec), top.optimizer_variables()
    slot_names = {k + "/" + s for k in w_names for s in F.OPTIMIZERS[name][2]}
    assert sorted(s_want) == sorted(slot_names)
    for path in paths:
        stored = dict(np.load(path)) if path.endswith(".npz") else read_tf_checkpoint(path)
        extra = set(stored) - set(w_names) - {top._ae.global_step.name}
        assert extra == slot_names, (path, sorted(extra ^ slot_names)[:6])
        assert not any(k.endswith("/Adam") or k.endswith("/Adam_1") or "beta1_power" in k or "beta2_power" in k for k in stored)
        enc2, dec2, top2 = _small_ae(name)
        F.Saver([enc2, dec2], global_step=top2._ae.global_step, train_op=top2).restore(sess, path)
        assert float(top2.step_device(xb, yb)) == loss_want, path
        w_got, s_got = _weights(enc2, dec2), top2.optimizer_variables()
        assert all(np.array_equal(w_got[k], w_want[k]) for k in w_want), path
        assert all(np.array_equal(s_got[k], s_want[k]) for k in s_want), path
        assert int(top2._ae.global_step.value()) == 3
    enc3, dec3, top3 = _small_ae(name)
    F.Saver([enc3, dec3], global_step=top3._ae.global_step, train_op=top3).restore(sess, weights_only)
    w = _weights(enc3, dec3)
    assert all(np.array_equal(w[k], v) for k, v in dict(np.load(weights_only)).items() if k in w)
    s = _initial_slots(name, w)
    _check_state(top3, enc3, dec3, w, s, name, "weights-only restore")
    top3.step_device(xb, yb)
    g = top3.gradients(sess.device)
    lr, hp = top3._opt.learning_rate, list(top3._opt.hp)
    for k in w:
        w[k], s[k] = RULES[name](w[k], g[k], s[k], lr, hp)
    _check_state(top3, enc3, dec3, w, s, name, "step after weights-only restore")


@pytest.mark.parametrize("variational", [0.1, 0.0])
def test_sigma_head_slots_follow_variational(sess, tmp_path, variational):
    """RMSProp with the sigma head: with VARIATIONAL the head's masters and slots update and are saved as dense_1/kernel/RMSProp;
    without it the head gets no gradient and stays untouched (masters and initial slots)."""
    from augmentedautoencoder_b200.ae import ae_factory as F
    from augmentedautoencoder_b200.ae.ae import AE
    from augmentedautoencoder_b200.ae.decoder import Decoder
    from augmentedautoencoder_b200.ae.encoder import Encoder
    from augmentedautoencoder_b200.ae.session import placeholder
    x, y = placeholder(np.float32, [None, 128, 128, 3]), placeholder(np.float32, [None, 128, 128, 3])
    enc = Encoder(x, 128, list(O.NUM_FILTER), 5, list(O.STRIDES), False, is_training=True, max_batch=2, precision=SPLIT)
    dec = Decoder(y, enc.sampled_z, list(reversed(O.NUM_FILTER)), 5, list(reversed(O.STRIDES)), "L2", 4, False, False, is_training=True,
                  max_batch=2, precision=SPLIT)
    head = _head(0.5)
    enc.load_weights({**O.make_encoder_params(42, bias_scale=0.02), "dense_1/kernel": head[0], "dense_1/bias": head[1]})
    dec.load_weights(_named(O.make_decoder_params(43, bias_scale=0.02), True))
    top = F.TrainOp(AE(enc, dec, 0, variational), 2e-4, optimizer="RMSProp")
    xb, yb = _batch(2, 128, seed=11)
    for e in (0.4, -1.2):
        top.step_device(xb, yb, eps=e)
    path = F.Saver([enc, dec], global_step=top._ae.global_step, train_op=top).save(sess, str(tmp_path / "chkpt"), global_step=2)
    stored = dict(np.load(path))
    w = enc.get_weights()
    for k, h0 in (("dense_1/kernel", head[0]), ("dense_1/bias", head[1])):
        rms, mom = stored[k + "/RMSProp"], stored[k + "/RMSProp_1"]
        if variational:     # (the bias's RMSProp steps, about lr * grad, stay below half an ulp of its 0.5)
            assert not np.all(rms == 1) and np.abs(mom).max() > 0, k
        else:
            assert np.array_equal(w[k], h0) and np.all(rms == 1) and np.all(mom == 0), k
    assert np.array_equal(w["dense_1/kernel"], head[0]) != bool(variational)
    assert not np.all(stored["dense/kernel/RMSProp"] == 1)


def test_refusals_leave_the_process_healthy(sess):
    """create_opt: a kind outside aae_optimizer_kind, an initial accumulator <= 0 (AAE_ERR_INVALID_ARG), an inference-only fp16
    encoder for every rule (AAE_ERR_UNSUPPORTED); get_state / set_state with a slot the rule does not have (AAE_ERR_INVALID_ARG).
    A trainer then still steps as before."""
    from augmentedautoencoder_b200 import _lib
    lib = _lib.lib()
    enc, dec, top = _small_ae("Adagrad")
    xb, yb = _batch(4, 16)
    first = top.step_device(xb, yb, update=False).item()
    eh, dh = enc.handle(sess.device), dec.handle(sess.device)

    def create(kind, hp0=0.1, e=eh, d=dh, gemm=FP32):
        th = C.c_void_p()
        opt = _lib.Optimizer(kind, 2e-4, (C.c_float * 4)(hp0, 0.999, 1e-8))
        st = lib.aae_trainer_create_opt(e, d, 4, C.byref(opt), gemm, C.byref(th))
        assert (st == 0) == bool(th.value)
        if th.value:
            lib.aae_trainer_destroy(th)
        return st
    assert create(7) == -1 and b"aae_optimizer_kind" in lib.aae_last_error_string()
    assert create(-1) == -1
    for kind in (_lib.OPT_ADAGRAD, _lib.OPT_PROXIMAL_ADAGRAD, _lib.OPT_FTRL):
        for hp0 in (0.0, -0.1):
            assert create(kind, hp0) == -1 and b"initial accumulator" in lib.aae_last_error_string()
    assert all(create(k) == 0 for k in range(7))
    cfg = _lib.make_cfg(128, 128, 3, list(O.NUM_FILTER), list(O.STRIDES), 5, 128, 4, FP16)
    cfg_d = _lib.make_cfg(128, 128, 3, list(O.NUM_FILTER), list(O.STRIDES), 5, 128, 4, SPLIT)
    fe, sd = C.c_void_p(), C.c_void_p()
    _lib.check(lib.aae_encoder_create(0, C.byref(cfg), C.byref(fe)), "fp16 encoder")
    _lib.check(lib.aae_decoder_create(0, C.byref(cfg_d), C.byref(sd)), "split decoder")
    try:
        for kind in range(7):
            for gemm in (FP16, SPLIT):
                assert create(kind, e=fe, d=sd, gemm=gemm) == -3, (kind, gemm)
    finally:
        lib.aae_encoder_destroy(fe)
        lib.aae_decoder_destroy(sd)
    h = top.trainer(sess.device)
    k, b = np.empty((5, 5, 3, 4), np.float32), np.empty(4, np.float32)
    assert lib.aae_trainer_get_state(h, 0, 0, None, _lib.ptr(k), None, None, None) == -1
    assert b"slot" in lib.aae_last_error_string()
    assert lib.aae_trainer_set_state(h, 0, 0, None, None, None, _lib.ptr(b), None) == -1
    assert lib.aae_trainer_get_state(h, 0, 0, _lib.ptr(k), None, _lib.ptr(b), None, None) == 0
    assert np.all(k == np.float32(0.1)) and np.all(b == np.float32(0.1))
    gd_enc, gd_dec, gd = _small_ae("GradientDescent")
    assert lib.aae_trainer_get_state(gd.trainer(sess.device), 0, 0, _lib.ptr(k), None, None, None, None) == -1
    assert gd.optimizer_variables() == {}
    assert top.step_device(xb, yb, update=False).item() == first
    torch.cuda.synchronize()
