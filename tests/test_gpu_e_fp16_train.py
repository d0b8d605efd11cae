"""GPU tests of the single-pass fp16 trainer (aae_trainer_create_prec / TrainOp(precision=PREC_TC_FP16)): the forward, dgrad
and wgrad GEMMs round every operand once to fp16 and issue one hi*hi product per K step.

The bounds come from the rounding model (include/aae_b200.h, DESIGN.md section 3), not from measurement.  One GEMM y = a w adds
at most U = 2^-9 (products: 2^-10 + 2^-22 each, doubled for the fp32 accumulation) + 2^-11 (hi-only storage of its result) of
its magnitude |a| |w|; relative to y in the L2 norm that is U k with k = ||(|a| |w|)|| / ||y||, the GEMM's condition, which the
float64 oracle evaluates for every forward, dgrad and wgrad GEMM on the exact operands.  Along a chain the per-GEMM terms add:
a gradient's bound is the sum of U k over the forward GEMMs, the loss-gradient perturbation that their error causes, and the
backward GEMMs from the loss to it, doubled for the second-order terms and the fp32 elementwise passes between the GEMMs.
This is the linearised error model, not a worst case: it takes the layers after a GEMM to pass its relative error on without
amplification.  Worst-case magnitudes compound by the condition of every later layer and say nothing after ten layers."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import aae_oracle as O
from tests.test_gpu_a_parity import sess  # noqa: F401

pytestmark = pytest.mark.gpu

FP32, SPLIT, FP16 = 0, 1, 2
U = 2.0 ** -9 + 2.0 ** -11
# forward order; kind: enc = 5x5/s2 conv, dense, dense1 = decoder dense + reshape, dec = x2 resize + 5x5 conv, out = output layer
LAYERS = [("conv2d", "enc"), ("conv2d_1", "enc"), ("conv2d_2", "enc"), ("conv2d_3", "enc"), ("dense", "dense"), ("dense_1", "dense1"),
          ("conv2d_4", "dec"), ("conv2d_5", "dec"), ("conv2d_6", "dec"), ("conv2d_7", "out")]


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to("cuda", torch.float64)


def _apply(kind, a, w, b):
    if kind == "enc":
        return O.conv2d_same(a, w, b, 2, None)
    if kind in ("dense", "dense1"):
        return a.reshape(a.shape[0], -1) @ w + b
    return O.conv2d_same(O.resize_nearest_2x(a, (2 * a.shape[1], 2 * a.shape[2])), w, b, 1, None)


def _cond(m, v):
    return float(m.norm() / max(float(v.norm()), 1e-300))


def _analyse(x, y, ep, dp, bootstrap):
    """float64 forward; the relative forward error of the rounded pre-activations, the loss gradient and its error, and the bound on
    the loss."""
    P = {k: _dev(v) for k, v in {**ep, **dp}.items()}
    a = _dev(x)
    ins, masks, fwd_rel, relu_need = [], [], 0.0, 0.0
    for name, kind in LAYERS:
        w, b = P[name + "/kernel"], P[name + "/bias"]
        ins.append(a)
        pre = _apply(kind, a, w, b)
        fwd_rel += U * _cond(_apply(kind, a.abs(), w.abs(), torch.zeros_like(b)), pre)   # the bias is added in fp32
        if kind == "out":
            break
        if kind == "dense":
            a = pre
            masks.append(None)
            continue
        relu_need = max(relu_need, fwd_rel * float(pre.abs().max()))
        m = (pre > 0).double()
        if kind == "dense1":
            pre, m = (t.reshape(-1, 8, 8, t.shape[1] // 64) for t in (pre, m))
        masks.append(m)
        a = pre * m
    rec = torch.sigmoid(pre)
    sig = rec * (1 - rec)
    B = rec.shape[0]
    yd = _dev(y)
    l2 = ((rec - yd) ** 2).reshape(B, -1)
    k = l2.shape[1] // bootstrap if bootstrap > 1 else l2.shape[1]
    sel = torch.zeros_like(l2).scatter_(1, torch.topk(l2, k, dim=1).indices, 1.0).reshape(rec.shape)
    d_rec = sig * fwd_rel * float(pre.abs().max())               # forward error of the reconstruction
    seed = (2.0 / (B * k)) * sel * (rec - yd) * sig
    d_seed = (2.0 / (B * k)) * sel * (sig + (rec - yd).abs()) * d_rec
    dl2 = (2 * (rec - yd).abs() * d_rec + d_rec ** 2).reshape(B, -1)
    loss_bound = float(torch.topk(dl2, k, dim=1).values.sum() / (B * k))   # top-k sums are subadditive
    return dict(P=P, ins=ins, masks=masks, seed=seed, seed_rel=_cond(d_seed, seed), fwd_rel=fwd_rel, loss_bound=loss_bound,
                relu_need=relu_need)


def _grad_bounds(A):
    """{variable: bound on the relative L2 error of its gradient}, walking the backward GEMM chain with the exact gradients"""
    out, g, bwd_rel = {}, A["seed"], 0.0
    for i in reversed(range(len(LAYERS))):
        name, kind = LAYERS[i]
        ops = (A["ins"][i], A["P"][name + "/kernel"], A["P"][name + "/bias"])
        val = [t.detach().clone().requires_grad_(True) for t in ops]
        mag = [t.abs().detach().clone().requires_grad_(True) for t in ops]
        yv = _apply(kind, *val)
        yv.backward(g.reshape(yv.shape))
        _apply(kind, *mag).backward(g.abs().reshape(yv.shape))
        base = A["fwd_rel"] + A["seed_rel"] + bwd_rel
        out[name + "/kernel"] = 2 * (base + U * _cond(mag[1].grad, val[1].grad))
        out[name + "/bias"] = 2 * (base + U * _cond(mag[2].grad, val[2].grad))
        if i > 0:
            bwd_rel += U * _cond(mag[0].grad, val[0].grad)          # the dgrad GEMM into the layer's input
            g = val[0].grad if A["masks"][i - 1] is None else val[0].grad * A["masks"][i - 1].reshape(val[0].grad.shape)
    return out


def _check_grads(grads, g64, bounds, tag):
    worst, worst_rel = 0.0, 0.0
    for name, gr in g64.items():
        assert np.all(np.isfinite(grads[name])), (tag, name)
        rel = float(np.linalg.norm(grads[name].astype(np.float64) - gr) / max(np.linalg.norm(gr), 1e-300))
        assert rel <= bounds[name], (tag, name, rel, bounds[name])
        worst, worst_rel = max(worst, rel / bounds[name]), max(worst_rel, rel)
    print("%s: largest relative L2 gradient error %.2e, largest share of its bound used %.3f" % (tag, worst_rel, worst))


def _clear_margin_params():
    """Weights scaled down and biases in [1, 2]: every ReLU unit is active with a margin far outside the fp16 rounding, so the
    exact and the rounded forward take the same ReLU path and every GEMM chain is exercised end to end."""
    ep, dp = O.make_encoder_params(42), O.make_decoder_params(43)
    rng = np.random.RandomState(5)
    for p in (ep, dp):
        for k in p:
            if k.endswith("kernel"):
                p[k] = (p[k] * 0.05).astype(np.float32)
            else:
                p[k] = rng.uniform(1.0, 2.0, p[k].shape).astype(np.float32)
    return ep, dp


def _pair(prec, B, ep, dp, bootstrap=4, handles=SPLIT):
    from augmentedautoencoder_b200.ae.ae import AE
    from augmentedautoencoder_b200.ae.ae_factory import TrainOp
    from augmentedautoencoder_b200.ae.decoder import Decoder
    from augmentedautoencoder_b200.ae.encoder import Encoder
    from augmentedautoencoder_b200.ae.session import placeholder
    x, y = placeholder(np.float32, [None, 128, 128, 3]), placeholder(np.float32, [None, 128, 128, 3])
    enc = Encoder(x, 128, list(O.NUM_FILTER), 5, list(O.STRIDES), False, is_training=True, max_batch=B, precision=handles)
    dec = Decoder(y, enc.z, list(reversed(O.NUM_FILTER)), 5, list(reversed(O.STRIDES)), "L2", bootstrap, False, False, is_training=True,
                  max_batch=B, precision=handles)
    enc.load_weights(ep)
    dec.load_weights(dp)
    return enc, dec, TrainOp(AE(enc, dec, 0, 0), 2e-4, precision=prec)


def _grads_of(prec, ep, dp, xb, yb, bootstrap, sess):
    enc, dec, top = _pair(prec, 2, ep, dp, bootstrap)
    loss = float(top.step_device(torch.from_numpy(xb).cuda(), torch.from_numpy(yb).cuda(), update=False))
    assert enc.precision == SPLIT and dec.precision == SPLIT
    return loss, top.gradients(sess.device)


def test_fp16_trainer_loss_and_gradients_meet_the_rounding_bound(sess):
    """One forward/backward at batch 1 without bootstrapping (a discrete top-k choice is no rounding error): the loss and all
    20 gradients of the single-pass trainer, and of the split trainer, within the bound of the rounding model."""
    ep, dp = _clear_margin_params()
    xb = np.random.RandomState(8).rand(1, 128, 128, 3).astype(np.float32)
    yb = np.random.RandomState(4).rand(1, 128, 128, 3).astype(np.float32)
    A = _analyse(xb, yb, ep, dp, 1)
    margin = O.relu_margin(xb, ep, dp)
    print("relu margin %.3e, largest forward rounding of a ReLU input %.3e, forward relative error bound %.2e"
          % (margin, A["relu_need"], A["fwd_rel"]))
    assert margin > 2 * A["relu_need"]
    loss64, _, g64 = O.ae_forward_loss(xb, yb, ep, dp, dtype=torch.float64, bootstrap_ratio=1, with_grads=True)
    bounds = _grad_bounds(A)
    for prec, tag in ((FP16, "fp16 trainer"), (SPLIT, "split trainer")):
        loss, grads = _grads_of(prec, ep, dp, xb, yb, 1, sess)
        print("%s: |loss - loss64| = %.3e, bound %.3e" % (tag, abs(loss - loss64), 2 * A["loss_bound"]))
        assert abs(loss - loss64) <= 2 * A["loss_bound"]
        _check_grads(grads, g64, bounds, tag)


@pytest.mark.parametrize("case", ["tiny", "large"])
def test_fp16_trainer_keeps_tiny_and_large_gradients_normal(sess, case):
    """The per-tensor power-of-two scale keeps a hi-only gradient a normal fp16 whatever its range: a target within 1e-4 of the
    reconstruction (loss gradients ~1e-9 and below, under fp16's smallest subnormal without the scale) and the complement of
    the reconstruction.  Both give finite, non-zero gradients within the bound of the test above."""
    ep, dp = _clear_margin_params()
    xb = np.random.RandomState(8).rand(1, 128, 128, 3).astype(np.float32)
    _, rec, _ = O.ae_forward_loss(xb, xb, ep, dp, dtype=torch.float64, bootstrap_ratio=1)
    noise = np.random.RandomState(6).uniform(-1e-4, 1e-4, rec.shape)
    yb = (rec + noise if case == "tiny" else 1.0 - rec).astype(np.float32)
    A = _analyse(xb, yb, ep, dp, 1)
    _, _, g64 = O.ae_forward_loss(xb, yb, ep, dp, dtype=torch.float64, bootstrap_ratio=1, with_grads=True)
    _, grads = _grads_of(FP16, ep, dp, xb, yb, 1, sess)
    for name, g in grads.items():
        assert np.any(g != 0), name
    print("%s target: largest |gradient| %.3e" % (case, max(float(np.abs(g).max()) for g in grads.values())))
    _check_grads(grads, g64, _grad_bounds(A), "fp16 trainer, %s target" % case)


def test_fp16_trainer_trajectory_follows_the_split_trainer(sess):
    """Five Adam steps at batch 3 (ragged against the 128-row tiles), bootstrapped loss.  The loss goes down, and at every step
    the two trainers' losses differ by at most twice the forward rounding bound of the loss plus the first-order change
    sum |dL/dw| |w_fp16 - w_split| that the different weights explain."""
    ep, dp = O.make_encoder_params(42, bias_scale=0.02), O.make_decoder_params(43, bias_scale=0.02)
    xn = np.random.RandomState(11).rand(3, 128, 128, 3).astype(np.float32)
    yn = np.random.RandomState(12).rand(3, 128, 128, 3).astype(np.float32)
    xb, yb = torch.from_numpy(xn).cuda(), torch.from_numpy(yn).cuda()
    run = {prec: _pair(prec, 4, ep, dp) for prec in (FP16, SPLIT)}
    losses = {FP16: [], SPLIT: []}
    for t in range(5):
        w = {prec: {**e.get_weights(short_names=True), **d.get_weights(short_names=True)} for prec, (e, d, _) in run.items()}
        for prec, (_, _, top) in run.items():
            losses[prec].append(float(top.step_device(xb, yb, update=True)))
        g = run[SPLIT][2].gradients(sess.device)
        drift = sum(float(np.sum(np.abs(g[k].astype(np.float64)) * np.abs(w[FP16][k].astype(np.float64) - w[SPLIT][k]))) for k in g)
        bound = 2 * (_analyse(xn, yn, w[SPLIT], {}, 4)["loss_bound"] + drift)
        diff = abs(losses[FP16][t] - losses[SPLIT][t])
        print("step %d: fp16 %.6f, split %.6f, |diff| %.3e, bound %.3e (weight drift term %.3e)"
              % (t + 1, losses[FP16][t], losses[SPLIT][t], diff, bound, drift))
        assert diff <= bound
    assert losses[FP16][-1] < losses[FP16][0]


def test_fp16_training_updates_the_masters_that_split_inference_reads(sess):
    """The trainer's Adam updates the handles' fp32 masters in place: after fp16 steps the handles' get_weights() equal a replay of
    TF-Adam over the trainer's own gradients, the handles stay split, and a forward on them equals fresh split handles loaded
    from those weights."""
    from augmentedautoencoder_b200.ae.decoder import Decoder
    from augmentedautoencoder_b200.ae.encoder import Encoder
    from augmentedautoencoder_b200.ae.session import placeholder
    ep, dp = O.make_encoder_params(42, bias_scale=0.02), O.make_decoder_params(43, bias_scale=0.02)
    enc, dec, top = _pair(FP16, 4, ep, dp)
    xb = torch.from_numpy(np.random.RandomState(11).rand(3, 128, 128, 3).astype(np.float32)).cuda()
    yb = torch.from_numpy(np.random.RandomState(12).rand(3, 128, 128, 3).astype(np.float32)).cuda()
    z_before = enc.encode_device(xb).clone()
    w = {**ep, **dp}
    m = {k: np.zeros_like(v) for k, v in w.items()}
    v = {k: np.zeros_like(v) for k, v in w.items()}
    moved = {k: np.zeros_like(v) for k, v in w.items()}         # sum over the steps of |update|
    for t in (1, 2):
        top.step_device(xb, yb, update=True)
        g = top.gradients(sess.device)
        for k in w:
            w_prev = w[k]
            w[k], m[k], v[k] = O.tf_adam_step(w[k], g[k], m[k], v[k], t)
            moved[k] += np.abs(w[k] - w_prev)
    got = {**enc.get_weights(short_names=True), **dec.get_weights(short_names=True)}
    # the kernel forms 1 - beta in fp32 and the replay in float64 (1.3e-5 apart for beta2 = 0.999), and may fuse multiply-adds:
    # the two agree to 2e-4 of the updates
    worst = 0.0
    for k in w:
        err = np.abs(got[k] - w[k])
        assert np.all(err <= 2e-4 * moved[k] + 4 * np.spacing(np.abs(w[k]))), k
        worst = max(worst, float(np.max(err / (moved[k] + 1e-30))))
    print("masters vs TF-Adam replay over the trainer's gradients: largest difference %.2e of the updates" % worst)
    assert enc.precision == SPLIT and dec.precision == SPLIT
    z_after = enc.encode_device(xb).clone()
    rec_after = dec.decode_device(z_after).clone()
    assert float((z_after - z_before).abs().max()) > 1e-4
    e2 = Encoder(placeholder(np.float32, [None, 128, 128, 3]), 128, list(O.NUM_FILTER), 5, list(O.STRIDES), False, max_batch=4, precision=SPLIT)
    d2 = Decoder(placeholder(np.float32, [None, 128, 128, 3]), e2.z, list(reversed(O.NUM_FILTER)), 5, list(reversed(O.STRIDES)), "L2", 4,
                 False, False, max_batch=4, precision=SPLIT)
    e2.load_weights(enc.get_weights())
    d2.load_weights(dec.get_weights())
    z_fresh = e2.encode_device(xb)
    assert torch.equal(z_after, z_fresh)
    assert torch.equal(rec_after, d2.decode_device(z_fresh))


def test_fp16_training_resumes_bit_identically(sess):
    """Adam slots and beta powers saved after two fp16 steps and restored into a new fp16 trainer: the third step is
    bit-identical to running three steps in one go (loss and every weight)."""
    ep, dp = O.make_encoder_params(42, bias_scale=0.02), O.make_decoder_params(43, bias_scale=0.02)
    xb = torch.from_numpy(np.random.RandomState(11).rand(3, 128, 128, 3).astype(np.float32)).cuda()
    yb = torch.from_numpy(np.random.RandomState(12).rand(3, 128, 128, 3).astype(np.float32)).cuda()
    enc, dec, top = _pair(FP16, 4, ep, dp)
    for _ in range(2):
        top.step_device(xb, yb)
    state = top.optimizer_variables()
    assert "conv2d_1/kernel/Adam" in state and abs(float(state["beta1_power"]) - 0.9 ** 3) < 1e-7
    ew, dw = enc.get_weights(short_names=True), dec.get_weights(short_names=True)
    l3 = float(top.step_device(xb, yb))
    enc2, dec2, top2 = _pair(FP16, 4, ew, dw)
    top2.load_optimizer_variables(state, sess.device)
    l3b = float(top2.step_device(xb, yb))
    assert l3 == l3b, (l3, l3b)
    for a, b in ((enc, enc2), (dec, dec2)):
        wa, wb = a.get_weights(short_names=True), b.get_weights(short_names=True)
        for k in wa:
            assert np.array_equal(wa[k], wb[k]), k


def test_fp16_trainer_refusals_leave_the_process_healthy(sess):
    """aae_trainer_create_prec refuses every combination but (handles' own precision) and (fp16 GEMMs, split handles), through the
    C ABI and through TrainOp, without switching any precision; after each refusal a split trainer still trains."""
    from augmentedautoencoder_b200 import _lib
    lib = _lib.lib()
    ep, dp = O.make_encoder_params(42, bias_scale=0.02), O.make_decoder_params(43, bias_scale=0.02)
    xb = torch.from_numpy(np.random.RandomState(11).rand(3, 128, 128, 3).astype(np.float32)).cuda()
    yb = torch.from_numpy(np.random.RandomState(12).rand(3, 128, 128, 3).astype(np.float32)).cuda()
    _, _, healthy = _pair(None, 4, ep, dp)
    first = float(healthy.step_device(xb, yb, update=False))

    def still_trains():
        assert float(healthy.step_device(xb, yb, update=False)) == first

    def cfg(prec):
        return _lib.make_cfg(128, 128, 3, list(O.NUM_FILTER), list(O.STRIDES), 5, 128, 4, prec)
    names = {FP32: b"AAE_PREC_FP32_SIMT", SPLIT: b"AAE_PREC_TC_SPLIT", FP16: b"AAE_PREC_TC_FP16"}
    cases = [((FP32, FP32), FP16, -3), ((FP16, SPLIT), FP16, -3), ((FP32, FP32), SPLIT, -3), ((SPLIT, SPLIT), FP32, -3),
             ((SPLIT, FP32), SPLIT, -3), ((SPLIT, SPLIT), 3, -1), ((SPLIT, SPLIT), -1, -1), ((SPLIT, SPLIT), SPLIT, 0),
             ((FP32, FP32), FP32, 0), ((SPLIT, SPLIT), FP16, 0)]
    for (pe, pd), gemm, want in cases:
        eh, dh, th = C.c_void_p(), C.c_void_p(), C.c_void_p()
        _lib.check(lib.aae_encoder_create(0, C.byref(cfg(pe)), C.byref(eh)), "encoder create")
        _lib.check(lib.aae_decoder_create(0, C.byref(cfg(pd)), C.byref(dh)), "decoder create")
        try:
            st = lib.aae_trainer_create_prec(eh, dh, 4, 2e-4, 0.9, 0.999, 1e-8, gemm, C.byref(th))
            assert st == want, ((pe, pd), gemm, st, lib.aae_last_error_string())
            if want == 0:
                assert th.value
                lib.aae_trainer_destroy(th)
            else:
                assert not th.value
                msg = lib.aae_last_error_string()
                if want == -3:
                    assert names[gemm] in msg and names[pe] in msg and names[pd] in msg, msg
                else:
                    assert b"gemm_precision" in msg, msg
        finally:
            lib.aae_encoder_destroy(eh)
            lib.aae_decoder_destroy(dh)
        still_trains()
    # TrainOp: explicit fp32 handles, and automatic handles that fell back to fp32 for their geometry (Cin 96 is no tensor-core
    # layer); both raise and keep the handles' precision
    for handles, filters in ((FP32, list(O.NUM_FILTER)), (None, [128, 96, 512, 512])):
        from augmentedautoencoder_b200.ae.ae import AE
        from augmentedautoencoder_b200.ae.ae_factory import TrainOp
        from augmentedautoencoder_b200.ae.decoder import Decoder
        from augmentedautoencoder_b200.ae.encoder import Encoder
        from augmentedautoencoder_b200.ae.session import placeholder
        x, y = placeholder(np.float32, [None, 128, 128, 3]), placeholder(np.float32, [None, 128, 128, 3])
        enc = Encoder(x, 128, filters, 5, list(O.STRIDES), False, is_training=True, max_batch=4, precision=handles)
        dec = Decoder(y, enc.z, list(reversed(filters)), 5, list(reversed(O.STRIDES)), "L2", 4, False, False, is_training=True, max_batch=4,
                      precision=handles)
        top = TrainOp(AE(enc, dec, 0, 0), 2e-4, precision=FP16)
        with pytest.raises(_lib.AaeError, match="AAE_PREC_TC_FP16.*AAE_PREC_FP32_SIMT"):
            top.trainer(sess.device)
        assert enc.precision == FP32 and dec.precision == FP32
        still_trains()


def test_fp16_trainer_reports_range_overflow_through_the_handles(sess):
    """The private single-pass plans share the handles' range guard: an activation of the training forward outside the fp16 range
    is reported by the handle's range check (the check Session.run makes after sess.run(train_op)), naming the layer."""
    from augmentedautoencoder_b200._lib import AaeError
    ep, dp = O.make_encoder_params(42, bias_scale=0.02), O.make_decoder_params(43, bias_scale=0.02)
    xb = torch.from_numpy(np.random.RandomState(11).rand(3, 128, 128, 3).astype(np.float32)).cuda()
    yb = torch.from_numpy(np.random.RandomState(12).rand(3, 128, 128, 3).astype(np.float32)).cuda()
    for which, name, index, layer in ((0, "conv2d_1/bias", 7, 1), (1, "dense_1/bias", 11, 0)):
        e, d = dict(ep), dict(dp)
        p = e if which == 0 else d
        p[name] = p[name].copy()
        p[name][index] = 5000.0
        enc, dec, top = _pair(FP16, 4, e, d)
        top.step_device(xb, yb, update=False)
        mod = enc if which == 0 else dec
        with pytest.raises(AaeError, match=r"activation.*layer\(s\) %d" % layer):
            mod.check_range(sess.device)
        mod.check_range(sess.device)                                  # the report cleared the word
