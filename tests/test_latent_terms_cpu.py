"""CPU tests of the latent terms of the AE loss (VARIATIONAL, NORM_REGULARIZE; auto_pose/ae/encoder.py:70-100, ae.py:43-53):
the oracle's known answers and gradients, and the TF variable names of the graph with and without the sigma head."""
import configparser

import numpy as np
import pytest
import torch

from oracle import latent_oracle as LO


def test_kl_and_norm_terms_meet_known_answers():
    z = torch.zeros(3, 8, dtype=torch.float64)
    assert float(LO.kl_div_loss(z, torch.ones_like(z))) == 0.0
    u = torch.randn(4, 8, dtype=torch.float64, generator=torch.Generator().manual_seed(0))
    assert abs(float(LO.norm_reg_loss(u / torch.linalg.vector_norm(u, dim=1, keepdim=True)))) < 1e-15
    # a zero head gives sigma = 1e-8 + ln 2 everywhere (kernel_initializer=zeros, zero bias)
    s = LO.q_sigma(torch.rand(2, 5, dtype=torch.float64), torch.zeros(5, 3, dtype=torch.float64), torch.zeros(3, dtype=torch.float64))
    assert torch.allclose(s, torch.full_like(s, 1e-8 + np.log(2.0)), rtol=0, atol=1e-15)
    # KL(N(z, s) || N(0, 1)) = z^2/2 + (s^2 - 1)/2 - log s, averaged
    z, s = torch.tensor([[0.5, -1.0]], dtype=torch.float64), torch.tensor([[2.0, 0.25]], dtype=torch.float64)
    want = np.mean([0.125 + 1.5 - np.log(2.0), 0.5 + 0.5 * (0.0625 - 1.0) - np.log(0.25)])
    assert abs(float(LO.kl_div_loss(z, s)) - want) < 1e-15
    # sampled z: one scalar eps for every sample and dimension
    assert torch.equal(LO.sampled_z(z, s, -0.5), z - 0.5 * s)


def _central_diff(f, x, h=1e-6):
    g = torch.zeros_like(x)
    flat = x.view(-1)
    for i in range(flat.numel()):
        old = float(flat[i])
        flat[i] = old + h
        fp = float(f(x))
        flat[i] = old - h
        fm = float(f(x))
        flat[i] = old
        g.view(-1)[i] = (fp - fm) / (2 * h)
    return g


def test_latent_term_gradients_match_central_differences():
    gen = torch.Generator().manual_seed(3)
    z = torch.randn(3, 6, dtype=torch.float64, generator=gen)
    pre = torch.randn(3, 6, dtype=torch.float64, generator=gen)
    flat = torch.rand(3, 4, dtype=torch.float64, generator=gen)
    w = 0.3 * torch.randn(4, 6, dtype=torch.float64, generator=gen)
    b = 0.1 * torch.randn(6, dtype=torch.float64, generator=gen)

    def total(z_, w_, b_):
        s = LO.q_sigma(flat, w_, b_)
        return 0.7 * LO.kl_div_loss(z_, s) + 0.4 * LO.norm_reg_loss(z_) + (LO.sampled_z(z_, s, 0.8) ** 2).sum()
    zz, ww, bb = (t.clone().requires_grad_(True) for t in (z, w, b))
    total(zz, ww, bb).backward()
    with torch.no_grad():
        for got, var, f in ((zz.grad, z.clone(), lambda v: total(v, w, b)), (ww.grad, w.clone(), lambda v: total(z, v, b)),
                            (bb.grad, b.clone(), lambda v: total(z, w, v))):
            assert torch.allclose(got, _central_diff(f, var), rtol=1e-6, atol=1e-8)
    # the closed forms the CUDA kernel uses: d KL / dz = z / (B J), d KL / d sigma = (sigma - 1/sigma) / (B J),
    # d reg / dz = sign(|z| - 1) z / (|z| B), d softplus = sigmoid
    B, J = z.shape
    s = (1e-8 + torch.nn.functional.softplus(pre)).requires_grad_(True)
    zz = z.clone().requires_grad_(True)
    LO.kl_div_loss(zz, s).backward()
    assert torch.allclose(zz.grad, z / (B * J), rtol=1e-12) and torch.allclose(s.grad, (s - 1 / s).detach() / (B * J), rtol=1e-12)
    zz = z.clone().requires_grad_(True)
    LO.norm_reg_loss(zz).backward()
    n = torch.linalg.vector_norm(z, dim=1, keepdim=True)
    assert torch.allclose(zz.grad, torch.sign(n - 1) * z / (n * B), rtol=1e-12)
    # the whole graph with both heads and both terms (vae_forward_loss with mask_head): every one of its 16 gradients (24 at the
    # template's depth), keyed by the TF names of that graph, against central differences of the float64 loss at sampled entries
    x, y, ep, dp, head, mhead = _small_graph()
    kw = dict(head=head, mask_head=mhead, variational=0.7, norm_regularize=0.4, eps=0.8, dtype=torch.float64, bootstrap_ratio=1)
    _, _, g = LO.vae_forward_loss(x, y, ep, dp, with_grads=True, **kw)
    assert len(g) == 16 and sorted(g) == sorted(_small_graph_names())
    var = {**ep, **dp}
    var = {("dense_2" + k[7:] if k.startswith("dense_1/") else "conv2d_4" + k[8:] if k.startswith("conv2d_3/") else k): v.astype(np.float64)
           for k, v in var.items()}
    var.update({"dense_1/kernel": head[0].astype(np.float64), "dense_1/bias": head[1].astype(np.float64),
                "conv2d_3/kernel": mhead[0].astype(np.float64), "conv2d_3/bias": mhead[1].astype(np.float64)})
    assert sorted(var) == sorted(g)

    def loss_of(v):
        e = {k: v[k] for k in ep}
        d = {("dense_1" + k[7:] if k.startswith("dense_2/") else "conv2d_3" + k[8:] if k.startswith("conv2d_4/") else k): v[k]
             for k in v if k not in ep and k not in ("dense_1/kernel", "dense_1/bias", "conv2d_3/kernel", "conv2d_3/bias")}
        return LO.vae_forward_loss(x, y, e, d, **{**kw, "head": (v["dense_1/kernel"], v["dense_1/bias"]),
                                                  "mask_head": (v["conv2d_3/kernel"], v["conv2d_3/bias"])})[0]
    rng = np.random.RandomState(0)
    h = 1e-6
    for name in sorted(var):
        for i in rng.choice(var[name].size, min(4, var[name].size), replace=False):
            old = var[name].flat[i]
            var[name].flat[i] = old + h
            fp = loss_of(var)
            var[name].flat[i] = old - h
            fm = loss_of(var)
            var[name].flat[i] = old
            want = (fp - fm) / (2 * h)
            assert abs(g[name].flat[i] - want) <= 1e-6 * max(abs(want), 1e-3), (name, i, g[name].flat[i], want)


def _small_graph():
    """16x16 input, encoder filters (4, 8), latent 8, with a sigma head and a mask head: every variable of the graph with both heads
    at a size where central differences of the whole loss are cheap."""
    from oracle import aae_oracle as O
    from oracle import mask_oracle as MO
    geo = dict(num_filters=(4, 8), strides=(2, 2), latent=8, bias_scale=0.1)
    ep = O.make_encoder_params(5, in_hw=16, **geo)
    dp = O.make_decoder_params(6, out_hw=16, n_encoder_convs=2, **geo)
    rng = np.random.RandomState(7)
    head = ((0.3 * rng.standard_normal((128, 8))).astype(np.float32), (0.1 * rng.standard_normal(8)).astype(np.float32))
    mhead = MO.make_mask_head(8, 4, bias_scale=0.1)
    x = rng.rand(2, 16, 16, 3).astype(np.float32)
    y = rng.rand(2, 16, 16, 3).astype(np.float32)
    y[rng.rand(2, 16, 16) < 0.3] = 0.0                   # background pixels: the mask target takes both values
    return x, y, ep, dp, head, mhead


def _small_graph_names():
    """TF's names for _small_graph's graph with both heads: the sigma head is dense_1 and the decoder dense dense_2; the mask head
    is conv2d_3 (created before the output conv) and the output conv conv2d_4"""
    layers = ["conv2d", "conv2d_1", "dense", "dense_1", "dense_2", "conv2d_2", "conv2d_3", "conv2d_4"]
    return [l + "/" + p for l in layers for p in ("kernel", "bias")]


@pytest.mark.parametrize("terms", [(0.0, 0.0), (0.3, 0.0), (0.0, 0.4), (0.3, 0.4)])
def test_vae_oracle_without_the_mask_head_is_unchanged(terms):
    """vae_forward_loss without mask_head: the loss and gradients of the graph without the mask head, bit for bit -- with the terms
    off, aae_oracle.ae_forward_loss; with them on, that reconstruction loss plus the weighted terms composed in the reference's
    order, on the sampled z."""
    from oracle import aae_oracle as O
    x, y, ep, dp, head, _ = _small_graph()
    variational, norm = terms
    loss, t, g = LO.vae_forward_loss(x, y, ep, dp, head=head, variational=variational, norm_regularize=norm, eps=0.8,
                                     dtype=torch.float64, with_grads=True)
    assert len(g) == (14 if variational else 12) and not any(k.startswith("conv2d_4/") for k in g)
    if not variational and not norm:
        want, _, gw = O.ae_forward_loss(x, y, ep, dp, dtype=torch.float64, with_grads=True)
        assert loss == want and all(np.array_equal(g[k], gw[k]) for k in gw)
        return
    tp = {k: torch.from_numpy(v).double() for k, v in dp.items()}
    zin = torch.from_numpy(t["sampled_z"])
    rec = O.decoder_layers(zin, tp, out_hw=16, strides=(2, 2), n_encoder_convs=2)[-1]
    want = O.bootstrapped_l2(rec, torch.from_numpy(y).double(), 4)
    if norm:
        want = want + t["reg"] * norm
    if variational:
        want = want + t["kl"] * variational
    assert loss == float(want)


def test_vae_oracle_with_the_mask_head_and_the_terms_off_is_the_mask_oracle():
    """vae_forward_loss with mask_head and VARIATIONAL = NORM_REGULARIZE = 0 equals mask_oracle.mask_forward_loss: the same loss and
    the same 14 gradients under the same names, bit for bit"""
    from oracle import mask_oracle as MO
    x, y, ep, dp, head, mhead = _small_graph()
    loss, _, g = LO.vae_forward_loss(x, y, ep, dp, mask_head=mhead, dtype=torch.float64, with_grads=True)
    want, _, _, gw = MO.mask_forward_loss(x, y, ep, dp, mhead, dtype=torch.float64, with_grads=True)
    assert loss == want and sorted(g) == sorted(gw) and len(g) == 14
    assert all(np.array_equal(g[k], gw[k]) for k in gw)
    assert "conv2d_3/kernel" in g and g["conv2d_3/kernel"].shape == (5, 5, 4, 1) and g["conv2d_4/kernel"].shape == (5, 5, 4, 3)
    # the sigma head given but VARIATIONAL 0: still the mask oracle (the head is not part of that loss)
    loss2, _, g2 = LO.vae_forward_loss(x, y, ep, dp, head=head, mask_head=mhead, dtype=torch.float64, with_grads=True)
    assert loss2 == want and all(np.array_equal(g2[k], gw[k]) for k in gw) and len(g2) == 14


def _cfg(variational, norm_regularize=0.0):
    c = configparser.ConfigParser()
    c.read_dict({"Network": {"LATENT_SPACE_SIZE": "128", "NUM_FILTER": "[128, 256, 512, 512]", "KERNEL_SIZE_ENCODER": "5",
                             "KERNEL_SIZE_DECODER": "5", "STRIDES": "[2, 2, 2, 2]", "BATCH_NORMALIZATION": "False", "LOSS": "L2",
                             "BOOTSTRAP_RATIO": "4", "VARIATIONAL": str(variational), "AUXILIARY_MASK": "False",
                             "NORM_REGULARIZE": str(norm_regularize)},
                 "Training": {"BATCH_SIZE": "4", "LEARNING_RATE": "2e-4", "OPTIMIZER": "Adam"}})
    return c


def _graph(variational, is_training):
    from augmentedautoencoder_b200.ae import ae_factory as F
    from augmentedautoencoder_b200.ae import session as S
    args = _cfg(variational)
    with S.variable_scope("obj_01"):
        x = S.placeholder(np.float32, [None, 128, 128, 3])
        y = S.placeholder(np.float32, [None, 128, 128, 3])
        enc = F.build_encoder(x, args, is_training=is_training)
        dec = F.build_decoder(y, enc, args, is_training=is_training)
        ae = F.build_ae(enc, dec, args) if is_training else None
    return enc, dec, ae


def test_variable_names_with_and_without_the_sigma_head():
    enc, dec, ae = _graph(0.1, True)
    assert enc.variable_names[-4:] == ["obj_01/dense/kernel", "obj_01/dense/bias", "obj_01/dense_1/kernel", "obj_01/dense_1/bias"]
    w = enc.get_weights()
    assert w["obj_01/dense_1/kernel"].shape == (32768, 128) and not w["obj_01/dense_1/kernel"].any()   # zeros initialiser
    assert w["obj_01/dense_1/bias"].shape == (128,) and not w["obj_01/dense_1/bias"].any()
    assert dec.variable_names == ["obj_01/dense_2/kernel", "obj_01/dense_2/bias"] + \
        ["obj_01/conv2d_%d/%s" % (k, v) for k in range(4, 8) for v in ("kernel", "bias")]
    assert dec._latent_code is enc.sampled_z and ae._variational == 0.1
    # without VARIATIONAL every name stays as it is
    enc0, dec0, _ = _graph(0.0, True)
    assert "obj_01/dense_1/kernel" not in enc0.variable_names and dec0.variable_names[0] == "obj_01/dense_1/kernel"
    assert dec0._latent_code is enc0.z
    # an inference graph never builds the head, whatever the cfg says (build_decoder reads VARIATIONAL only when training)
    enc1, dec1, _ = _graph(0.1, False)
    assert enc1.variable_names == enc0.variable_names and dec1.variable_names == dec0.variable_names


def test_inference_graph_restores_a_variational_checkpoint(tmp_path):
    from augmentedautoencoder_b200.ae import ae_factory as F
    enc, dec, _ = _graph(0.1, True)
    head = np.random.RandomState(0).standard_normal((32768, 128)).astype(np.float32) * 1e-3
    enc.load_weights({"obj_01/dense_1/kernel": head}, strict=False)
    path = F.Saver([enc, dec]).save(None, str(tmp_path / "chkpt"), global_step=5)
    stored = np.load(path)
    assert "obj_01/dense_1/kernel" in stored.files and "obj_01/dense_2/kernel" in stored.files
    assert np.array_equal(stored["obj_01/dense_1/kernel"], head)
    # the encoder of an inference graph restores strictly (the head is simply not read)
    enc1, dec1, _ = _graph(0.1, False)
    F.Saver([enc1]).restore(None, path)
    assert np.array_equal(enc1.get_weights()["obj_01/dense/kernel"], enc.get_weights()["obj_01/dense/kernel"])
    # its decoder would read the head as its dense_1: refused, naming the shape, and nothing is loaded
    before = dec1.get_weights()["obj_01/dense_1/kernel"].copy()
    with pytest.raises(ValueError, match=r"dense_1/kernel: shape \(32768, 128\) != expected \(128, 32768\)"):
        F.Saver([enc1, dec1]).restore(None, path)
    assert np.array_equal(dec1.get_weights()["obj_01/dense_1/kernel"], before)


def test_variational_training_needs_the_decoder_on_the_sampled_z():
    from augmentedautoencoder_b200.ae.ae import AE
    from augmentedautoencoder_b200.ae.ae_factory import TrainOp
    enc0, dec0, _ = _graph(0.0, True)
    top = TrainOp(AE(enc0, dec0, 0.0, 0.1), 2e-4)
    with pytest.raises(NotImplementedError, match="sampled_z"):
        top.trainer(torch.device("cuda", 0))
