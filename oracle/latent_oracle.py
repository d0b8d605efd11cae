"""CPU oracle of the latent terms of the AE loss (VARIATIONAL and NORM_REGULARIZE).  TEST INFRASTRUCTURE ONLY, like
aae_oracle.py, whose TF op restatements it builds on: torch on the CPU, float64 = "truth", float32 = "TF stand-in".
Restates auto_pose/ae/encoder.py:70-100, ae.py:43-53 and ae_factory.py:50-77 (paths relative to /root/reference)."""
from __future__ import annotations

from typing import Dict, Optional, Tuple

import numpy as np
import torch
import torch.nn.functional as F

from oracle.aae_oracle import BOOTSTRAP_RATIO, STRIDES, _check_device, _t, bootstrapped_l2, conv2d_same, decoder_layers
from oracle.mask_oracle import decoder_with_mask, mask_loss, mask_target


def q_sigma(flat: torch.Tensor, kernel: torch.Tensor, bias: torch.Tensor) -> torch.Tensor:
    """1e-8 + tf.layers.dense(encoder_out, latent, activation=tf.nn.softplus) (encoder.py:70-79)."""
    return 1e-8 + F.softplus(flat @ kernel + bias)


def sampled_z(z: torch.Tensor, sigma: torch.Tensor, eps: float) -> torch.Tensor:
    """z + q_sigma * eps with eps = tf.random_normal(tf.shape(<python int>)): ONE scalar for the whole batch
    (encoder.py:81-84)."""
    return z + sigma * eps


def kl_div_loss(z: torch.Tensor, sigma: torch.Tensor) -> torch.Tensor:
    """reduce_mean(kl_divergence(Normal(z, sigma), Normal(0, 1))) in TF's form (z^2 + sigma^2 - 1 - log sigma^2) / 2
    (encoder.py:87-94)."""
    s2 = sigma * sigma
    return (0.5 * z * z + 0.5 * (s2 - 1.0 - torch.log(s2))).mean()


def norm_reg_loss(z: torch.Tensor) -> torch.Tensor:
    """reduce_mean(|norm(z, axis=1) - 1|) (encoder.py:97-100)."""
    return (torch.linalg.vector_norm(z, dim=1) - 1.0).abs().mean()


def vae_forward_loss(x: np.ndarray, target: np.ndarray, enc: Dict[str, np.ndarray], dec: Dict[str, np.ndarray],
                     head: Optional[Tuple[np.ndarray, np.ndarray]] = None, variational: float = 0.0,
                     norm_regularize: float = 0.0, eps: float = 0.0, dtype: torch.dtype = torch.float32,
                     bootstrap_ratio: int = BOOTSTRAP_RATIO, with_grads: bool = False, device: str = "cpu",
                     mask_head: Optional[Tuple[np.ndarray, np.ndarray]] = None):
    """AE.loss with the latent terms (ae.py:43-53): reconstr_loss, + reg_loss * norm_regularize if that is > 0, + kl_div_loss *
    variational if that is non-zero; the decoder reads sampled_z when variational is set (ae_factory.py:58).
    ``enc`` / ``dec`` as for aae_oracle.ae_forward_loss (decoder dense under "dense_1"); ``head`` = (kernel [flat, latent],
    bias [latent]) of the sigma head, required when variational.  ``mask_head`` = (kernel [k, k, cin, 1], bias [1]) of the
    decoder's AUXILIARY_MASK head: the decoder is then mask_oracle.decoder_with_mask and reconstr_loss includes the mask loss
    (decoder.py:134-142), before the latent terms are added.
    Returns (loss, terms, grads or None).  terms: z, q_sigma, sampled_z, xmask (numpy), kl, reg (floats).  Gradients are keyed by the
    TF names of the graph built: with variational the head is "dense_1" and the decoder dense "dense_2"; with the mask head that
    head is conv2d_<k> and the output conv conv2d_<k+1> (k = encoder convs + decoder hidden convs: conv2d_7 / conv2d_8 for the
    template); otherwise the plain names.
    device="cuda" evaluates the graph on the GPU (float64 only), as aae_oracle.ae_forward_loss."""
    if variational and head is None:
        raise ValueError("variational needs the sigma head")
    _check_device(dtype, device)
    tp = {k: _t(v, dtype, device).requires_grad_(with_grads) for k, v in {**enc, **dec}.items()}
    hk = hb = None
    if head is not None:
        hk, hb = (_t(a, dtype, device).requires_grad_(with_grads) for a in head)
    if mask_head is not None:
        mk, mb = (_t(a, dtype, device).requires_grad_(with_grads) for a in mask_head)
    strides = STRIDES[:sum(1 for k in enc if k.startswith("conv2d") and k.endswith("kernel"))]
    with torch.set_grad_enabled(with_grads):
        h = _t(x, dtype, device)
        for i, s in enumerate(strides):
            name = "conv2d" if i == 0 else f"conv2d_{i}"
            h = conv2d_same(h, tp[f"{name}/kernel"], tp[f"{name}/bias"], s, "relu")
        flat = h.reshape(h.shape[0], -1)
        z = flat @ tp["dense/kernel"] + tp["dense/bias"]
        sigma = q_sigma(flat, hk, hb) if head is not None else None
        zin = sampled_z(z, sigma, eps) if variational else z
        if mask_head is None:
            rec = decoder_layers(zin, tp, out_hw=x.shape[1], strides=strides, n_encoder_convs=len(strides))[-1]
        else:
            rec, xmask = decoder_with_mask(zin, tp, mk, mb, x.shape[1], strides, len(strides))
        loss = bootstrapped_l2(rec, _t(target, dtype, device), bootstrap_ratio)
        if mask_head is not None:
            loss = loss + mask_loss(xmask, _t(mask_target(target), dtype, device))
        reg = norm_reg_loss(z)
        kl = kl_div_loss(z, sigma) if sigma is not None else None
        if norm_regularize > 0:
            loss = loss + reg * norm_regularize
        if variational:
            loss = loss + kl * variational
        grads = None
        if with_grads:
            loss.backward()
            grads = {k: v.grad.cpu().numpy() for k, v in tp.items()}
            if mask_head is not None:
                k = 2 * len(strides) - 1                 # the output conv's name without the head
                grads[f"conv2d_{k + 1}/kernel"], grads[f"conv2d_{k + 1}/bias"] = grads.pop(f"conv2d_{k}/kernel"), grads.pop(f"conv2d_{k}/bias")
                grads[f"conv2d_{k}/kernel"], grads[f"conv2d_{k}/bias"] = mk.grad.cpu().numpy(), mb.grad.cpu().numpy()
            if variational:
                grads["dense_2/kernel"], grads["dense_2/bias"] = grads.pop("dense_1/kernel"), grads.pop("dense_1/bias")
                grads["dense_1/kernel"], grads["dense_1/bias"] = hk.grad.cpu().numpy(), hb.grad.cpu().numpy()
    terms = {"z": z.detach().cpu().numpy(), "q_sigma": None if sigma is None else sigma.detach().cpu().numpy(),
             "sampled_z": zin.detach().cpu().numpy(), "kl": None if kl is None else float(kl.detach()), "reg": float(reg.detach()),
             "xmask": None if mask_head is None else xmask.detach().cpu().numpy()}
    return float(loss.item()), terms, grads
