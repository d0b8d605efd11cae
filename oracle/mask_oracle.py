"""CPU oracle of the decoder's mask head and mask loss (AUXILIARY_MASK).  TEST INFRASTRUCTURE ONLY, like aae_oracle.py, whose
TF op restatements it builds on: torch, float64 = "truth", float32 = "TF stand-in".
Restates auto_pose/ae/decoder.py:66-83 (the head) and 134-142 (the mask loss) (paths relative to /root/reference)."""
from __future__ import annotations

from typing import Dict, Tuple

import numpy as np
import torch

from oracle.aae_oracle import (BOOTSTRAP_RATIO, STRIDES, _check_device, _t, bootstrapped_l2, conv2d_same, glorot_uniform,
                               resize_nearest_2x)

MASK_THRESHOLD = np.float32(0.0001)


def mask_target(target: np.ndarray) -> np.ndarray:
    """m = float(reduce_sum(target, axis=3, keepdims=True) > 0.0001) on the float32 target, the channels summed in channel
    order: [B, H, W, 1] float32."""
    t = np.asarray(target, dtype=np.float32)
    s = t[..., 0].copy()
    for c in range(1, t.shape[-1]):
        s = (s + t[..., c]).astype(np.float32)
    return (s > MASK_THRESHOLD).astype(np.float32)[..., None]


def mask_loss(xmask: torch.Tensor, m: torch.Tensor) -> torch.Tensor:
    """tf.losses.mean_squared_error(m, xmask, reduction=MEAN): the mean over B*H*W of (xmask - m)^2."""
    return ((xmask - m) ** 2).mean()


def make_mask_head(seed: int, cin: int, ksize: int = 5, bias_scale: float = 0.0) -> Tuple[np.ndarray, np.ndarray]:
    """Head kernel [k, k, cin, 1] (glorot-uniform, the tf.layers default) and bias [1]."""
    rng = np.random.RandomState(seed)
    return glorot_uniform(rng, (ksize, ksize, cin, 1)), (bias_scale * rng.standard_normal(1)).astype(np.float32)


def decoder_with_mask(z: torch.Tensor, p: Dict[str, torch.Tensor], head_k: torch.Tensor, head_b: torch.Tensor, out_hw: int,
                      strides, n_encoder_convs: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """decoder.py:44-83 with the head: (x, xmask).  ``p`` holds the decoder variables under the names of a decoder WITHOUT the
    head (dense_1, conv2d_k0 .. conv2d_k0+nl-1, the last being the output conv)."""
    st = list(reversed(strides))
    dims = [int(out_hw / np.prod(st[i:])) for i in range(len(st))]
    h = torch.relu(z @ p["dense_1/kernel"] + p["dense_1/bias"])
    nf0 = p["dense_1/kernel"].shape[1] // (dims[0] * dims[0])
    h = h.reshape(-1, dims[0], dims[0], nf0)
    k = n_encoder_convs
    for d in dims[1:]:
        h = resize_nearest_2x(h, (d, d))
        h = conv2d_same(h, p[f"conv2d_{k}/kernel"], p[f"conv2d_{k}/bias"], 1, "relu")
        k += 1
    h = resize_nearest_2x(h, (out_hw, out_hw))
    # built first: TF's conv2d_<k>.  The kernel goes in through a contiguous OIHW copy: torch's CPU conv backward wants its weight
    # gradient contiguous, and the OIHW view of a [k, k, cin, 1] kernel is not
    head_k = head_k.permute(3, 2, 0, 1).contiguous().permute(2, 3, 1, 0)
    xmask = conv2d_same(h, head_k, head_b, 1, "sigmoid")
    x = conv2d_same(h, p[f"conv2d_{k}/kernel"], p[f"conv2d_{k}/bias"], 1, "sigmoid")
    return x, xmask


def mask_forward_loss(x: np.ndarray, target: np.ndarray, enc: Dict[str, np.ndarray], dec: Dict[str, np.ndarray],
                      head: Tuple[np.ndarray, np.ndarray], dtype: torch.dtype = torch.float32,
                      bootstrap_ratio: int = BOOTSTRAP_RATIO, with_grads: bool = False, device: str = "cpu"):
    """AE.loss with AUXILIARY_MASK (NORM_REGULARIZE = VARIATIONAL = 0): reconstr_loss = bootstrapped L2 + mask loss.
    ``enc`` / ``dec`` as for aae_oracle.ae_forward_loss, ``head`` = (kernel, bias).  Returns (loss, x, xmask, grads or None),
    the gradients keyed by the TF names of the graph with the head: the head is conv2d_<k> and the output conv conv2d_<k+1>,
    k = encoder convs + decoder hidden convs.  device="cuda" evaluates on the GPU (float64 only)."""
    _check_device(dtype, device)
    tp = {k: _t(v, dtype, device).requires_grad_(with_grads) for k, v in {**enc, **dec}.items()}
    hk, hb = (_t(a, dtype, device).requires_grad_(with_grads) for a in head)
    n_enc = sum(1 for k in enc if k.startswith("conv2d") and k.endswith("kernel"))
    strides = STRIDES[:n_enc]
    with torch.set_grad_enabled(with_grads):
        h = _t(x, dtype, device)
        for i, s in enumerate(strides):
            name = "conv2d" if i == 0 else f"conv2d_{i}"
            h = conv2d_same(h, tp[f"{name}/kernel"], tp[f"{name}/bias"], s, "relu")
        z = h.reshape(h.shape[0], -1) @ tp["dense/kernel"] + tp["dense/bias"]
        rec, xmask = decoder_with_mask(z, tp, hk, hb, x.shape[1], strides, n_enc)
        loss = bootstrapped_l2(rec, _t(target, dtype, device), bootstrap_ratio)
        loss = loss + mask_loss(xmask, _t(mask_target(target), dtype, device))
        grads = None
        if with_grads:
            loss.backward()
            grads = {k: v.grad.cpu().numpy() for k, v in tp.items()}
            k = n_enc + len(strides) - 1                         # the output conv's name without the head
            grads[f"conv2d_{k + 1}/kernel"], grads[f"conv2d_{k + 1}/bias"] = grads.pop(f"conv2d_{k}/kernel"), grads.pop(f"conv2d_{k}/bias")
            grads[f"conv2d_{k}/kernel"], grads[f"conv2d_{k}/bias"] = hk.grad.cpu().numpy(), hb.grad.cpu().numpy()
    return float(loss.item()), rec.detach().cpu().numpy(), xmask.detach().cpu().numpy(), grads


def mask_loss_grad(xmask: np.ndarray, target: np.ndarray) -> Tuple[float, np.ndarray]:
    """float64 mask loss and its gradient wrt xmask, 2 (xmask - m) / (B H W), from the closed form."""
    xm = np.asarray(xmask, dtype=np.float64).reshape(np.asarray(target).shape[:3] + (1,))
    d = xm - mask_target(target).astype(np.float64)
    return float(np.mean(d * d)), 2.0 * d / d.size
