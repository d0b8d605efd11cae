"""CPU oracle for the Augmented-Autoencoder hot path.  TEST INFRASTRUCTURE ONLY.

This file is the *checker*, never the product: only ``tests/``,
``__graft_entry__.smoke()`` and ``bench.py``'s CPU-baseline / ``--impl reference``
legs may import it.  The product package (``augmentedautoencoder_b200``) must never
import anything under ``oracle/``.

PARITY STATUS
-------------
* Network arithmetic (conv / dense / l2-normalise / matmul / top_k / Adam): the
  reference delegates these to TensorFlow (env pin ``tensorflow=2.6.0``,
  ``tf-slim==1.1.0`` -- /root/reference/aae_py37_tf26.yml:29-30,102-105,142).
  TensorFlow is NOT installable in this image (no network) and the reference
  ships no golden vectors, tests or checkpoints for the path, so this part of the
  oracle restates TensorFlow's *published* op semantics and is
  **parity unpinned** against TF itself.  It is cross-checked three ways instead
  (tests/test_oracle.py): float32 vs float64 evaluation, an independent
  pure-numpy loop implementation on small cases, and structural known-answer
  tests (asymmetric SAME padding, NHWC flatten order, lowest-index ties, ...).
* Host logic (uint8 /255, argmax / upright / top_n selection, idx -> R lookup,
  ``auto_pose6d`` pose lift, ``extract_square_patch``, the view-sphere table):
  **pinned** against the reference's own Python, executed in the build container
  with TensorFlow stubbed out (tests/golden/make_golden.py -> tests/golden/*.npz).

Every function cites the reference lines it restates (paths relative to
/root/reference).
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch
import torch.nn.functional as F

# ----------------------------------------------------------------------------------------
# Template configuration -- auto_pose/ae/cfg/train_template.cfg:5-9,41-55
# ----------------------------------------------------------------------------------------
H = W = 128
C = 3
LATENT = 128
NUM_FILTER = (128, 256, 512, 512)
STRIDES = (2, 2, 2, 2)
KSIZE = 5
NUM_VIEWS = 2562
NUM_CYCLO = 36
N_CODEBOOK = NUM_VIEWS * NUM_CYCLO  # 92 232
BOOTSTRAP_RATIO = 4


# ----------------------------------------------------------------------------------------
# Deterministic synthetic parameters (SURVEY.md section 8d)
# ----------------------------------------------------------------------------------------
def glorot_uniform(rng: np.random.RandomState, shape: Sequence[int]) -> np.ndarray:
    """tf.layers default kernel initialiser (glorot_uniform); no initialiser is passed at
    auto_pose/ae/encoder.py:43-50,62-66.  fan_in/fan_out follow TF: receptive field x channels."""
    if len(shape) == 4:  # HWIO
        rf = shape[0] * shape[1]
        fan_in, fan_out = rf * shape[2], rf * shape[3]
    else:  # [in, out]
        fan_in, fan_out = shape
    limit = math.sqrt(6.0 / (fan_in + fan_out))
    return rng.uniform(-limit, limit, size=shape).astype(np.float32)


def make_encoder_params(seed: int = 42, num_filters=NUM_FILTER, ksize=KSIZE, latent=LATENT,
                        in_ch=C, in_hw=H, strides=STRIDES, bias_scale: float = 0.0,
                        in_w: Optional[int] = None) -> Dict[str, np.ndarray]:
    """Variable names / layouts of auto_pose/ae/encoder.py:43-66 (conv kernels HWIO, dense [in,out]).
    TF zero-initialises biases; ``bias_scale`` > 0 draws small random biases so that parity tests
    actually exercise the bias path.  ``in_w``: crop width when it differs from the height ``in_hw``.  Each conv's output is
    ceil(in / stride) per axis, as TF's SAME padding makes it (127 -> 64 -> 32 -> 16 -> 8)."""
    rng = np.random.RandomState(seed)
    p: Dict[str, np.ndarray] = {}
    cin, hh, ww = in_ch, in_hw, in_hw if in_w is None else in_w
    for i, (f, s) in enumerate(zip(num_filters, strides)):
        name = "conv2d" if i == 0 else f"conv2d_{i}"
        p[f"{name}/kernel"] = glorot_uniform(rng, (ksize, ksize, cin, f))
        p[f"{name}/bias"] = (bias_scale * rng.standard_normal(f)).astype(np.float32)
        cin, hh, ww = f, -(-hh // s), -(-ww // s)
    p["dense/kernel"] = glorot_uniform(rng, (hh * ww * cin, latent))
    p["dense/bias"] = (bias_scale * rng.standard_normal(latent)).astype(np.float32)
    return p


def make_decoder_params(seed: int = 43, num_filters=NUM_FILTER, ksize=KSIZE, latent=LATENT,
                        out_ch=C, out_hw=H, strides=STRIDES, bias_scale: float = 0.0,
                        n_encoder_convs: int = 4) -> Dict[str, np.ndarray]:
    """Decoder variables (auto_pose/ae/decoder.py:44-83): dense_1, conv2d_4..conv2d_7 when built after a
    4-conv encoder inside the same variable scope.  Filters are the encoder's reversed
    (auto_pose/ae/ae_factory.py:59-70)."""
    rng = np.random.RandomState(seed)
    nf = list(reversed(num_filters))
    st = list(reversed(strides))
    hw0 = out_hw // int(np.prod(st))
    p: Dict[str, np.ndarray] = {}
    p["dense_1/kernel"] = glorot_uniform(rng, (latent, hw0 * hw0 * nf[0]))
    p["dense_1/bias"] = (bias_scale * rng.standard_normal(hw0 * hw0 * nf[0])).astype(np.float32)
    cin = nf[0]
    k = n_encoder_convs
    for f in nf[1:]:
        p[f"conv2d_{k}/kernel"] = glorot_uniform(rng, (ksize, ksize, cin, f))
        p[f"conv2d_{k}/bias"] = (bias_scale * rng.standard_normal(f)).astype(np.float32)
        cin = f
        k += 1
    p[f"conv2d_{k}/kernel"] = glorot_uniform(rng, (ksize, ksize, cin, out_ch))
    p[f"conv2d_{k}/bias"] = (bias_scale * rng.standard_normal(out_ch)).astype(np.float32)
    return p


def make_crops_u8(seed: int, batch: int, hw: int = H, ch: int = C, structured: bool = True, w: Optional[int] = None) -> np.ndarray:
    """Synthetic BGR crops, NHWC uint8 (auto_pose/ae/ae_factory.py:133 placeholder shape).  structured=True draws a
    different coarse random pattern per crop (8x8 blocks + pixel noise) so that the latents -- and therefore the
    matched codebook rows -- differ from crop to crop; structured=False is i.i.d. U{0..255} (every crop then encodes
    to almost the same latent).  ``w``: crop width when it differs from the height ``hw``.  A size that the cell count does
    not divide takes ceil(size / cells) pixels per cell, the last cell cut short."""
    rng = np.random.RandomState(seed)
    w = hw if w is None else w
    if not structured:
        return rng.randint(0, 256, size=(batch, hw, w, ch), dtype=np.uint8)
    cells, cells_w = max(hw // 16, 1), max(w // 16, 1)
    coarse = rng.randint(0, 256, size=(batch, cells, cells_w, ch)).astype(np.int32)
    img = np.repeat(np.repeat(coarse, -(-hw // cells), axis=1), -(-w // cells_w), axis=2)[:, :hw, :w]
    img = img + rng.randint(-40, 41, size=(batch, hw, w, ch))
    return np.clip(img, 0, 255).astype(np.uint8)


def make_codebook(seed: int, n: int = N_CODEBOOK, j: int = LATENT, num_cyclo: int = NUM_CYCLO,
                  duplicate_cyclo_endpoints: bool = True) -> np.ndarray:
    """Unit-norm Gaussian rows, normalised in float64 then rounded to float32 exactly as
    auto_pose/ae/codebook.py:213-216 does.  With ``duplicate_cyclo_endpoints`` rows v*num_cyclo+(num_cyclo-1)
    are bit-copies of rows v*num_cyclo+0, reproducing the duplicate rows real codebooks contain because
    np.linspace(0, 2pi, num_cyclo) includes both end points (auto_pose/ae/dataset.py:54-57)."""
    rng = np.random.RandomState(seed)
    e = rng.standard_normal((n, j))
    e = e / np.linalg.norm(e, axis=1, keepdims=True)
    e = e.astype(np.float32)
    if duplicate_cyclo_endpoints and n % num_cyclo == 0 and num_cyclo > 1:
        e[num_cyclo - 1::num_cyclo] = e[0::num_cyclo]
    return e


# ----------------------------------------------------------------------------------------
# Pre-processing -- auto_pose/ae/codebook.py:58-61
# ----------------------------------------------------------------------------------------
def preprocess(x: np.ndarray) -> np.ndarray:
    """``if x.dtype == 'uint8': x = x/255.`` (numpy float64) then fed to a float32 placeholder."""
    if x.dtype == np.uint8:
        x = x / 255.0
    if x.ndim == 3:
        x = np.expand_dims(x, 0)
    return np.asarray(x, dtype=np.float32)


# ----------------------------------------------------------------------------------------
# TF op restatements (torch CPU; dtype float32 = "TF stand-in", float64 = "truth")
# ----------------------------------------------------------------------------------------
def _same_pads(in_size: int, k: int, stride: int) -> Tuple[int, int]:
    """TensorFlow 'SAME': out = ceil(in/stride); pad_total = max((out-1)*stride + k - in, 0);
    before = pad_total // 2, after = pad_total - before."""
    out = -(-in_size // stride)
    total = max((out - 1) * stride + k - in_size, 0)
    return total // 2, total - total // 2


def conv2d_same(x_nhwc: torch.Tensor, kernel_hwio: torch.Tensor, bias: torch.Tensor, stride: int,
                activation: Optional[str]) -> torch.Tensor:
    """tf.layers.conv2d(padding='same', activation=...) on NHWC input with an HWIO kernel
    (auto_pose/ae/encoder.py:43-50, auto_pose/ae/decoder.py:56-62,77-83)."""
    kh, kw = kernel_hwio.shape[0], kernel_hwio.shape[1]
    pt, pb = _same_pads(x_nhwc.shape[1], kh, stride)
    pl, pr = _same_pads(x_nhwc.shape[2], kw, stride)
    x = x_nhwc.permute(0, 3, 1, 2)
    x = F.pad(x, (pl, pr, pt, pb))
    w = kernel_hwio.permute(3, 2, 0, 1)
    y = F.conv2d(x, w, bias, stride=stride)
    if activation == "relu":
        y = torch.relu(y)
    elif activation == "sigmoid":
        y = torch.sigmoid(y)
    elif activation is not None:
        raise ValueError(activation)
    return y.permute(0, 2, 3, 1).contiguous()


def resize_nearest_2x(x_nhwc: torch.Tensor, out_hw: Tuple[int, int]) -> torch.Tensor:
    """tf.image.resize_nearest_neighbor (align_corners=False): out[i] = in[floor(i * in/out)]
    (auto_pose/ae/decoder.py:54,66)."""
    ih, iw = x_nhwc.shape[1], x_nhwc.shape[2]
    oh, ow = out_hw
    dev = x_nhwc.device
    ri = torch.clamp((torch.arange(oh, dtype=torch.float64, device=dev) * (ih / oh)).floor().long(), max=ih - 1)
    ci = torch.clamp((torch.arange(ow, dtype=torch.float64, device=dev) * (iw / ow)).floor().long(), max=iw - 1)
    return x_nhwc[:, ri][:, :, ci]


def _t(a: np.ndarray, dtype: torch.dtype, device: str = "cpu") -> torch.Tensor:
    return torch.from_numpy(np.ascontiguousarray(a)).to(device, dtype)


def _check_device(dtype: torch.dtype, device: str) -> None:
    """Only float64 runs on the GPU: torch's float32 convolutions and matmuls there may use TF32, which is no fp32 reference."""
    if torch.device(device).type != "cpu" and dtype != torch.float64:
        raise ValueError("the oracle runs %s on the CPU only; on %s it evaluates float64" % (dtype, device))


def encoder_layers(x: np.ndarray, params: Dict[str, np.ndarray], strides=STRIDES,
                   dtype: torch.dtype = torch.float32, device: str = "cpu") -> List[torch.Tensor]:
    """All intermediate activations of the encoder: [conv1, conv2, ..., flatten, z]
    (auto_pose/ae/encoder.py:37-68).  device="cuda" evaluates float64 on the GPU."""
    _check_device(dtype, device)
    h = _t(x, dtype, device)
    outs: List[torch.Tensor] = []
    for i, s in enumerate(strides):
        name = "conv2d" if i == 0 else f"conv2d_{i}"
        h = conv2d_same(h, _t(params[f"{name}/kernel"], dtype, device), _t(params[f"{name}/bias"], dtype, device), s, "relu")
        outs.append(h)
    flat = h.reshape(h.shape[0], -1)  # tf.layers.flatten on NHWC: (h, w, c) order
    outs.append(flat)
    z = flat @ _t(params["dense/kernel"], dtype, device) + _t(params["dense/bias"], dtype, device)
    outs.append(z)
    return outs


def encoder_forward(x: np.ndarray, params: Dict[str, np.ndarray], strides=STRIDES,
                    dtype: torch.dtype = torch.float32, device: str = "cpu") -> np.ndarray:
    """crop batch (float NHWC in [0,1]) -> z [B, latent]."""
    with torch.no_grad():
        return encoder_layers(x, params, strides, dtype, device)[-1].cpu().numpy()


def l2_normalize(z: np.ndarray, eps: float = 1e-12) -> np.ndarray:
    """tf.nn.l2_normalize(z, 1) = z * rsqrt(max(sum(z^2), eps)) (auto_pose/ae/codebook.py:27)."""
    z = np.asarray(z)
    ss = np.sum(z * z, axis=1, keepdims=True, dtype=z.dtype)
    return (z * (1.0 / np.sqrt(np.maximum(ss, z.dtype.type(eps))))).astype(z.dtype)


def cos_similarity(z: np.ndarray, codebook: np.ndarray) -> np.ndarray:
    """tf.matmul(l2_normalize(z), embedding_normalized, transpose_b=True) (auto_pose/ae/codebook.py:50)."""
    zq = l2_normalize(z)
    with torch.no_grad():
        return (torch.from_numpy(zq) @ torch.from_numpy(np.ascontiguousarray(codebook)).to(torch.from_numpy(zq).dtype).T).numpy()


def select_indices(cos: np.ndarray, top_n: int = 1, upright: bool = False, num_cyclo: int = NUM_CYCLO) -> np.ndarray:
    """Host-side index selection of Codebook.nearest_rotation (auto_pose/ae/codebook.py:64-71).
    np.argmax -> lowest index on ties."""
    if top_n == 1:
        if upright:
            return np.argmax(cos[:, ::int(num_cyclo)], axis=1) * int(num_cyclo)
        return np.argmax(cos, axis=1)
    c = cos.squeeze()
    unsorted_max_idcs = np.argpartition(-c, top_n)[:top_n]
    return unsorted_max_idcs[np.argsort(-c[unsorted_max_idcs])]


def nearest_rotation_idcs(x: np.ndarray, enc_params: Dict[str, np.ndarray], codebook: np.ndarray,
                          top_n: int = 1, upright: bool = False, num_cyclo: int = NUM_CYCLO,
                          dtype: torch.dtype = torch.float32, return_cos: bool = False, device: str = "cpu"):
    """Codebook.nearest_rotation(..., return_idcs=True) end to end (auto_pose/ae/codebook.py:55-73).  device="cuda" runs
    the float64 encoder on the GPU; the cosines and the selection stay on the host."""
    xf = preprocess(x)
    z = encoder_forward(xf, enc_params, dtype=dtype, device=device)
    cb = codebook.astype(np.float64 if dtype == torch.float64 else np.float32)
    cos = cos_similarity(z, cb)
    idcs = select_indices(cos, top_n, upright, num_cyclo)
    return (idcs, cos) if return_cos else idcs


# ----------------------------------------------------------------------------------------
# Decoder + loss -- auto_pose/ae/decoder.py:36-101
# ----------------------------------------------------------------------------------------
def decoder_layers(z: torch.Tensor, params: Dict[str, torch.Tensor], out_hw: int = H, strides=STRIDES,
                   n_encoder_convs: int = 4) -> List[torch.Tensor]:
    st = list(reversed(strides))
    dims = [int(out_hw / np.prod(st[i:])) for i in range(len(st))]  # decoder.py:41
    outs = []
    h = torch.relu(z @ params["dense_1/kernel"] + params["dense_1/bias"])
    outs.append(h)
    nf0 = params["dense_1/kernel"].shape[1] // (dims[0] * dims[0])
    h = h.reshape(-1, dims[0], dims[0], nf0)
    k = n_encoder_convs
    for d in dims[1:]:
        h = resize_nearest_2x(h, (d, d))
        h = conv2d_same(h, params[f"conv2d_{k}/kernel"], params[f"conv2d_{k}/bias"], 1, "relu")
        outs.append(h)
        k += 1
    h = resize_nearest_2x(h, (out_hw, out_hw))
    h = conv2d_same(h, params[f"conv2d_{k}/kernel"], params[f"conv2d_{k}/bias"], 1, "sigmoid")
    outs.append(h)
    return outs


def bootstrapped_l2(x: torch.Tensor, target: torch.Tensor, bootstrap_ratio: int = BOOTSTRAP_RATIO) -> torch.Tensor:
    """LOSS: L2, BOOTSTRAP_RATIO > 1 (auto_pose/ae/decoder.py:90-101): per-sample top_k of the flattened
    squared error with k = numel // ratio, then the mean over the [B, k] survivors."""
    b = x.shape[0]
    l2 = (target.reshape(b, -1) - x.reshape(b, -1)) ** 2
    if bootstrap_ratio > 1:
        k = l2.shape[1] // bootstrap_ratio
        vals, _ = torch.topk(l2, k, dim=1)
        return vals.mean()
    return l2.mean()


def ae_forward_loss(x: np.ndarray, target: np.ndarray, enc: Dict[str, np.ndarray], dec: Dict[str, np.ndarray],
                    dtype: torch.dtype = torch.float32, bootstrap_ratio: int = BOOTSTRAP_RATIO,
                    with_grads: bool = False, device: str = "cpu", strides=None):
    """encode -> decode -> bootstrapped L2 (auto_pose/ae/ae.py:42-53 with NORM_REGULARIZE=0, VARIATIONAL=0).
    Returns (loss, reconstruction, grads-dict or None) as numpy.  device="cuda" evaluates the same graph on the GPU (float64
    only), which makes the reference affordable at training batch sizes.  ``strides``: the encoder's, one per conv (default: the
    template's for as many convs as ``enc`` has)."""
    _check_device(dtype, device)
    tp = {k: _t(v, dtype, device).requires_grad_(with_grads) for k, v in {**enc, **dec}.items()}
    if strides is None:
        strides = STRIDES[:_n_convs(enc)]
    hw = x.shape[1]
    with torch.set_grad_enabled(with_grads):
        h = _t(x, dtype, device)
        for i, s in enumerate(strides):
            name = "conv2d" if i == 0 else f"conv2d_{i}"
            h = conv2d_same(h, tp[f"{name}/kernel"], tp[f"{name}/bias"], s, "relu")
        z = h.reshape(h.shape[0], -1) @ tp["dense/kernel"] + tp["dense/bias"]
        rec = decoder_layers(z, tp, out_hw=hw, strides=strides, n_encoder_convs=len(strides))[-1]
        loss = bootstrapped_l2(rec, _t(target, dtype, device), bootstrap_ratio)
        grads = None
        if with_grads:
            loss.backward()
            grads = {k: v.grad.cpu().numpy() for k, v in tp.items()}
    return float(loss.item()), rec.detach().cpu().numpy(), grads


def _n_convs(enc: Dict[str, np.ndarray]) -> int:
    return sum(1 for k in enc if k.startswith("conv2d") and k.endswith("kernel"))


def relu_margin(x: np.ndarray, enc: Dict[str, np.ndarray], dec: Dict[str, np.ndarray], device: str = "cpu",
                latent: Optional[np.ndarray] = None, strides=None) -> float:
    """Smallest |pre-activation| over every ReLU unit of encoder + decoder, in float64.  A unit closer to zero than fp32
    rounding can land on either side of the ReLU in any fp32 implementation (TF included), which changes its gradient
    path discretely; gradient parity tests pick inputs whose margin is comfortably above that.  ``latent``: the decoder's
    input when it is not the encoder's z (the sampled z of the variational AE).  ``strides``: as in ae_forward_loss."""
    dt = torch.float64
    tp = {k: _t(v, dt, device) for k, v in {**enc, **dec}.items()}
    n_enc = _n_convs(enc)
    if strides is None:
        strides = STRIDES[:n_enc]
    m = float("inf")
    with torch.no_grad():
        h = _t(x, dt, device)
        for i, s_ in enumerate(strides):
            name = "conv2d" if i == 0 else f"conv2d_{i}"
            pre = conv2d_same(h, tp[f"{name}/kernel"], tp[f"{name}/bias"], s_, None)
            m = min(m, float(pre.abs().min()))
            h = torch.relu(pre)
        z = h.reshape(h.shape[0], -1) @ tp["dense/kernel"] + tp["dense/bias"]
        if latent is not None:
            z = _t(latent, dt, device)
        pre = z @ tp["dense_1/kernel"] + tp["dense_1/bias"]
        m = min(m, float(pre.abs().min()))
        st = list(reversed(strides))
        hw = x.shape[1]
        dims = [int(hw / np.prod(st[i:])) for i in range(len(st))]
        nf0 = tp["dense_1/kernel"].shape[1] // (dims[0] * dims[0])
        h = torch.relu(pre).reshape(-1, dims[0], dims[0], nf0)
        k = n_enc
        for d in dims[1:]:
            h = resize_nearest_2x(h, (d, d))
            pre = conv2d_same(h, tp[f"conv2d_{k}/kernel"], tp[f"conv2d_{k}/bias"], 1, None)
            m = min(m, float(pre.abs().min()))
            h = torch.relu(pre)
            k += 1
    return m


def tf_adam_step(p: np.ndarray, g: np.ndarray, m: np.ndarray, v: np.ndarray, t: int, lr: float = 2e-4,
                 beta1: float = 0.9, beta2: float = 0.999, eps: float = 1e-8):
    """tf.train.AdamOptimizer update (auto_pose/ae/ae_factory.py:86-88):
    lr_t = lr*sqrt(1-b2^t)/(1-b1^t); m = b1 m + (1-b1) g; v = b2 v + (1-b2) g^2; p -= lr_t*m/(sqrt(v)+eps).
    All arithmetic in the parameter dtype, as TF's ApplyAdam kernel does."""
    dt = p.dtype.type
    lr_t = dt(lr * math.sqrt(1.0 - beta2 ** t) / (1.0 - beta1 ** t))
    m = (dt(beta1) * m + dt(1.0 - beta1) * g).astype(p.dtype)
    v = (dt(beta2) * v + dt(1.0 - beta2) * g * g).astype(p.dtype)
    p = (p - lr_t * m / (np.sqrt(v) + dt(eps))).astype(p.dtype)
    return p, m, v


# ----------------------------------------------------------------------------------------
# Independent slow implementation (pure numpy loops) used to pin the torch restatement
# ----------------------------------------------------------------------------------------
def conv2d_same_loops(x: np.ndarray, k: np.ndarray, b: np.ndarray, stride: int) -> np.ndarray:
    """Direct definition of an NHWC / HWIO 'SAME' convolution in float64, no library conv."""
    n, ih, iw, ci = x.shape
    kh, kw, _, co = k.shape
    oh, ow = -(-ih // stride), -(-iw // stride)
    pt, _ = _same_pads(ih, kh, stride)
    pl, _ = _same_pads(iw, kw, stride)
    y = np.zeros((n, oh, ow, co), dtype=np.float64)
    for r in range(oh):
        for c in range(ow):
            for dy in range(kh):
                iy = r * stride + dy - pt
                if iy < 0 or iy >= ih:
                    continue
                for dx in range(kw):
                    ix = c * stride + dx - pl
                    if ix < 0 or ix >= iw:
                        continue
                    y[:, r, c, :] += x[:, iy, ix, :].astype(np.float64) @ k[dy, dx].astype(np.float64)
    return y + b.astype(np.float64)


# ----------------------------------------------------------------------------------------
# View sphere (idx -> R table) -- auto_pose/ae/dataset.py:39-58 + pysixd_stuff/view_sampler.py:19-188
# ----------------------------------------------------------------------------------------
def hinter_sampling(min_n_pts: int, radius: float = 1.0):
    """Icosphere refinement of Hinterstoisser et al. (auto_pose/ae/pysixd_stuff/view_sampler.py:19-92):
    start from an icosahedron, subdivide every triangle into four until >= min_n_pts vertices, project
    onto the sphere, order by (a) descending z then (b) azimuth -- returns (pts, pts_level)."""
    a, b, c = 0.0, 1.0, (1.0 + math.sqrt(5.0)) / 2.0
    pts = [(-b, c, a), (b, c, a), (-b, -c, a), (b, -c, a), (a, -b, c), (a, b, c),
           (a, -b, -c), (a, b, -c), (c, a, -b), (c, a, b), (-c, a, -b), (-c, a, b)]
    faces = [(0, 11, 5), (0, 5, 1), (0, 1, 7), (0, 7, 10), (0, 10, 11), (1, 5, 9),
             (5, 11, 4), (11, 10, 2), (10, 7, 6), (7, 1, 8), (3, 9, 4), (3, 4, 2),
             (3, 2, 6), (3, 6, 8), (3, 8, 9), (4, 9, 5), (2, 4, 11), (6, 2, 10),
             (8, 6, 7), (9, 8, 1)]
    pts_level = [0 for _ in range(len(pts))]
    ref_level = 0
    while len(pts) < min_n_pts:
        ref_level += 1
        edge_pt_map = {}
        faces_new = []
        for face in faces:
            pt_inds = list(face)
            for i in range(3):
                edge = (face[i], face[(i + 1) % 3])
                edge = (min(edge), max(edge))
                if edge not in edge_pt_map:
                    pt_new_id = len(pts)
                    edge_pt_map[edge] = pt_new_id
                    pt_inds.append(pt_new_id)
                    pt_new = 0.5 * (np.array(pts[edge[0]]) + np.array(pts[edge[1]]))
                    pts.append(pt_new.tolist())
                    pts_level.append(ref_level)
                else:
                    pt_inds.append(edge_pt_map[edge])
            faces_new += [(pt_inds[0], pt_inds[3], pt_inds[5]), (pt_inds[3], pt_inds[1], pt_inds[4]),
                          (pt_inds[3], pt_inds[4], pt_inds[5]), (pt_inds[5], pt_inds[4], pt_inds[2])]
        faces = faces_new
    pts = np.array(pts)
    pts *= np.reshape(radius / np.linalg.norm(pts, axis=1), (pts.shape[0], 1))
    # Spiral ordering starting from the top pole, walking neighbours (view_sampler.py:68-90)
    pt_conns = {}
    for face in faces:
        for i in range(len(face)):
            pt_conns.setdefault(face[i], set()).add(face[(i + 1) % len(face)])
            pt_conns[face[i]].add(face[(i + 2) % len(face)])
    top_pt_id = int(np.argmax(pts[:, 2]))
    pts_ordered = []
    pts_todo = [top_pt_id]
    pts_done = [False for _ in range(pts.shape[0])]

    def calc_azimuth(x, y):
        two_pi = 2.0 * math.pi
        return (math.atan2(y, x) + two_pi) % two_pi

    while len(pts_ordered) != pts.shape[0]:
        pts_todo = sorted(pts_todo, key=lambda i: calc_azimuth(pts[i][0], pts[i][1]))
        nxt = []
        for pt_id in pts_todo:
            pts_ordered.append(pt_id)
            pts_done[pt_id] = True
            nxt.extend(pt_conns[pt_id])
        # the reference de-duplicates through a Python set; its iteration order breaks azimuth ties
        pts_todo = [i for i in set(nxt) if not pts_done[i]]
    pts = pts[np.array(pts_ordered), :]
    pts_level = [pts_level[i] for i in pts_ordered]
    return pts, pts_level


def sample_view_rotations(min_n_views: int, radius: float = 700.0) -> np.ndarray:
    """R of every view returned by view_sampler.sample_views with the full azimuth/elevation range
    (auto_pose/ae/pysixd_stuff/view_sampler.py:122-188): camera looks at the origin, f = -pt/|pt|,
    u = (0,0,1), s = f x u (s = (1,0,0) at the poles), u = s x f, R = Ryz180 . [s;u;-f]."""
    pts, _ = hinter_sampling(min_n_views, radius=radius)
    rs = []
    for pt in pts:
        f = -np.array(pt)
        f /= np.linalg.norm(f)
        u = np.array([0.0, 0.0, 1.0])
        s = np.cross(f, u)
        if np.count_nonzero(s) == 0:
            s = np.array([1.0, 0.0, 0.0])
        s /= np.linalg.norm(s)
        u = np.cross(s, f)
        r = np.array([[s[0], s[1], s[2]], [u[0], u[1], u[2]], [-f[0], -f[1], -f[2]]])
        r_yz_flip = np.array([[1.0, 0.0, 0.0], [0.0, math.cos(math.pi), -math.sin(math.pi)],
                              [0.0, math.sin(math.pi), math.cos(math.pi)]])  # transform.rotation_matrix(pi,[1,0,0])
        rs.append(r_yz_flip.dot(r))
    return np.array(rs)


def viewsphere_for_embedding(min_n_views: int = NUM_VIEWS, num_cyclo: int = NUM_CYCLO,
                             radius: float = 700.0) -> np.ndarray:
    """Dataset.viewsphere_for_embedding (auto_pose/ae/dataset.py:39-58): [views*num_cyclo, 3, 3] float64,
    in-plane angles from np.linspace(0, 2pi, num_cyclo) (both end points included)."""
    view_rs = sample_view_rotations(min_n_views, radius)
    rs = np.empty((len(view_rs) * num_cyclo, 3, 3))
    i = 0
    for r_view in view_rs:
        for cyclo in np.linspace(0, 2.0 * np.pi, num_cyclo):
            rot_z = np.array([[np.cos(-cyclo), -np.sin(-cyclo), 0], [np.sin(-cyclo), np.cos(-cyclo), 0], [0, 0, 1]])
            rs[i] = rot_z.dot(r_view)
            i += 1
    return rs


# ----------------------------------------------------------------------------------------
# Pose lift -- auto_pose/ae/codebook.py:79-129
# ----------------------------------------------------------------------------------------
def auto_pose6d_lift(idcs: np.ndarray, rs_table: np.ndarray, embed_obj_bbs: np.ndarray, predicted_bb,
                     k_test: np.ndarray, k_train: np.ndarray, render_radius: float,
                     depth_pred: Optional[float] = None) -> Tuple[np.ndarray, np.ndarray]:
    """Everything of Codebook.auto_pose6d after the index lookup: translation from the bbox-diagonal
    ratio and the rotation correction R_corr_y . R_corr_x . R."""
    idcs = np.atleast_1d(idcs)
    rs_est = rs_table[idcs].copy()
    k_diag_ratio = np.sqrt(k_test[0, 0] ** 2 + k_test[1, 1] ** 2) / np.sqrt(k_train[0, 0] ** 2 + k_train[1, 1] ** 2)
    ts_est = np.empty((len(idcs), 3))
    for i, idx in enumerate(idcs):
        rendered_bb = embed_obj_bbs[idx].squeeze()
        if depth_pred is None:
            diag = np.linalg.norm(np.float32(rendered_bb[2:])) / np.linalg.norm(np.float32(predicted_bb[2:]))
            z = diag * k_diag_ratio * render_radius
        else:
            z = depth_pred
        cx_tr = rendered_bb[0] + rendered_bb[2] / 2.0 - k_train[0, 2]
        cy_tr = rendered_bb[1] + rendered_bb[3] / 2.0 - k_train[1, 2]
        cx_te = predicted_bb[0] + predicted_bb[2] / 2 - k_test[0, 2]
        cy_te = predicted_bb[1] + predicted_bb[3] / 2 - k_test[1, 2]
        tx = cx_te * z / k_test[0, 0] - cx_tr * render_radius / k_train[0, 0]
        ty = cy_te * z / k_test[1, 1] - cy_tr * render_radius / k_train[1, 1]
        t_est = np.array([tx, ty, z])
        ts_est[i] = t_est
        d_alpha_y = np.arctan(t_est[0] / np.sqrt(t_est[2] ** 2 + t_est[1] ** 2))
        d_alpha_x = -np.arctan(t_est[1] / t_est[2])
        r_corr_x = np.array([[1, 0, 0], [0, np.cos(d_alpha_x), -np.sin(d_alpha_x)], [0, np.sin(d_alpha_x), np.cos(d_alpha_x)]])
        r_corr_y = np.array([[np.cos(d_alpha_y), 0, np.sin(d_alpha_y)], [0, 1, 0], [-np.sin(d_alpha_y), 0, np.cos(d_alpha_y)]])
        rs_est[i] = np.dot(r_corr_y, np.dot(r_corr_x, rs_est[i]))
    return rs_est, ts_est


# ----------------------------------------------------------------------------------------
# The same inference data flow with the variables held resident, as a tf.Session holds them:
# the timed CPU baseline (bench.py cpu_baseline / --impl reference).  Arithmetic = nearest_rotation_idcs.
# ----------------------------------------------------------------------------------------
class ResidentCpuPath:
    """Codebook.nearest_rotation(x, return_idcs=True) on the CPU (auto_pose/ae/codebook.py:55-73 + encoder.py:37-68) with
    every variable converted ONCE to the layout the convolution library wants (OIHW kernels in channels_last memory, the dense
    kernel re-indexed from TF's NHWC flatten order to the NCHW order the activations are in, the codebook transposed) --
    a fair CPU baseline must not re-wrap 59 MB of weights per call.  The full [B, N] cosine matrix is materialised and scanned
    on the host, as the reference does."""

    def __init__(self, enc_params: Dict[str, np.ndarray], codebook: np.ndarray, strides=STRIDES):
        self.layers = []
        i = 0
        hw = None
        while True:
            name = "conv2d" if i == 0 else f"conv2d_{i}"
            if f"{name}/kernel" not in enc_params or i >= len(strides):
                break
            k = torch.from_numpy(np.ascontiguousarray(enc_params[f"{name}/kernel"])).permute(3, 2, 0, 1)
            k = k.contiguous(memory_format=torch.channels_last)
            self.layers.append((k, torch.from_numpy(np.ascontiguousarray(enc_params[f"{name}/bias"])), int(strides[i])))
            i += 1
        cout = self.layers[-1][0].shape[0]
        dk = enc_params["dense/kernel"]                       # rows in (h, w, c) order (tf.layers.flatten of NHWC)
        hw = int(round(math.sqrt(dk.shape[0] // cout)))
        self.dense_w = torch.from_numpy(np.ascontiguousarray(dk.reshape(hw, hw, cout, -1).transpose(2, 0, 1, 3).reshape(dk.shape[0], -1)))
        self.dense_b = torch.from_numpy(np.ascontiguousarray(enc_params["dense/bias"]))
        self.codebook_t = torch.from_numpy(np.ascontiguousarray(codebook.astype(np.float32).T))

    def cos(self, crops: np.ndarray) -> np.ndarray:
        x = torch.from_numpy(preprocess(crops)).permute(0, 3, 1, 2).contiguous(memory_format=torch.channels_last)
        with torch.no_grad():
            for k, b, s in self.layers:
                pt, pb = _same_pads(x.shape[2], k.shape[2], s)
                pl, pr = _same_pads(x.shape[3], k.shape[3], s)
                x = torch.relu(F.conv2d(F.pad(x, (pl, pr, pt, pb)), k, b, stride=s))
            z = x.reshape(x.shape[0], -1) @ self.dense_w + self.dense_b     # NCHW flatten against the re-indexed kernel
            ss = torch.clamp((z * z).sum(1, keepdim=True), min=1e-12)
            zq = z * torch.rsqrt(ss)
            return (zq @ self.codebook_t).numpy()

    def __call__(self, crops: np.ndarray) -> np.ndarray:
        return np.argmax(self.cos(crops), axis=1)


def best_thread_count(fn, candidates=(1, 2, 4, 8, 16, 32, 64, 128, 256), repeats: int = 2, min_threads: int = 1):
    """Times ``fn()`` under torch.set_num_threads(t) for every candidate min_threads <= t <= the machine's cores and leaves
    torch set to the fastest.  Returns (threads, seconds per call at that setting, {t: seconds})."""
    import os
    import time
    ncpu = len(os.sched_getaffinity(0)) if hasattr(os, "sched_getaffinity") else (os.cpu_count() or 1)   # the cores this process may use
    cands = sorted({t for t in candidates if min_threads <= t <= ncpu} | {ncpu})
    table = {}
    for t in cands:
        torch.set_num_threads(t)
        fn()
        best = float("inf")
        for _ in range(repeats):
            t0 = time.perf_counter()
            fn()
            best = min(best, time.perf_counter() - t0)
        table[t] = best
    win = min(table, key=table.get)
    torch.set_num_threads(win)
    return win, table[win], table
