"""Encoder: 128x128x3 crop -> latent z.  Mirrors auto_pose/ae/encoder.py:12-68 (class name, constructor arguments,
``x`` / ``z`` / ``encoder_out`` / ``latent_space_size``); the TF layers are replaced by the CUDA kernels behind
``aae_encoder_*`` (include/aae_b200.h)."""
import ctypes as C
import math

import numpy as np
import torch

from .. import _lib
from .session import Tensor, scoped, to_device_input
from .utils import lazy_property

DEFAULT_MAX_BATCH = 256


def glorot_uniform(rng, shape):
    """tf.layers default kernel_initializer (none is passed at encoder.py:43-50,62-66)."""
    if len(shape) == 4:
        rf = shape[0] * shape[1]
        fan_in, fan_out = rf * shape[2], rf * shape[3]
    else:
        fan_in, fan_out = shape
    limit = math.sqrt(6.0 / (fan_in + fan_out))
    return rng.uniform(-limit, limit, size=shape).astype(np.float32)


class _RawCudaArray:
    """Wraps a raw device pointer owned by a C handle through the CUDA array interface (zero copy)."""

    def __init__(self, ptr, shape, typestr="<f4"):
        self.__cuda_array_interface__ = {"shape": tuple(shape), "typestr": typestr, "data": (int(ptr), False), "version": 2}


def tensor_from_ptr(ptr, shape, device, typestr="<f4"):
    return torch.as_tensor(_RawCudaArray(ptr, shape, typestr), device=device)


class _DeviceModule:
    """Shared plumbing for Encoder / Decoder: named variables + one C handle per device."""

    _create = _destroy = _set = _get = None

    def _init_module(self, cfg_args, var_shapes, seed):
        self._cfg_args = cfg_args
        self._var_shapes = var_shapes                 # list of (kernel_name, kernel_shape, bias_name, bias_shape)
        rng = np.random.RandomState(seed)
        self._host = {}
        for kn, ks, bn, bs in var_shapes:
            self._host[kn] = glorot_uniform(rng, ks)
            self._host[bn] = np.zeros(bs, np.float32)
        self._handles = {}

    # -- variables -------------------------------------------------------------------------
    @property
    def variable_names(self):
        return [n for kn, _, bn, _ in self._var_shapes for n in (kn, bn)]

    def load_weights(self, weights, strict=True):
        """weights: {variable name (full scoped name, or without the scope prefix): array in the reference layout}.
        Like ``tf.train.Saver.restore``, a variable of this module that the dict does not hold is an error (KeyError naming every
        missing one; nothing is modified then) unless ``strict=False`` (partial update)."""
        found, missing = {}, []
        for kn, ks, bn, bs in self._var_shapes:
            for name, shape in ((kn, ks), (bn, bs)):
                short = "/".join(name.split("/")[-2:])
                src = weights.get(name, weights.get(short))
                if src is None:
                    missing.append(name)
                    continue
                arr = np.ascontiguousarray(np.asarray(src, dtype=np.float32))
                if arr.shape != tuple(shape):
                    raise ValueError("%s: shape %s != expected %s" % (name, arr.shape, tuple(shape)))
                found[name] = arr
        if missing and strict:
            raise KeyError("variables not found in the checkpoint / weight dict (wrong experiment scope?): %s" % ", ".join(missing))
        self._host.update(found)
        for dev, h in self._handles.items():
            self._upload(dev, h)

    def get_weights(self, device=None, short_names=False):
        """Current values; once a device handle exists (e.g. after training) they are read back from it."""
        if self._handles:
            dev = device if device is not None else next(iter(self._handles))
            h = self._handles[dev]
            with torch.cuda.device(dev):
                stream = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)     # behind the steps the caller launched on it
                for i, (kn, ks, bn, bs) in enumerate(self._var_shapes):
                    k = np.empty(ks, np.float32)
                    b = np.empty(bs, np.float32)
                    _lib.check(self._get(h, i, _lib.ptr(k), _lib.ptr(b), stream), "get_weights")
                    self._host[kn], self._host[bn] = k, b
        if short_names:
            return {"/".join(k.split("/")[-2:]): v for k, v in self._host.items()}
        return dict(self._host)

    def _upload(self, dev, h):
        with torch.cuda.device(dev):
            stream = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)         # ahead of the forwards the caller launches on it
            for i, (kn, ks, bn, bs) in enumerate(self._var_shapes):
                _lib.check(self._set(h, i, _lib.ptr(self._host[kn]), _lib.ptr(self._host[bn]), stream), "set_weights(%s)" % kn)

    def handle(self, device):
        dev = device.index if isinstance(device, torch.device) else int(device)
        if dev not in self._handles:
            cfg = _lib.make_cfg(*self._cfg_args)
            h = C.c_void_p()
            st = self._create(dev, C.byref(cfg), C.byref(h))
            if st == -3 and getattr(self, "_auto_precision", False) and cfg.precision == _lib.PREC_TC_SPLIT:
                # geometry outside what the tensor-core kernels are built for (e.g. a toy network): both paths are this
                # library's CUDA kernels, the fp32 CUDA-core one handles every geometry
                self.precision = _lib.PREC_FP32_SIMT
                self._cfg_args = self._cfg_args[:-1] + (self.precision,)
                cfg = _lib.make_cfg(*self._cfg_args)
                st = self._create(dev, C.byref(cfg), C.byref(h))
            _lib.check(st, type(self).__name__ + " create")
            try:
                self._prepare(h)
                self._upload(dev, h)
            except Exception:          # e.g. a weight outside the tensor-core range: no half-initialised handle may stay behind
                self._destroy(h)
                raise
            self._handles[dev] = h
        return self._handles[dev]

    def _prepare(self, h):
        """Called on a new handle before the variables are uploaded to it."""

    def check_range(self, device=None):
        """Raises AaeError if a forward / training step launched so far on this module left the range of the split-fp16
        tensor-core arithmetic (|activation| >= 4095, or weights an optimizer step carried out of range; include/aae_b200.h: aae_*_range_status).  Synchronises the current
        stream, so the asynchronous device entry points (encode_device / decode_device) do not call it; every path that
        hands results to the host does."""
        for dev, h in self._handles.items():
            if device is not None and dev != (device.index if isinstance(device, torch.device) else int(device)):
                continue
            with torch.cuda.device(dev):
                _lib.check(self._range_status(h, C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)), type(self).__name__ + " range check")

    def set_precision(self, precision):
        """Re-create the device handles with another aae_precision (weights are kept; device-side values are read back first)."""
        precision = int(precision)
        if precision == self.precision:
            return
        if self._handles:
            self.get_weights()
        self.close()
        self.precision = precision
        self._auto_precision = False
        self._cfg_args = self._cfg_args[:-1] + (precision,)

    def close(self):
        for h in self._handles.values():
            self._destroy(h)
        self._handles = {}

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class Encoder(_DeviceModule):

    def __init__(self, input, latent_space_size, num_filters, kernel_size, strides, batch_norm, is_training=False,
                 precision=None, max_batch=DEFAULT_MAX_BATCH, seed=42):
        if batch_norm:
            raise NotImplementedError("BATCH_NORMALIZATION: True is not supported (False in every shipped config, "
                                      "auto_pose/ae/cfg/train_template.cfg:45)")
        L = _lib.lib()
        self._create, self._destroy = L.aae_encoder_create, L.aae_encoder_destroy
        self._set, self._get = L.aae_encoder_set_weights, L.aae_encoder_get_weights
        self._range_status = L.aae_encoder_range_status
        self._input = input
        self._latent_space_size = int(latent_space_size)
        self._num_filters = list(num_filters)
        self._kernel_size = int(kernel_size)
        self._strides = list(strides)
        self._batch_normalization = batch_norm
        self._is_training = is_training
        shape = input.get_shape().as_list()
        h, w, c = shape[1:]
        self._in_shape = (h, w, c)
        self.max_batch = int(max_batch)
        # default: tensor cores (fp32-grade split-fp16 arithmetic) for inference and training; precision=_lib.PREC_FP32_SIMT
        # selects the fp32 CUDA-core path (exact fp32 operation order; ~10x slower), precision=_lib.PREC_TC_FP16 the inference-only
        # single-pass fp16 path (TF32-class rounding; never chosen automatically, and never replaced by another precision)
        self._auto_precision = precision is None
        if precision is None:
            precision = _lib.PREC_TC_SPLIT
        self.precision = int(precision)
        var_shapes = []
        cin, hh, ww = c, h, w
        for i, (f, s) in enumerate(zip(self._num_filters, self._strides)):
            base = scoped("conv2d" if i == 0 else "conv2d_%d" % i)
            var_shapes.append((base + "/kernel", (self._kernel_size, self._kernel_size, cin, f), base + "/bias", (f,)))
            cin, hh, ww = f, -(-hh // s), -(-ww // s)
        self._flat = hh * ww * cin
        var_shapes.append((scoped("dense/kernel"), (self._flat, self._latent_space_size), scoped("dense/bias"), (self._latent_space_size,)))
        self._init_module((h, w, c, self._num_filters, self._strides, self._kernel_size, self._latent_space_size,
                           self.max_batch, self.precision), var_shapes, seed)
        self._scope_prefix = scoped("dense/kernel")[:-len("dense/kernel")]
        self._has_sigma_head = False
        self._eps_rng = np.random.RandomState(seed)
        self.encoder_out
        self.z

    @property
    def x(self):
        return self._input

    @property
    def latent_space_size(self):
        return self._latent_space_size

    # -- device entry point (torch tensors in, torch tensor out; no host round trip) -------------
    def encode_device(self, x_dev, out=None):
        """x_dev: CUDA tensor [B,H,W,C], uint8 (divided by 255 inside the kernel) or float32.  Returns z [B, latent]."""
        dev = x_dev.device
        h = self.handle(dev)
        B = x_dev.shape[0]
        if tuple(x_dev.shape[1:]) != self._in_shape:
            raise ValueError("crop shape %s != %s" % (tuple(x_dev.shape[1:]), self._in_shape))
        if out is None:
            out = torch.empty((B, self._latent_space_size), dtype=torch.float32, device=dev)
        fwd = _lib.lib().aae_encoder_forward_u8 if x_dev.dtype == torch.uint8 else _lib.lib().aae_encoder_forward_f32
        stream = torch.cuda.current_stream(dev).cuda_stream
        for a in range(0, B, self.max_batch):
            e = min(B, a + self.max_batch)
            _lib.check(fwd(h, _lib.ptr(x_dev[a:e]), e - a, _lib.ptr(out[a:e]), C.c_void_p(stream)), "encoder forward")
        return out

    def _eval_input(self, ctx):
        if self not in ctx.touched:
            ctx.touched.append(self)
        x = to_device_input(ctx.get(self._input), ctx.session.device)
        if x.ndim == 3:
            x = x.unsqueeze(0)
        return x

    def range_word(self, device):
        """The range guard's device word as an int32 tensor view (None on the fp32 path): see aae_encoder_range_word."""
        h = self.handle(device)
        p = C.c_void_p()
        _lib.check(_lib.lib().aae_encoder_range_word(h, C.byref(p)), "range word")
        return tensor_from_ptr(p.value, (1,), device, typestr="<i4") if p.value else None

    @lazy_property
    def z(self):
        return Tensor("dense/BiasAdd", (None, self._latent_space_size), np.float32,
                      lambda ctx: self.encode_device(self._eval_input(ctx)))

    @lazy_property
    def encoder_out(self):
        def fn(ctx):
            ctx.get(self.z)
            h = self.handle(ctx.session.device)
            p, n = C.c_void_p(), C.c_int64()
            _lib.check(_lib.lib().aae_encoder_activation(h, len(self._num_filters), C.byref(p), C.byref(n)), "encoder_out")
            B = n.value // self._flat
            return tensor_from_ptr(p.value, (B, self._flat), ctx.session.device).clone()
        return Tensor("flatten/Reshape", (None, self._flat), np.float32, fn)

    def activation_device(self, layer, device):
        """NHWC fp32 activation of conv layer `layer` from the last forward on `device` (fp32 SIMT path only)."""
        h = self.handle(device)
        p, n = C.c_void_p(), C.c_int64()
        _lib.check(_lib.lib().aae_encoder_activation(h, layer, C.byref(p), C.byref(n)), "activation")
        f = self._num_filters[layer]
        hh, ww = self._in_shape[0], self._in_shape[1]
        for s in self._strides[:layer + 1]:
            hh, ww = -(-hh // s), -(-ww // s)
        B = n.value // (hh * ww * f)
        return tensor_from_ptr(p.value, (B, hh, ww, f), device).clone()

    # -- variational AE: sigma head, sampled z, KL term (auto_pose/ae/encoder.py:70-95) -------------------------------
    def _register_sigma_head(self):
        """Creates the head's variables, zero-initialised (kernel_initializer=zeros, default zero bias).  TF numbers dense layers
        per scope: the head is the second one, "<scope>/dense_1" (the decoder's dense layer then becomes "dense_2")."""
        if self._has_sigma_head:
            return
        J = self._latent_space_size
        kn, bn = self._scope_prefix + "dense_1/kernel", self._scope_prefix + "dense_1/bias"
        self._var_shapes.append((kn, (self._flat, J), bn, (J,)))
        self._host[kn] = np.zeros((self._flat, J), np.float32)
        self._host[bn] = np.zeros((J,), np.float32)
        self._has_sigma_head = True
        layer = len(self._num_filters) + 1
        for dev, h in self._handles.items():
            with torch.cuda.device(dev):
                self._prepare(h)
                _lib.check(self._set(h, layer, _lib.ptr(self._host[kn]), _lib.ptr(self._host[bn]),
                                     C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)), "set_weights(%s)" % kn)

    def _prepare(self, h):
        if self._has_sigma_head:
            _lib.check(_lib.lib().aae_encoder_enable_sigma_head(h), "enable sigma head")

    def _sigma_of_last_forward(self, device, B):
        out = torch.empty((B, self._latent_space_size), dtype=torch.float32, device=device)
        _lib.check(_lib.lib().aae_encoder_sigma_forward(self.handle(device), B, _lib.ptr(out),
                                                        C.c_void_p(torch.cuda.current_stream(device).cuda_stream)), "sigma forward")
        return out

    def run_eps(self, ctx, draw=None):
        """eps of sampled_z in this Session.run: one scalar N(0,1) per run (tf.shape of the Python int latent_space_size is an
        empty shape, so tf.random_normal draws a single value), shared by every fetch of the run.  ``draw`` (a callable)
        supplies it when this run has none yet; else the encoder's own seeded stream does."""
        key = ("latent_eps", id(self))                 # the Encoder outlives every RunContext, so its id is stable
        if key not in ctx.memo:
            ctx.memo[key] = np.float32(draw() if draw is not None else self._eps_rng.standard_normal())
        return ctx.memo[key]

    @lazy_property
    def q_sigma(self):
        """1e-8 + softplus(encoder_out . W + b) on the device (aae_encoder_sigma_forward)."""
        self._register_sigma_head()

        def fn(ctx):
            dev = ctx.session.device
            x = self._eval_input(ctx)
            if x.shape[0] <= self.max_batch:
                ctx.get(self.z)
                return self._sigma_of_last_forward(dev, x.shape[0])
            parts = []
            for a in range(0, x.shape[0], self.max_batch):
                chunk = x[a:a + self.max_batch]
                self.encode_device(chunk)
                parts.append(self._sigma_of_last_forward(dev, chunk.shape[0]))
            return torch.cat(parts)
        return Tensor("add", (None, self._latent_space_size), np.float32, fn)

    @lazy_property
    def sampled_z(self):
        """z + q_sigma * eps, eps one scalar per Session.run (run_eps)."""
        q_sigma = self.q_sigma
        t = Tensor("add_1", (None, self._latent_space_size), np.float32,
                   lambda ctx: ctx.get(self.z) + ctx.get(q_sigma) * float(self.run_eps(ctx)))
        t.sigma_head = True                            # a decoder built on it is the scope's third dense layer
        return t

    @lazy_property
    def kl_div_loss(self):
        """mean over [B, latent] of KL(N(z, q_sigma) || N(0, 1)) in TF's form z^2/2 + (s^2 - 1 - log s^2)/2; torch on the device
        tensors, like reg_loss."""
        q_sigma = self.q_sigma

        def fn(ctx):
            z, s2 = ctx.get(self.z), ctx.get(q_sigma) ** 2
            return (0.5 * z * z + 0.5 * (s2 - 1.0 - torch.log(s2))).mean()
        return Tensor("kl_div_loss", (), np.float32, fn)

    @lazy_property
    def reg_loss(self):
        """mean(| ||z|| - 1 |) (auto_pose/ae/encoder.py:97-100); evaluated with torch on the device z."""
        return Tensor("reg_loss", (), np.float32,
                      lambda ctx: (torch.linalg.vector_norm(ctx.get(self.z), dim=1) - 1.0).abs().mean())
