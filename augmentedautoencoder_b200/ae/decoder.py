"""Decoder + reconstruction loss.  Mirrors auto_pose/ae/decoder.py:13-144 (constructor arguments, ``x``,
``reconstr_loss``, ``reconstruction_target``)."""
import ctypes as C

import numpy as np
import torch

from .. import _lib
from .encoder import _DeviceModule
from .session import Tensor, scoped, to_device_input
from .utils import lazy_property


class Decoder(_DeviceModule):

    def __init__(self, reconstruction_target, latent_code, num_filters, kernel_size, strides, loss, bootstrap_ratio,
                 auxiliary_mask, batch_norm, is_training=False, max_batch=64, seed=43, n_encoder_convs=None, precision=None):
        if batch_norm:
            raise NotImplementedError("BATCH_NORMALIZATION: True is not supported")
        if loss != "L2":
            raise NotImplementedError("LOSS: %s is not supported (template cfg uses L2)" % loss)
        L = _lib.lib()
        self._create, self._destroy = L.aae_decoder_create, L.aae_decoder_destroy
        self._set, self._get = L.aae_decoder_set_weights, L.aae_decoder_get_weights
        self._range_status = L.aae_decoder_range_status
        self._reconstruction_target = reconstruction_target
        self._latent_code = latent_code
        self._auxiliary_mask = bool(auxiliary_mask)
        self._num_filters = list(num_filters)      # already reversed by build_decoder (ae_factory.py:62)
        self._kernel_size = int(kernel_size)
        self._strides = list(strides)
        self._loss = loss
        self._bootstrap_ratio = int(bootstrap_ratio)
        self._batch_normalization = batch_norm
        self._is_training = is_training
        self.max_batch = int(max_batch)
        h, w, c = reconstruction_target.get_shape().as_list()[1:]
        self._out_shape = (h, w, c)
        latent = latent_code.get_shape().as_list()[-1]
        self._latent = latent
        nl = len(self._num_filters)
        dims = [int(h / np.prod(self._strides[i:])) for i in range(nl)]
        k0 = n_encoder_convs if n_encoder_convs is not None else nl
        # TF numbers dense layers per scope: after the encoder's sigma head (built when the decoder reads the sampled z) this is
        # the third one
        dense = "dense_2" if getattr(latent_code, "sigma_head", False) else "dense_1"
        var_shapes = [(scoped(dense + "/kernel"), (latent, dims[0] * dims[0] * self._num_filters[0]),
                       scoped(dense + "/bias"), (dims[0] * dims[0] * self._num_filters[0],))]
        cin = self._num_filters[0]
        for j, f in enumerate(self._num_filters[1:] + [c]):
            # the mask head is created before the output conv, so TF numbers it conv2d_<k0+nl-1> and the output conv one higher
            base = scoped("conv2d_%d" % (k0 + j + (1 if self._auxiliary_mask and j == nl - 1 else 0)))
            var_shapes.append((base + "/kernel", (self._kernel_size, self._kernel_size, cin, f), base + "/bias", (f,)))
            cin = f
        if self._auxiliary_mask:
            # C ABI layer num_layers + 1 (aae_decoder_enable_mask_head): conv over the output conv's input, one sigmoid channel.
            # Appended last, so its initial values come after every other variable's in the seeded stream.
            base = scoped("conv2d_%d" % (k0 + nl - 1))
            var_shapes.append((base + "/kernel", (self._kernel_size, self._kernel_size, self._num_filters[-1], 1), base + "/bias", (1,)))
        # same default as the encoder: tensor cores unless precision=_lib.PREC_FP32_SIMT is asked for
        self._auto_precision = precision is None
        if precision is None:
            precision = _lib.PREC_TC_SPLIT
        self.precision = int(precision)
        # the C ABI takes the encoder-order filters/strides and reverses them itself (aae_net_cfg)
        self._init_module((h, w, c, list(reversed(self._num_filters)), list(reversed(self._strides)), self._kernel_size,
                           latent, self.max_batch, self.precision), var_shapes, seed)
        if self._auxiliary_mask:
            # [B, H, W, 1] sigmoid output of the mask head (decoder.py:68-75), from the same forward as x in a Session.run
            self._xmask = Tensor("conv2d_mask/Sigmoid", (None, h, w, 1), np.float32, lambda ctx: self._forward(ctx)[1])
        self.reconstr_loss

    @property
    def reconstruction_target(self):
        return self._reconstruction_target

    def _prepare(self, h):
        if self._auxiliary_mask:
            _lib.check(_lib.lib().aae_decoder_enable_mask_head(h), "enable mask head")

    def decode_device(self, z_dev, with_mask=False):
        """x [B, H, W, C]; with_mask=True (a decoder with the mask head): (x, xmask [B, H, W, 1]) from one forward."""
        dev = z_dev.device
        h = self.handle(dev)
        B = z_dev.shape[0]
        out = torch.empty((B,) + self._out_shape, dtype=torch.float32, device=dev)
        mask = torch.empty((B,) + self._out_shape[:2] + (1,), dtype=torch.float32, device=dev) if with_mask else None
        stream = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
        for a in range(0, B, self.max_batch):
            e = min(B, a + self.max_batch)
            z = z_dev[a:e].contiguous()         # kept alive until the call has been enqueued
            if with_mask:
                _lib.check(_lib.lib().aae_decoder_forward_mask(h, _lib.ptr(z), e - a, _lib.ptr(out[a:e]), _lib.ptr(mask[a:e]), stream), "decoder forward")
            else:
                _lib.check(_lib.lib().aae_decoder_forward(h, _lib.ptr(z), e - a, _lib.ptr(out[a:e]), stream), "decoder forward")
        return (out, mask) if with_mask else out

    def _forward(self, ctx):
        """(x, xmask) of this Session.run, computed once for both fetches (decoder with the mask head)."""
        key = ("decoder_forward", id(self))
        if key not in ctx.memo:
            if self not in ctx.touched:
                ctx.touched.append(self)
            ctx.memo[key] = self.decode_device(to_device_input(ctx.get(self._latent_code), ctx.session.device), with_mask=True)
        return ctx.memo[key]

    @lazy_property
    def x(self):
        if self._auxiliary_mask:
            return Tensor("conv2d_out/Sigmoid", (None,) + self._out_shape, np.float32, lambda ctx: self._forward(ctx)[0])

        def fn(ctx):
            if self not in ctx.touched:
                ctx.touched.append(self)
            return self.decode_device(to_device_input(ctx.get(self._latent_code), ctx.session.device))   # a fed latent may be numpy
        return Tensor("conv2d_out/Sigmoid", (None,) + self._out_shape, np.float32, fn)

    @staticmethod
    def loss_device(x_dev, target_dev, bootstrap_ratio, with_grad=False):
        """Bootstrapped L2 on device tensors -> (loss 0-d tensor, grad or None)."""
        if target_dev.dtype == torch.uint8:          # the kernel reads float*: a uint8 target is the image / 255 (as the trainer's feed)
            target_dev = target_dev.to(torch.float32) / 255.0
        if x_dev.dtype != torch.float32 or target_dev.dtype != torch.float32 or x_dev.shape != target_dev.shape:
            raise ValueError("bootstrapped L2 wants float32 tensors of one shape, got %s %s / %s %s"
                             % (x_dev.dtype, tuple(x_dev.shape), target_dev.dtype, tuple(target_dev.shape)))
        B = x_dev.shape[0]
        numel = x_dev[0].numel()
        loss = torch.empty((1,), dtype=torch.float32, device=x_dev.device)
        grad = torch.empty_like(x_dev) if with_grad else None
        stream = C.c_void_p(torch.cuda.current_stream(x_dev.device).cuda_stream)
        _lib.check(_lib.lib().aae_bootstrap_l2_loss(_lib.ptr(x_dev.contiguous()), _lib.ptr(target_dev.contiguous()), B, numel,
                                                    int(bootstrap_ratio), _lib.ptr(loss), _lib.ptr(grad), stream), "bootstrap_l2")
        return loss[0], grad

    @staticmethod
    def mask_loss_device(xmask_dev, target_dev, loss=None, with_grad=False):
        """Mask loss of AUXILIARY_MASK (decoder.py:134-140) on device tensors: mean of (xmask - m)^2 with m = float(sum of the
        target's channels > 0.0001), added to ``loss`` (a 1-element float32 tensor; None: a new zero).  -> (loss 0-d, grad or None)."""
        if target_dev.dtype == torch.uint8:          # as loss_device: the image / 255
            target_dev = target_dev.to(torch.float32) / 255.0
        B, H, W = target_dev.shape[:3]
        if xmask_dev.dtype != torch.float32 or target_dev.dtype != torch.float32 or xmask_dev.numel() != B * H * W:
            raise ValueError("mask loss wants float32 tensors [B,H,W,1] / [B,H,W,C], got %s %s / %s %s"
                             % (xmask_dev.dtype, tuple(xmask_dev.shape), target_dev.dtype, tuple(target_dev.shape)))
        if loss is None:
            loss = torch.zeros((1,), dtype=torch.float32, device=xmask_dev.device)
        grad = torch.empty_like(xmask_dev) if with_grad else None
        stream = C.c_void_p(torch.cuda.current_stream(xmask_dev.device).cuda_stream)
        _lib.check(_lib.lib().aae_mask_loss(_lib.ptr(xmask_dev.contiguous()), _lib.ptr(target_dev.contiguous()), B, H * W,
                                            target_dev.shape[3], _lib.ptr(loss), _lib.ptr(grad), stream), "mask loss")
        return loss[0], grad

    @lazy_property
    def reconstr_loss(self):
        def fn(ctx):
            x = ctx.get(self.x)
            y = to_device_input(ctx.get(self._reconstruction_target), ctx.session.device)
            loss = self.loss_device(x, y, self._bootstrap_ratio)[0]
            if self._auxiliary_mask:                 # reconstr_loss = bootstrapped L2 + mask_loss, fp32 add on the device
                loss = self.mask_loss_device(ctx.get(self._xmask), y, loss=loss.reshape(1))[0]
            return loss
        return Tensor("reconstr_loss", (), np.float32, fn)
