"""AE: total loss + global step.  Mirrors auto_pose/ae/ae.py:11-53."""
import numpy as np

from .session import Tensor, Variable
from .utils import lazy_property


class AE(object):

    def __init__(self, encoder, decoder, norm_regularize, variational):
        self._encoder = encoder
        self._decoder = decoder
        self._norm_regularize = norm_regularize
        self._variational = variational
        self.loss
        self.global_step

    @property
    def x(self):
        return self._encoder.x

    @property
    def z(self):
        return self._encoder.z

    @property
    def reconstruction(self):
        return self._decoder.x

    @property
    def reconstruction_target(self):
        return self._decoder.reconstruction_target

    @lazy_property
    def global_step(self):
        return Variable(0, dtype=np.int64, trainable=False, name="global_step")

    @lazy_property
    def loss(self):
        def fn(ctx):
            loss = ctx.get(self._decoder.reconstr_loss)
            if self._norm_regularize > 0:
                loss = loss + ctx.get(self._encoder.reg_loss) * float(self._norm_regularize)
            if self._variational:
                loss = loss + ctx.get(self._encoder.kl_div_loss) * float(self._variational)
            return loss
        return Tensor("total_loss", (), np.float32, fn)
