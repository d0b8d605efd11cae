"""Config -> object constructors.  Mirrors auto_pose/ae/ae_factory.py:11-172: same function names, argument order and
cfg keys; ``tf.placeholder`` / ``tf.variable_scope`` / ``tf.train.Saver`` are served by augmentedautoencoder_b200.ae.session
and the checkpoint helpers below."""
import ctypes as C
import glob
import os

import numpy as np
import torch

from .. import _lib
from . import session as S
from . import utils as u
from .ae import AE
from .codebook import Codebook
from .dataset import Dataset
from .decoder import Decoder
from .encoder import Encoder
from .session import Tensor


def build_dataset(dataset_path, args):
    dataset_args = {k: v for k, v in
                    args.items('Dataset') + args.items('Paths') + args.items('Augmentation') +
                    args.items('Queue') + args.items('Embedding')}
    return Dataset(dataset_path, **dataset_args)


class Queue(object):
    """Stand-in for auto_pose/ae/queue.py:14-74 (TF FIFOQueue fed by Python threads): ``x`` / ``y`` evaluate to the next
    (augmented input, reconstruction target) batch from ``dataset.batch(batch_size)`` or a user-supplied callable.

    Until ``start(session)`` every run makes its batch synchronously.  ``start`` with the default source runs a producer thread
    (batch_producer.BatchProducer) that makes batches ahead on its own CUDA stream into QUEUE_SIZE device slots, from the
    training set kept on the device (``Dataset.upload``; ``start`` uploads it if it is not there yet).  The batches are the
    ones repeated synchronous calls would make, in the same order and with the same bits.  NUM_THREADS is accepted and does not
    change them: one thread makes every batch.  While the producer runs it is the only user of numpy's global random stream.
    ``stop`` joins the thread (batches made ahead are dropped); start / stop can be repeated.  With a ``source`` callable,
    start / stop do nothing.  A ``Session.run_device`` fetch of ``x`` / ``y`` of a started queue is the slot itself: valid
    until the next run that pulls a batch."""

    def __init__(self, dataset, num_threads, queue_size, batch_size, source=None):
        self._dataset = dataset
        self._batch_size = batch_size
        self._num_threads = num_threads
        self._queue_size = queue_size
        self._custom_source = source is not None
        self._source = source or (lambda n: dataset.batch(n))
        self._producer = None
        shape = (None,) + tuple(dataset.shape)
        self.x = Tensor("queue_x", shape, np.float32, lambda ctx: self._pull(ctx)[0])
        self.y = Tensor("queue_y", shape, np.float32, lambda ctx: self._pull(ctx)[1])

    def _pull(self, ctx):
        """One dequeue per ``Session.run``: x and y fetched in the same run see the same batch, the next run pulls the next
        one.  The batch lives in the run's own memo (not keyed by ``id(ctx)``: a freed context's address is reused)."""
        key = ("queue_batch", id(self))            # the Queue outlives every RunContext, so its id is stable
        if key not in ctx.memo:
            if self._producer is not None:
                ctx.memo[key] = self._producer.pull()
            else:
                x, y = self._source(self._batch_size)
                ctx.memo[key] = (S.to_device_input(x, ctx.session.device), S.to_device_input(y, ctx.session.device))
        return ctx.memo[key]

    def start(self, session):
        if self._custom_source or self._producer is not None:
            return
        from .batch_producer import BatchProducer
        self._producer = BatchProducer(self._dataset, self._batch_size, self._queue_size, session.device)

    def stop(self, session):
        if self._producer is not None:
            self._producer.close()
            self._producer = None


def build_queue(dataset, args, source=None):
    NUM_THREADS = args.getint('Queue', 'NUM_THREADS')
    QUEUE_SIZE = args.getint('Queue', 'QUEUE_SIZE')
    BATCH_SIZE = args.getint('Training', 'BATCH_SIZE')
    return Queue(dataset, NUM_THREADS, QUEUE_SIZE, BATCH_SIZE, source=source)


def build_encoder(x, args, is_training=False, precision=None, max_batch=None):
    LATENT_SPACE_SIZE = args.getint('Network', 'LATENT_SPACE_SIZE')
    NUM_FILTER = eval(args.get('Network', 'NUM_FILTER'))
    KERNEL_SIZE_ENCODER = args.getint('Network', 'KERNEL_SIZE_ENCODER')
    STRIDES = eval(args.get('Network', 'STRIDES'))
    BATCH_NORM = args.getboolean('Network', 'BATCH_NORMALIZATION')
    kw = {}
    if max_batch is not None:
        kw["max_batch"] = max_batch
    elif is_training:
        kw["max_batch"] = args.getint('Training', 'BATCH_SIZE')
    return Encoder(x, LATENT_SPACE_SIZE, NUM_FILTER, KERNEL_SIZE_ENCODER, STRIDES, BATCH_NORM, is_training=is_training,
                   precision=precision, **kw)


def build_decoder(reconstruction_target, encoder, args, is_training=False):
    NUM_FILTER = eval(args.get('Network', 'NUM_FILTER'))
    KERNEL_SIZE_DECODER = args.getint('Network', 'KERNEL_SIZE_DECODER')
    STRIDES = eval(args.get('Network', 'STRIDES'))
    LOSS = args.get('Network', 'LOSS')
    BOOTSTRAP_RATIO = args.getint('Network', 'BOOTSTRAP_RATIO')
    VARIATIONAL = args.getfloat('Network', 'VARIATIONAL') if is_training else False
    AUXILIARY_MASK = args.getboolean('Network', 'AUXILIARY_MASK')
    BATCH_NORM = args.getboolean('Network', 'BATCH_NORMALIZATION')
    return Decoder(reconstruction_target, encoder.sampled_z if VARIATIONAL else encoder.z, list(reversed(NUM_FILTER)), KERNEL_SIZE_DECODER,
                   list(reversed(STRIDES)),
                   LOSS, BOOTSTRAP_RATIO, AUXILIARY_MASK, BATCH_NORM, is_training=is_training, max_batch=encoder.max_batch,
                   n_encoder_convs=len(NUM_FILTER))


def build_ae(encoder, decoder, args):
    NORM_REGULARIZE = args.getfloat('Network', 'NORM_REGULARIZE')
    VARIATIONAL = args.getfloat('Network', 'VARIATIONAL')
    return AE(encoder, decoder, NORM_REGULARIZE, VARIATIONAL)


# cfg OPTIMIZER -> (aae_optimizer_kind, aae_optimizer.hp at TF's defaults, slot names in TF's creation order).  The reference builds
# tf.train.<OPTIMIZER>Optimizer(LEARNING_RATE) (ae_factory.py:79-95), so every other constructor argument keeps TF's default.
# Formulas, initial slot values and what is unverified: DESIGN.md section 3.
OPTIMIZERS = {
    "Adam": (_lib.OPT_ADAM, (0.9, 0.999, 1e-8), ("Adam", "Adam_1")),
    "GradientDescent": (_lib.OPT_GRADIENT_DESCENT, (), ()),
    "ProximalGradientDescent": (_lib.OPT_GRADIENT_DESCENT, (), ()),      # l1 = l2 = 0: gradient descent bit for bit
    "Adagrad": (_lib.OPT_ADAGRAD, (0.1,), ("Adagrad",)),                   # initial_accumulator_value
    "ProximalAdagrad": (_lib.OPT_PROXIMAL_ADAGRAD, (0.1,), ("ProximalAdagrad",)),
    "Adadelta": (_lib.OPT_ADADELTA, (0.95, 1e-8), ("Adadelta", "Adadelta_1")),       # rho, epsilon
    "RMSProp": (_lib.OPT_RMSPROP, (0.9, 0.0, 1e-10), ("RMSProp", "RMSProp_1")),      # decay, momentum, epsilon
    "Ftrl": (_lib.OPT_FTRL, (0.1,), ("Ftrl", "Ftrl_1")),                            # initial_accumulator_value
}
# tf.train optimizers whose constructor needs an argument besides the learning rate: the reference's call fails for them
_NEEDS_ARGUMENT = {"Momentum": "momentum", "AdagradDA": "global_step"}


def optimizer_spec(name):
    """(kind, hp, slot names) of a cfg OPTIMIZER; ValueError for a name no reference cfg can train with."""
    if name in _NEEDS_ARGUMENT:
        raise ValueError("OPTIMIZER: %s: tf.train.%sOptimizer needs `%s`, which a cfg cannot pass, so the reference cannot build it from a "
                         "cfg either" % (name, name, _NEEDS_ARGUMENT[name]))
    if name not in OPTIMIZERS:
        raise ValueError("OPTIMIZER: %s is not one of the tf.train optimizers a cfg can build: %s" % (name, ", ".join(OPTIMIZERS)))
    return OPTIMIZERS[name]


class TrainOp(Tensor):
    """``session.run(train_op)``: encoder fwd, decoder fwd, bootstrapped L2, backward, the optimizer update, global_step += 1 -- one
    call into aae_train_step (replaces slim.learning.create_train_op, ae_factory.py:86-88).  Evaluates to the loss.

    ``optimizer`` is a cfg OPTIMIZER name (OPTIMIZERS).  beta1, beta2 and epsilon are Adam's; every other rule runs at TF's
    defaults, the only values a cfg reaches.

    ``precision`` picks the GEMM arithmetic of the step apart from the handles' (aae_trainer_create_prec).  None follows the
    handles.  ``_lib.PREC_TC_FP16`` is the single-pass trainer: it needs PREC_TC_SPLIT encoder and decoder handles, which keep
    that precision for inference, and raises for any other handles instead of switching their precision."""

    def __init__(self, ae, learning_rate, beta1=0.9, beta2=0.999, epsilon=1e-8, precision=None, noise_seed=0, optimizer="Adam"):
        """noise_seed seeds the stream of VARIATIONAL's eps, one N(0,1) draw per step (Encoder.run_eps)."""
        super().__init__("train_op", (), np.float32, self._run)
        self._ae = ae
        self._hp = (float(learning_rate), float(beta1), float(beta2), float(epsilon))
        kind, hp, self._slots = optimizer_spec(optimizer)
        hp = self._hp[1:] if kind == _lib.OPT_ADAM else hp
        self._opt = _lib.Optimizer(kind, self._hp[0], (C.c_float * 4)(*hp))
        self._precision = None if precision is None else int(precision)
        self._trainers = {}
        self._eps_rng = np.random.RandomState(noise_seed)

    def trainer(self, device):
        dev = device.index
        if dev not in self._trainers:
            ae = self._ae
            enc, dec = ae._encoder, ae._decoder
            if _lib.PREC_TC_FP16 in (enc.precision, dec.precision):
                # never switch a precision the caller chose: the fp16 mode has no backward pass
                raise _lib.AaeError("training needs precision PREC_TC_SPLIT or PREC_FP32_SIMT; PREC_TC_FP16 is inference-only "
                                    "(create the encoder with another precision for training)")
            if ae._variational and dec._latent_code is not enc.sampled_z:
                # the fused step feeds the decoder the sampled z exactly when VARIATIONAL is set, as build_decoder wires it
                raise NotImplementedError("VARIATIONAL != 0 trains a decoder built on encoder.sampled_z (build_decoder(..., "
                                          "is_training=True)); this decoder reads %s" % dec._latent_code.name)
            h = C.c_void_p()
            with torch.cuda.device(dev):
                eh, dh = enc.handle(device), dec.handle(device)       # settles automatic precisions
                def create(eh, dh, gemm):
                    return _lib.lib().aae_trainer_create_opt(eh, dh, dec._bootstrap_ratio, C.byref(self._opt), gemm, C.byref(h))
                if self._precision is not None:
                    # an explicit GEMM precision: the handles must suit it as they are (an automatic fp32 fallback does not)
                    _lib.check(create(eh, dh, self._precision), "trainer create (GEMM precision %d)" % self._precision)
                else:
                    # GEMMs at the handles' own precision (aae_trainer_create)
                    st = -3 if enc.precision != dec.precision else create(eh, dh, enc.precision)
                    if st == -3 and (enc._auto_precision or dec._auto_precision or enc.precision != dec.precision) and \
                            (enc.precision, dec.precision) != (_lib.PREC_FP32_SIMT, _lib.PREC_FP32_SIMT):
                        # a geometry the tensor-core trainer is not built for: the fp32 CUDA-core trainer handles every geometry
                        enc.set_precision(_lib.PREC_FP32_SIMT)
                        dec.set_precision(_lib.PREC_FP32_SIMT)
                        st = create(enc.handle(device), dec.handle(device), _lib.PREC_FP32_SIMT)
                    _lib.check(st, "trainer create")
                if ae._variational or ae._norm_regularize > 0:
                    # AE.loss adds reg_loss only for NORM_REGULARIZE > 0 and the KL term for VARIATIONAL != 0 (ae.py:43-53)
                    st = _lib.lib().aae_trainer_set_latent_terms(h, float(ae._variational), float(max(ae._norm_regularize, 0.0)))
                    if st != 0:
                        msg = _lib.lib().aae_last_error_string().decode("utf-8", "replace")
                        _lib.lib().aae_trainer_destroy(h)
                        raise _lib.AaeError("latent terms (VARIATIONAL %g, NORM_REGULARIZE %g) failed (status %d): %s"
                                            % (ae._variational, ae._norm_regularize, st, msg))
            self._trainers[dev] = h
        return self._trainers[dev]

    def close(self):
        """Frees this op's device trainers: their gradient, scratch and optimizer-slot buffers.  Call it while the encoder and decoder
        are still open (a trainer is destroyed through their handles).  A later step creates a new trainer with fresh optimizer
        state."""
        for dev, h in self._trainers.items():
            with torch.cuda.device(dev):
                _lib.lib().aae_trainer_destroy(h)
        self._trainers = {}

    def _io(self, ctx):
        ae = self._ae
        x = S.to_device_input(ctx.get(ae._encoder.x), ctx.session.device)
        y = S.to_device_input(ctx.get(ae._decoder.reconstruction_target), ctx.session.device)
        if x.dtype == torch.uint8:
            x = x.to(torch.float32) / 255.0
        if y.dtype == torch.uint8:
            y = y.to(torch.float32) / 255.0
        return x.contiguous(), y.contiguous()

    def step_device(self, x, y, update=True, eps=None):
        """One step on device tensors; returns the total loss.  With VARIATIONAL, ``eps`` is the step's noise scalar (None: the
        next draw of this TrainOp's seeded stream)."""
        dev = x.device
        h = self.trainer(dev)
        if self._ae._variational:
            eps = self._eps_rng.standard_normal() if eps is None else eps
            _lib.check(_lib.lib().aae_trainer_set_latent_noise(h, float(np.float32(eps))), "latent noise")
        loss = torch.empty((1,), dtype=torch.float32, device=dev)
        fn = _lib.lib().aae_train_step if update else _lib.lib().aae_trainer_forward_backward
        _lib.check(fn(h, _lib.ptr(x), _lib.ptr(y), x.shape[0], _lib.ptr(loss), C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)),
                   "train step")
        if update:
            self._ae.global_step._host = np.asarray(self._ae.global_step.value() + 1, dtype=np.int64)
        return loss[0]

    def _run(self, ctx):
        x, y = self._io(ctx)
        for m in (self._ae._encoder, self._ae._decoder):
            if m not in ctx.touched:
                ctx.touched.append(m)
        eps = self._ae._encoder.run_eps(ctx, draw=self._eps_rng.standard_normal) if self._ae._variational else None
        return self.step_device(x, y, update=True, eps=eps)

    # -- optimizer state under TensorFlow's names: "<var>/<slot>" (OPTIMIZERS), and Adam's "<scope>/beta1_power", "<scope>/beta2_power"
    def _scope_prefix(self):
        name = self._ae._encoder._var_shapes[0][0]                    # e.g. "obj_05/conv2d/kernel"
        return name.rsplit("/", 2)[0] + "/" if name.count("/") >= 2 else ""

    def _slot_arrays(self, ks, bs):
        """(kernel slot 0, kernel slot 1, bias slot 0, bias slot 1): arrays for the rule's slots, None for the others"""
        n = len(self._slots)
        return [np.empty(shape, np.float32) if k < n else None for shape in (ks, bs) for k in (0, 1)]

    def optimizer_variables(self, device=None):
        """{TF name: array} of the optimizer's slots, and Adam's beta powers (what tf.train.Saver stores beside the weights,
        ae_train.py:82).  Empty until a trainer exists (no step has run): a fresh optimizer has nothing to save."""
        if not self._trainers:
            return {}
        dev = next(iter(self._trainers)) if device is None else (device.index if isinstance(device, torch.device) else int(device))
        h = self._trainers[dev]
        out = {}
        with torch.cuda.device(dev):
            stream = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)     # behind the steps the caller launched on it
            for which, mod in ((0, self._ae._encoder), (1, self._ae._decoder)):
                for i, (kn, ks, bn, bs) in enumerate(mod._var_shapes):
                    km, kv, bm, bv = self._slot_arrays(ks, bs)
                    _lib.check(_lib.lib().aae_trainer_get_state(h, which, i, _lib.ptr(km), _lib.ptr(kv), _lib.ptr(bm), _lib.ptr(bv), stream), "get_state")
                    for name, arrs in ((kn, (km, kv)), (bn, (bm, bv))):
                        for suffix, a in zip(self._slots, arrs):
                            out[name + "/" + suffix] = a
            step = int(_lib.lib().aae_trainer_global_step(h))
        if self._opt.kind != _lib.OPT_ADAM:
            return out
        lr, b1, b2, eps = self._hp
        # TF keeps beta^(t+1) after t updates (initialised to beta, multiplied once per apply)
        out[self._scope_prefix() + "beta1_power"] = np.asarray(b1 ** (step + 1), dtype=np.float32)
        out[self._scope_prefix() + "beta2_power"] = np.asarray(b2 ** (step + 1), dtype=np.float32)
        return out

    def load_optimizer_variables(self, weights, device, global_step=None):
        """Restore the optimizer's slots (and the update count) from a checkpoint dict; returns the names it used.  Variables
        without slots in the dict keep their current ones -- for a new trainer the rule's initial values, so a weights-only
        checkpoint restarts the optimizer, as in TF.  The step comes from ``global_step``, or for Adam from beta1_power."""
        h = self.trainer(device)
        used = []
        with torch.cuda.device(device):
            stream = C.c_void_p(torch.cuda.current_stream(device).cuda_stream)
            for which, mod in ((0, self._ae._encoder), (1, self._ae._decoder)):
                for i, (kn, ks, bn, bs) in enumerate(mod._var_shapes):
                    arrs = []
                    names = [base + "/" + self._slots[k] if k < len(self._slots) else None for base in (kn, bn) for k in (0, 1)]
                    for name, shape in zip(names, (ks, ks, bs, bs)):
                        a = weights.get(name) if name else None
                        if a is not None:
                            a = np.ascontiguousarray(np.asarray(a, dtype=np.float32))
                            if a.shape != tuple(shape):
                                raise ValueError("%s: shape %s != expected %s" % (name, a.shape, tuple(shape)))
                            used.append(name)
                        arrs.append(a)
                    if any(a is not None for a in arrs):
                        _lib.check(_lib.lib().aae_trainer_set_state(h, which, i, *[_lib.ptr(a) for a in arrs], stream), "set_state")
            step = global_step
            b1p = weights.get(self._scope_prefix() + "beta1_power") if self._opt.kind == _lib.OPT_ADAM else None
            if step is None and b1p is not None and 0.0 < float(b1p) < 1.0:
                step = int(round(np.log(float(b1p)) / np.log(self._hp[1]))) - 1
            if step is not None:
                _lib.check(_lib.lib().aae_trainer_set_global_step(h, int(max(step, 0))), "set_global_step")
                self._ae.global_step._host = np.asarray(int(max(step, 0)), dtype=np.int64)
        return used

    def gradients(self, device):
        """{variable name: gradient} from the last forward/backward (for parity tests)."""
        h = self.trainer(device)
        out = {}
        stream = C.c_void_p(torch.cuda.current_stream(device).cuda_stream)      # behind the step the caller launched on it
        for which, mod in ((0, self._ae._encoder), (1, self._ae._decoder)):
            for i, (kn, ks, bn, bs) in enumerate(mod._var_shapes):
                k, b = np.empty(ks, np.float32), np.empty(bs, np.float32)
                with torch.cuda.device(device):
                    _lib.check(_lib.lib().aae_trainer_get_grads(h, which, i, _lib.ptr(k), _lib.ptr(b), stream), "get_grads")
                out[kn], out[bn] = k, b
        return out


def build_train_op(ae, args, precision=None):
    """precision: the GEMM arithmetic of the training step (see TrainOp); None follows the encoder and decoder handles."""
    LEARNING_RATE = args.getfloat('Training', 'LEARNING_RATE')
    OPTIMIZER_NAME = args.get('Training', 'OPTIMIZER')
    optimizer_spec(OPTIMIZER_NAME)
    return TrainOp(ae, LEARNING_RATE, precision=precision, optimizer=OPTIMIZER_NAME)


def build_codebook(encoder, dataset, args):
    embed_bb = args.getboolean('Embedding', 'EMBED_BB')
    return Codebook(encoder, dataset, embed_bb)


def build_codebook_from_name(experiment_name, experiment_group='', return_dataset=False, return_decoder=False,
                             precision=None, max_batch=None):
    import configparser
    workspace_path = os.environ.get('AE_WORKSPACE_PATH')
    if workspace_path is None:
        raise EnvironmentError('Please define a workspace path: export AE_WORKSPACE_PATH=/path/to/workspace')
    log_dir = u.get_log_dir(workspace_path, experiment_name, experiment_group)
    cfg_file_path = u.get_train_config_exp_file_path(log_dir, experiment_name)
    dataset_path = u.get_dataset_path(workspace_path)
    if not os.path.exists(cfg_file_path):
        raise FileNotFoundError('Config File not found: %s' % cfg_file_path)
    args = configparser.ConfigParser()
    args.read(cfg_file_path)
    with S.variable_scope(experiment_name):
        dataset = build_dataset(dataset_path, args)
        x = S.placeholder(np.float32, [None, ] + list(dataset.shape))
        encoder = build_encoder(x, args, precision=precision, max_batch=max_batch)
        codebook = build_codebook(encoder, dataset, args)
        if return_decoder:
            reconst_target = S.placeholder(np.float32, [None, ] + list(dataset.shape))
            decoder = build_decoder(reconst_target, encoder, args)
    if return_dataset:
        return (codebook, dataset, decoder) if return_decoder else (codebook, dataset)
    return codebook


class Saver(object):
    """tf.train.Saver stand-in over a list of modules (Encoder / Decoder / Codebook).  Checkpoints are ``chkpt-<step>.npz``
    files holding the reference's variable names (encoder.py / decoder.py / codebook.py scopes) in the reference's layouts."""

    def __init__(self, modules, global_step=None, train_op=None):
        """modules: Encoder / Decoder / Codebook objects.  train_op (a TrainOp): also save / restore the optimizer state under
        TensorFlow's slot names, so that training resumes where it stopped (a tf.train.Saver built after build_train_op stores
        them too: ae_train.py:81-82)."""
        self._modules = list(modules)
        self._global_step = global_step
        self._train_op = train_op

    def variables(self):
        out = {}
        for m in self._modules:
            if isinstance(m, Codebook):
                out[m.embedding_normalized.name] = m.embedding_normalized.value()
                if m.embed_bb:
                    out[m.embed_obj_bbs_var.name] = m.embed_obj_bbs_var.value()
            else:
                out.update(m.get_weights())
        if self._global_step is not None:
            out[self._global_step.name] = self._global_step.value()
        if self._train_op is not None:
            out.update(self._train_op.optimizer_variables())
        return out

    def save(self, session, save_path, global_step=None):
        path = "%s-%d.npz" % (save_path, int(global_step)) if global_step is not None else save_path + ".npz"
        os.makedirs(os.path.dirname(path), exist_ok=True)
        np.savez(path, **self.variables())
        return path

    def save_tf(self, session, save_path, global_step=None):
        """Same variables as a TensorFlow tensor bundle (``<save_path>-<step>.index`` / ``.data-00000-of-00001``) plus the
        ``checkpoint`` state file, i.e. what the reference's ``saver.save`` leaves behind (ae_train.py:134-135)."""
        from .tf_checkpoint import write_tf_checkpoint
        prefix = "%s-%d" % (save_path, int(global_step)) if global_step is not None else save_path
        write_tf_checkpoint(prefix, self.variables())
        with open(os.path.join(os.path.dirname(prefix), "checkpoint"), "w") as f:
            f.write('model_checkpoint_path: "%s"\nall_model_checkpoint_paths: "%s"\n' % (os.path.basename(prefix), os.path.basename(prefix)))
        return prefix

    def restore(self, session, path, strict=True):
        """path: ``chkpt-<step>.npz`` or the prefix of a TensorFlow checkpoint (``.../chkpt-30000``).  As with
        ``tf.train.Saver.restore`` (NotFoundError), every variable of every module must be in the checkpoint: a checkpoint of
        another experiment scope must not leave seeded weights and an all-zero codebook behind silently.  ``strict=False``
        restores what is there (e.g. a training checkpoint written by a Saver that did not include the codebook)."""
        if path.endswith(".npz"):
            data = np.load(path)
            weights = {k: data[k] for k in data.files}
        else:
            from .tf_checkpoint import read_tf_checkpoint
            weights = read_tf_checkpoint(path)
        missing = []
        for m in self._modules:
            if isinstance(m, Codebook):
                missing += [v.name for v in ([m.embedding_normalized] + ([m.embed_obj_bbs_var] if m.embed_bb else [])) if v.name not in weights]
            else:
                missing += [n for n in m.variable_names if n not in weights and "/".join(n.split("/")[-2:]) not in weights]
        if missing and strict:
            raise KeyError("%s does not hold: %s" % (path, ", ".join(missing)))
        for m in self._modules:
            if isinstance(m, Codebook):
                if m.embedding_normalized.name in weights:
                    m.embedding_normalized.assign(weights[m.embedding_normalized.name])
                if m.embed_bb and m.embed_obj_bbs_var.name in weights:
                    m.embed_obj_bbs_var.assign(weights[m.embed_obj_bbs_var.name])
                    m.embed_obj_bbs_values = None
            else:
                m.load_weights(weights, strict=strict)
        if self._global_step is not None and self._global_step.name in weights:
            self._global_step._host = np.asarray(weights[self._global_step.name], dtype=np.int64)
        if self._train_op is not None and session is not None:
            gs = int(weights[self._global_step.name]) if self._global_step is not None and self._global_step.name in weights else None
            self._train_op.load_optimizer_variables(weights, session.device, global_step=gs)


def restore_checkpoint(session, saver, ckpt_dir, at_step=None):
    """Latest checkpoint in ckpt_dir, or the one whose name contains ``at_step`` (ae_factory.py:149-172).  A TensorFlow
    ``checkpoint`` state file takes precedence (the reference's own layout); otherwise ``chkpt-<step>.npz`` files."""
    from .tf_checkpoint import latest_checkpoint
    latest, every = latest_checkpoint(ckpt_dir)
    if latest is not None:
        if at_step is None:
            saver.restore(session, latest)
            return latest
        for p in every:
            if str(at_step) in str(p):
                saver.restore(session, p)
                return p
        raise FileNotFoundError('No checkpoint for step %s in %s' % (at_step, ckpt_dir))
    paths = sorted(glob.glob(os.path.join(ckpt_dir, "chkpt-*.npz")), key=lambda p: int(p.rsplit("-", 1)[1][:-4]))
    if not paths:
        raise FileNotFoundError('No checkpoint found. Expected one in: %s' % ckpt_dir)
    if at_step is None:
        saver.restore(session, paths[-1])
        return paths[-1]
    for p in paths:
        if str(at_step) in os.path.basename(p):
            saver.restore(session, p)
            return p
    raise FileNotFoundError('No checkpoint for step %s in %s' % (at_step, ckpt_dir))
