"""ctypes binding of libaae_b200.so (the C ABI declared in include/aae_b200.h).  Fails loudly: no fallback."""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libaae_b200.so")
HEADER_PATH = os.path.join(_HERE, "..", "include", "aae_b200.h")

AAE_MAX_LAYERS = 8
PREC_FP32_SIMT = 0
PREC_TC_SPLIT = 1
PREC_TC_FP16 = 2      # encoder + codebook match handles, and the trainer's GEMMs (TrainOp(precision=...)): one fp16 product per K step
# aae_optimizer_kind: the update rule of the training step (ae_factory.OPTIMIZERS maps cfg names to these)
OPT_ADAM = 0
OPT_GRADIENT_DESCENT = 1
OPT_ADAGRAD = 2
OPT_PROXIMAL_ADAGRAD = 3
OPT_ADADELTA = 4
OPT_RMSPROP = 5
OPT_FTRL = 6


class AaeError(RuntimeError):
    pass


class NetCfg(C.Structure):
    _fields_ = [("in_h", C.c_int32), ("in_w", C.c_int32), ("in_c", C.c_int32), ("num_layers", C.c_int32),
                ("filters", C.c_int32 * AAE_MAX_LAYERS), ("strides", C.c_int32 * AAE_MAX_LAYERS),
                ("kernel_size", C.c_int32), ("latent", C.c_int32), ("max_batch", C.c_int32), ("precision", C.c_int32)]


class Optimizer(C.Structure):
    _fields_ = [("kind", C.c_int32), ("learning_rate", C.c_float), ("hp", C.c_float * 4)]


class _Args(C.Structure):
    """Argument struct of an input-pipeline call: struct_size is filled in, and a field given a tensor or array takes its
    address (None: NULL)."""

    def __init__(self, **fields):
        super().__init__(struct_size=C.sizeof(type(self)))
        self.set(**fields)

    def set(self, **fields):
        for name, v in fields.items():
            setattr(self, name, v if v is None or isinstance(v, (int, float)) else ptr(v).value)
        return self

    def copy(self):
        return type(self).from_buffer_copy(self)


class AugmentArgs(_Args):
    """aae_augment_args"""
    _fields_ = [("struct_size", C.c_int32),
                ("batch", C.c_int32), ("h", C.c_int32), ("w", C.c_int32), ("c", C.c_int32), ("low_w", C.c_int32),
                ("x", C.c_void_p), ("mask", C.c_void_p), ("bg", C.c_void_p), ("y", C.c_void_p), ("idx", C.c_void_p),
                ("idx_bg", C.c_void_p), ("n_images", C.c_int64), ("n_bg", C.c_int64), ("mask_batch", C.c_void_p),
                ("geom", C.c_void_p), ("lut", C.c_void_p), ("crop", C.c_void_p),
                ("bilinear_tab", C.c_void_p), ("row_cell", C.c_void_p), ("col_cell", C.c_void_p), ("blur_kernel_q8", C.c_void_p),
                ("u8_to_float", C.c_void_p), ("y_to_float", C.c_void_p), ("resample", C.c_void_p), ("resample_len", C.c_int64),
                ("max_src_rows", C.c_int32), ("max_src_w", C.c_int32),
                ("tmp", C.c_void_p), ("crop_tmp", C.c_void_p),
                ("out_u8", C.c_void_p), ("out_f32", C.c_void_p), ("y_out", C.c_void_p)]


class OcclusionArgs(_Args):
    """aae_occlusion_args"""
    _fields_ = [("struct_size", C.c_int32),
                ("batch", C.c_int32), ("h", C.c_int32), ("w", C.c_int32),
                ("realistic", C.c_int32), ("square", C.c_int32), ("max_occl", C.c_double), ("min_kept", C.c_double),
                ("mask", C.c_void_p), ("idx", C.c_void_p), ("n_images", C.c_int64),
                ("cand", C.c_void_p), ("n_cand", C.c_int32),
                ("n_bank", C.c_int32), ("bank", C.c_void_p), ("row_cell", C.c_void_p), ("col_cell", C.c_void_p),
                ("low_h", C.c_int32), ("low_w", C.c_int32),
                ("mask_out", C.c_void_p), ("fallbacks", C.c_void_p)]


_P = C.c_void_p
_I = C.c_int
_L = C.c_int64
_F = C.c_float
_D = C.c_double
_SIGS = {
    "aae_version": (_I, []),
    "aae_last_error_string": (C.c_char_p, []),
    "aae_device_supported": (_I, [_I]),
    "aae_launch_count": (_L, []),
    "aae_encoder_create": (_I, [_I, C.POINTER(NetCfg), C.POINTER(_P)]),
    "aae_encoder_destroy": (_I, [_P]),
    "aae_encoder_set_weights": (_I, [_P, _I, _P, _P, _P]),
    "aae_encoder_get_weights": (_I, [_P, _I, _P, _P, _P]),
    "aae_encoder_forward_u8": (_I, [_P, _P, _I, _P, _P]),
    "aae_encoder_forward_f32": (_I, [_P, _P, _I, _P, _P]),
    "aae_encoder_range_status": (_I, [_P, _P]),
    "aae_encoder_range_word": (_I, [_P, C.POINTER(_P)]),
    "aae_encoder_activation": (_I, [_P, _I, C.POINTER(_P), C.POINTER(_L)]),
    "aae_encoder_profile": (_I, [_P, _I, _P, _I]),
    "aae_encoder_enable_sigma_head": (_I, [_P]),
    "aae_encoder_sigma_forward": (_I, [_P, _I, _P, _P]),
    "aae_codebook_profile": (_I, [_P, _I, _P, _I]),
    "aae_codebook_create": (_I, [_I, _P, _L, _I, _I, _L, _I, _I, C.POINTER(_P)]),
    "aae_codebook_destroy": (_I, [_P]),
    "aae_l2_normalize": (_I, [_P, _I, _I, _P, _P]),
    "aae_codebook_match": (_I, [_P, _P, _I, _I, _I, _P, _P, _P]),
    "aae_codebook_cosine": (_I, [_P, _P, _I, _P, _P]),
    "aae_topk_merge": (_I, [_P, _P, _I, _I, _I, _P, _P, _P]),
    "aae_topk_merge_packed": (_I, [_P, _I, _I, _I, _P, _P, _P]),
    "aae_codebook_rows": (_L, [_P]),
    "aae_launch_floor_probe": (_I, [_I, _I, _P]),
    "aae_decoder_create": (_I, [_I, C.POINTER(NetCfg), C.POINTER(_P)]),
    "aae_decoder_destroy": (_I, [_P]),
    "aae_decoder_set_weights": (_I, [_P, _I, _P, _P, _P]),
    "aae_decoder_get_weights": (_I, [_P, _I, _P, _P, _P]),
    "aae_decoder_forward": (_I, [_P, _P, _I, _P, _P]),
    "aae_decoder_range_status": (_I, [_P, _P]),
    "aae_decoder_enable_mask_head": (_I, [_P]),
    "aae_decoder_forward_mask": (_I, [_P, _P, _I, _P, _P, _P]),
    "aae_mask_loss": (_I, [_P, _P, _I, _I, _I, _P, _P, _P]),
    "aae_bootstrap_l2_loss": (_I, [_P, _P, _I, _I, _I, _P, _P, _P]),
    "aae_trainer_create": (_I, [_P, _P, _I, _F, _F, _F, _F, C.POINTER(_P)]),
    "aae_trainer_create_prec": (_I, [_P, _P, _I, _F, _F, _F, _F, _I, C.POINTER(_P)]),
    "aae_trainer_create_opt": (_I, [_P, _P, _I, C.POINTER(Optimizer), _I, C.POINTER(_P)]),
    "aae_trainer_destroy": (_I, [_P]),
    "aae_train_step": (_I, [_P, _P, _P, _I, _P, _P]),
    "aae_trainer_forward_backward": (_I, [_P, _P, _P, _I, _P, _P]),
    "aae_trainer_get_grads": (_I, [_P, _I, _I, _P, _P, _P]),
    "aae_trainer_global_step": (_L, [_P]),
    "aae_trainer_profile": (_I, [_P, _I, _P, _I]),
    "aae_trainer_get_state": (_I, [_P, _I, _I, _P, _P, _P, _P, _P]),
    "aae_trainer_set_state": (_I, [_P, _I, _I, _P, _P, _P, _P, _P]),
    "aae_trainer_set_global_step": (_I, [_P, _L]),
    "aae_trainer_set_latent_terms": (_I, [_P, _F, _F]),
    "aae_trainer_set_latent_noise": (_I, [_P, _F]),
    "aae_extract_square_patches": (_I, [_P, _I, _I, _P, _I, _I, _P, _P]),
    "aae_augment": (_I, [C.POINTER(AugmentArgs), _P]),
    "aae_occlusion": (_I, [C.POINTER(OcclusionArgs), _P]),
}

_lib = None


def lib():
    """The loaded library.  Raises AaeError if it has not been built (python __graft_entry__.py / build_ext.py)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise AaeError(f"{LIB_PATH} is missing: build it with `python -m augmentedautoencoder_b200.build_ext` "
                           "(there is no CPU or PyTorch fallback for the hot path)")
        l = C.CDLL(LIB_PATH)
        for name, (res, args) in _SIGS.items():
            fn = getattr(l, name)
            fn.restype = res
            fn.argtypes = args
        _lib = l
    return _lib


def check(status: int, what: str = ""):
    if status != 0:
        msg = lib().aae_last_error_string().decode("utf-8", "replace")
        raise AaeError(f"{what or 'aae call'} failed (status {status}): {msg}")


def make_cfg(h, w, c, filters, strides, kernel_size, latent, max_batch, precision) -> NetCfg:
    if len(filters) != len(strides) or not 1 <= len(filters) <= AAE_MAX_LAYERS:
        raise ValueError("NUM_FILTER / STRIDES must have the same length in [1, %d]" % AAE_MAX_LAYERS)
    cfg = NetCfg()
    cfg.in_h, cfg.in_w, cfg.in_c = int(h), int(w), int(c)
    cfg.num_layers = len(filters)
    for i, (f, s) in enumerate(zip(filters, strides)):
        cfg.filters[i], cfg.strides[i] = int(f), int(s)
    cfg.kernel_size, cfg.latent, cfg.max_batch, cfg.precision = int(kernel_size), int(latent), int(max_batch), int(precision)
    return cfg


def ptr(t):
    """Device (or host) pointer of a torch tensor / numpy array as c_void_p; None -> NULL."""
    if t is None:
        return None
    if hasattr(t, "data_ptr"):
        return C.c_void_p(t.data_ptr())
    return C.c_void_p(t.ctypes.data)
