"""CPU tests of the input-pipeline ABI (aae_augment / aae_occlusion, include/aae_b200.h):

  * the ctypes mirrors _lib.AugmentArgs / _lib.OcclusionArgs have the header's layout: every field at the offset and with the
    size the C++ compiler gives it, and the same struct size.  A field out of order, of the wrong width or missing fails here
    instead of being read from the wrong place;
  * every refusal the header documents is returned, with its status and message, before anything is launched."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
import torch

from augmentedautoencoder_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STRUCTS = {"aae_augment_args": _lib.AugmentArgs, "aae_occlusion_args": _lib.OcclusionArgs}
INVALID_ARG, CUDA, UNSUPPORTED = -1, -2, -3


def test_ctypes_structs_match_the_header_layout(tmp_path):
    lines = ["#include <cstddef>", "#include <cstdio>", '#include "aae_b200.h"', "int main() {"]
    for name, cls in STRUCTS.items():
        lines.append('  std::printf("%s %%zu\\n", sizeof(%s));' % (name, name))
        for field, _ in cls._fields_:
            lines.append('  std::printf("%s.%s %%zu %%zu\\n", offsetof(%s, %s), sizeof(((%s*)0)->%s));' % (name, field, name, field, name, field))
    lines += ["  return 0;", "}"]
    src, exe = tmp_path / "layout.cpp", tmp_path / "layout"
    src.write_text("\n".join(lines) + "\n")
    subprocess.run(["g++", "-std=c++17", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    got = dict(line.split(" ", 1) for line in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines())
    want = {}
    for name, cls in STRUCTS.items():
        want[name] = str(C.sizeof(cls))
        for field, _ in cls._fields_:
            want["%s.%s" % (name, field)] = "%d %d" % (getattr(cls, field).offset, getattr(cls, field).size)
    assert got == want


# A fake device address per pointer field: the cases below never reach a launch (a case that did would fail for want of a
# device, with AAE_ERR_CUDA, which is what the accepted cases check).
def _fake(i):
    return 0x10000 * (i + 1)


def _augment_base():
    return dict(batch=2, h=128, w=128, c=3, low_w=4, x=_fake(0), mask=_fake(1), bg=_fake(2), geom=_fake(3), lut=_fake(4),
                bilinear_tab=_fake(5), row_cell=_fake(6), col_cell=_fake(7), u8_to_float=_fake(8), tmp=_fake(9), out_f32=_fake(10))


CROP = dict(crop=_fake(11), resample=_fake(12), resample_len=4096, max_src_rows=16, max_src_w=141, crop_tmp=_fake(13))
INDEXED = dict(idx=_fake(14), idx_bg=_fake(15), n_images=40, n_bg=30)
BLUR_255 = np.array([16, 64, 95, 64, 16], np.int32)
BLUR_256 = np.array([16, 64, 96, 64, 16], np.int32)

AUGMENT_CASES = [
    # (what, changed fields, status, message substring)
    ("struct_size", dict(struct_size=C.sizeof(_lib.AugmentArgs) - 8), INVALID_ARG, "struct_size"),
    ("idx without idx_bg", dict(idx=_fake(14), n_images=40, n_bg=30), INVALID_ARG, "idx and idx_bg"),
    ("idx_bg without idx", dict(idx_bg=_fake(15), n_images=40, n_bg=30), INVALID_ARG, "idx and idx_bg"),
    ("an empty image stack", dict(INDEXED, n_images=0), INVALID_ARG, "empty image stack"),
    ("an empty background stack", dict(INDEXED, n_bg=0), INVALID_ARG, "empty image stack"),
    ("no x", dict(x=None), INVALID_ARG, "null argument"),
    ("no mask and no mask_batch", dict(mask=None), INVALID_ARG, "null argument"),
    ("no geom", dict(geom=None), INVALID_ARG, "null argument"),
    ("no scratch", dict(tmp=None), INVALID_ARG, "null argument"),
    ("no output", dict(out_f32=None), INVALID_ARG, "no output requested"),
    ("y_out without y", dict(y_out=_fake(16), y_to_float=_fake(17)), INVALID_ARG, "y_out needs y and y_to_float"),
    ("y_out without y_to_float", dict(y_out=_fake(16), y=_fake(18)), INVALID_ARG, "y_out needs y and y_to_float"),
    ("out_f32 without u8_to_float", dict(u8_to_float=None), INVALID_ARG, "out_f32 needs u8_to_float"),
    ("batch 0", dict(batch=0), INVALID_ARG, "bad geometry"),
    ("low_w 0", dict(low_w=0), INVALID_ARG, "bad geometry"),
    ("5 channels", dict(c=5), INVALID_ARG, "5 channels unsupported"),
    ("0 channels", dict(c=0), INVALID_ARG, "0 channels unsupported"),
    ("a blur kernel summing to 255", dict(blur_kernel_q8=BLUR_255), INVALID_ARG, "got 255"),
    ("crop without resample", dict(CROP, resample=None), INVALID_ARG, "null argument"),
    ("crop without crop_tmp", dict(CROP, crop_tmp=None), INVALID_ARG, "null argument"),
    ("crop with an empty table", dict(CROP, resample_len=0), INVALID_ARG, "bad crop-pad bounds"),
    ("crop with no source rows", dict(CROP, max_src_rows=0), INVALID_ARG, "bad crop-pad bounds"),
    ("crop-pad rows over 48 KB", dict(CROP, max_src_rows=200, max_src_w=154), UNSUPPORTED, "shared memory"),
    # accepted: these pass every check and fail only at the launch
    ("gathered", {}, CUDA, ""),
    ("gathered with u8 output only", dict(out_f32=None, u8_to_float=None, out_u8=_fake(19)), CUDA, ""),
    ("mask_batch in place of mask", dict(mask=None, mask_batch=_fake(20)), CUDA, ""),
    ("indexed with y_out and crop-pad", dict(INDEXED, **CROP, y=_fake(18), y_out=_fake(16), y_to_float=_fake(17)), CUDA, ""),
    ("a blur kernel summing to 256", dict(blur_kernel_q8=BLUR_256), CUDA, ""),
]


def _occlusion_base():
    return dict(batch=2, h=128, w=128, realistic=1, max_occl=0.25, square=1, min_kept=0.75, mask=_fake(0), cand=_fake(1), n_cand=64,
                n_bank=10, bank=_fake(2), row_cell=_fake(3), col_cell=_fake(4), low_h=3, low_w=3, mask_out=_fake(5), fallbacks=_fake(6))


OCCLUSION_CASES = [
    ("struct_size", dict(struct_size=C.sizeof(_lib.OcclusionArgs) + 8), INVALID_ARG, "struct_size"),
    ("no mask", dict(mask=None), INVALID_ARG, "null argument"),
    ("no fallback counters", dict(fallbacks=None), INVALID_ARG, "null argument"),
    ("an empty mask stack", dict(idx=_fake(7), n_images=0), INVALID_ARG, "empty mask stack"),
    ("no candidates", dict(n_cand=0), INVALID_ARG, "candidate count"),
    ("realistic without a bank", dict(bank=None), INVALID_ARG, "occluder bank"),
    ("realistic with an empty bank", dict(n_bank=0), INVALID_ARG, "occluder bank"),
    ("square without the cell maps", dict(col_cell=None), INVALID_ARG, "dropout cell maps"),
    ("width not a multiple of 32", dict(w=112), UNSUPPORTED, "not a multiple of 32"),
    ("more than 32 cells", dict(low_h=6, low_w=6), UNSUPPORTED, "32 keep bits"),
    ("masks over 48 KB", dict(h=2048), UNSUPPORTED, "shared memory"),
    ("gathered", {}, CUDA, ""),
    ("indexed", dict(idx=_fake(7), n_images=40), CUDA, ""),
    ("steps off without their fields", dict(realistic=0, square=0, bank=None, n_bank=0, row_cell=None, col_cell=None), CUDA, ""),
    ("more than 32 cells with square off", dict(square=0, low_h=6, low_w=6), CUDA, ""),
]


@pytest.mark.skipif(torch.cuda.is_available(), reason="the cases pass fake device pointers: run only where nothing can be launched")
def test_refusals_are_returned_before_any_launch():
    from augmentedautoencoder_b200 import build_ext
    build_ext.build()
    lib = _lib.lib()
    wrong = []
    for entry, cls, base, cases in ((lib.aae_augment, _lib.AugmentArgs, _augment_base, AUGMENT_CASES),
                                    (lib.aae_occlusion, _lib.OcclusionArgs, _occlusion_base, OCCLUSION_CASES)):
        assert entry(None, None) == INVALID_ARG and b"null argument" in lib.aae_last_error_string()
        for what, change, status, message in cases:
            st = entry(C.byref(cls(**base()).set(**change)), None)
            msg = lib.aae_last_error_string().decode()
            if st != status or message not in msg:
                wrong.append((entry.__name__, what, st, msg))
    assert not wrong, wrong
