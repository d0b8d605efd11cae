"""CropAndPad on the device (aae_augment with a crop table, gathered and indexed) against the CPU restatement, which
tests/test_crop_pad_cpu.py pins to OpenCV: forced firing patterns at every input geometry, the gathered, resident and queued
batches bit for bit, ae_train from a cfg with the template's CropAndPad line uncommented, and the stream contract."""
import configparser
import ctypes as C
import gc
import os

import cv2
import numpy as np
import pytest
import torch

from augmentedautoencoder_b200 import _lib
from augmentedautoencoder_b200.ae import ae_factory as F
from augmentedautoencoder_b200.ae import augment as A
from augmentedautoencoder_b200.ae.dataset import Dataset
from tests import crop_pad_oracle as CP
from tests.test_crop_pad_cpu import CROP_CODE, GEOMETRIES
from tests.test_gpu_a_parity import sess  # noqa: F401
from tests.test_gpu_g_occlusion import _bank, _objects
from tests.test_gpu_n_streams import S, delay, dev, ok, poisoned, returns_before_the_device, run_on_side_stream  # noqa: F401

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)


@pytest.fixture(autouse=True)
def _quiet_device():
    torch.cuda.synchronize()
    yield
    torch.cuda.synchronize()
    gc.collect()
    torch.cuda.empty_cache()


def _force(P, H, W):
    """images 0..11: every case of the op; the rest keep their draws.  Returns the cases by image."""
    c, p = -int(round(0.05 * H)), int(round(0.1 * H))
    cw, pw = -int(round(0.05 * W)), int(round(0.1 * W))
    cases = {"crop only": (c, cw, c, cw), "pad only": (p, pw, p, pw), "mixed: rows cropped, columns padded": (c, pw, c, pw),
             "mixed: rows padded, columns cropped": (p, cw, p, cw), "area, both axes larger": (p, 1, 2, pw),
             "pure shift": (c, 0, -c, 0), "pure shift, both axes": (3, -2, -3, 2), "one side": (0, 0, 0, cw),
             "copy (all zero)": (0, 0, 0, 0), "uneven": (c, pw, 1, -1)}
    for b, px in enumerate(cases.values()):
        P["crop_on"][b], P["crop_px"][b] = True, px
        P["crop_cval"][b] = 0 if b % 2 else 77 + b
    P["crop_on"][len(cases):len(cases) + 2] = False
    P["affine_on"][:len(cases):3] = True                   # the warp reads the crop-pad output
    P["affine_on"][1:len(cases):3] = False
    return cases


def _inputs(rng, B, H, W, C):
    x = rng.randint(0, 256, (B, H, W, C), dtype=np.uint8)
    bg = rng.randint(0, 256, (B, H, W, C), dtype=np.uint8)
    mask = rng.rand(B, H, W) < 0.4
    return x, mask, bg


@pytest.mark.parametrize("geometry", sorted(GEOMETRIES))
def test_augment_device_matches_the_restatement(geometry):
    H, W, C = GEOMETRIES[geometry]
    rng = np.random.RandomState(len(geometry))
    B = 64
    aug = A.Augmenter(CROP_CODE, (H, W, C), seed=3)
    P = aug.sample(B)
    cases = _force(P, H, W)
    modes = aug.pack_crop(P)[:, 0]
    assert set(modes[:len(cases)]) == {1, 2} and not modes[len(cases):len(cases) + 2].any()
    x, mask, bg = _inputs(rng, B, H, W, C)
    out_f, out_u = aug.augment_device(dev(x), dev(mask), dev(bg), params=P, want_u8=True)
    want = CP.augment_batch(x, mask, bg, P, aug.sigma, low=aug.low)
    got = out_u.cpu().numpy()
    bad = np.nonzero((got != want).any((1, 2, 3)))[0]
    assert not len(bad), [(b, list(cases)[b] if b < len(cases) else "drawn") for b in bad]
    assert np.array_equal(out_f.cpu().numpy(), (want / 255.).astype(np.float32))


def _arrays(c, seed=5, n=40, n_bg=30, H=128, W=128):
    rng = np.random.RandomState(seed)
    x = rng.randint(0, 256, (n, H, W, c), dtype=np.uint8)
    y = rng.randint(0, 256, (n, H, W, c), dtype=np.uint8)
    bg = rng.randint(0, 256, (n_bg, H, W, c), dtype=np.uint8)
    return x, _objects(rng, n), y, bg


def _dataset(arrays, occl=None, bank_path=None, resident=True, c=3):
    kw = dict(code=CROP_CODE, h=128, w=128, c=c, seed=6)
    if occl:
        kw.update(realistic_occlusion="0.25", square_occlusion="0.25")
    ds = Dataset(None, **kw)
    ds.train_x, ds.mask_x, ds.train_y, ds.bg_imgs = arrays
    if bank_path is not None:
        ds.load_occlusion_masks(bank_path)
    if resident:
        ds.upload(DEV)
    return ds


@pytest.mark.parametrize("occl", [False, True])
def test_gathered_resident_and_queued_batches_agree(sess, tmp_path, occl):
    arrays = _arrays(3)
    bank = _bank(tmp_path, np.random.RandomState(9))[0] if occl else None
    sizes = [16, 16, 16, 16]
    a = _dataset(arrays, occl, bank, resident=False)
    np.random.seed(21)
    want = [tuple(t.cpu().numpy() for t in a.batch_device(n)) for n in sizes]
    assert a._aug.crop is not None
    b = _dataset(arrays, occl, bank)
    np.random.seed(21)
    for k, n in enumerate(sizes):
        x, y = b.batch_resident(n)
        assert np.array_equal(x.cpu().numpy(), want[k][0]) and np.array_equal(y.cpu().numpy(), want[k][1]), k
    assert b.occlusion_fallbacks() == a.occlusion_fallbacks()
    ds = _dataset(arrays, occl, bank)
    q = F.Queue(ds, 10, 2, 16)
    np.random.seed(21)
    q.start(sess)
    try:
        for k in range(len(sizes)):
            x, y = sess.run_device([q.x, q.y])
            assert np.array_equal(x.cpu().numpy(), want[k][0]) and np.array_equal(y.cpu().numpy(), want[k][1]), k
    finally:
        q.stop(sess)


def test_resident_outside_the_stack_still_crops_and_pads(sess):
    """An image whose row is outside its stack is pasted as zeros; its pad value still shows."""
    x, mask, y, bg = _arrays(3, n=8, n_bg=8)
    aug = A.Augmenter(CROP_CODE, (128, 128, 3), seed=2)
    B = 8
    P = aug.sample(B)
    for key in ("affine_on", "drop_on", "blur_on", "add_on", "invert_on", "mul1_on", "mul2_on", "contrast_on"):
        P[key][:] = False
    P["crop_on"][:], P["crop_px"][:], P["crop_cval"][:] = True, (5, 4, 3, 2), 200
    geom, lut = aug.pack(P)
    stacks = {"x": dev(x), "mask": dev(mask.astype(np.uint8)), "y": dev(y), "bg": dev(bg)}
    idx = np.arange(B, dtype=np.int32)
    idx[3] = 99
    out_f = torch.empty((B, 128, 128, 3), dtype=torch.float32, device=DEV)
    y_out = torch.empty_like(out_f)
    aug.augment_indexed(stacks, dev(idx), dev(np.arange(B, dtype=np.int32)), dev(geom), dev(lut), out_f, y_out,
                        torch.cuda.current_stream(DEV), crop_d=dev(aug.pack_crop(P)))
    xs, ms = x[np.minimum(idx, 7)].copy(), mask[np.minimum(idx, 7)].copy()
    xs[3], ms[3] = 0, False
    want = CP.augment_batch(xs, ms, bg, P, aug.sigma, low=aug.low)
    assert np.array_equal(out_f.cpu().numpy(), (want / 255.).astype(np.float32))
    assert want[3].max() > 0 and (want[3][0, 0] > 0).all()


def test_ae_train_with_crop_and_pad_uncommented(sess, golden_dir, tmp_path, monkeypatch):
    from augmentedautoencoder_b200.ae import ae_train
    ws = tmp_path / "ws"
    (ws / "cfg" / "grp").mkdir(parents=True)
    (ws / "bg").mkdir()
    text = open(os.path.join(golden_dir, "train_template.cfg")).read()
    assert "#Sometimes(0.5, CropAndPad" in text                 # a comment line: configparser drops it from CODE
    args = configparser.ConfigParser()
    args.read_string(text.replace("#Sometimes(0.5, CropAndPad", "Sometimes(0.5, CropAndPad"))
    assert "CropAndPad(percent=(-0.05, 0.1))" in args.get("Augmentation", "CODE")
    args.set("Paths", "BACKGROUND_IMAGES_GLOB", str(ws / "bg" / "*.png"))
    args.set("Dataset", "NOOF_TRAINING_IMGS", "40")
    args.set("Dataset", "NOOF_BG_IMGS", "18")
    args.set("Embedding", "MIN_N_VIEWS", "12")
    args.set("Embedding", "NUM_CYCLO", "4")
    args.set("Training", "SAVE_INTERVAL", "10")
    args.set("Training", "BATCH_SIZE", "16")

    def write(num_iter):
        args.set("Training", "NUM_ITER", str(num_iter))
        with open(ws / "cfg" / "grp" / "exp.cfg", "w") as f:
            args.write(f)
    write(20)
    monkeypatch.setenv("AE_WORKSPACE_PATH", str(ws))
    rng = np.random.RandomState(3)
    for i in range(20):
        cv2.imwrite(str(ws / "bg" / ("%02d.png" % i)), rng.randint(0, 256, (160, 180, 3), dtype=np.uint8))
    x, masks, y, _ = _arrays(3)
    cache = Dataset(None, h=128, w=128, c=3).training_images_path(str(ws / "tmp_datasets"), args)
    os.makedirs(os.path.dirname(cache))
    np.savez(cache, train_x=x, mask_x=masks, train_y=y)
    np.random.seed(0)
    assert ae_train.main(["grp/exp"]) == 20
    log_dir = ws / "experiments" / "grp" / "exp"
    for step in (10, 20):
        assert (log_dir / "checkpoints" / ("chkpt-%d.index" % step)).exists()
    lines = [l for l in (log_dir / "train_loss.txt").read_text().split("\n") if l]
    assert [int(l.split()[0]) for l in lines] == [0, 10] and all(np.isfinite(float(l.split()[1])) for l in lines)
    write(30)
    run = ae_train.prepare(["grp/exp"])
    assert run.restored.endswith("chkpt-20") and int(run.ae.global_step.value()) == 20
    assert ae_train.train(run) == 30
    assert (log_dir / "checkpoints" / "chkpt-30.index").exists()
    run.train_op.close()
    for m in (run.encoder, run.decoder):
        m.close()


def test_augment_with_a_crop_table_on_a_side_stream(sess, delay):
    lib, B = _lib.lib(), 24
    rng = np.random.RandomState(0)
    x, mask, bg = _inputs(rng, B, 128, 128, 3)
    aug = A.Augmenter(CROP_CODE, seed=1)
    P = aug.sample(B)
    _force(P, 128, 128)
    geom, lut = aug.pack(P)
    crop = aug.pack_crop(P)
    k = aug._constants(DEV)
    rs, taps = k["resample"], k["taps"]
    const = dict(batch=B, h=128, w=128, c=3, low_w=aug.low[1], bilinear_tab=k["tab"], row_cell=k["rows"], col_cell=k["cols"],
                 blur_kernel_q8=taps, u8_to_float=k["to_float"], resample=rs, resample_len=int(rs.numel()),
                 max_src_rows=aug.crop["max_rows"], max_src_w=aug.crop["max_w"])

    def gathered(xd, md, bd, gd, ld, cd):
        tmp, ct, of = poisoned(xd.shape, torch.uint8), poisoned(xd.shape, torch.uint8), poisoned(xd.shape, torch.float32)
        ok(lib.aae_augment(C.byref(_lib.AugmentArgs(x=xd, mask=md, bg=bd, geom=gd, lut=ld, crop=cd, tmp=tmp, crop_tmp=ct, out_f32=of,
                                                    **const)), S()))
        return of
    inputs = [dev(x), dev(mask.astype(np.uint8)), dev(bg), dev(geom), dev(lut), dev(crop)]
    want = aug.augment_device(inputs[0], inputs[1], inputs[2], params=P)
    of = run_on_side_stream(gathered, inputs, delay, "augment crop-pad")[0]
    assert np.array_equal(of, want.cpu().numpy())
    returns_before_the_device(lambda: gathered(*inputs), delay)

    idx = np.arange(B, dtype=np.int32)[::-1].copy()

    def indexed(xd, md, bd, yd, id_, gd, ld, cd):
        tmp, ct = poisoned(xd.shape, torch.uint8), poisoned(xd.shape, torch.uint8)
        of, yo = poisoned(xd.shape, torch.float32), poisoned(xd.shape, torch.float32)
        ok(lib.aae_augment(C.byref(_lib.AugmentArgs(
            x=xd, mask=md, bg=bd, y=yd, idx=id_, idx_bg=id_, n_images=B, n_bg=B, geom=gd, lut=ld, crop=cd, y_to_float=k["y_to_float"],
            tmp=tmp, crop_tmp=ct, out_f32=of, y_out=yo, **const)), S()))
        return of, yo
    ins = [dev(x), dev(mask.astype(np.uint8)), dev(bg), dev(x), dev(idx), dev(geom), dev(lut), dev(crop)]
    of, yo = run_on_side_stream(indexed, ins, delay, "augment indexed crop-pad")
    want = CP.augment_batch(x[idx], mask[idx], bg[idx], P, aug.sigma, low=aug.low)
    assert np.array_equal(of, (want / 255.).astype(np.float32))
    returns_before_the_device(lambda: indexed(*ins), delay)


def test_augment_refuses_a_geometry_whose_rows_do_not_fit(monkeypatch):
    """Below four area taps (ratio < 3) the staged rows of a 128-wide crop stay under 48 KB, so the limit is lowered to reach
    the construction check; the library's own check takes a bound above it."""
    with monkeypatch.context() as m:
        m.setattr(A, "CROP_PAD_SMEM_LIMIT", 4096)
        with pytest.raises(NotImplementedError, match="shared memory"):
            A.Augmenter(CROP_CODE, (128, 128, 3))
    aug = A.Augmenter(CROP_CODE, seed=0)
    x = torch.zeros((2, 128, 128, 3), dtype=torch.uint8, device=DEV)
    k = aug._constants(DEV)
    st = _lib.lib().aae_augment(C.byref(_lib.AugmentArgs(
        batch=2, h=128, w=128, c=3, low_w=aug.low[1], x=x, mask=x[..., 0], bg=x, geom=x, lut=x, crop=x, bilinear_tab=k["tab"],
        row_cell=k["rows"], col_cell=k["cols"], u8_to_float=k["to_float"], resample=k["resample"], resample_len=int(k["resample"].numel()),
        max_src_rows=200, max_src_w=154, tmp=x, crop_tmp=x, out_u8=x)), S())
    assert st == -3 and b"shared memory" in _lib.lib().aae_last_error_string()
