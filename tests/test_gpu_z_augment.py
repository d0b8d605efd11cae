"""Device training-input pipeline (aae_augment) against the CPU restatement, which tests/test_augment_cpu.py pins to OpenCV."""
import numpy as np
import pytest
import torch

from augmentedautoencoder_b200.ae import augment as A
from oracle import augment_oracle as AO
from tests.test_augment_cpu import TEMPLATE_CODE

pytestmark = pytest.mark.gpu


def _inputs(seed, B):
    rng = np.random.RandomState(seed)
    x = rng.randint(0, 256, (B, 128, 128, 3), dtype=np.uint8)
    bg = rng.randint(0, 256, (B, 128, 128, 3), dtype=np.uint8)
    yy, xx = np.mgrid[:128, :128]
    mask = np.stack([((yy - 64) ** 2 + (xx - 60 - b) ** 2) > (30 + 2 * b) ** 2 for b in range(B)])       # True = background
    return x, mask, bg


def test_device_pipeline_is_bit_identical_to_the_restatement():
    B = 24
    x, mask, bg = _inputs(0, B)
    for seed in (1, 2):
        aug = A.Augmenter(TEMPLATE_CODE, seed=seed)
        aug.sigma = [0.5, 1.17][seed - 1]                       # the cfg draws sigma once per run; cover two kernels
        P = aug.sample(B)
        if seed == 1:                                           # make sure every op fires somewhere, alone and combined
            for k in ("affine_on", "drop_on", "blur_on", "add_on", "invert_on", "mul1_on", "mul2_on", "contrast_on"):
                P[k][:4] = True
                P[k][4:8] = False
            P["affine_on"][4], P["drop_on"][5], P["blur_on"][6], P["contrast_on"][7] = True, True, True, True
        want = AO.augment_batch(x, mask, bg, P, aug.sigma, low=aug.low)
        got_f, got_u = aug.augment_device(torch.from_numpy(x).cuda(), torch.from_numpy(mask).cuda(), torch.from_numpy(bg).cuda(), params=P, want_u8=True)
        got_u = got_u.cpu().numpy()
        assert np.array_equal(got_u, want), (seed, np.argwhere(got_u != want)[:5])
        assert np.array_equal(got_f.cpu().numpy(), (want / 255.).astype(np.float32))      # batch_x / 255. then the float32 feed


def test_no_op_parameters_reduce_to_the_background_paste():
    B = 3
    x, mask, bg = _inputs(3, B)
    aug = A.Augmenter(TEMPLATE_CODE, seed=0)
    P = aug.sample(B)
    for k in P:
        if k.endswith("_on"):
            P[k][:] = False
    out, out_u = aug.augment_device(torch.from_numpy(x).cuda(), torch.from_numpy(mask).cuda(), torch.from_numpy(bg).cuda(), params=P, want_u8=True)
    want = x.copy()
    want[mask] = bg[mask]
    assert np.array_equal(out_u.cpu().numpy(), want)


def test_dataset_batch_device_shapes(tmp_path):
    from augmentedautoencoder_b200.ae.dataset import Dataset
    x, mask, bg = _inputs(5, 12)
    np.savez(tmp_path / "train.npz", train_x=x, mask_x=mask, train_y=x)
    np.save(tmp_path / "bg.npy", bg)
    ds = Dataset(None, code=TEMPLATE_CODE, h=128, w=128, c=3, seed=4)
    ds.load_training_images(str(tmp_path / "train.npz"), str(tmp_path / "bg.npy"))
    bx, by = ds.batch(8)
    assert bx.shape == (8, 128, 128, 3) and by.shape == (8, 128, 128, 3) and bx.dtype == np.float32
    assert 0.0 <= bx.min() and bx.max() <= 1.0
