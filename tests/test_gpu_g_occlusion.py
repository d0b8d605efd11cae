"""Occlusion-mask augmentations on the device (aae_occlusion) against the CPU restatement, which
tests/test_occlusion_cpu.py pins to the reference's own output and to OpenCV."""
import numpy as np
import pytest
import torch

from augmentedautoencoder_b200.ae import augment as A
from augmentedautoencoder_b200.ae.dataset import Dataset
from oracle import augment_oracle as AO
from oracle import occlusion_oracle as OO
from tests.test_augment_cpu import TEMPLATE_CODE

pytestmark = pytest.mark.gpu
H = W = 128


def _objects(rng, B, h=H, w=W):
    """True = background: random ellipses and rectangles of very different sizes.  Centres and radii are drawn on the 128 x 128
    grid and scaled to h x w, so the default draws the same masks from the same stream."""
    yy, xx = np.mgrid[:h, :w]
    masks = np.ones((B, h, w), bool)
    for b in range(B):
        cy, cx = 10 + rng.randint(0, 108, 2) * np.array([h - 20, w - 20]) // 108
        ry, rx = 6 + rng.randint(0, 54, 2) * np.array([h, w]) // 128
        if b % 4 == 3:
            masks[b] = ~((np.abs(yy - cy) <= ry) & (np.abs(xx - cx) <= rx))
        else:
            masks[b] = ((yy - cy) / float(ry)) ** 2 + ((xx - cx) / float(rx)) ** 2 > 1.0
    return masks


def _bank(tmp_path, rng, n=12, h=H, w=W):
    side = A.OCCLUSION_BANK_SIDE
    yy, xx = np.mgrid[:side, :side]
    bits = np.zeros((n, side, side), bool)
    for i in range(n):
        for _ in range(rng.randint(1, 4)):
            cy, cx = rng.randint(30, 194, 2)
            ry, rx = rng.randint(10, 70, 2)
            bits[i] |= ((yy - cy) / float(ry)) ** 2 + ((xx - cx) / float(rx)) ** 2 <= 1.0
    path = tmp_path / "arbitrary_syn_masks.bin"
    np.packbits(bits.reshape(-1)).tofile(path)
    words = A.load_occlusion_bank(str(path), (h, w))
    f32 = np.unpackbits(words.view(np.uint8), axis=-1, bitorder="little").reshape(n, h, w).astype(np.float32)
    return str(path), words, f32


def _overlap(mask, occ, tx, ty):
    obj = ~mask
    return np.count_nonzero(obj & OO.shift_zero_fill(occ, tx, ty).astype(bool)) / float(np.count_nonzero(obj))


def _run(occl, masks, words, P):
    out = occl.apply_device(torch.from_numpy(masks).cuda(), words, params=P)
    return out.cpu().numpy().astype(bool), occl.fallbacks()


def test_kernel_matches_the_restatement_with_edge_cases(tmp_path):
    rng = np.random.RandomState(0)
    B, R, S = 64, 0.4, 0.2                     # realistic limit above the square one: step 2 can leave nothing step 3 accepts
    _, words, bank = _bank(tmp_path, rng)
    masks = _objects(rng, B)
    occl = A.Occlusion((H, W), R, S, seed=1)
    K = occl.K
    P = occl.sample(B, len(words))
    yy, xx = np.mgrid[:H, :W]
    masks[0] = True                                                    # no object pixels
    masks[1] = (yy - 15) ** 2 + (xx - 15) ** 2 > 12 ** 2               # object in the top-left corner ...
    P["tx"][1], P["ty"][1] = 89, 89                                    # ... and every shift moves the occluder away from it
    ov = lambda b, k: _overlap(masks[b], bank[P["occluder"][b]], P["tx"][b, k], P["ty"][b, k])     # noqa: E731
    # late accepts (rounds 2..8 of the kernel), and a first accept whose overlap is above the square step's limit
    arranged, targets = {}, [20, K - 1, 9]
    for b in range(2, B):
        o = np.array([ov(b, k) for k in range(K)])
        ok = (o > 0) & (o < R)
        good, bad, over = np.nonzero(ok)[0], np.nonzero(~ok)[0], np.nonzero((o > S) & (o < R))[0]
        if targets and len(good) and len(bad):
            k = targets.pop(0)                                         # rejected candidates (repeated as needed) first
            order = np.concatenate([np.resize(bad, k), good, bad])[:K]
            arranged[b] = k
        elif "over" not in arranged and len(over):
            order = np.concatenate([over, np.nonzero(~((o > S) & (o < R)))[0]])
            arranged["over"] = b
        else:
            continue
        P["tx"][b], P["ty"][b] = P["tx"][b][order], P["ty"][b][order]
    assert len(arranged) == 4, arranged
    got, fb = _run(occl, masks, words, P)
    want, wfb = OO.occlude(masks, bank, P, R, S)
    assert np.array_equal(got, want), np.nonzero((got != want).any((1, 2)))[0]
    assert fb == wfb, (fb, wfb)
    # the cases did what they are there for
    _, taken = OO.realistic_occlusion(masks, bank[P["occluder"]], P["tx"], P["ty"], R)
    assert taken[0] == -1 and taken[1] == -1 and (taken == 0).any()
    for b, k in arranged.items():
        if b != "over":
            assert taken[b] == k, (b, taken[b], k)
    b = arranged["over"]
    assert taken[b] == 0
    noof = np.count_nonzero(~masks, axis=(1, 2))
    mid, _ = OO.realistic_occlusion(masks[b:b + 1], bank[P["occluder"][b:b + 1]], P["tx"][b:b + 1], P["ty"][b:b + 1], R)
    _, taken_sq = OO.square_occlusion(mid, noof[b:b + 1], P["square_on"][b:b + 1], P["square_keep"][b:b + 1], S)
    assert taken_sq[0] == -1 and np.array_equal(got[b], mid[0])
    assert wfb["realistic"] >= 2 and wfb["square"] >= 1


def test_each_step_alone_and_the_fallback_counter_clears(tmp_path):
    rng = np.random.RandomState(3)
    _, words, bank = _bank(tmp_path, rng)
    masks = _objects(rng, 32)
    for R, S in ((0.25, 0.0), (0.0, 0.3)):
        occl = A.Occlusion((H, W), R, S, seed=5)
        P = occl.sample(32, len(words))
        got, fb = _run(occl, masks, words if R else None, P)
        want, wfb = OO.occlude(masks, bank, P, R, S)
        assert np.array_equal(got, want) and fb == wfb
        assert occl.fallbacks() == {"realistic": 0, "square": 0}


def test_accepted_images_satisfy_the_acceptance_tests(tmp_path):
    rng = np.random.RandomState(7)
    _, words, bank = _bank(tmp_path, rng, n=40)
    B = 4096
    masks = _objects(rng, B)
    n0 = np.count_nonzero(~masks, axis=(1, 2))
    occl = A.Occlusion((H, W), 0.25, 0.0, seed=11)
    got, fb = _run(occl, masks, words, occl.sample(B, len(words)))
    assert not (got < masks).any()                                    # only object pixels become background
    n1 = np.count_nonzero(~got, axis=(1, 2))
    changed = n1 != n0
    frac = (n0 - n1) / np.maximum(n0, 1)
    assert ((frac[changed] > 0) & (frac[changed] < 0.25)).all()
    assert fb["realistic"] == int((~changed).sum()) and fb["square"] == 0
    occl = A.Occlusion((H, W), 0.25, 0.25, seed=12)
    P = occl.sample(B, len(words))
    got, fb = _run(occl, masks, words, P)
    assert not (got < masks).any()
    kept = np.count_nonzero(~got, axis=(1, 2)) / n0.astype(np.float32)
    assert int((kept < 0.75).sum()) <= fb["square"]
    print("fallbacks per %d images: %s" % (B, fb))
    # a slice of the same batch bit for bit
    sl = slice(0, 256)
    want, _ = OO.occlude(masks[sl], bank, {k: v[sl] for k, v in P.items()}, 0.25, 0.25)
    assert np.array_equal(got[sl], want)


def test_batch_device_with_both_switches_matches_the_restated_chain(tmp_path):
    rng = np.random.RandomState(9)
    path, words, bank = _bank(tmp_path, rng)
    n = 40
    x = rng.randint(0, 256, (n, H, W, 3), dtype=np.uint8)
    bg = rng.randint(0, 256, (n, H, W, 3), dtype=np.uint8)
    np.savez(tmp_path / "train.npz", train_x=x, mask_x=_objects(rng, n), train_y=x[::-1].copy())
    np.save(tmp_path / "bg.npy", bg)
    ds = Dataset(None, code=TEMPLATE_CODE, h=H, w=W, c=3, seed=6, realistic_occlusion="0.25", square_occlusion="0.25")
    ds.load_training_images(str(tmp_path / "train.npz"), str(tmp_path / "bg.npy"))
    assert ds.load_occlusion_masks(path) == len(words)
    aug, occl = ds._aug, ds._occlusion
    aug_state, occl_state = aug.rng.get_state(), occl.rng.get_state()
    np.random.seed(21)
    xf, yf = ds.batch_device(24)
    fb = ds.occlusion_fallbacks()
    np.random.seed(21)
    idx = np.random.choice(n, 24, replace=False)
    idx_bg = np.random.choice(n, 24, replace=False)
    aug.rng.set_state(aug_state)
    occl.rng.set_state(occl_state)
    P_occl = occl.sample(24, len(words))
    P_aug = aug.sample(24)
    masks, wfb = OO.occlude(ds.mask_x[idx], bank, P_occl, 0.25, 0.25)
    want = AO.augment_batch(x[idx], masks, bg[idx_bg], P_aug, aug.sigma, low=aug.low)
    assert np.array_equal(xf.cpu().numpy(), (want / 255.).astype(np.float32))
    assert np.allclose(yf.cpu().numpy(), x[::-1][idx] / 255., rtol=0, atol=1e-7)         # the targets are not occluded
    assert fb == wfb
