"""Occlusion-mask augmentations (REALISTIC_OCCLUSION / SQUARE_OCCLUSION, auto_pose/ae/dataset.py:405-454) without a GPU: the
bank loader and the shift against OpenCV, the restatement against the reference's own output (tests/golden/occlusion_realistic.npz,
tests/golden/make_occlusion_golden.py), the host draws, cfg parsing, and batch_device's random streams."""
import os

import numpy as np
import pytest
import torch

from augmentedautoencoder_b200.ae import augment as A
from augmentedautoencoder_b200.ae.dataset import Dataset
from oracle import occlusion_oracle as OO

cv2 = pytest.importorskip("cv2")
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "occlusion_realistic.npz")


def _unpack_bank(words, h, w):
    return np.unpackbits(words.view(np.uint8), axis=-1, bitorder="little").reshape(-1, h, w).astype(bool)


def test_bank_loader_follows_the_reference_arithmetic(tmp_path):
    bits = np.random.RandomState(0).rand(3, 224, 224) < 0.3
    path = tmp_path / "masks.bin"
    np.packbits(bits.reshape(-1)).tofile(path)
    # dataset.py:411-416: bitarray unpack (big-endian bits), reshape(-1, 224, 224, 1), float32, cv2.resize NEAREST to (H, W)
    ref = np.unpackbits(np.fromfile(path, np.uint8)).astype(bool).reshape(-1, 224, 224, 1).astype(np.float32)
    for h in (128, 64, 96):
        want = np.array([cv2.resize(m, (h, h), interpolation=cv2.INTER_NEAREST) for m in ref])
        got = A.load_occlusion_bank(str(path), (h, h, 3))
        assert got.dtype == np.uint32 and got.shape == (3, h, h // 32)
        assert np.array_equal(_unpack_bank(got, h, h), want.astype(bool)), h
    with open(path, "rb") as f:
        data = f.read()
    (tmp_path / "short.bin").write_bytes(data[:-1])
    with pytest.raises(ValueError):
        A.load_occlusion_bank(str(tmp_path / "short.bin"), (128, 128, 3))
    with pytest.raises(NotImplementedError):
        A.load_occlusion_bank(str(path), (80, 80, 3))


def test_bank_loader_reads_the_golden_bank(tmp_path):
    g = np.load(GOLDEN)
    path = tmp_path / "bank.bin"
    g["bank_raw"].tofile(path)
    got = _unpack_bank(A.load_occlusion_bank(str(path), (128, 128, 1)), 128, 128)
    assert np.array_equal(got, np.unpackbits(g["bank_f32"], axis=-1).astype(bool))


def test_shift_restatement_equals_warp_affine_for_every_reachable_shift():
    rng = np.random.RandomState(1)
    m = (rng.rand(128, 128) < 0.5).astype(np.float32)
    m[:, :3] = m[:3, :] = m[-3:, :] = m[:, -3:] = 1.0            # borders set: the fill has to come from the shift
    for t in range(25, 90):
        for tx, ty in ((t, -t), (-t, t), (t, 114 - t), (-t, t - 114)):
            ref = cv2.warpAffine(m, np.float32([[1, 0, tx], [0, 1, ty]]), (128, 128))
            assert np.array_equal(OO.shift_zero_fill(m, tx, ty), ref), (tx, ty)


def _golden():
    g = np.load(GOLDEN)
    h, w = (int(v) for v in g["shape"])
    unpack = lambda a: np.unpackbits(a, axis=-1)[..., :w].astype(bool)      # noqa: E731
    return g, unpack(g["masks_in"]), unpack(g["masks_out"]), unpack(g["bank_f32"]).astype(np.float32), h, w


def test_restatement_replays_the_reference_bit_for_bit():
    g, masks, want, bank, h, w = _golden()
    d = g["draws"]
    tx, ty = OO.translations(d[:, 0], d[:, 1], d[:, 2], d[:, 3], h, w)
    first = np.concatenate([[0], np.cumsum(g["attempts"])])
    assert first[-1] == len(d) and (g["attempts"] == 1).any() and g["attempts"].max() >= 20     # first and late accepts
    for b in range(len(masks)):
        s, e = first[b], first[b + 1]
        got, taken = OO.realistic_occlusion(masks[b:b + 1], bank[g["occluder"][b:b + 1]], tx[None, s:e], ty[None, s:e], float(g["max_occl"]))
        assert taken[0] == e - s - 1, b                               # the reference stopped at its first accept
        assert np.array_equal(got[0], want[b]), b
        # ... and the product's candidate arithmetic makes the same shifts from the same draws
        span = A.OCCLUSION_MAX_TRANS - A.OCCLUSION_MIN_TRANS
        assert np.array_equal(np.trunc(d[s:e, 0] * (d[s:e, 1] * span + A.OCCLUSION_MIN_TRANS) * h).astype(int), tx[s:e])


def test_restatement_fallbacks_and_square_step():
    _, masks, _, bank, h, w = _golden()
    empty = np.ones((1, h, w), bool)
    got, taken = OO.realistic_occlusion(empty, bank[:1], np.array([[30]]), np.array([[30]]), 0.25)
    assert taken[0] == -1 and np.array_equal(got, empty)
    # square: a no-op candidate passes, a grid that drops everything fails, and the denominator is the unoccluded count
    lh, lw = A.square_grid(h, w)
    keep_none = np.zeros((1, 2, lh, lw), bool)
    noof = np.count_nonzero(masks[:1] == 0, axis=(1, 2))
    out, taken = OO.square_occlusion(masks[:1], noof, np.array([[True, False]]), keep_none, 0.25)
    assert taken[0] == 1 and np.array_equal(out, masks[:1])
    out, taken = OO.square_occlusion(masks[:1], noof, np.array([[True, True]]), keep_none, 0.25)
    assert taken[0] == -1 and np.array_equal(out, masks[:1])


def test_host_draws_follow_the_reference_distributions():
    occl = A.Occlusion((128, 128, 3), 0.25, 0.3, seed=3)
    assert occl.low == (A.SQUARE_OCCLUSION_MIN_SIZE,) * 2
    P = occl.sample(512, n_bank=10)
    K = A.OCCLUSION_CANDIDATES
    assert P["tx"].shape == P["ty"].shape == P["square_on"].shape == (512, K)
    assert P["square_keep"].shape == (512, K) + occl.low
    for t in (P["tx"], P["ty"]):
        assert np.abs(t).min() == 25 and np.abs(t).max() == 89            # int((u * 0.5 + 0.2) * 128), u in [0, 1)
        assert abs((t > 0).mean() - 0.5) < 0.01
    counts = np.bincount(P["occluder"], minlength=10)
    assert counts.min() > 25 and P["occluder"].max() == 9
    assert abs(P["square_on"].mean() - A.SQUARE_P_ON) < 0.01
    assert abs(P["square_keep"].mean() - (1 - A.SQUARE_P_DROP)) < 0.01
    cand = occl.pack(P)
    assert cand.shape == (512, 1 + 3 * K) and cand.dtype == np.int32
    assert np.array_equal(cand[:, 0], P["occluder"]) and np.array_equal(cand[:, 1:K + 1], P["tx"])
    assert np.array_equal(cand[:, K + 1:2 * K + 1], P["ty"])
    cells = occl.low[0] * occl.low[1]
    keep = cand[:, 2 * K + 1:].view(np.uint32)
    bits = (keep[..., None] >> np.arange(cells, dtype=np.uint32)) & 1
    want = np.where(P["square_on"][..., None], P["square_keep"].reshape(512, K, cells), True)
    assert np.array_equal(bits.astype(bool), want) and not (keep >> np.uint32(cells)).any()


@pytest.mark.parametrize("value,want", [("False", 0.0), ("0", 0.0), ("0.25", 0.25), (None, 0.0), (0.3, 0.3)])
def test_occlusion_switches_parse_like_the_reference(value, want):
    assert A.occlusion_limit(value) == want


def test_switches_build_the_step_and_refuse_unsupported_shapes():
    assert Dataset(None, realistic_occlusion="False", square_occlusion="0")._occlusion is None
    occl = Dataset(None, realistic_occlusion="0.25", square_occlusion="False", seed=2)._occlusion
    assert occl.realistic == 0.25 and occl.square == 0.0
    with pytest.raises(NotImplementedError):
        Dataset(None, h=128, w=96, realistic_occlusion="0.25")._occlusion
    with pytest.raises(NotImplementedError):
        Dataset(None, h=80, w=80, square_occlusion="0.25")._occlusion


def _dataset(tmp_path, **kw):
    rng = np.random.RandomState(5)
    x = rng.randint(0, 256, (12, 128, 128, 3), dtype=np.uint8)
    mask = rng.rand(12, 128, 128) < 0.5
    np.savez(tmp_path / "train.npz", train_x=x, mask_x=mask, train_y=x)
    np.save(tmp_path / "bg.npy", x[::-1].copy())
    ds = Dataset(None, code="Sequential([Sometimes(0.5, Add((-25, 25)))])", seed=4, **kw)
    ds.load_training_images(str(tmp_path / "train.npz"), str(tmp_path / "bg.npy"))
    return ds


def test_batch_device_random_streams(tmp_path, monkeypatch):
    """Switches off (or absent): the global stream gives exactly the two index draws, the mask reaches the augmenter unchanged
    and no occlusion step exists.  Switches on: the same global draws; the occlusion draws come from a stream of their own."""
    seen = []

    def fake_augment(self, x, m, bg, params=None, want_u8=False):
        seen.append(m.cpu().numpy().copy())
        return x.to(torch.float32)

    def fake_occlusion(self, m, bank=None, params=None):
        self.sample(len(m), len(bank))
        return m

    monkeypatch.setattr(A.Augmenter, "augment_device", fake_augment)
    monkeypatch.setattr(A.Occlusion, "apply_device", fake_occlusion)
    for kw in ({"realistic_occlusion": "False", "square_occlusion": "False"}, {}, {"realistic_occlusion": "0.25", "square_occlusion": "0.3"}):
        on = bool(kw) and kw["realistic_occlusion"] != "False"
        ds = _dataset(tmp_path, **kw)
        if on:
            bank = tmp_path / "bank.bin"
            np.packbits(np.random.RandomState(0).rand(2, 224, 224) < 0.2).tofile(bank)
            assert ds.load_occlusion_masks(str(bank)) == 2
        np.random.seed(11)
        ds.batch_device(8, device=torch.device("cpu"))
        after = np.random.rand()
        np.random.seed(11)
        idx = np.random.choice(12, 8, replace=False)
        np.random.choice(12, 8, replace=False)
        assert np.random.rand() == after
        assert (ds._occlusion is None) == (not on)
        if not on:
            assert np.array_equal(seen[-1], ds.mask_x[idx].astype(np.uint8))
        else:
            # the occlusion draws left the augmenter's RandomState(seed) alone, and their stream is not a copy of it
            assert ds._occlusion.rng is not ds._aug.rng
            assert ds._aug.rng.rand() == np.random.RandomState(4).rand()
            assert A.Occlusion((128, 128), 0.25, seed=4).rng.rand() != np.random.RandomState(4).rand()
