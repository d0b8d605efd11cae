#!/usr/bin/env python
"""Generate tests/golden/occlusion_realistic.npz by running the REFERENCE's own ``Dataset.augment_occlusion_mask``
(auto_pose/ae/dataset.py:421-444, REALISTIC_OCCLUSION) on synthetic masks and a small synthetic occluder bank.

Run in the build container only (needs /root/reference; the GPU box has no copy):

    python tests/golden/make_occlusion_golden.py

The function needs only numpy and cv2.  Its random draws (one ``np.random.choice(n_bank, B)``, then per attempt
``choice([-1, 1])``, ``rand()``, ``choice([-1, 1])``, ``rand()``) come from a seeded RandomState through recording wrappers,
so the file holds inputs, every draw in call order and the reference's output masks.  The bank is stored as the raw bits of
the reference's file format (224 x 224 bits per mask, big-endian bit order) together with the float32 128 x 128 masks the
reference's loader arithmetic makes of them (unpack, reshape, float32, cv2.resize INTER_NEAREST).
"""
import os
import sys

import numpy as np

sys.dont_write_bytecode = True  # /root/reference is read-only
OUT = os.path.dirname(os.path.abspath(__file__))
H = W = 128


def synthetic_masks():
    """True = background.  Discs, an ellipse, a rectangle, a ring and objects at the border, sized so that every image has
    shifts the reference accepts (its loop has no bound)."""
    yy, xx = np.mgrid[:H, :W]
    objs = []
    for cy, cx, r in ((64, 64, 40), (60, 70, 25), (40, 40, 30), (90, 30, 18), (64, 64, 55), (20, 100, 15)):
        objs.append((yy - cy) ** 2 + (xx - cx) ** 2 <= r * r)
    objs.append(((yy - 64) / 50.0) ** 2 + ((xx - 64) / 20.0) ** 2 <= 1.0)
    objs.append((yy >= 20) & (yy < 110) & (xx >= 30) & (xx < 100))
    objs.append(((yy - 64) ** 2 + (xx - 64) ** 2 <= 45 ** 2) & ((yy - 64) ** 2 + (xx - 64) ** 2 > 25 ** 2))
    objs.append((yy < 50) & (xx < 60))
    return ~np.stack(objs)


def synthetic_bank(rng, n=5, side=224):
    """Occluder blobs in the reference's 224 x 224 format: unions of random ellipses."""
    yy, xx = np.mgrid[:side, :side]
    bank = np.zeros((n, side, side), bool)
    for i in range(n):
        for _ in range(rng.randint(1, 4)):
            cy, cx = rng.randint(40, 184, 2)
            ry, rx = rng.randint(15, 60, 2)
            bank[i] |= ((yy - cy) / float(ry)) ** 2 + ((xx - cx) / float(rx)) ** 2 <= 1.0
    return bank


def main():
    import cv2
    if not hasattr(np, "bool"):
        np.bool = bool  # auto_pose/ae/dataset.py:423-433 uses the alias numpy removed in 1.24
    sys.path.insert(0, OUT)
    from make_golden import install_stubs      # TensorFlow / progressbar / m3vision stubs for importing auto_pose
    install_stubs()
    from auto_pose.ae.dataset import Dataset

    rng = np.random.RandomState(2024)
    bank_bits = synthetic_bank(rng)
    raw = np.packbits(bank_bits.reshape(-1))                                        # the .bin file's bytes
    # the reference's loader arithmetic (dataset.py:411-416) on those bytes
    occl = np.unpackbits(raw).astype(bool).reshape(-1, 224, 224, 1).astype(np.float32)
    occl = np.array([cv2.resize(m, (H, W), interpolation=cv2.INTER_NEAREST) for m in occl])

    masks = synthetic_masks()
    ds = Dataset.__new__(Dataset)
    ds.shape = (H, W, 1)
    ds._cache_random_syn_masks = occl                                               # lazy_property's cache slot

    calls = []
    draw_rng = np.random.RandomState(7)
    real_choice, real_rand = np.random.choice, np.random.rand

    def choice(a, size=None, *args, **kw):
        v = draw_rng.choice(a, size, *args, **kw)
        calls.append(("choice", np.array(v)))
        if len(calls) > 200000:
            raise RuntimeError("no accept after 50000 attempts: change the synthetic inputs")
        return v

    def rand(*shape):
        v = draw_rng.rand(*shape)
        calls.append(("rand", np.array(v)))
        return v

    # one call per image, so that the attempts of each image are the draws of its own call (the loop treats the images of a
    # batch independently; a batch call would make the same draws with the occluder indices up front)
    out, occl_idx, draws, per_img = [], [], [], []
    np.random.choice, np.random.rand = choice, rand
    try:
        for b in range(len(masks)):
            calls.clear()
            out.append(ds.augment_occlusion_mask(masks[b:b + 1].copy(), max_occl=0.25)[0])
            assert calls[0][0] == "choice" and (len(calls) - 1) % 4 == 0
            assert [c[0] for c in calls[1:]] == ["choice", "rand"] * ((len(calls) - 1) // 2)
            occl_idx.append(int(calls[0][1][0]))
            draws += [float(c[1]) for c in calls[1:]]
            per_img.append((len(calls) - 1) // 4)
    finally:
        np.random.choice, np.random.rand = real_choice, real_rand
    out, occl_idx = np.stack(out), np.array(occl_idx)
    draws = np.array(draws).reshape(-1, 4)                                         # [attempts, (sx, ux, sy, uy)] in call order
    print("attempts per image:", per_img)
    np.savez_compressed(
        os.path.join(OUT, "occlusion_realistic.npz"), masks_in=np.packbits(masks, axis=-1), masks_out=np.packbits(out, axis=-1),
        shape=np.array([H, W]), bank_raw=raw, bank_n=np.array(len(bank_bits)), bank_f32=np.packbits(occl.astype(bool), axis=-1),
        max_occl=np.array(0.25), occluder=occl_idx, draws=draws, attempts=np.array(per_img))
    print("wrote", os.path.join(OUT, "occlusion_realistic.npz"), os.path.getsize(os.path.join(OUT, "occlusion_realistic.npz")), "B")


if __name__ == "__main__":
    main()
