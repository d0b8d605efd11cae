"""The training input kernels (aae_augment and aae_occlusion, gathered and indexed) against the CPU restatement at
the cfg geometries beyond the template (tests/geometry_table.py): px64 (64 x 64 x 3), gray (128 x 128 x 1) and rect (64 x 128 x 3),
where tests/test_input_geometry_cpu.py pins the restatement to OpenCV.  Every comparison is bit for bit: the pipelines are
integer, and the float outputs are table look-ups.

  * gray reads one lane of the kernel's four-lane fetch and one LUT channel per image; with size_percent 0.0625 its 8 x 8
    CoarseDropout grid reaches keep bit 63 (the template's 6 x 6 grid never sets the top of the high keep word);
  * px64 runs the occlusion kernel with two words per row, occluder shifts past one word (up to +-44 px) and a 3 x 3 square grid;
  * the chains scale with Affine(scale=(0.5, 1.5)): below 1 the source coordinates go negative and the bilinear fetch reads the
    zero border; the blur runs at sigma 0.0005 (flag off), 0.01 (taps 0, 0, 256, 0, 0 with the flag on) and 1.49;
  * the out-of-stack contract of include/aae_b200.h for both indexed entry points, and stack rows past 2^31 and 2^32 bytes;
  * aae_extract_square_patches at the px64 patch size."""
import gc

import numpy as np
import pytest
import torch

from augmentedautoencoder_b200.ae import augment as A
from augmentedautoencoder_b200.ae.dataset import Dataset
from oracle import augment_oracle as AO
from oracle import occlusion_oracle as OO
from tests import geometry_table as GT
from tests.test_gpu_g_occlusion import _bank, _objects, _overlap, _run

pytestmark = pytest.mark.gpu
GEOMS = ["px64", "gray", "rect"]
SIGMAS = [0.0005, 0.01, 1.49]
SCALE = (0.5, 1.5)
DROP = {"px64": 0.0625, "gray": 0.0625, "rect": 0.05}        # size_percent of the CoarseDropout in each geometry's chain
GRID = {"px64": (4, 4), "gray": (8, 8), "rect": (4, 6)}     # ... and the grid it gives there
ON_KEYS = ("affine_on", "drop_on", "blur_on", "add_on", "invert_on", "mul1_on", "mul2_on", "contrast_on")
DEV = torch.device("cuda", 0)


@pytest.fixture(autouse=True)
def _quiet_device():
    torch.cuda.synchronize()
    yield
    torch.cuda.synchronize()
    gc.collect()
    torch.cuda.empty_cache()


def _shape(geom):
    r = GT.row(geom)
    return r["h"], r["w"], r["c"]


def _code(size_percent, sigma, scale=SCALE):
    """the template's chain with a wider scale range, every value op per channel, and the given dropout grid and blur sigma"""
    return """Sequential([
    Sometimes(0.5, Affine(scale=(%r, %r))),
    Sometimes(0.5, CoarseDropout(p=0.2, size_percent=%r)),
    Sometimes(0.5, GaussianBlur(%r)),
    Sometimes(0.5, Add((-25, 25), per_channel=True)),
    Sometimes(0.3, Invert(0.2, per_channel=True)),
    Sometimes(0.5, Multiply((0.6, 1.4), per_channel=0.5)),
    Sometimes(0.5, Multiply((0.6, 1.4))),
    Sometimes(0.5, ContrastNormalization((0.5, 2.2), per_channel=0.3))
    ], random_order=False)""" % (scale[0], scale[1], size_percent, sigma)


def _augmenter(geom, sigma, seed):
    h, w, c = _shape(geom)
    aug = A.Augmenter(_code(DROP[geom], sigma), (h, w, c), seed=seed)
    assert aug.low == GRID[geom] and aug.sigma == sigma
    return aug


def _images(rng, n, h, w, c):
    return rng.randint(0, 256, (n, h, w, c), dtype=np.uint8)


def _force(P):
    """every op fires somewhere: all of them on images 0-3, each one alone on images 4-11, the draws elsewhere"""
    for i, k in enumerate(ON_KEYS):
        P[k][:4] = True
        P[k][4:4 + len(ON_KEYS)] = False
        P[k][4 + i] = True
    return P


def _sampled(aug, B):
    """a batch of draws with every op forced on somewhere, both sides of scale 1, and (8 x 8 grid) keep bit 63 both ways"""
    P = _force(aug.sample(B))
    s = P["affine_M"][:, 0, 0]
    assert (P["affine_on"] & (s < 0.9)).any() and (P["affine_on"] & (s > 1.1)).any()
    if aug.c > 1:                                              # per-channel values that differ between channels
        assert (P["add_on"] & (P["add_val"] != P["add_val"][:, :1]).any(1)).any()
        assert (P["mul1_on"] & (P["mul1_val"] != P["mul1_val"][:, :1]).any(1)).any()
    if aug.low == (8, 8):
        P["drop_keep"][0, 7, 7], P["drop_keep"][1, 7, 7] = 0, 1
    return P


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def _y_target(y):
    """the target y / 255. of uint8 values as Dataset.batch_device computes it: torch's float32 division by a scalar on the
    device, which multiplies by the float32 reciprocal and so differs from numpy's y / np.float32(255) in the last bit"""
    return (torch.arange(256, dtype=torch.float32, device=DEV) / 255.0).cpu().numpy()[y]


# ---- aae_augment --------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("sigma", SIGMAS)
@pytest.mark.parametrize("geom", GEOMS)
def test_augment_batch_matches_the_restatement(geom, sigma):
    """rect (64 x 128) is the only shape where a swapped row / column table shows: adelta / bdelta have W entries and X0 / Y0
    H, the dropout maps H and W entries, and the scale centre differs between the axes.  No decoder trains at rect, but the
    augment kernels accept it, so they are checked there."""
    h, w, c = _shape(geom)
    B = 32
    rng = np.random.RandomState(1)
    x, bg, mask = _images(rng, B, h, w, c), _images(rng, B, h, w, c), _objects(rng, B, h, w)
    aug = _augmenter(geom, sigma, seed=3)
    P = _sampled(aug, B)
    want = AO.augment_batch(x, mask, bg, P, aug.sigma, low=aug.low)
    got_f, got_u = aug.augment_device(_dev(x), _dev(mask), _dev(bg), params=P, want_u8=True)
    got_u = got_u.cpu().numpy()
    assert np.array_equal(got_u, want), (geom, sigma, np.argwhere(got_u != want)[:5])
    assert np.array_equal(got_f.cpu().numpy(), (want / 255.).astype(np.float32))


# ---- aae_occlusion at 64 x 64 -------------------------------------------------------------------------------------------------------
FAR = [(1, 1), (1, -1), (-1, 1), (-1, -1)]                    # signs of (tx, ty) of the arranged accepts
LATE = [0, 9, 20, A.OCCLUSION_CANDIDATES - 1]                # ... and the candidate they sit at


def _arrange_far_accepts(masks, bank, P, R, first):
    """For each sign pair of FAR, an image from `first` on whose accepted candidate is a shift of 33..44 px in both axes, placed
    at the LATE position after candidates the image rejects.  Returns {image: accepted candidate}."""
    K = P["tx"].shape[1]
    arranged = {}
    b = first
    for (sx, sy), k in zip(FAR, LATE):
        found = None
        while found is None and b < len(masks):
            occ = bank[P["occluder"][b]]
            o = np.array([_overlap(masks[b], occ, P["tx"][b, j], P["ty"][b, j]) for j in range(K)])
            bad = np.nonzero(~((o > 0) & (o < R)))[0]
            for t in ((tx, ty) for tx in range(33, 45) for ty in range(33, 45)):
                if len(bad) and 0 < _overlap(masks[b], occ, sx * t[0], sy * t[1]) < R:
                    found = (b, sx * t[0], sy * t[1], bad)
                    break
            b += 1
        assert found is not None, (sx, sy)
        i, tx, ty, bad = found
        tx_i, ty_i = P["tx"][i].copy(), P["ty"][i].copy()
        order = np.resize(bad, k)                              # rejected candidates first (repeated as needed)
        P["tx"][i, :k], P["ty"][i, :k] = tx_i[order], ty_i[order]
        P["tx"][i, k], P["ty"][i, k] = tx, ty
        arranged[i] = k
    return arranged


@pytest.mark.parametrize("R,S", [(0.4, 0.0), (0.0, 0.2), (0.4, 0.2)], ids=["realistic", "square", "both"])
def test_occlusion_at_64_matches_the_restatement(tmp_path, R, S):
    h = 64
    B = 48
    rng = np.random.RandomState(4)
    _, words, bank = _bank(tmp_path, rng, h=h, w=h)
    masks = _objects(rng, B, h, h)
    occl = A.Occlusion((h, h), R, S, seed=2)
    assert occl.low == (3, 3)
    K = occl.K
    P = occl.sample(B, len(words))
    yy, xx = np.mgrid[:h, :h]
    masks[0] = True                                             # no object pixels: realistic falls back, square accepts its NaN
    masks[1:3] = (yy - 7) ** 2 + (xx - 7) ** 2 > 6 ** 2          # object in the top-left corner ...
    arranged = {}
    if R:
        assert np.abs(P["tx"]).max() > 32 and np.abs(P["ty"]).max() > 32
        P["tx"][1:3], P["ty"][1:3] = 44, 44                      # ... every shift moves the occluder off it: a fallback
        arranged = _arrange_far_accepts(masks, bank, P, R, first=4)
    if S:
        P["square_on"][2, :17], P["square_keep"][2, :17] = True, False     # a late accept: 17 candidates drop every cell,
        P["square_on"][2, 17] = False                                      # the 18th is the Sometimes draw that did not fire
        P["square_on"][3], P["square_keep"][3] = True, False               # ... and a fallback: every candidate drops every cell
    got, fb = _run(occl, masks, words if R else None, P)
    want, wfb = OO.occlude(masks, bank, P, R, S)
    assert np.array_equal(got, want), np.nonzero((got != want).any((1, 2)))[0]
    assert fb == wfb, (fb, wfb)
    # the cases did what they are there for
    mid = masks
    if R:
        mid, taken = OO.realistic_occlusion(masks, bank[P["occluder"]], P["tx"], P["ty"], R)
        assert (taken[:3] == -1).all() and wfb["realistic"] >= 3
        for b, k in arranged.items():
            assert taken[b] == k and abs(P["tx"][b, k]) > 32 and abs(P["ty"][b, k]) > 32, (b, taken[b], k)
        assert {(np.sign(P["tx"][b, k]), np.sign(P["ty"][b, k])) for b, k in arranged.items()} == set(FAR)
    if S:
        noof = np.count_nonzero(~masks, axis=(1, 2))
        _, taken_sq = OO.square_occlusion(mid, noof, P["square_on"], P["square_keep"], S)
        assert taken_sq[0] == 0 and taken_sq[2] == 17 and taken_sq[3] == -1 and wfb["square"] >= 1


# ---- Dataset.batch_device / batch_resident ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("geom", ["px64", "gray"])
def test_batch_device_and_batch_resident_match_the_restated_chain(tmp_path, geom):
    """Both batch paths against the chain restated on the host (not against each other): px64 with both occlusion switches on,
    gray (C = 1) with them off. """
    h, w, c = _shape(geom)
    on = geom == "px64"
    n, n_bg, B = 40, 30, 24
    rng = np.random.RandomState(9)
    x, y, bg, mask = _images(rng, n, h, w, c), _images(rng, n, h, w, c), _images(rng, n_bg, h, w, c), _objects(rng, n, h, w)
    kw = dict(code=_code(DROP[geom], 1.49), h=h, w=w, c=c, seed=6)
    if on:
        kw.update(realistic_occlusion="0.25", square_occlusion="0.25")
    ds = Dataset(None, **kw)
    ds.train_x, ds.mask_x, ds.train_y, ds.bg_imgs = x, mask, y, bg
    bank = None
    if on:
        path, words, bank = _bank(tmp_path, rng, h=h, w=w)
        assert ds.load_occlusion_masks(path) == len(words)
    ds.upload(DEV)
    aug, occl = ds._aug, ds._occlusion
    assert (occl is not None) == on and aug.low == GRID[geom]
    states = aug.rng.get_state(), (occl.rng.get_state() if on else None)

    def rewind(seed):
        np.random.seed(seed)
        aug.rng.set_state(states[0])
        if on:
            occl.rng.set_state(states[1])

    rewind(21)                                                  # Dataset.batch's draws in its order
    idx = np.random.choice(n, B, replace=False)
    idx_bg = np.random.choice(n_bg, B, replace=False)
    P_occl = occl.sample(B, len(bank)) if on else None
    P_aug = aug.sample(B)
    masks, wfb = OO.occlude(mask[idx], bank, P_occl, 0.25, 0.25) if on else (mask[idx], {"realistic": 0, "square": 0})
    want_x = (AO.augment_batch(x[idx], masks, bg[idx_bg], P_aug, aug.sigma, low=aug.low) / 255.).astype(np.float32)
    want_y = _y_target(y[idx])
    assert P_aug["blur_on"].any() and P_aug["affine_on"].any() and P_aug["drop_on"].any()
    for run in (ds.batch_device, ds.batch_resident):
        rewind(21)
        xf, yf = run(B)
        assert np.array_equal(xf.cpu().numpy(), want_x), run.__name__
        assert np.array_equal(yf.cpu().numpy(), want_y), run.__name__
        assert ds.occlusion_fallbacks() == wfb, run.__name__


# ---- indices outside the stack ------------------------------------------------------------------------------------------------------
def _gathered(x, mask, bg, idx, idx_bg, mask_batch=None):
    """the batch the header's contract describes: image b is x[idx[b]] pasted on bg[idx_bg[b]], or all zeros when either index
    is outside its stack; the mask is mask[idx[b]] or row b of mask_batch"""
    ok = (idx >= 0) & (idx < len(x)) & (idx_bg >= 0) & (idx_bg < len(bg))
    xg, bgg = np.zeros((len(idx),) + x.shape[1:], np.uint8), np.zeros((len(idx),) + bg.shape[1:], np.uint8)
    xg[ok], bgg[ok] = x[idx[ok]], bg[idx_bg[ok]]
    if mask_batch is not None:
        mg = mask_batch.astype(bool)
    else:
        mg = np.ones((len(idx),) + mask.shape[1:], bool)
        mg[ok] = mask[idx[ok]]
    return xg, mg, bgg, ok


@pytest.mark.parametrize("geom", GEOMS)
def test_augment_indexed_outside_the_stack(geom):
    """include/aae_b200.h: an image whose idx OR idx_bg is outside its stack is pasted and warped as all zeros, its value tables
    still apply, and its target is y_to_float[0] (0.0); an image whose idx alone is inside keeps its target.  Indices -1, n and
    2^31 - 1; a duplicated (idx, idx_bg) pair with the same draws gives identical rows."""
    h, w, c = _shape(geom)
    n, n_bg, B = 12, 9, 16
    big = 2 ** 31 - 1
    rng = np.random.RandomState(13)
    x, y, bg, mask = _images(rng, n, h, w, c), _images(rng, n, h, w, c), _images(rng, n_bg, h, w, c), _objects(rng, n, h, w)
    idx = np.array([3, -1, 5, n, 7, big, 3, 0, 11, 4, 5, 6, 8, 9, 10, 1], np.int32)
    idx_bg = np.array([0, 1, -1, 2, n_bg, 3, 0, big, 4, 5, 6, 7, 8, 0, 1, 2], np.int32)
    aug = _augmenter(geom, 1.0, seed=5)
    P = _sampled(aug, B)
    for k in P:
        P[k][6] = P[k][0]                                       # image 6 repeats image 0: same rows, same draws
    geom_t, lut = aug.pack(P)
    stacks = {"x": _dev(x), "mask": _dev(mask.astype(np.uint8)), "y": _dev(y), "bg": _dev(bg)}
    idx_in = (idx >= 0) & (idx < n)
    want_y = np.zeros((B, h, w, c), np.float32)
    want_y[idx_in] = _y_target(y[idx[idx_in]])
    for mask_batch in (None, _objects(rng, B, h, w)):
        xg, mg, bgg, ok = _gathered(x, mask, bg, idx, idx_bg, mask_batch)
        assert ok.tolist() == [b not in (1, 2, 3, 4, 5, 7) for b in range(B)]
        want = AO.augment_batch(xg, mg, bgg, P, aug.sigma, low=aug.low)
        # the header's wording: a zero image through the value tables
        assert np.array_equal(want[~ok], np.broadcast_to(lut[~ok][:, None, None, :, 0], (int((~ok).sum()), h, w, c)))
        out_f = torch.empty((B, h, w, c), dtype=torch.float32, device=DEV)
        y_out = torch.full_like(out_f, -1.0)
        mb = _dev(mask_batch.astype(np.uint8)) if mask_batch is not None else None
        aug.augment_indexed(stacks, _dev(idx), _dev(idx_bg), _dev(geom_t), _dev(lut), out_f, y_out, torch.cuda.current_stream(DEV),
                            mask_batch=mb)
        got, got_y = out_f.cpu().numpy(), y_out.cpu().numpy()
        assert np.array_equal(got, (want / 255.).astype(np.float32)), (geom, mask_batch is not None, np.argwhere(got != want / 255.)[:5])
        assert np.array_equal(got_y, want_y)
        assert not got_y[~idx_in].any()
        if mask_batch is None:
            assert np.array_equal(got[0], got[6])


def test_occlusion_indexed_outside_the_stack(tmp_path):
    """A mask row outside the stack is a mask without object pixels: the realistic step falls back (its overlap is 0 / 0) and
    the square step accepts its NaN ratio, so the row comes out all background.  A duplicated index with the same draws gives
    identical rows."""
    h, n, B = 64, 12, 12
    big = 2 ** 31 - 1
    rng = np.random.RandomState(17)
    _, words, bank = _bank(tmp_path, rng, h=h, w=h)
    mask = _objects(rng, n, h, h)
    idx = np.array([2, -1, 5, n, big, 2, 7, 0, 9, 11, 3, 4], np.int32)
    occl = A.Occlusion((h, h), 0.4, 0.2, seed=3)
    P = occl.sample(B, len(words))
    for k in P:
        P[k][5] = P[k][0]
    out = torch.empty((B, h, h), dtype=torch.uint8, device=DEV)
    occl.apply_indexed(_dev(mask.astype(np.uint8)), _dev(idx), _dev(occl.pack(P)), words, out, torch.cuda.current_stream(DEV))
    got, fb = out.cpu().numpy().astype(bool), occl.fallbacks()
    inside = (idx >= 0) & (idx < n)
    mg = np.ones((B, h, h), bool)
    mg[inside] = mask[idx[inside]]
    want, wfb = OO.occlude(mg, bank, P, 0.4, 0.2)
    assert np.array_equal(got, want), np.nonzero((got != want).any((1, 2)))[0]
    assert fb == wfb, (fb, wfb)
    assert got[~inside].all() and np.array_equal(got[0], got[5])
    mid, taken = OO.realistic_occlusion(mg, bank[P["occluder"]], P["tx"], P["ty"], 0.4)
    _, taken_sq = OO.square_occlusion(mid, np.count_nonzero(~mg, axis=(1, 2)), P["square_on"], P["square_keep"], 0.2)
    assert (taken[~inside] == -1).all() and (taken_sq[~inside] == 0).all() and wfb["realistic"] >= 3


# ---- stacks past 2^31 and 2^32 bytes ------------------------------------------------------------------------------------------------
NEED_FREE = 12e9


def _skip_unless_free():
    free = torch.cuda.mem_get_info(DEV)[0]
    if free < NEED_FREE:
        pytest.skip("%.1f GB free on the device; the large-stack test needs %.0f GB" % (free / 1e9, NEED_FREE / 1e9))


def test_augment_reads_stack_rows_past_2_and_4_gib():
    """A 128 x 128 x 3 stack of 87 400 rows (4.30 GB) passed as x, y and bg, and its 1.43 GB mask stack: row 43 690 straddles
    2^31 bytes, row 87 381 straddles 2^32.  Only the indexed rows are filled."""
    _skip_unless_free()
    h, w, c, n = 128, 128, 3, 87400
    rows = np.array([0, 43690, 43691, 87381, 87399], np.int32)
    first = [int(r) * h * w * c for r in rows]                  # byte offset of each row
    assert first[1] < 2 ** 31 < first[2] and first[3] < 2 ** 32 < first[4]
    rng = np.random.RandomState(23)
    x, m = _images(rng, len(rows), h, w, c), _objects(rng, len(rows), h, w)
    stack = torch.empty((n, h, w, c), dtype=torch.uint8, device=DEV)
    mstack = torch.empty((n, h, w), dtype=torch.uint8, device=DEV)
    try:
        for i, r in enumerate(rows):
            stack[int(r)].copy_(torch.from_numpy(x[i]))
            mstack[int(r)].copy_(torch.from_numpy(m[i].astype(np.uint8)))
        B = 15
        sel, sel_bg = np.resize(np.arange(len(rows)), B), np.resize(np.roll(np.arange(len(rows))[::-1], 2), B)
        aug = A.Augmenter(_code(0.05, 1.0), (h, w, c), seed=7)
        P = _sampled(aug, B)
        geom_t, lut = aug.pack(P)
        want = AO.augment_batch(x[sel], m[sel], x[sel_bg], P, aug.sigma, low=aug.low)
        out_f = torch.empty((B, h, w, c), dtype=torch.float32, device=DEV)
        y_out = torch.empty_like(out_f)
        stacks = {"x": stack, "mask": mstack, "y": stack, "bg": stack}
        aug.augment_indexed(stacks, _dev(rows[sel]), _dev(rows[sel_bg]), _dev(geom_t), _dev(lut), out_f, y_out,
                            torch.cuda.current_stream(DEV))
        assert np.array_equal(out_f.cpu().numpy(), (want / 255.).astype(np.float32))
        assert np.array_equal(y_out.cpu().numpy(), _y_target(x[sel]))
    finally:
        del stack, mstack
        gc.collect()
        torch.cuda.empty_cache()


def test_occlusion_reads_stack_rows_past_2_and_4_gib(tmp_path):
    """A 262 200-row 128 x 128 mask stack (4.30 GB): row 131 072 starts at 2^31 bytes, row 262 144 at 2^32."""
    _skip_unless_free()
    h, n = 128, 262200
    rows = np.array([131071, 131072, 262143, 262144, 262199], np.int32)
    assert int(rows[1]) * h * h == 2 ** 31 and int(rows[3]) * h * h == 2 ** 32
    rng = np.random.RandomState(29)
    _, words, bank = _bank(tmp_path, rng)
    m = _objects(rng, len(rows), h, h)
    mstack = torch.empty((n, h, h), dtype=torch.uint8, device=DEV)
    try:
        for i, r in enumerate(rows):
            mstack[int(r)].copy_(torch.from_numpy(m[i].astype(np.uint8)))
        B = 10
        sel = np.resize(np.arange(len(rows)), B)
        occl = A.Occlusion((h, h), 0.4, 0.2, seed=8)
        P = occl.sample(B, len(words))
        out = torch.empty((B, h, h), dtype=torch.uint8, device=DEV)
        occl.apply_indexed(mstack, _dev(rows[sel]), _dev(occl.pack(P)), words, out, torch.cuda.current_stream(DEV))
        got, fb = out.cpu().numpy().astype(bool), occl.fallbacks()
        want, wfb = OO.occlude(m[sel], bank, P, 0.4, 0.2)
        assert np.array_equal(got, want) and fb == wfb
        assert (got != m[sel]).any()                              # the steps changed something
    finally:
        del mstack
        gc.collect()
        torch.cuda.empty_cache()


# ---- crops at the px64 patch size ---------------------------------------------------------------------------------------------------
def test_square_patches_at_the_px64_patch_size():
    """aae_extract_square_patches at out_size 64, the patch size process() passes for a 64 x 64 model, against the plugin's
    extract_square_patch + cv2.resize(INTER_LINEAR) on the random boxes of the 128 test.  A 128 px square at pad factor 1.0 is
    an exact 2x reduction, which cv2 runs through its INTER_AREA path."""
    import cv2
    from augmentedautoencoder_b200.m3_interface.ae_pose_estimator import AePoseEstimator
    scene = np.random.RandomState(7).randint(0, 256, (480, 640, 3), dtype=np.uint8)
    est = AePoseEstimator.__new__(AePoseEstimator)
    frame = torch.from_numpy(scene).to(DEV)
    rng = np.random.RandomState(3)
    boxes = []
    for _ in range(200):
        w, h = rng.randint(8, 400), rng.randint(8, 400)
        x, y = rng.randint(0, 640 - min(w, 639)), rng.randint(0, 480 - min(h, 479))
        w, h = min(w, 640 - x), min(h, 480 - y)
        boxes.append([x + rng.rand() * 0.9, y + rng.rand() * 0.9, w + rng.rand() * 0.9, h + rng.rand() * 0.9])
    boxes += [[0, 0, 640, 480], [0, 0, 1, 1], [639, 479, 1, 1], [100, 100, 128, 128], [10, 20, 256, 256], [5, 7, 64, 64]]
    for pf in (1.2, 1.0, 1.37):
        got = est.extract_square_patches_device(frame, boxes, pf, (64, 64)).cpu().numpy()
        assert got.shape == (len(boxes), 64, 64, 3)
        for b, g_ in zip(boxes, got):
            want = est.extract_square_patch(scene, b, pf, resize=(64, 64), interpolation=cv2.INTER_LINEAR, black_borders=True)
            assert np.array_equal(g_, want), (b, pf, int((g_ != want).sum()))
