"""CPU restatement of the occlusion-mask augmentations of auto_pose/ae/dataset.py (REALISTIC_OCCLUSION: ``augment_occlusion_mask``,
dataset.py:421-444; SQUARE_OCCLUSION: ``augment_squares`` + ``_aug_occl``, dataset.py:392-402, 445-454), written after the
reference line by line with its random draws passed in explicitly.  TEST INFRASTRUCTURE ONLY -- imported by tests/.

Masks are True on BACKGROUND pixels, as ``mask_x`` of the reference.  The reference loops until a draw is accepted; here each
image gets a finite list of candidates in draw order, and an image whose candidates all fail keeps its mask (``fell_back``).

Pinning status:
* realistic   tests/golden/occlusion_realistic.npz holds masks, draws and results of the reference's own
              ``augment_occlusion_mask``; ``realistic_occlusion`` replays the recorded draws and must reproduce them bit for bit.
* square      imgaug (0.4.0 in the reference's environment) is not installable here, so the step stays a restatement:
              Sometimes(0.7) over CoarseDropout(p=0.4, size_percent=0.01) = a low-resolution Binomial(0.6) keep grid upsampled
              with cv2.resize(INTER_NEAREST) and multiplied into the object plane.  The grid size is the product's
              SQUARE_OCCLUSION_MIN_SIZE, unverified (see there).
"""
import numpy as np


def shift_zero_fill(mask, tx, ty):
    """cv2.warpAffine(mask, [[1, 0, tx], [0, 1, ty]], ...) for integer shifts: out[y, x] = mask[y - ty, x - tx], 0 outside."""
    h, w = mask.shape
    out = np.zeros_like(mask)
    ys, yd = max(-ty, 0), max(ty, 0)
    xs, xd = max(-tx, 0), max(tx, 0)
    nh, nw = h - abs(ty), w - abs(tx)
    if nh > 0 and nw > 0:
        out[yd:yd + nh, xd:xd + nw] = mask[ys:ys + nh, xs:xs + nw]
    return out


def realistic_occlusion(masks, occluders, tx, ty, max_occl, min_occl=0.0):
    """augment_occlusion_mask with the draws given: masks bool [B,H,W]; occluders float32 [B,H,W] (the bank entry drawn for
    each image, ``random_syn_masks[choice]``); tx, ty int [B, K] (``trans_x``, ``trans_y`` of each attempt).
    Returns (new masks, index of the accepted candidate per image, -1 = none)."""
    import cv2
    new_masks = np.array(masks, dtype=bool, copy=True)
    taken = np.full(len(masks), -1)
    for idx, mask in enumerate(masks):
        occl_mask = occluders[idx]
        obj = len(mask[mask == 0])
        for k in range(tx.shape[1]):
            M = np.float32([[1, 0, int(tx[idx, k])], [0, 1, int(ty[idx, k])]])
            transl_occl_mask = cv2.warpAffine(occl_mask, M, (occl_mask.shape[0], occl_mask.shape[1]))
            overlap_matrix = np.invert(mask.astype(bool)) * transl_occl_mask.astype(bool)
            if obj == 0:                 # the reference raises ZeroDivisionError here; no candidate can be accepted
                break
            overlap = len(overlap_matrix[overlap_matrix == True]) / float(obj)        # noqa: E712 (the reference's form)
            if overlap < max_occl and overlap > min_occl:
                new_masks[idx] = np.logical_xor(mask.astype(bool), overlap_matrix)
                taken[idx] = k
                break
    return new_masks, taken


def translations(sign_x, u_x, sign_y, u_y, h, w, min_trans=0.2, max_trans=0.7):
    """trans_x / trans_y of augment_occlusion_mask from its four draws per attempt (choice([-1, 1]), rand(), choice, rand)."""
    tx = np.array([int(s * (u * (max_trans - min_trans) + min_trans) * h) for s, u in zip(np.ravel(sign_x), np.ravel(u_x))])
    ty = np.array([int(s * (u * (max_trans - min_trans) + min_trans) * w) for s, u in zip(np.ravel(sign_y), np.ravel(u_y))])
    return tx.reshape(np.shape(sign_x)), ty.reshape(np.shape(sign_y))


def upsample_keep(keep, h, w):
    """CoarseDropout's low-resolution keep grid [rows, cols] (bool) -> [h, w] through cv2.resize(INTER_NEAREST)."""
    import cv2
    return cv2.resize(keep.astype(np.uint8), (w, h), interpolation=cv2.INTER_NEAREST).astype(bool)


def square_occlusion(masks, noof_obj_pixels, square_on, square_keep, max_occl):
    """augment_squares with the draws given: masks bool [B,H,W] (after the realistic step); noof_obj_pixels [B] of the
    unoccluded images; square_on bool [B, K] (the Sometimes draws); square_keep bool [B, K, rows, cols] (the dropout cells).
    Returns (new masks, index of the accepted candidate per image, -1 = none)."""
    B, h, w = masks.shape
    new_masks = np.invert(masks)
    taken = np.full(B, -1)
    denom = np.asarray(noof_obj_pixels).astype(np.float32)
    for idx in range(B):
        for k in range(square_on.shape[1]):
            obj = np.invert(masks[idx])
            if square_on[idx, k]:
                obj = obj & upsample_keep(square_keep[idx, k], h, w)
            with np.errstate(invalid="ignore", divide="ignore"):
                kept = np.count_nonzero(obj) / denom[idx]
            if not kept < 1 - max_occl:          # the reference re-draws the images with kept < 1 - max_occl
                new_masks[idx] = obj
                taken[idx] = k
                break
    return np.invert(new_masks), taken


def occlude(masks, bank_f32, P, realistic, square):
    """Both steps in the order of Dataset.batch (dataset.py:468-471) with the candidates of ``Occlusion.sample``.
    Returns (masks, fallbacks {"realistic": n, "square": n})."""
    masks = np.array(masks, dtype=bool)
    noof = np.count_nonzero(masks == 0, axis=(1, 2))          # dataset.py:94
    fb = {"realistic": 0, "square": 0}
    if realistic:
        masks, taken = realistic_occlusion(masks, bank_f32[P["occluder"]], P["tx"], P["ty"], realistic)
        fb["realistic"] = int((taken < 0).sum())
    if square:
        masks, taken = square_occlusion(masks, noof, P["square_on"], P["square_keep"], square)
        fb["square"] = int((taken < 0).sum())
    return masks, fb
