"""The slice of auto_pose/ae/dataset.py the hot path touches: crop shape, the idx -> rotation table
(``viewsphere_for_embedding``, dataset.py:39-58, built on pysixd_stuff/view_sampler.py:19-188), ``embedding_size``
and the square-patch crop helper (dataset.py:354-373).  Rendering / augmentation (OpenGL, imgaug) are out of scope
(SURVEY.md section 2 rows 7, 11): ``render_embedding_image_batch`` delegates to a user-supplied renderer."""
import glob
import hashlib
import math
import os

import numpy as np

from .utils import lazy_property

_GOLDEN = (1.0 + math.sqrt(5.0)) / 2.0
_ICO_VERTS = [(-1.0, _GOLDEN, 0.0), (1.0, _GOLDEN, 0.0), (-1.0, -_GOLDEN, 0.0), (1.0, -_GOLDEN, 0.0),
              (0.0, -1.0, _GOLDEN), (0.0, 1.0, _GOLDEN), (0.0, -1.0, -_GOLDEN), (0.0, 1.0, -_GOLDEN),
              (_GOLDEN, 0.0, -1.0), (_GOLDEN, 0.0, 1.0), (-_GOLDEN, 0.0, -1.0), (-_GOLDEN, 0.0, 1.0)]
_ICO_FACES = [(0, 11, 5), (0, 5, 1), (0, 1, 7), (0, 7, 10), (0, 10, 11), (1, 5, 9), (5, 11, 4), (11, 10, 2), (10, 7, 6),
              (7, 1, 8), (3, 9, 4), (3, 4, 2), (3, 2, 6), (3, 6, 8), (3, 8, 9), (4, 9, 5), (2, 4, 11), (6, 2, 10),
              (8, 6, 7), (9, 8, 1)]


def icosphere_points(min_n_pts, radius=1.0):
    """Hinterstoisser view sphere: subdivide an icosahedron until it has >= min_n_pts vertices, push the vertices
    to the sphere and order them ring by ring from the top pole, each ring sorted by azimuth.  The vertex numbering,
    midpoint arithmetic and ring construction reproduce view_sampler.hinter_sampling exactly (checked bit-for-bit
    against tests/golden/viewsphere_*.npz)."""
    verts = [list(v) for v in _ICO_VERTS]
    faces = list(_ICO_FACES)
    while len(verts) < min_n_pts:
        midpoint = {}
        refined = []
        for tri in faces:
            mids = []
            for a, b in ((tri[0], tri[1]), (tri[1], tri[2]), (tri[2], tri[0])):
                key = (a, b) if a < b else (b, a)
                if key not in midpoint:
                    midpoint[key] = len(verts)
                    verts.append((0.5 * (np.array(verts[key[0]]) + np.array(verts[key[1]]))).tolist())
                mids.append(midpoint[key])
            v0, v1, v2 = tri
            m01, m12, m20 = mids
            refined += [(v0, m01, m20), (m01, v1, m12), (m01, m12, m20), (m20, m12, v2)]
        faces = refined
    pts = np.array(verts)
    pts *= np.reshape(radius / np.linalg.norm(pts, axis=1), (pts.shape[0], 1))
    neighbours = {}
    for tri in faces:
        for i in range(3):
            neighbours.setdefault(tri[i], set()).update((tri[(i + 1) % 3], tri[(i + 2) % 3]))
    two_pi = 2.0 * math.pi
    azimuth = [(math.atan2(p[1], p[0]) + two_pi) % two_pi for p in pts]
    visited = [False] * len(pts)
    ring = [int(np.argmax(pts[:, 2]))]
    order = []
    while len(order) != len(pts):
        ring = sorted(ring, key=azimuth.__getitem__)
        reach = []
        for v in ring:
            order.append(v)
            visited[v] = True
            reach += [i for i in neighbours[v]]
        ring = [i for i in set(reach) if not visited[i]]  # set iteration order decides azimuth ties, as upstream
    return pts[np.array(order), :]


def look_at_rotations(pts):
    """Camera rotation for every view point: the camera looks at the origin with world +z up (OpenGL look-at), then a
    180 degree flip about x converts to the OpenCV convention (view_sampler.sample_views, view_sampler.py:160-181)."""
    c, s = math.cos(math.pi), math.sin(math.pi)
    flip = np.array([[1.0, 0.0, 0.0], [0.0, c, -s], [0.0, s, c]])
    up = np.array([0.0, 0.0, 1.0])
    out = np.empty((len(pts), 3, 3))
    for i, pt in enumerate(pts):
        fwd = -np.array(pt)
        fwd /= np.linalg.norm(fwd)
        side = np.cross(fwd, up)
        if np.count_nonzero(side) == 0:
            side = np.array([1.0, 0.0, 0.0])
        side /= np.linalg.norm(side)
        upv = np.cross(side, fwd)
        out[i] = flip.dot(np.array([[side[0], side[1], side[2]], [upv[0], upv[1], upv[2]], [-fwd[0], -fwd[1], -fwd[2]]]))
    return out


def viewsphere_rotations(min_n_views, num_cyclo, radius):
    views = look_at_rotations(icosphere_points(min_n_views, radius=radius))
    rs = np.empty((len(views) * num_cyclo, 3, 3))
    angles = np.linspace(0, 2.0 * np.pi, num_cyclo)  # both end points included -> first and last in-plane step coincide
    i = 0
    for view in views:
        for cyclo in angles:
            rot_z = np.array([[np.cos(-cyclo), -np.sin(-cyclo), 0], [np.sin(-cyclo), np.cos(-cyclo), 0], [0, 0, 1]])
            rs[i] = rot_z.dot(view)
            i += 1
    return rs


class Dataset(object):
    """Constructor signature of auto_pose/ae/dataset.py:16-36 (``Dataset(dataset_path, **kw)`` with the lower-cased
    cfg keys).  Only what the encoder / codebook path needs is kept."""

    def __init__(self, dataset_path=None, renderer=None, **kw):
        self.shape = (int(kw.get("h", 128)), int(kw.get("w", 128)), int(kw.get("c", 3)))
        self.dataset_path = dataset_path
        self._kw = dict(kw)
        self._kw.setdefault("num_cyclo", 36)
        self._kw.setdefault("min_n_views", 2562)
        self._kw.setdefault("radius", 700)
        self._renderer = renderer

    @lazy_property
    def viewsphere_for_embedding(self):
        kw = self._kw
        return viewsphere_rotations(int(kw["min_n_views"]), int(kw["num_cyclo"]), float(kw["radius"]))

    @property
    def embedding_size(self):
        return len(self.viewsphere_for_embedding)

    def render_embedding_image_batch(self, start, end):
        """(batch [n,H,W,C] float in [0,1], obj_bbs [n,4]) for codebook rows start..end (dataset.py:308-352).  Needs a
        renderer callable ``renderer(R) -> (bgr uint8 image, depth)``; OpenGL rendering is out of scope here."""
        if self._renderer is None:
            raise NotImplementedError("no renderer attached: pass renderer=callable(R)->(bgr, depth) to Dataset, or "
                                      "build the codebook with Codebook.update_embedding_from_crops")
        import cv2
        kw = self._kw
        h, w = self.shape[:2]
        pad_factor = float(kw.get("pad_factor", 1.2))
        batch = np.empty((end - start,) + self.shape)
        obj_bbs = np.empty((end - start, 4))
        for i, R in enumerate(self.viewsphere_for_embedding[start:end]):
            bgr, depth = self._renderer(R)
            ys, xs = np.nonzero(depth > 0)
            size = (depth.shape[1], depth.shape[0])
            x0, y0 = max(xs.min() - 1, 0), max(ys.min() - 1, 0)
            x1, y1 = min(xs.max() + 1, size[0] - 1), min(ys.max() + 1, size[1] - 1)
            obj_bbs[i] = [x0, y0, x1 - x0, y1 - y0]
            crop = self.extract_square_patch(bgr, obj_bbs[i], pad_factor, resize=(w, h), interpolation=cv2.INTER_NEAREST)
            batch[i] = crop / 255.
        return batch, obj_bbs

    def extract_square_patch(self, scene_img, bb_xywh, pad_factor, resize=(128, 128), interpolation=None, black_borders=False):
        """Square crop around a bbox, clipped to the image, optional blackening outside the bbox (dataset.py:354-373)."""
        import cv2
        if interpolation is None:
            interpolation = cv2.INTER_NEAREST
        x, y, w, h = np.array(bb_xywh).astype(np.int32)
        size = int(np.maximum(h, w) * pad_factor)
        left = int(np.maximum(x + w / 2 - size / 2, 0))
        right = int(np.minimum(x + w / 2 + size / 2, scene_img.shape[1]))
        top = int(np.maximum(y + h / 2 - size / 2, 0))
        bottom = int(np.minimum(y + h / 2 + size / 2, scene_img.shape[0]))
        crop = scene_img[top:bottom, left:right].copy()
        if black_borders:
            crop[:(y - top), :] = 0
            crop[(y + h - top):, :] = 0
            crop[:, :(x - left)] = 0
            crop[:, (x + w - left):] = 0
        return cv2.resize(crop, resize, interpolation=interpolation)

    # ------------------------------------------------------------------------------------------------ training batches
    def load_training_images(self, path, bg_path=None, device=None):
        """The cache the reference writes after rendering (``np.savez(current_file_name, train_x=, mask_x=, train_y=)``,
        dataset.py:101-113) and, optionally, the background image stack (``.npy``, dataset.py:229-255).  With ``device`` the
        stacks are also uploaded once and kept there (``upload``) for ``batch_resident`` and the started ``Queue``; the host
        arrays stay as they are either way."""
        data = np.load(path)
        self.train_x, self.mask_x, self.train_y = data["train_x"].astype(np.uint8), data["mask_x"], data["train_y"].astype(np.uint8)
        self.noof_training_imgs = len(self.train_x)
        if bg_path is not None:
            self.bg_imgs = np.load(bg_path).astype(np.uint8)
            self.noof_bg_imgs = len(self.bg_imgs)
        if device is not None:
            self.upload(device)

    def training_images_path(self, dataset_path, args):
        """Where the reference caches the rendered training set of a cfg: md5 of ``str(args.items('Dataset') +
        args.items('Paths'))`` (dataset.py:91-92), so a cache the reference rendered is found under the same name."""
        digest = hashlib.md5((str(args.items('Dataset') + args.items('Paths'))).encode('utf-8')).hexdigest()
        return os.path.join(dataset_path, digest + '.npz')

    def get_training_images(self, dataset_path, args, device=None):
        """dataset.py:90-103 without rendering: loads the cache of ``training_images_path``; a missing cache raises and names it."""
        path = self.training_images_path(dataset_path, args)
        if not os.path.exists(path):
            raise FileNotFoundError("no training-image cache for this cfg: %s (rendering the training set is not part of this "
                                    "package; render it with the reference's ae_train -gen and copy the .npz there)" % path)
        self.load_training_images(path)
        self.noof_obj_pixels = np.count_nonzero(np.asarray(self.mask_x) == 0, axis=(1, 2))
        if device is not None:
            self.upload(device, which=("x", "mask", "y"))
        return path

    def bg_images_path(self, dataset_path):
        """Where the reference caches the background stack (dataset.py:146-147): md5 of ``str(shape) + str(noof_bg_imgs) +
        BACKGROUND_IMAGES_GLOB``, noof_bg_imgs = min(NOOF_BG_IMGS, files the glob matches) (dataset.py:24-25)."""
        pattern = str(self._kw['background_images_glob'])
        n = min(int(self._kw['noof_bg_imgs']), len(glob.glob(pattern)))
        digest = hashlib.md5((str(self.shape) + str(n) + pattern).encode('utf-8')).hexdigest()
        return os.path.join(dataset_path, digest + '.npy')

    def load_bg_images(self, dataset_path, device=None):
        """The background stack of dataset.py:145-170: the cache of ``bg_images_path``, or, when it is missing, built from
        BACKGROUND_IMAGES_GLOB with the reference's rule and saved there: the first noof_bg_imgs files in a shuffled order, each
        cropped to H x W at a random anchor (grey for C = 1).  An image smaller than the crop leaves its row zero (the
        reference leaves it uninitialised).  With ``device`` the stack is also kept on the device (``upload``)."""
        path = self.bg_images_path(dataset_path)
        if os.path.exists(path):
            self.bg_imgs = np.load(path).astype(np.uint8)
        else:
            import random
            import cv2
            h, w, c = self.shape
            files = glob.glob(str(self._kw['background_images_glob']))
            n = min(int(self._kw['noof_bg_imgs']), len(files))
            if n == 0:
                raise FileNotFoundError("no background images match BACKGROUND_IMAGES_GLOB %s (and no cache at %s)"
                                        % (self._kw['background_images_glob'], path))
            files = files[:n]
            random.shuffle(files)
            bg = np.zeros((n, h, w, c), np.uint8)
            for j, fname in enumerate(files):
                bgr = cv2.imread(fname)
                if bgr is None:
                    raise IOError("cannot read background image %s" % fname)
                H, W = bgr.shape[:2]
                y0 = int(np.random.rand() * (H - h))
                x0 = int(np.random.rand() * (W - w))
                bgr = bgr[y0:y0 + h, x0:x0 + w, :]
                if bgr.shape[0] != h or bgr.shape[1] != w:
                    continue
                if c == 1:
                    bgr = cv2.cvtColor(np.uint8(bgr), cv2.COLOR_BGR2GRAY)[:, :, np.newaxis]
                bg[j] = bgr
            os.makedirs(os.path.dirname(path), exist_ok=True)
            np.save(path, bg)
            self.bg_imgs = bg
        self.noof_bg_imgs = len(self.bg_imgs)
        if device is not None:
            self.upload(device, which=("bg",))
        return path

    # -- the training set resident on the device --------------------------------------------------------------------
    def upload(self, device, which=("x", "mask", "y", "bg")):
        """Keeps train_x, mask_x (as uint8), train_y and bg_imgs on ``device``, uploaded once: N H W (2C + 1) + N_bg H W C bytes.
        ``batch_resident`` and the started ``Queue`` read batches from there through index arrays instead of gathering them."""
        import torch
        dev = torch.device(device) if not isinstance(device, torch.device) else device
        if dev.index is None:
            dev = torch.device("cuda", torch.cuda.current_device())
        sources = {"x": "train_x", "mask": "mask_x", "y": "train_y", "bg": "bg_imgs"}
        res = self.__dict__.setdefault("_resident", {})
        for key in which:
            arr = getattr(self, sources[key], None)
            if arr is None:
                raise RuntimeError("Dataset.%s is not loaded (load_training_images / load_bg_images)" % sources[key])
            host = np.ascontiguousarray(np.asarray(arr).astype(np.uint8, copy=False))
            res[key] = (arr, torch.from_numpy(host).to(dev))
        return dev

    def resident(self, device):
        """{"x", "mask", "y", "bg"} -> the device stacks of ``upload`` on ``device``; RuntimeError naming what is missing or stale
        (a host array replaced after the upload)."""
        res = self.__dict__.get("_resident", {})
        sources = {"x": "train_x", "mask": "mask_x", "y": "train_y", "bg": "bg_imgs"}
        out = {}
        for key, name in sources.items():
            if key not in res or res[key][0] is not getattr(self, name, None) or res[key][1].device != device:
                raise RuntimeError("Dataset.%s is not resident on %s: call upload(device) (or load_*(..., device=))" % (name, device))
            out[key] = res[key][1]
        return out

    @lazy_property
    def _aug(self):
        from .augment import Augmenter
        code = self._kw.get("code")
        if code is None:
            raise NotImplementedError("no [Augmentation] CODE in the dataset arguments")
        return Augmenter(code, self.shape, seed=self._kw.get("seed"))

    @lazy_property
    def _occlusion(self):
        """The [Augmentation] switches REALISTIC_OCCLUSION / SQUARE_OCCLUSION (dataset.py:468-471); None when both are off."""
        from .augment import Occlusion, occlusion_limit
        realistic = occlusion_limit(self._kw.get("realistic_occlusion"))
        square = occlusion_limit(self._kw.get("square_occlusion"))
        if not realistic and not square:
            return None
        return Occlusion(self.shape, realistic, square, seed=self._kw.get("seed"))

    def load_occlusion_masks(self, path=None):
        """The occluder bank of REALISTIC_OCCLUSION (``random_syn_masks``, dataset.py:405-418), kept bit-packed (2 KB per
        128 x 128 mask).  Default path: $AE_WORKSPACE_PATH/random_tless_masks/arbitrary_syn_masks_1000.bin, as the reference."""
        from .augment import load_occlusion_bank
        if path is None:
            ws = os.environ.get("AE_WORKSPACE_PATH")
            if not ws:
                raise RuntimeError("REALISTIC_OCCLUSION needs the occluder bank: set AE_WORKSPACE_PATH or call load_occlusion_masks(path)")
            path = os.path.join(ws, "random_tless_masks", "arbitrary_syn_masks_1000.bin")
        self.occlusion_masks = load_occlusion_bank(path, self.shape)
        return len(self.occlusion_masks)

    def occlusion_fallbacks(self):
        """Images that kept their mask because all their occlusion candidates failed, since the last call: {"realistic": n,
        "square": n}.  The reference re-draws without bound instead (and never returns for an image without object pixels or
        whose realistic occlusion already took more than SQUARE_OCCLUSION of it).  Clears the counts; synchronises."""
        occl = self._occlusion
        return occl.fallbacks() if occl is not None else {"realistic": 0, "square": 0}

    def batch_device(self, batch_size, device=None):
        """Dataset.batch (dataset.py:456-495) with the image work on the GPU: draws the rendering / background indices like the
        reference, uploads the uint8 images once and returns (x, y) float32 CUDA tensors in [0, 1].  With REALISTIC_OCCLUSION or
        SQUARE_OCCLUSION set, the masks are occluded on the device before the paste (see ``occlusion_fallbacks``)."""
        import torch
        for name in ("train_x", "mask_x", "train_y", "bg_imgs"):
            if not hasattr(self, name):
                raise RuntimeError("Dataset.%s is not loaded (load_training_images / set the arrays)" % name)
        occl = self._occlusion
        if occl is not None and occl.realistic and getattr(self, "occlusion_masks", None) is None:
            self.load_occlusion_masks()
        dev = torch.device("cuda", torch.cuda.current_device()) if device is None else device
        idx = np.random.choice(len(self.train_x), batch_size, replace=False)
        idx_bg = np.random.choice(len(self.bg_imgs), batch_size, replace=False)
        x = torch.from_numpy(self.train_x[idx]).to(dev, non_blocking=True)
        m = torch.from_numpy(np.ascontiguousarray(self.mask_x[idx]).astype(np.uint8)).to(dev, non_blocking=True)
        bg = torch.from_numpy(self.bg_imgs[idx_bg]).to(dev, non_blocking=True)
        y = torch.from_numpy(self.train_y[idx]).to(dev, non_blocking=True)
        if occl is not None:
            m = occl.apply_device(m, getattr(self, "occlusion_masks", None))
        xf = self._aug.augment_device(x, m, bg)
        return xf, y.to(torch.float32) / 255.0

    def _draws(self, batch_size):
        """The random draws of one batch in ``batch_device``'s order and from its generators: rendering and background indices
        (numpy's global stream), occlusion candidates (the Occlusion's own stream), augmentation parameters (the Augmenter's);
        then the packed tables: (idx, idx_bg, cand or None, geom, lut, crop or None -- the CropAndPad table)."""
        occl = self._occlusion
        if occl is not None and occl.realistic and getattr(self, "occlusion_masks", None) is None:
            self.load_occlusion_masks()
        idx = np.random.choice(len(self.train_x), batch_size, replace=False)
        idx_bg = np.random.choice(len(self.bg_imgs), batch_size, replace=False)
        cand = None
        if occl is not None:
            bank = getattr(self, "occlusion_masks", None)
            cand = occl.pack(occl.sample(batch_size, len(bank) if bank is not None else 0))
        aug = self._aug                 # built here on first use, as in batch_device: CODE may draw from numpy's stream
        P = aug.sample(batch_size)
        geom, lut = aug.pack(P)
        return idx, idx_bg, cand, geom, lut, aug.pack_crop(P)

    def _chain_has_crop_pad(self):
        """Whether [Augmentation] CODE has CropAndPad, without building the Augmenter: the first batch's draws build it (CODE
        may draw from numpy's global stream there), so the stream is left as it was."""
        if "_cache__aug" in self.__dict__:
            return self._aug.crop is not None
        if self._kw.get("code") is None:
            return False
        from .augment import parse_code
        state = np.random.get_state()
        try:
            return any(op.kind == "CropAndPad" for _, op in parse_code(self._kw["code"]))
        finally:
            np.random.set_state(state)

    def _resident_scratch(self, batch_size, device):
        """Device buffers of one batch of ``_enqueue_resident``: the uploaded draws, the augment scratch and the occluded masks.
        The batch producer keeps one set per slot, so its loop allocates no device memory."""
        import torch
        B = int(batch_size)
        (h, w, c), occl = self.shape, self._occlusion
        n_cand = B * (1 + 3 * occl.K) if occl is not None else 0
        crop = self._chain_has_crop_pad()
        return {"draws": torch.empty(2 * B + B * (4 + 2 * w + 2 * h) + n_cand + (8 * B if crop else 0), dtype=torch.int32, device=device),
                "lut": torch.empty(B * c * 256, dtype=torch.uint8, device=device),
                "tmp": torch.empty((B, h, w, c), dtype=torch.uint8, device=device),
                "mask": torch.empty((B, h, w), dtype=torch.uint8, device=device) if occl is not None else None,
                "crop": torch.empty((B, h, w, c), dtype=torch.uint8, device=device) if crop else None}

    def _enqueue_resident(self, stacks, draws, x_out, y_out, stream, scratch=None):
        """One batch from the resident stacks into x_out / y_out (float32 [B,H,W,C]) on ``stream``: the draws go up from pinned
        staging (torch's caching host allocator keeps a block until its copy has run), then the indexed occlusion and augment
        kernels.  ``scratch`` (``_resident_scratch``, ordered by the caller) replaces the device buffers allocated here.  Nothing
        waits for the device."""
        import torch
        idx, idx_bg, cand, geom, lut, crop = draws
        B = len(idx)
        dev = x_out.device
        n_cand = cand.size if cand is not None else 0
        n_crop = crop.size if crop is not None else 0
        if scratch is None:
            with torch.cuda.stream(stream):
                scratch = self._resident_scratch(B, dev)
        with torch.cuda.stream(stream):
            host = torch.empty(2 * B + geom.size + n_cand + n_crop, dtype=torch.int32, pin_memory=True)
            h = host.numpy()
            h[:B], h[B:2 * B], h[2 * B:2 * B + geom.size] = idx, idx_bg, geom.ravel()
            if cand is not None:
                h[2 * B + geom.size:2 * B + geom.size + n_cand] = cand.ravel()
            if crop is not None:
                h[2 * B + geom.size + n_cand:] = crop.ravel()
            host_lut = torch.empty(lut.size, dtype=torch.uint8, pin_memory=True)
            host_lut.numpy()[:] = lut.ravel()
            d = scratch["draws"][:host.numel()]
            d.copy_(host, non_blocking=True)
            lut_d = scratch["lut"]
            lut_d.copy_(host_lut, non_blocking=True)
            idx_d, idx_bg_d, geom_d = d[:B], d[B:2 * B], d[2 * B:2 * B + geom.size]
            mask = None
            if cand is not None:
                mask = scratch["mask"]
                self._occlusion.apply_indexed(stacks["mask"], idx_d, d[2 * B + geom.size:2 * B + geom.size + n_cand],
                                              getattr(self, "occlusion_masks", None), mask, stream)
            crop_d = d[2 * B + geom.size + n_cand:] if crop is not None else None
            self._aug.augment_indexed(stacks, idx_d, idx_bg_d, geom_d, lut_d, x_out, y_out, stream, mask_batch=mask,
                                      tmp=scratch["tmp"], crop_d=crop_d, crop_tmp=scratch["crop"])

    def batch_resident(self, batch_size, device=None):
        """``batch_device`` on the stacks kept on the device by ``upload``: the same draws in the same order, so the same
        (x, y), bit for bit, and the same occlusion fallback counts; only the draws (indices and packed tables, ~0.2 MB at
        batch 64) are uploaded, and the target y / 255. comes out of the same launch.  Asynchronous on the current stream."""
        import torch
        dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        stacks = self.resident(dev)
        draws = self._draws(batch_size)
        x = torch.empty((batch_size,) + self.shape, dtype=torch.float32, device=dev)
        y = torch.empty_like(x)
        self._enqueue_resident(stacks, draws, x, y, torch.cuda.current_stream(dev))
        return x, y

    def batch(self, batch_size):
        """numpy (batch_x, batch_y) like the reference's ``Dataset.batch``."""
        x, y = self.batch_device(batch_size)
        return x.cpu().numpy(), y.cpu().numpy()
