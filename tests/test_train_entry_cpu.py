"""CPU tests of ae_train's host side: the reference's cache file names, the errors for a missing cfg / cache / unsupported flag,
and utils.tiles."""
import configparser
import hashlib
import os
import shutil

import cv2
import numpy as np
import pytest

from augmentedautoencoder_b200.ae import ae_factory as factory
from augmentedautoencoder_b200.ae import ae_train
from augmentedautoencoder_b200.ae import utils as u


def _template(golden_dir):
    args = configparser.ConfigParser()
    args.read(os.path.join(golden_dir, "train_template.cfg"))
    return args


def test_cache_names_are_the_reference_hashes_of_the_template(golden_dir, tmp_path):
    args = _template(golden_dir)
    ds = factory.build_dataset(str(tmp_path), args)
    # dataset.py:91-92, the expression as the reference writes it, and its value for the template
    want = hashlib.md5((str(args.items('Dataset') + args.items('Paths'))).encode('utf-8')).hexdigest()
    assert want == "bd4bcd90d31d24f2e52c504a2288537f"
    assert ds.training_images_path(str(tmp_path), args) == os.path.join(str(tmp_path), want + ".npz")
    # dataset.py:146-147 with noof_bg_imgs = min(NOOF_BG_IMGS, files matched): the template's glob matches nothing here
    want_bg = hashlib.md5((str((128, 128, 3)) + str(0) + "/path/to/VOCdevkit/VOC2012/JPEGImages/*.jpg").encode('utf-8')).hexdigest()
    assert want_bg == "7667d9b5b8c4b34c19d081aca26eb5d6"
    assert ds.bg_images_path(str(tmp_path)) == os.path.join(str(tmp_path), want_bg + ".npy")
    # with files: the count is min(NOOF_BG_IMGS, matches)
    for i in range(3):
        cv2.imwrite(str(tmp_path / ("bg%d.jpg" % i)), np.zeros((8, 8, 3), np.uint8))
    args.set("Paths", "BACKGROUND_IMAGES_GLOB", str(tmp_path / "*.jpg"))
    ds = factory.build_dataset(str(tmp_path), args)
    want_bg = hashlib.md5((str((128, 128, 3)) + str(3) + str(tmp_path / "*.jpg")).encode('utf-8')).hexdigest()
    assert ds.bg_images_path(str(tmp_path)) == os.path.join(str(tmp_path), want_bg + ".npy")


def _workspace(golden_dir, tmp_path, monkeypatch):
    ws = tmp_path / "ws"
    (ws / "cfg" / "grp").mkdir(parents=True)
    shutil.copy(os.path.join(golden_dir, "train_template.cfg"), ws / "cfg" / "grp" / "exp.cfg")
    monkeypatch.setenv("AE_WORKSPACE_PATH", str(ws))
    return ws


def test_missing_cfg_and_missing_cache_name_their_paths(golden_dir, tmp_path, monkeypatch):
    ws = _workspace(golden_dir, tmp_path, monkeypatch)
    with pytest.raises(FileNotFoundError) as e:
        ae_train.prepare(["grp/nope"])
    assert str(ws / "cfg" / "grp" / "nope.cfg") in str(e.value)
    with pytest.raises(FileNotFoundError) as e:
        ae_train.prepare(["grp/exp"])
    want = os.path.join(str(ws), "tmp_datasets", "bd4bcd90d31d24f2e52c504a2288537f.npz")
    assert want in str(e.value)
    assert not (ws / "experiments").exists()             # nothing is written before the inputs are found
    monkeypatch.delenv("AE_WORKSPACE_PATH")
    with pytest.raises(EnvironmentError, match="AE_WORKSPACE_PATH"):
        ae_train.prepare(["grp/exp"])


def test_unsupported_flags_raise_with_a_reason(golden_dir, tmp_path, monkeypatch):
    _workspace(golden_dir, tmp_path, monkeypatch)
    with pytest.raises(NotImplementedError, match="-gen"):
        ae_train.prepare(["grp/exp", "-gen"])
    with pytest.raises(NotImplementedError, match="-d"):
        ae_train.prepare(["grp/exp", "-d"])
    assert ae_train.split_name("grp/exp") == ("exp", "grp") and ae_train.split_name("exp") == ("exp", "")


def test_tiles_layout():
    rng = np.random.RandomState(0)
    b = rng.rand(5, 6, 4, 3)
    t = u.tiles(b, 2, 3)
    assert t.shape == (12, 12, 3)
    for i in range(5):
        r, c = divmod(i, 3)
        assert np.array_equal(t[r * 6:(r + 1) * 6, c * 4:(c + 1) * 4], b[i])
    assert (t[6:, 8:] == 1).all()                              # the sixth cell has no image
    t = u.tiles(b, 2, 2, spacing_x=2, spacing_y=1)
    assert t.shape == (13, 10, 3)
    assert (t[6, :] == 1).all() and (t[:, 4:6] == 1).all()     # spacing rows / columns
    assert np.array_equal(t[7:13, 6:10], b[3])
    g = rng.rand(4, 6, 4).astype(np.float32)                   # [N, H, W] -> one channel
    t = u.tiles(g, 2, 2)
    assert t.shape == (12, 8, 1) and np.array_equal(t[6:, 4:, 0], g[3])
    t = u.tiles(b[..., :1], 1, 2, scale=0.5)                   # [N, H, W, 1], scaled with cv2.resize
    assert t.shape == (3, 4, 1) and np.array_equal(t[:, 2:, 0], cv2.resize(b[1, :, :, 0], (2, 3)))
    with pytest.raises(ValueError):
        u.tiles(np.zeros((2, 3)), 1, 1)
