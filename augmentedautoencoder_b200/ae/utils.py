"""Workspace path conventions and helpers mirroring auto_pose/ae/utils.py:6-90 (same names, same results)."""
import functools
import os

import numpy as np


def lazy_property(function):
    attribute = "_cache_" + function.__name__

    @property
    @functools.wraps(function)
    def decorator(self):
        if not hasattr(self, attribute):
            setattr(self, attribute, function(self))
        return getattr(self, attribute)

    return decorator


def batch_iteration_indices(N, batch_size):
    """(start, end) pairs covering range(N) -- auto_pose/ae/utils.py:19-25."""
    for a in range(0, int(N), int(batch_size)):
        yield (a, min(a + int(batch_size), int(N)))


def get_dataset_path(workspace_path):
    return os.path.join(workspace_path, "tmp_datasets")


def get_checkpoint_dir(log_dir):
    return os.path.join(log_dir, "checkpoints")


def get_log_dir(workspace_path, experiment_name, experiment_group=""):
    return os.path.join(workspace_path, "experiments", experiment_group, experiment_name)


def get_train_fig_dir(log_dir):
    return os.path.join(log_dir, "train_figures")


def get_train_config_exp_file_path(log_dir, experiment_name):
    return os.path.join(log_dir, "{}.cfg".format(experiment_name))


def get_checkpoint_basefilename(log_dir):
    return os.path.join(log_dir, "checkpoints", "chkpt")


def get_config_file_path(workspace_path, experiment_name, experiment_group=""):
    return os.path.join(workspace_path, "cfg", experiment_group, "{}.cfg".format(experiment_name))


def get_eval_config_file_path(workspace_path, eval_cfg="eval.cfg"):
    return os.path.join(workspace_path, "cfg_eval", eval_cfg)


def get_eval_dir(log_dir, evaluation_name, data):
    return os.path.join(log_dir, "eval", evaluation_name, data)


def tiles(batch, rows, cols, spacing_x=0, spacing_y=0, scale=1.0):
    """One image of the first rows * cols images of ``batch`` ([N, H, W, C] or [N, H, W]) laid out row by row, each resized to
    (H * scale, W * scale) with cv2.resize, ``spacing_x`` / ``spacing_y`` pixels apart; cells without an image and the spacing
    are 1.  Always [rows * h + (rows - 1) * spacing_y, cols * w + (cols - 1) * spacing_x, C] float64 (auto_pose/ae/utils.py:93)."""
    import cv2
    batch = np.asarray(batch)
    if batch.ndim not in (3, 4):
        raise ValueError("Invalid batch shape: {}".format(batch.shape))
    n, h, w = batch.shape[:3]
    c = batch.shape[3] if batch.ndim == 4 else 1
    h, w = int(h * scale), int(w * scale)
    out = np.ones((rows * h + (rows - 1) * spacing_y, cols * w + (cols - 1) * spacing_x, c))
    for i in range(min(n, rows * cols)):
        r, q = divmod(i, cols)
        y0, x0 = r * (h + spacing_y), q * (w + spacing_x)
        img = cv2.resize(batch[i], (w, h))
        out[y0:y0 + h, x0:x0 + w, :] = img if img.ndim == 3 else img[:, :, None]
    return out
