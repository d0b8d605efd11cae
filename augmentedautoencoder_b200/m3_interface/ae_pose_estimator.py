"""AePoseEstimator: the m3vision pose-estimation plugin.  Mirrors auto_pose/m3_interface/ae_pose_estimator.py:16-232
(constructor from a test-config path, attributes read by other tools, ``process`` signature and result type).

B200-first difference: the reference runs one B=1 ``session.run`` per detection (ae_pose_estimator.py:143-170); here all
detections of a frame that share an object class are cropped, stacked and sent through encoder + fused codebook match
in ONE batch per class, on the device that owns that class' (encoder, codebook) pair (multi-object routing, F14).
"""
import configparser
import ctypes as C
import os

import cv2
import numpy as np
import torch

from .. import _lib
from ..ae import factory, utils
from ..ae.codebook import lift_pose, lift_pose_batch
from ..ae.session import Session
from .m3_interfaces import PoseEstimate, PoseEstInterface


def square_patch_boxes(boxes_xywh, pad_factor):
    """int32 [n, 5] table of (x, y, w, h, size) per box, with the reference's own expressions (ae_pose_estimator.py:108-109):
    ``np.array(bb_xywh).astype(np.int32)`` on the float64 box and ``int(np.maximum(h, w) * pad_factor)``, a float64 product
    with the Python float ``pad_factor``.  Neither goes through float32: a box side such as 21.999999999999996 rounds up to
    22 in float32, and float32(1.3) is below 1.3.  Raises ValueError for a box whose square would be smaller than its
    longest side (a pad factor below 1), where the reference pastes outside its square."""
    b = np.asarray(boxes_xywh, dtype=np.float64).reshape(-1, 4).astype(np.int32)
    pad_factor = float(pad_factor)
    longest = np.maximum(b[:, 3], b[:, 2])
    size = (longest * pad_factor).astype(np.int64)          # int() of each float64 product: truncation toward zero
    bad = np.flatnonzero(size < longest)
    if len(bad):
        raise ValueError("pad factor %r makes a %d px square for the box %s (x, y, w, h = %s), smaller than its longest side"
                         % (pad_factor, size[bad[0]], np.asarray(boxes_xywh, dtype=np.float64).reshape(-1, 4)[bad[0]].tolist(),
                            b[bad[0]].tolist()))
    return np.ascontiguousarray(np.concatenate([b, size[:, None].astype(np.int32)], axis=1))


class AePoseEstimator(PoseEstInterface):

    def __init__(self, test_config_path, devices=None, precision=None):
        test_args = self.get_params(test_config_path)
        workspace_path = os.environ.get('AE_WORKSPACE_PATH')
        if workspace_path is None:
            raise EnvironmentError('Please define a workspace path: export AE_WORKSPACE_PATH=/path/to/workspace')
        self._process_requirements = ['color_img', 'camK', 'bboxes']
        if test_args.getboolean('auto_pose', 'camPose'):
            self._process_requirements.append('camPose')
        self._camPose = test_args.getboolean('auto_pose', 'camPose')
        self._upright = test_args.getboolean('auto_pose', 'upright')
        self._topk = test_args.getint('auto_pose', 'topk')
        if self._topk > 1:
            raise NotImplementedError('topk > 1 not implemented yet')  # reference: print + exit (ae_pose_estimator.py:37-39)
        self._image_format = {'color_format': test_args.get('auto_pose', 'color_format'),
                              'color_data_type': eval(test_args.get('auto_pose', 'color_data_type'), {"np": np}),
                              'depth_data_type': eval(test_args.get('auto_pose', 'depth_data_type'), {"np": np})}
        self.class_2_encoder = eval(test_args.get('auto_pose', 'class_2_encoder'))
        self.all_codebooks = {}
        self.all_train_args = {}
        self.pad_factors = {}
        self.patch_sizes = {}
        n_dev = torch.cuda.device_count()
        if devices is None:
            devices = list(range(max(n_dev, 1)))
        self.sess = Session(device=devices[0])
        self._sessions = {}
        self._class_streams = {}   # one CUDA stream per object class (process() overlaps the classes)
        for i, (clas_name, experiment) in enumerate(self.class_2_encoder.items()):
            full_name = experiment.split('/')
            experiment_name = full_name.pop()
            experiment_group = full_name.pop() if len(full_name) > 0 else ''
            log_dir = utils.get_log_dir(workspace_path, experiment_name, experiment_group)
            ckpt_dir = utils.get_checkpoint_dir(log_dir)
            train_cfg_file_path = utils.get_train_config_exp_file_path(log_dir, experiment_name)
            train_args = configparser.ConfigParser(inline_comment_prefixes="#")
            train_args.read(train_cfg_file_path)
            self.all_train_args[clas_name] = train_args
            self.pad_factors[clas_name] = train_args.getfloat('Dataset', 'PAD_FACTOR')
            self.patch_sizes[clas_name] = (train_args.getint('Dataset', 'W'), train_args.getint('Dataset', 'H'))
            cb = factory.build_codebook_from_name(experiment_name, experiment_group, return_dataset=False, precision=precision)
            self.all_codebooks[clas_name] = cb
            self._sessions[clas_name] = Session(device=devices[i % len(devices)])  # one object per GPU, round robin
            saver = factory.Saver([cb._encoder, cb])
            factory.restore_checkpoint(self._sessions[clas_name], saver, ckpt_dir)

    def set_parameter(self, string_name, string_val):
        pass

    def query_process_requirements(self):
        return self._process_requirements

    def query_image_format(self):
        return self._image_format

    def extract_square_patch(self, scene_img, bb_xywh, pad_factor, resize=(128, 128), interpolation=cv2.INTER_NEAREST, black_borders=False):
        """Square, zero-padded patch around a detection, bbox content centred (ae_pose_estimator.py:106-131; ``process``
        always uses black_borders=True).  The reference's other branch slices with float indices and cannot run."""
        x, y, w, h, size = (int(v) for v in square_patch_boxes(bb_xywh, pad_factor)[0])
        scene_crop = np.zeros((size, size, 3), dtype=np.uint8)
        if not black_borders:
            raise NotImplementedError("black_borders=False is broken upstream (float slice indices, ae_pose_estimator.py:118-127)")
        scene_crop[(size - h) // 2:(size - h) // 2 + h, (size - w) // 2:(size - w) // 2 + w] = scene_img[y:y + h, x:x + w].copy()
        return cv2.resize(scene_crop, resize, interpolation=interpolation)

    def extract_square_patches_device(self, frame_dev, boxes_xywh, pad_factor, patch_size):
        """All crops of a frame in one launch (aae_extract_square_patches): the same pixels as ``extract_square_patch(...,
        interpolation=cv2.INTER_LINEAR, black_borders=True)`` per box, bit for bit.  frame_dev: CUDA uint8 [H,W,3].  The
        box integers and square sizes are computed here (``square_patch_boxes``), the pixels on the device.  A box past the
        frame's right or bottom edge, which the reference refuses, is cropped from the frame padded with black."""
        if patch_size[0] != patch_size[1]:
            raise NotImplementedError("non-square patches")
        table = square_patch_boxes(boxes_xywh, pad_factor)
        n, ps = len(table), int(patch_size[0])
        dev = frame_dev.device
        boxes = torch.from_numpy(table).to(dev)
        out = torch.empty((n, ps, ps, 3), dtype=torch.uint8, device=dev)
        _lib.check(_lib.lib().aae_extract_square_patches(_lib.ptr(frame_dev), frame_dev.shape[0], frame_dev.shape[1], _lib.ptr(boxes), n,
                                                         ps, _lib.ptr(out), C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)),
                   "extract_square_patches")
        return out

    def process(self, bboxes, color_img, camK, depth_img=None, camPose=None, rois3ds=[], mm=False):
        H, W = color_img.shape[:2]
        jobs = {}  # class -> list of (order, box_xywh)
        order = 0
        for box in bboxes:
            pred_clas = max(box.classes, key=box.classes.get)
            if pred_clas not in self.class_2_encoder:
                continue
            box_xywh = [box.xmin * W, box.ymin * H, (box.xmax - box.xmin) * W, (box.ymax - box.ymin) * H]
            if np.any(np.array(box_xywh) < 0):
                continue
            jobs.setdefault(pred_clas, []).append((order, box_xywh))
            order += 1
        results = [None] * order
        pending = []
        frame_u8 = np.ascontiguousarray(color_img if color_img.dtype == np.uint8 else color_img.astype(np.uint8))
        frames = {}   # device -> the frame, uploaded once per GPU
        # Launch every class' batch first, each on ITS OWN stream: an object class is an independent (encoder, codebook) pair, and a
        # handful of crops per class does not fill 148 SMs -- the classes' kernels overlap on one GPU and run in parallel on
        # different GPUs.  Results are collected afterwards.
        for clas, items in jobs.items():
            cb, sess = self.all_codebooks[clas], self._sessions[clas]
            dev = sess.device
            with torch.cuda.device(dev):
                cur = torch.cuda.current_stream(dev)
                if dev not in frames:
                    frames[dev] = torch.from_numpy(frame_u8).to(dev, non_blocking=True)
                st = self._class_streams.get(clas)
                if st is None:
                    st = self._class_streams[clas] = torch.cuda.Stream(device=dev)
                st.wait_stream(cur)                              # the frame upload (and whatever the caller queued before)
                with torch.cuda.stream(st):
                    crops = self.extract_square_patches_device(frames[dev], [it[1] for it in items], self.pad_factors[clas],
                                                               self.patch_sizes[clas])
                    _, idx = cb.nearest_idx_device(crops, k=1, upright=self._upright)
                frames[dev].record_stream(st)
            pending.append((clas, items, idx, st))
        for clas, items, idx, st in pending:     # ... then collect
            cb, sess = self.all_codebooks[clas], self._sessions[clas]
            with torch.cuda.device(sess.device), torch.cuda.stream(st):
                idcs = idx.cpu().numpy().astype(np.int64)[:, 0]
                cb._encoder.check_range(sess.device)
            train_args = self.all_train_args[clas]
            K_train = np.array(eval(train_args.get('Dataset', 'K'))).reshape(3, 3)
            radius = train_args.getfloat('Dataset', 'RADIUS')
            if cb.embed_obj_bbs_values is None:
                cb.embed_obj_bbs_values = sess.run(cb.embed_obj_bbs_var)
            # pose lift of all detections of this class in one vectorised call (SURVEY 8f N3; codebook.py:82-129)
            Rs, ts = lift_pose_batch(idcs[:, None], cb._dataset.viewsphere_for_embedding, cb.embed_obj_bbs_values,
                                     np.array([it[1] for it in items]), np.asarray(camK), K_train, radius)
            for j, (o, _) in enumerate(items):
                H_est = np.eye(4)
                H_est[:3, :3] = Rs[j, 0]
                H_est[:3, 3] = ts[j, 0] if mm else ts[j, 0] / 1000.
                if self._camPose:
                    H_est = np.dot(camPose, H_est)
                results[o] = PoseEstimate(name=clas, trafo=H_est)
        return results
