"""``ae_train <group>/<name>``: trains an experiment from its workspace cfg, as auto_pose/ae/ae_train.py does.

    python -m augmentedautoencoder_b200.ae.ae_train exp_group/my_autoencoder [--precision fp16]

Reads $AE_WORKSPACE_PATH/cfg/<group>/<name>.cfg and copies it into the experiment's log dir, builds the model through the
factory, loads the training set from the cache the reference renders (same file name, so a cache rendered by the reference is
used as it is) and the background stack (built from BACKGROUND_IMAGES_GLOB when its cache is missing), keeps both on the GPU,
resumes from ``checkpoints/`` and trains until NUM_ITER with the Queue started: batches are made ahead on a stream of their
own.  Every SAVE_INTERVAL steps it writes ``checkpoints/chkpt-<step>`` (TensorFlow bundle, with the optimizer slots and
global_step) and ``train_figures/training_images_<i>.png`` (input, reconstruction and target tiles); every 10 steps it appends
the loss to ``train_loss.txt`` in the log dir.  Apart from those, the loop never waits for the device.  Ctrl-C stops after the
current step.

Not supported: rendering the training set (``-gen``; without a cache the run stops and names the file it looked for), the
cv2 debug window (``-d``), TensorBoard summaries."""
import argparse
import configparser
import os
import shutil
import signal
import sys

import numpy as np

from .. import _lib
from . import ae_factory as factory
from . import session as S
from . import utils as u

LOSS_LOG = "train_loss.txt"
LOG_EVERY = 10
PRECISIONS = {"auto": None, "fp16": _lib.PREC_TC_FP16}


def parse_args(argv=None):
    parser = argparse.ArgumentParser(prog="ae_train", description=__doc__.split("\n\n")[0])
    parser.add_argument("experiment_name", help="<group>/<name> of $AE_WORKSPACE_PATH/cfg/<group>/<name>.cfg")
    parser.add_argument("-d", action="store_true", default=False, help="not supported (the reference's cv2 debug window)")
    parser.add_argument("-gen", action="store_true", default=False, help="not supported (the reference renders the training set)")
    parser.add_argument("--precision", choices=sorted(PRECISIONS), default="auto",
                        help="GEMM arithmetic of the training step: auto follows the handles (split fp16 on the tensor cores where "
                             "the geometry allows it, else fp32); fp16 is the single-pass trainer")
    return parser.parse_args(argv)


def split_name(full):
    parts = full.split("/")
    name = parts.pop()
    group = parts.pop() if parts else ""
    return name, group


class Run(object):
    """What ``prepare`` builds: session, dataset, queue, modules, train op, saver, paths and the cfg's NUM_ITER / SAVE_INTERVAL."""

    def __init__(self, **kw):
        self.__dict__.update(kw)


def prepare(argv=None):
    """Everything ae_train does before its loop: cfg, log dir, model, training set and backgrounds on the GPU, and the state of
    the latest checkpoint in ``checkpoints/`` (weights, optimizer slots, global_step) when there is one."""
    arguments = parse_args(argv)
    if arguments.d:
        raise NotImplementedError("ae_train -d (the cv2 window of sample batches) is not supported: train without it and look at "
                                  "train_figures/")
    if arguments.gen:
        raise NotImplementedError("ae_train -gen renders the training set, and rendering is not part of this package: render the "
                                  "cache with the reference's ae_train -gen; this one finds it under the same name")
    workspace_path = os.environ.get("AE_WORKSPACE_PATH")
    if workspace_path is None:
        raise EnvironmentError("Please define a workspace path: export AE_WORKSPACE_PATH=/path/to/workspace")
    experiment_name, experiment_group = split_name(arguments.experiment_name)
    cfg_file_path = u.get_config_file_path(workspace_path, experiment_name, experiment_group)
    log_dir = u.get_log_dir(workspace_path, experiment_name, experiment_group)
    ckpt_dir = u.get_checkpoint_dir(log_dir)
    train_fig_dir = u.get_train_fig_dir(log_dir)
    dataset_path = u.get_dataset_path(workspace_path)
    if not os.path.exists(cfg_file_path):
        raise FileNotFoundError("Could not find config file: %s" % cfg_file_path)
    args = configparser.ConfigParser()
    args.read(cfg_file_path)
    with S.variable_scope(experiment_name):
        dataset = factory.build_dataset(dataset_path, args)
    training_images = dataset.training_images_path(dataset_path, args)
    if not os.path.exists(training_images):      # before anything is built or written
        raise FileNotFoundError("no training-image cache for this cfg: %s (rendering the training set is not part of this package; "
                                "render it with the reference's ae_train -gen and copy the .npz there)" % training_images)
    for d in (ckpt_dir, train_fig_dir, dataset_path):
        os.makedirs(d, exist_ok=True)
    shutil.copy2(cfg_file_path, log_dir)

    sess = S.Session()
    with S.variable_scope(experiment_name):
        queue = factory.build_queue(dataset, args)
        encoder = factory.build_encoder(queue.x, args, is_training=True)
        decoder = factory.build_decoder(queue.y, encoder, args, is_training=True)
        ae = factory.build_ae(encoder, decoder, args)
        codebook = factory.build_codebook(encoder, dataset, args)
        train_op = factory.build_train_op(ae, args, precision=PRECISIONS[arguments.precision])
        saver = factory.Saver([encoder, decoder, codebook], global_step=ae.global_step, train_op=train_op)
    dataset.get_training_images(dataset_path, args, device=sess.device)
    dataset.load_bg_images(dataset_path, device=sess.device)

    from .tf_checkpoint import latest_checkpoint
    latest, _ = latest_checkpoint(ckpt_dir)
    if latest is not None:
        saver.restore(sess, latest)
    return Run(name=arguments.experiment_name, sess=sess, dataset=dataset, queue=queue, encoder=encoder, decoder=decoder, ae=ae,
               codebook=codebook, train_op=train_op, saver=saver, log_dir=log_dir, checkpoint_file=u.get_checkpoint_basefilename(log_dir),
               train_fig_dir=train_fig_dir, restored=latest, num_iter=args.getint("Training", "NUM_ITER"),
               save_interval=args.getint("Training", "SAVE_INTERVAL"))


def train(run):
    """The loop of ae_train.py:117-146 from global_step to NUM_ITER with the queue started; returns the final global_step."""
    import cv2
    sess, queue, ae = run.sess, run.queue, run.ae
    gentle_stop = [False]

    def on_ctrl_c(signum, frame):
        gentle_stop[0] = True

    previous = signal.signal(signal.SIGINT, on_ctrl_c)
    first = int(ae.global_step.value())
    print("Training %s from step %d to %d" % (run.name, first, run.num_iter))
    queue.start(sess)
    try:
        with open(os.path.join(run.log_dir, LOSS_LOG), "a") as log:
            for i in range(first, run.num_iter):
                loss = sess.run_device(run.train_op)
                if i % LOG_EVERY == 0:
                    log.write("%d %.9g\n" % (i, float(loss)))      # the one wait for the device every LOG_EVERY steps
                    log.flush()
                    for m in (run.encoder, run.decoder):            # the results are on the host: check the range guard
                        m.check_range(sess.device)
                if (i + 1) % run.save_interval == 0:
                    run.saver.save_tf(sess, run.checkpoint_file, global_step=int(ae.global_step.value()))
                    this_x, this_y = sess.run([queue.x, queue.y])
                    reconstr_train = sess.run(run.decoder.x, feed_dict={queue.x: this_x})
                    train_imgs = np.hstack((u.tiles(this_x, 4, 4), u.tiles(reconstr_train, 4, 4), u.tiles(this_y, 4, 4)))
                    cv2.imwrite(os.path.join(run.train_fig_dir, "training_images_%s.png" % i),
                                np.clip(np.rint(train_imgs * 255), 0, 255).astype(np.uint8))
                if gentle_stop[0]:
                    break
    finally:
        queue.stop(sess)
        signal.signal(signal.SIGINT, previous)
    if not gentle_stop[0]:
        print("To create the embedding run:\n\nae_embed %s\n" % run.name)
    return int(ae.global_step.value())


def main(argv=None):
    return train(prepare(argv))


if __name__ == "__main__":
    try:
        main()
    except (FileNotFoundError, NotImplementedError, EnvironmentError) as e:
        sys.exit("ae_train: %s" % e)
