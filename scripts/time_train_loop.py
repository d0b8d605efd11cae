"""Period of the training loop at batch 64 (template network) with each input path, for the split and the single-pass fp16
trainers, with the occlusion switches off and on:

  serial     Dataset.batch_device + TrainOp.step_device: host gather, pageable upload and host draws in series with the step
  resident   Dataset.batch_resident + step_device: the training set on the device, only the draws uploaded, still in series
  async      Queue.start + Session.run(train_op) on the device (run_device): the producer thread makes batches ahead
  bare       step_device on one fixed batch: the step alone, the period the async loop should reach

The modes alternate in rounds; each round times STEPS steps between two CUDA events on the consumer's stream after a warm-up
(for async, after five untimed steps of the started queue, so the first fills of the ring are not counted).
Also: batch_device's parts (host draws, host gather of the four arrays, their pageable upload), host clock over synchronised
calls.  Synthetic data (20 000 training images, 15 000 backgrounds as in the template cfg).  Prints one JSON document (and
writes it to --out); writes nothing else."""
import argparse
import configparser
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from augmentedautoencoder_b200 import _lib
from augmentedautoencoder_b200.ae import augment as A
from augmentedautoencoder_b200.ae import ae_factory as F
from augmentedautoencoder_b200.ae import session as S
from augmentedautoencoder_b200.ae.ae import AE
from augmentedautoencoder_b200.ae.dataset import Dataset
from augmentedautoencoder_b200.ae.decoder import Decoder
from augmentedautoencoder_b200.ae.encoder import Encoder
from oracle import aae_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

B, H, N_IMG, N_BG, N_BANK = 64, 128, 20000, 15000, 1000


def gpu_query(fields):
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=" + fields, "--format=csv,noheader", "-i", "0"], capture_output=True,
                              text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return "not readable"


def synthetic(tmp):
    """20 000 / 15 000 images tiled from 500 random ones (content does not change the cost), elliptic objects, an occluder bank"""
    rng = np.random.RandomState(0)
    yy, xx = np.mgrid[:H, :H]
    k = 500
    cy, cx, ry, rx = (rng.randint(a, b, (k, 1, 1)) for a, b in ((40, 88), (40, 88), (20, 55), (20, 55)))
    mask = ((yy - cy) / ry.astype(float)) ** 2 + ((xx - cx) / rx.astype(float)) ** 2 > 1.0          # True = background
    x = rng.randint(0, 256, (k, H, H, 3), dtype=np.uint8)
    arrays = (np.tile(x, (N_IMG // k, 1, 1, 1)), np.tile(mask, (N_IMG // k, 1, 1)), np.tile(x[::-1], (N_IMG // k, 1, 1, 1)),
              np.tile(x, (N_BG // k, 1, 1, 1)))
    s = A.OCCLUSION_BANK_SIDE
    yy, xx = np.mgrid[:s, :s]
    cy, cx, ry, rx = (rng.randint(a, b, (N_BANK, 1, 1)) for a, b in ((40, 184), (40, 184), (15, 70), (15, 70)))
    bits = ((yy - cy) / ry.astype(float)) ** 2 + ((xx - cx) / rx.astype(float)) ** 2 <= 1.0
    path = os.path.join(tmp, "bank.bin")
    np.packbits(bits.reshape(-1)).tofile(path)
    return arrays, path


def template_code():
    """[Augmentation] CODE of the template training cfg (tests/golden/train_template.cfg, the reference's train_template.cfg)"""
    args = configparser.ConfigParser()
    args.read(os.path.join(ROOT, "tests", "golden", "train_template.cfg"))
    return args.get("Augmentation", "CODE")


def dataset(arrays, bank, occlusion):
    kw = {"realistic_occlusion": "0.25", "square_occlusion": "0.25"} if occlusion else {}
    ds = Dataset(None, code=template_code(), seed=1, **kw)
    ds.train_x, ds.mask_x, ds.train_y, ds.bg_imgs = arrays
    if occlusion:
        ds.load_occlusion_masks(bank)
    return ds


def model(ds, precision):
    q = F.Queue(ds, 10, 3, B)
    enc = Encoder(q.x, 128, list(O.NUM_FILTER), 5, list(O.STRIDES), False, is_training=True, max_batch=B, precision=_lib.PREC_TC_SPLIT)
    dec = Decoder(q.y, enc.z, list(reversed(O.NUM_FILTER)), 5, list(reversed(O.STRIDES)), "L2", 4, False, False, is_training=True,
                  max_batch=B, precision=_lib.PREC_TC_SPLIT)
    enc.load_weights(O.make_encoder_params(42, bias_scale=0.02))
    dec.load_weights(O.make_decoder_params(43, bias_scale=0.02))
    return q, enc, dec, F.TrainOp(AE(enc, dec, 0.0, 0.0), 2e-4, precision=precision)


def timed(fn, steps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / steps


def batch_device_parts(ds, dev, n=30):
    """host ms of batch_device's draws, of its host gather, and of the gather's pageable upload; the whole call (synchronised)"""
    draws, gather, upload, whole = [], [], [], []
    for _ in range(n):
        t0 = time.perf_counter()
        idx, idx_bg = ds._draws(B)[:2]
        t1 = time.perf_counter()
        parts = [ds.train_x[idx], np.ascontiguousarray(ds.mask_x[idx]).astype(np.uint8), ds.bg_imgs[idx_bg], ds.train_y[idx]]
        t2 = time.perf_counter()
        for p in parts:
            torch.from_numpy(p).to(dev, non_blocking=True)
        torch.cuda.synchronize(dev)
        t3 = time.perf_counter()
        ds.batch_device(B)
        torch.cuda.synchronize(dev)
        t4 = time.perf_counter()
        draws.append(t1 - t0)
        gather.append(t2 - t1)
        upload.append(t3 - t2)
        whole.append(t4 - t3)
    med = lambda v: round(1e3 * float(np.median(v)), 3)
    return {"draws_ms": med(draws), "gather_ms": med(gather), "upload_ms": med(upload), "batch_device_ms": med(whole)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=40)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    sess = S.Session(device=0)
    out = {"card": gpu_query("name,power.limit"), "sm_clock_before": gpu_query("clocks.sm,clocks.max.sm"), "batch": B,
           "steps_per_round": a.steps, "rounds": a.rounds, "configs": {}}
    with tempfile.TemporaryDirectory() as tmp:
        arrays, bank = synthetic(tmp)
        for occlusion in (False, True):
            ds = dataset(arrays, bank, occlusion)
            ds.upload(dev)
            np.random.seed(0)
            out["configs"]["batch_device_parts" + ("_occlusion" if occlusion else "")] = batch_device_parts(ds, dev)
            for prec_name, prec in (("split", None), ("fp16", _lib.PREC_TC_FP16)):
                q, enc, dec, top = model(ds, prec)
                x0, y0 = ds.batch_resident(B)
                modes = {
                    "serial": lambda: top.step_device(*ds.batch_device(B)),
                    "resident": lambda: top.step_device(*ds.batch_resident(B)),
                    "async": lambda: sess.run_device(top),
                    "bare": lambda: top.step_device(x0, y0),
                }
                res = {m: [] for m in modes}
                for r in range(a.rounds + 1):              # round 0 warms every path up and is not reported
                    for m, fn in modes.items():
                        if m == "async":
                            q.start(sess)
                            for _ in range(5):             # untimed: the first fills of the ring, ahead of the timed steps
                                fn()
                        ms = timed(fn, a.steps if r else 5)
                        if m == "async":
                            q.stop(sess)
                        if r:
                            res[m].append(ms)
                summary = {m: {"median_ms": round(float(np.median(v)), 3), "min_ms": round(min(v), 3), "max_ms": round(max(v), 3)}
                           for m, v in res.items()}
                key = "%s_%s" % (prec_name, "occlusion" if occlusion else "plain")
                out["configs"][key] = summary
                print(key, json.dumps(summary), flush=True)
                top.close()
                enc.close()
                dec.close()
            ds.occlusion_fallbacks()
    out["sm_clock_after"] = gpu_query("clocks.sm,clocks.max.sm")
    text = json.dumps(out, indent=1)
    print(text)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
