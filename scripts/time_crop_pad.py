"""Cost of CropAndPad in the device input pipeline at batch 64, the template chain with and without the template's
Sometimes(0.5, CropAndPad(percent=(-0.05, 0.1))) line, alternated in rounds (medians reported):

  batch        Dataset.batch_device(64) and Dataset.batch_resident(64), device time between CUDA events
  kernel       the crop-pad pass: aae_augment with the crop table minus without it, on the same draws (events, half the images fired)
  steps        the split and single-pass fp16 trainers through the started queue (Session.run on the device), per step

Synthetic data; the card's name and power limit are read in the same run.  Writes nothing unless --out is given."""
import argparse
import configparser
import ctypes as C
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from augmentedautoencoder_b200 import _lib
from augmentedautoencoder_b200.ae import session as S
from scripts.time_train_loop import B, ROOT, gpu_query, model, synthetic, template_code, timed

ROUNDS = 5


def codes():
    """CODE of the template cfg as shipped (the CropAndPad line is a comment, which configparser drops) and with the line
    uncommented"""
    text = open(os.path.join(ROOT, "tests", "golden", "train_template.cfg")).read()
    assert "#Sometimes(0.5, CropAndPad" in text
    args = configparser.ConfigParser()
    args.read_string(text.replace("#Sometimes(0.5, CropAndPad", "Sometimes(0.5, CropAndPad"))
    return {"plain": template_code(), "crop_pad": args.get("Augmentation", "CODE")}


def datasets(arrays, dev):
    from augmentedautoencoder_b200.ae.dataset import Dataset
    out = {}
    for name, code in codes().items():
        ds = Dataset(None, code=code, seed=1)
        ds.train_x, ds.mask_x, ds.train_y, ds.bg_imgs = arrays
        ds.upload(dev)
        out[name] = ds
    return out


def kernel_only(ds, dev, launches=200):
    """us per launch of the gathered call with and without the crop-pad pass, on one batch of draws with about half the images fired"""
    aug = ds._aug
    rng = np.random.RandomState(3)
    x = torch.from_numpy(ds.train_x[:B]).to(dev)
    m = torch.from_numpy(np.ascontiguousarray(ds.mask_x[:B]).astype(np.uint8)).to(dev)
    bg = torch.from_numpy(ds.bg_imgs[:B]).to(dev)
    P = aug.sample(B)
    P["crop_on"][:] = rng.rand(B) < 0.5
    geom, lut = aug.pack(P)
    k = aug._constants(dev)
    gd, ld, cd = (torch.from_numpy(np.ascontiguousarray(a)).to(dev) for a in (geom, lut, aug.pack_crop(P)))
    tmp, ct, of = torch.empty_like(x), torch.empty_like(x), torch.empty(x.shape, dtype=torch.float32, device=dev)
    stream = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    plain = _lib.AugmentArgs(batch=B, h=128, w=128, c=3, low_w=aug.low[1], x=x, mask=m, bg=bg, geom=gd, lut=ld, bilinear_tab=k["tab"],
                             row_cell=k["rows"], col_cell=k["cols"], blur_kernel_q8=k["taps"], u8_to_float=k["to_float"], tmp=tmp,
                             out_f32=of)
    crop = plain.copy().set(crop=cd, resample=k["resample"], resample_len=int(k["resample"].numel()), max_src_rows=aug.crop["max_rows"],
                            max_src_w=aug.crop["max_w"], crop_tmp=ct)
    calls = {"without": lambda: _lib.check(_lib.lib().aae_augment(C.byref(plain), stream)),
             "with": lambda: _lib.check(_lib.lib().aae_augment(C.byref(crop), stream))}
    res = {n: [] for n in calls}
    for r in range(ROUNDS + 1):
        for n, fn in calls.items():
            ms = timed(fn, launches if r else 10)
            if r:
                res[n].append(ms * 1e3)
    med = {n: float(np.median(v)) for n, v in res.items()}
    return {"augment_us": round(med["without"], 2), "augment_crop_pad_us": round(med["with"], 2),
            "crop_pad_pass_us": round(med["with"] - med["without"], 2), "images_fired": int(P["crop_on"].sum())}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=40)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    sess = S.Session(device=0)
    out = {"card": gpu_query("name,power.limit"), "batch": B, "rounds": ROUNDS}
    import tempfile
    with tempfile.TemporaryDirectory() as tmp:
        arrays, _ = synthetic(tmp)
    sets = datasets(arrays, dev)
    np.random.seed(0)
    batches = {"%s_%s" % (kind, n): [] for n in sets for kind in ("batch_device", "batch_resident")}
    for r in range(ROUNDS + 1):
        for n, ds in sets.items():
            for kind in ("batch_device", "batch_resident"):
                ms = timed(lambda: getattr(ds, kind)(B), 50 if r else 5)
                if r:
                    batches["%s_%s" % (kind, n)].append(ms)
    out["batch_ms"] = {k: round(float(np.median(v)), 4) for k, v in batches.items()}
    print("batch", json.dumps(out["batch_ms"]), flush=True)
    out["kernel"] = kernel_only(sets["crop_pad"], dev)
    print("kernel", json.dumps(out["kernel"]), flush=True)
    steps = {}
    for prec_name, prec in (("split", None), ("fp16", _lib.PREC_TC_FP16)):
        built = {n: model(ds, prec) for n, ds in sets.items()}
        res = {n: [] for n in built}
        for r in range(ROUNDS + 1):
            for n, (q, enc, dec, top) in built.items():
                q.start(sess)
                for _ in range(5):
                    sess.run_device(top)
                ms = timed(lambda: sess.run_device(top), a.steps if r else 5)
                q.stop(sess)
                if r:
                    res[n].append(ms)
        for n, (q, enc, dec, top) in built.items():
            steps["%s_%s" % (prec_name, n)] = round(float(np.median(res[n])), 4)
            top.close()
            enc.close()
            dec.close()
    out["async_step_ms"] = steps
    print("steps", json.dumps(steps), flush=True)
    out["card_after"] = gpu_query("name,power.limit,clocks.sm,clocks.max.sm")
    text = json.dumps(out, indent=1)
    print(text)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
