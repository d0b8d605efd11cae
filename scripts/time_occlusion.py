"""Cost of the occlusion switches in the device input pipeline at batch 64: Dataset.batch_device with both switches off,
REALISTIC_OCCLUSION only, and both (alternated in rounds, host clock around synchronised batches), the
aae_occlusion kernel alone (CUDA events), and the host's candidate draws + packing.  Synthetic data; writes nothing."""
import ctypes as C
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
from augmentedautoencoder_b200.ae.dataset import Dataset
from tests.test_augment_cpu import TEMPLATE_CODE

B, N_IMG, N_BANK, H = 64, 1024, 1000, 128


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                           text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = ""
    return q or "%s (power limit not readable)" % torch.cuda.get_device_name(0)


def synthetic(tmp):
    rng = np.random.RandomState(0)
    yy, xx = np.mgrid[:H, :H]
    cy, cx, ry, rx = (rng.randint(a, b, (N_IMG, 1, 1)) for a, b in ((40, 88), (40, 88), (20, 55), (20, 55)))
    mask = ((yy - cy) / ry.astype(float)) ** 2 + ((xx - cx) / rx.astype(float)) ** 2 > 1.0          # True = background
    x = rng.randint(0, 256, (N_IMG, H, H, 3), dtype=np.uint8)
    np.savez(os.path.join(tmp, "train.npz"), train_x=x, mask_x=mask, train_y=x)
    np.save(os.path.join(tmp, "bg.npy"), rng.randint(0, 256, (N_IMG, H, H, 3), dtype=np.uint8))
    s = A.OCCLUSION_BANK_SIDE
    yy, xx = np.mgrid[:s, :s]
    cy, cx, ry, rx = (rng.randint(a, b, (N_BANK, 1, 1)) for a, b in ((40, 184), (40, 184), (15, 70), (15, 70)))
    bits = ((yy - cy) / ry.astype(float)) ** 2 + ((xx - cx) / rx.astype(float)) ** 2 <= 1.0
    np.packbits(bits.reshape(-1)).tofile(os.path.join(tmp, "bank.bin"))


def main():
    dev = torch.device("cuda", 0)
    print("card:", card())
    with tempfile.TemporaryDirectory() as tmp:
        synthetic(tmp)
        sets = {}
        for name, kw in (("off", {}), ("realistic", {"realistic_occlusion": "0.25"}),
                         ("both", {"realistic_occlusion": "0.25", "square_occlusion": "0.25"})):
            ds = Dataset(None, code=TEMPLATE_CODE, seed=1, **kw)
            ds.load_training_images(os.path.join(tmp, "train.npz"), os.path.join(tmp, "bg.npy"))
            if kw:
                ds.load_occlusion_masks(os.path.join(tmp, "bank.bin"))
            sets[name] = ds
    n, rounds = 50, 5
    times = {k: [] for k in sets}
    for ds in sets.values():                                  # warm-up: module load, bank upload
        for _ in range(5):
            ds.batch_device(B)
    torch.cuda.synchronize()
    for _ in range(rounds):
        for name, ds in sets.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(n):
                ds.batch_device(B)
            torch.cuda.synchronize()
            times[name].append((time.perf_counter() - t0) / n * 1e3)
    for name in sets:
        print("batch_device %-9s %.3f ms per batch of %d (median of %d rounds of %d; all: %s)" % (
            name, np.median(times[name]), B, rounds, n, " ".join("%.3f" % t for t in times[name])))
    fb = sets["both"].occlusion_fallbacks()
    print("fallbacks over the 'both' batches: %s of %d images" % (fb, (5 + rounds * n) * B))

    # the kernel alone: both steps, candidates uploaded once
    ds = sets["both"]
    occl = ds._occlusion
    st = occl._state(dev)
    idx = np.random.RandomState(3).choice(N_IMG, B, replace=False)
    mask = torch.from_numpy(ds.mask_x[idx].astype(np.uint8)).to(dev)
    out = torch.empty_like(mask)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    for label, R, S in (("realistic", occl.realistic, 0.0), ("both", occl.realistic, occl.square)):
        cand = torch.from_numpy(occl.pack(occl.sample(B, N_BANK))).to(dev)
        stream = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)

        args = _lib.OcclusionArgs(batch=B, h=H, w=H, realistic=1, max_occl=R, square=int(S != 0), min_kept=1.0 - S, mask=mask, cand=cand,
                                  n_cand=occl.K, n_bank=N_BANK, bank=st["bank"], row_cell=st["rows"], col_cell=st["cols"],
                                  low_h=occl.low[0], low_w=occl.low[1], mask_out=out, fallbacks=st["fallbacks"])

        def launch():
            _lib.check(_lib.lib().aae_occlusion(C.byref(args), stream))

        for _ in range(10):
            launch()
        res = []
        for _ in range(rounds):
            ev[0].record()
            for _ in range(200):
                launch()
            ev[1].record()
            ev[1].synchronize()
            res.append(ev[0].elapsed_time(ev[1]) / 200 * 1e3)
        print("aae_occlusion %-9s %.1f us per batch of %d (median of %d x 200 launches)" % (label, np.median(res), B, rounds))
    occl.fallbacks()

    # host side: candidate draws + packing
    t0 = time.perf_counter()
    for _ in range(200):
        occl.pack(occl.sample(B, N_BANK))
    print("host draws + pack (both steps, K = %d): %.3f ms per batch" % (occl.K, (time.perf_counter() - t0) / 200 * 1e3))


if __name__ == "__main__":
    main()
