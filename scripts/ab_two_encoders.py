"""In-process A/B of a switch that is read when an encoder plan is CREATED: builds one encoder without and one with the variable,
alternates them batch by batch and compares the stage times.   python scripts/ab_two_encoders.py AAE_C1_V1 1"""
import ctypes as C
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from augmentedautoencoder_b200 import _lib  # noqa: E402
from bench import make_model  # noqa: E402

var, val = sys.argv[1], sys.argv[2]
n = int(sys.argv[sys.argv.index("--batches") + 1]) if "--batches" in sys.argv else 40
dev = torch.device("cuda", 0)
encs = {}
os.environ.pop(var, None)
encs["base"], _ = make_model(_lib.PREC_TC_SPLIT, 256, 42, with_codebook=False)
encs["base"].handle(dev)
os.environ[var] = val
encs["variant"], _ = make_model(_lib.PREC_TC_SPLIT, 256, 42, with_codebook=False)
encs["variant"].handle(dev)
os.environ.pop(var, None)
x = torch.randint(0, 256, (256, 128, 128, 3), dtype=torch.uint8, device="cuda")
flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
lib = _lib.lib()
buf = (C.c_float * 16)()
res = {k: [] for k in encs}
for k, e in encs.items():
    for _ in range(5):
        e.encode_device(x)
    lib.aae_encoder_profile(e.handle(dev), 1, None, 0)
for i in range(2 * n):
    k = "base" if i % 2 == 0 else "variant"
    flush.zero_()
    encs[k].encode_device(x)
    torch.cuda.synchronize()
    m = lib.aae_encoder_profile(encs[k].handle(dev), 1, buf, 16)
    res[k].append([buf[j] for j in range(m)])
for k in res:
    med = [statistics.median(col) for col in zip(*res[k])]
    print("%-8s median stage ms (conv1..conv4, dense): %s  sum %.4f" % (k, ["%.4f" % v for v in med], sum(med)))
