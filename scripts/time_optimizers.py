"""Cost of each OPTIMIZER rule in the split trainer's step, with bench.py's --workload train protocol: batch 64, a ring of 4
device-resident (input, target) batches, warm-up steps, one CUDA-event pair per step.  One trainer per rule, each on its own
AAE_PREC_TC_SPLIT handles from the same seeds, alternated in rounds (the order reversed every other round) so that the clock drift
of a power-capped card falls on all alike.

Reports per rule: step-time medians of every round with their median, p10 and p90; phase 6 of aae_trainer_profile (the optimizer
update, median of profiled steps in a separate run from the timed ones) with the bytes/s it achieves -- (12, 20 or 28 B per
parameter: parameter read and write, gradient read, each slot read and written) x parameters / phase time -- and that rate's
fraction of the 3.35 TB/s HBM3 data-sheet figure of the H100 SXM; the device memory taken by creating the trainer; kernel launches
per step.  The card's name, power limit and SM clocks come from read-only nvidia-smi queries; no device setting is changed.

    python scripts/time_optimizers.py [--rounds 4] [--steps 20] [--warmup 5] [--out result.json]
"""
import argparse
import ctypes as C
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from scripts.time_fp16_inference import gpu_state, stats  # noqa: E402
from augmentedautoencoder_b200 import _lib, build_ext  # noqa: E402

B = 64
DATASHEET_BYTES_PER_S = 3.35e12
RULES = ["Adam", "GradientDescent", "Adagrad", "ProximalAdagrad", "Adadelta", "RMSProp", "Ftrl"]


def make_trainer(name, dev):
    from augmentedautoencoder_b200.ae.ae import AE
    from augmentedautoencoder_b200.ae.ae_factory import TrainOp
    from augmentedautoencoder_b200.ae.decoder import Decoder
    from augmentedautoencoder_b200.ae.encoder import Encoder
    from augmentedautoencoder_b200.ae.session import placeholder
    x, y = placeholder(np.float32, [None, 128, 128, 3]), placeholder(np.float32, [None, 128, 128, 3])
    enc = Encoder(x, 128, [128, 256, 512, 512], 5, [2, 2, 2, 2], False, is_training=True, max_batch=B, precision=_lib.PREC_TC_SPLIT, seed=42)
    dec = Decoder(y, enc.z, [512, 512, 256, 128], 5, [2, 2, 2, 2], "L2", 4, False, False, is_training=True, max_batch=B,
                  precision=_lib.PREC_TC_SPLIT, seed=43)
    top = TrainOp(AE(enc, dec, 0, 0), 2e-4, optimizer=name)
    enc.handle(dev), dec.handle(dev)
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info(dev)[0]
    top.trainer(dev)
    torch.cuda.synchronize()
    params = sum(int(np.prod(ks)) + int(np.prod(bs)) for m in (enc, dec) for _, ks, _, bs in m._var_shapes)
    return top, (free0 - torch.cuda.mem_get_info(dev)[0]) / 2 ** 20, params


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=4)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    build_ext.build()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    lib = _lib.lib()
    state = [gpu_state()]
    tops, mem = {}, {}
    params = 0
    for name in RULES:
        tops[name], mem[name], params = make_trainer(name, dev)
    g = torch.Generator(device="cpu").manual_seed(1234)
    ring = [(torch.rand((B, 128, 128, 3), generator=g).to(dev), torch.rand((B, 128, 128, 3), generator=g).to(dev)) for _ in range(4)]
    launches = {}
    for name in RULES:
        for i in range(max(args.warmup, 3)):
            tops[name].step_device(*ring[i % 4])
        torch.cuda.synchronize()
        n0 = lib.aae_launch_count()
        tops[name].step_device(*ring[0])
        torch.cuda.synchronize()
        launches[name] = int(lib.aae_launch_count() - n0)
    rounds = {n: [] for n in RULES}
    for r in range(args.rounds):
        for name in (RULES if r % 2 == 0 else RULES[::-1]):
            evs = []
            for i in range(args.steps):
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                tops[name].step_device(*ring[i % 4])
                b.record()
                evs.append((a, b))
            torch.cuda.synchronize()
            rounds[name].append(stats([a.elapsed_time(b) for a, b in evs])["median"])
        state.append(gpu_state())
    update = {}
    for name in RULES:
        h = tops[name].trainer(dev)
        buf = (C.c_float * 8)()
        lib.aae_trainer_profile(h, 1, None, 0)
        ms = []
        for i in range(args.steps):
            tops[name].step_device(*ring[i % 4])
            torch.cuda.synchronize()
            n = lib.aae_trainer_profile(h, 1, buf, 8)
            if n >= 7:
                ms.append(buf[6])
        lib.aae_trainer_profile(h, 0, None, 0)
        phase = float(np.median(ms))
        nbytes = (12 + 8 * len(tops[name]._slots)) * params
        rate = nbytes / (phase * 1e-3)
        update[name] = {"phase6_ms_median": round(phase, 4), "bytes_per_param": nbytes // params, "achieved_TB_per_s": round(rate / 1e12, 3),
                        "fraction_of_3.35_TB_per_s_datasheet": round(rate / DATASHEET_BYTES_PER_S, 3)}
    out = {"gpu": state,
           "protocol": "batch %d, ring of 4 device-resident batches, %d warm-up steps, CUDA events per step; per-round medians of %d "
                       "steps, %d rounds alternating the rule order; split trainer per rule on its own handles" %
                       (B, max(args.warmup, 3), args.steps, args.rounds),
           "parameters": params,
           "step_ms": {n: {"round_medians": v, **stats(v)} for n, v in rounds.items()},
           "optimizer_update": update, "trainer_device_memory_MiB": {n: round(v, 1) for n, v in mem.items()}, "launches_per_step": launches}
    print(json.dumps(out, indent=1))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
