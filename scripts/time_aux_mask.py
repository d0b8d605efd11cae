"""Cost of AUXILIARY_MASK in the training step: the mask head joined with the output conv (N = 256 instead of 128 in the output
layer's GEMMs) and the mask loss, against the step without the head, on the split and the single-pass fp16 trainers.  bench.py's
--workload train protocol: batch 64, a ring of 4 device-resident (input, target) batches (targets with background pixels, so the
mask has both values), warm-up steps, one CUDA-event pair per step.  All four trainers start from the same seeds on their own
AAE_PREC_TC_SPLIT handles and are alternated (ABCD, then DCBA) over the rounds, so the clock drift of a power-capped card falls on
all alike.

Reports per trainer: step-time medians of every round with their median, p10 and p90; the seven phases of aae_trainer_profile
(median of profiled steps, a separate run from the timed ones); the device memory taken by the handles and the trainer; kernel
launches per step.  The card's name, power limit and SM clocks come from read-only nvidia-smi queries; no device setting is changed.

    python scripts/time_aux_mask.py [--rounds 4] [--steps 20] [--warmup 5] [--out result.json]
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
PHASES = ["operand_packs", "forward_and_loss", "wgrad_gemms", "dgrad_gemms", "glue", "fp32_dense_and_conv1_backward", "optimizer"]
MODES = {"split_mask_off": (None, False), "split_mask_on": (None, True), "fp16_mask_off": (_lib.PREC_TC_FP16, False),
         "fp16_mask_on": (_lib.PREC_TC_FP16, True)}


def make_trainer(gemm, mask, dev):
    from augmentedautoencoder_b200.ae.ae import AE
    from augmentedautoencoder_b200.ae.ae_factory import TrainOp
    from augmentedautoencoder_b200.ae.decoder import Decoder
    from augmentedautoencoder_b200.ae.encoder import Encoder
    from augmentedautoencoder_b200.ae.session import placeholder
    x, y = placeholder(np.float32, [None, 128, 128, 3]), placeholder(np.float32, [None, 128, 128, 3])
    enc = Encoder(x, 128, [128, 256, 512, 512], 5, [2, 2, 2, 2], False, is_training=True, max_batch=B, precision=_lib.PREC_TC_SPLIT, seed=42)
    dec = Decoder(y, enc.z, [512, 512, 256, 128], 5, [2, 2, 2, 2], "L2", 4, mask, False, is_training=True, max_batch=B,
                  precision=_lib.PREC_TC_SPLIT, seed=43)
    top = TrainOp(AE(enc, dec, 0, 0), 2e-4, precision=gemm)
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info(dev)[0]
    enc.handle(dev), dec.handle(dev)
    torch.cuda.synchronize()
    free1 = torch.cuda.mem_get_info(dev)[0]
    top.trainer(dev)
    torch.cuda.synchronize()
    free2 = torch.cuda.mem_get_info(dev)[0]
    return (enc, dec, top), {"handles": (free0 - free1) / 2 ** 20, "trainer": (free1 - free2) / 2 ** 20}


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
    graphs, tops, mem = {}, {}, {}
    for name, (gemm, mask) in MODES.items():
        graphs[name], mem[name] = make_trainer(gemm, mask, dev)
        tops[name] = graphs[name][2]
    g = torch.Generator(device="cpu").manual_seed(1234)
    ring = []
    for _ in range(4):
        x = torch.rand((B, 128, 128, 3), generator=g)
        y = torch.rand((B, 128, 128, 3), generator=g)
        y[torch.rand((B, 128, 128), generator=g) < 0.4] = 0.0      # background pixels: m = 0 there
        ring.append((x.to(dev), y.to(dev)))
    launches = {}
    for name in MODES:
        for i in range(max(args.warmup, 3)):
            tops[name].step_device(*ring[i % 4])
        torch.cuda.synchronize()
        n0 = lib.aae_launch_count()
        tops[name].step_device(*ring[0])
        torch.cuda.synchronize()
        launches[name] = int(lib.aae_launch_count() - n0)
    names = list(MODES)
    rounds = {n: [] for n in names}
    for r in range(args.rounds):
        for name in (names if r % 2 == 0 else names[::-1]):
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
    phases = {}
    for name in names:
        h = tops[name].trainer(dev)
        buf = (C.c_float * 8)()
        lib.aae_trainer_profile(h, 1, None, 0)
        rows = []
        for i in range(args.steps):
            tops[name].step_device(*ring[i % 4])
            torch.cuda.synchronize()
            n = lib.aae_trainer_profile(h, 1, buf, 8)
            if n:
                rows.append([buf[j] for j in range(n)])
        lib.aae_trainer_profile(h, 0, None, 0)
        phases[name] = {k: round(float(v), 4) for k, v in zip(PHASES, np.median(np.array(rows), axis=0))}
    med = {n: stats(v)["median"] for n, v in rounds.items()}
    out = {"gpu": state,
           "protocol": "batch %d, ring of 4 device-resident batches, %d warm-up steps, CUDA events per step; per-round medians of %d "
                       "steps, %d alternating rounds" % (B, max(args.warmup, 3), args.steps, args.rounds),
           "step_ms": {n: {"round_medians": v, **stats(v)} for n, v in rounds.items()},
           "added_ms_median": {"split": round(med["split_mask_on"] - med["split_mask_off"], 4),
                               "fp16": round(med["fp16_mask_on"] - med["fp16_mask_off"], 4)},
           "phase_ms_median": phases, "device_memory_MiB": mem, "launches_per_step": launches}
    print(json.dumps(out, indent=1))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
