"""AAE_PREC_TC_FP16 against AAE_PREC_TC_SPLIT on the inference hot path, with bench.py's protocol: batches of 256 uint8
crops resident on the device, a 256 MiB memset between timed batches (untimed) so weights and codebook come from HBM, one
CUDA-event pair per batch, median / p10 / p90.  Both precisions are created from the same weights and codebook and are
alternated (ABBA) over the rounds, so clock drift of a power-capped card falls on both alike.

Reports: encoder + fused match per 256-crop batch, the match alone at B in {1, 32, 128, 256}, the encoder's per-layer stages
(aae_encoder_profile), the device memory taken by creating each precision's encoder + codebook handles, and the card's power
limit and SM clocks (read-only nvidia-smi queries; no device setting is changed).

    python scripts/time_fp16_inference.py [--rounds 4] [--batches 20] [--out result.json]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bench import BATCH, make_model  # noqa: E402
from augmentedautoencoder_b200 import _lib  # noqa: E402

NAMES = {_lib.PREC_TC_SPLIT: "tc_split", _lib.PREC_TC_FP16: "tc_fp16"}


def gpu_state():
    q = "name,power.limit,clocks.sm,clocks.max.sm,temperature.gpu"
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30)
        return dict(zip(q.split(","), [v.strip() for v in r.stdout.strip().split(",")]))
    except (OSError, subprocess.SubprocessError) as e:
        return {"error": str(e)}


def stats(xs):
    xs = sorted(xs)
    return {"median": statistics.median(xs), "p10": xs[int(0.1 * (len(xs) - 1))], "p90": xs[int(0.9 * (len(xs) - 1))], "n": len(xs)}


def timed(fn, n, flush):
    out = []
    for _ in range(n):
        flush.zero_()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        out.append((a, b))
    torch.cuda.synchronize()
    return [a.elapsed_time(b) for a, b in out]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=4)
    ap.add_argument("--batches", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    state = [gpu_state()]
    precs = (_lib.PREC_TC_SPLIT, _lib.PREC_TC_FP16)
    models, mem = {}, {}
    for prec in precs:                                 # same seed: same weights and codebook
        enc, cb = make_model(prec, BATCH, 42)
        torch.cuda.synchronize()
        free0 = torch.cuda.mem_get_info(dev)[0]
        cb.handle(dev)                                 # creates the encoder handle first, then the codebook's
        torch.cuda.synchronize()
        mem[NAMES[prec]] = (free0 - torch.cuda.mem_get_info(dev)[0]) / 2 ** 20
        models[prec] = (enc, cb)
    g = torch.Generator(device="cpu").manual_seed(1234)
    crops = [torch.randint(0, 256, (BATCH, 128, 128, 3), dtype=torch.uint8, generator=g).to(dev) for _ in range(4)]
    z = {B: torch.randn((B, 128), generator=g).to(dev) for B in (1, 32, 128, 256)}
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    for prec in precs:                                 # warm-up: handles, operand packing, kernel attributes
        enc, cb = models[prec]
        for i in range(3):
            cb.nearest_idx_device(crops[i % 4])
            for B in z:
                cb.match_device(z[B])
    torch.cuda.synchronize()
    e2e = {NAMES[p]: [] for p in precs}
    match = {NAMES[p]: {B: [] for B in z} for p in precs}
    for r in range(args.rounds):
        for prec in (precs if r % 2 == 0 else precs[::-1]):
            enc, cb = models[prec]
            k = [0]

            def batch():
                cb.nearest_idx_device(crops[k[0] % 4])
                k[0] += 1
            e2e[NAMES[prec]].append(stats(timed(batch, args.batches, flush))["median"])
            for B in z:
                match[NAMES[prec]][B].append(stats(timed(lambda: cb.match_device(z[B]), args.batches, flush))["median"])
        state.append(gpu_state())
    stages = {}
    for prec in precs:
        enc, cb = models[prec]
        h = enc.handle(dev)
        lib = _lib.lib()
        lib.aae_encoder_profile(h, 1, None, 0)
        rows = []
        for i in range(args.batches):
            flush.zero_()
            enc.encode_device(crops[i % 4])
            torch.cuda.synchronize()
            buf = (torch.zeros(16, dtype=torch.float32)).numpy()
            n = lib.aae_encoder_profile(h, 1, _lib.ptr(buf), 16)
            rows.append(buf[:n].copy())
        lib.aae_encoder_profile(h, 0, None, 0)
        med = np.median(np.array(rows), axis=0)
        stages[NAMES[prec]] = {("conv%d" % (j + 1) if j < len(med) - 1 else "dense"): round(float(v), 4) for j, v in enumerate(med)}
    # agreement of the two precisions on one batch (informational)
    (s1, i1), (s2, i2) = (models[p][1].nearest_idx_device(crops[0]) for p in precs)
    agree = {"top1_index_differs": int((i1 != i2).sum()), "of": int(i1.numel()), "max_abs_score_diff": float((s1 - s2).abs().max())}
    out = {"gpu": state, "protocol": "B=%d uint8 crops on device, 256 MiB memset between batches, CUDA events; per-round medians of %d batches, "
                                     "%d ABBA rounds" % (BATCH, args.batches, args.rounds),
           "handle_memory_MiB_encoder_plus_codebook": mem,
           "encoder_plus_match_ms_per_batch": {n: {"round_medians": v, **stats(v)} for n, v in e2e.items()},
           "match_only_ms": {n: {str(B): {"round_medians": v, **stats(v)} for B, v in d.items()} for n, d in match.items()},
           "encoder_stage_ms_median": stages, "agreement": agree}
    print(json.dumps(out, indent=1))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
