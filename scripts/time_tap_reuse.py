"""L2 -> shared-memory traffic of the tensor-core encoder GEMMs (conv2..conv4), before and after tap groups.

tc_gemm_kernel loads, per (tap group, 64-channel chunk), one A box, and per tap one W box of 128 output channels.  Before tap
groups every tap was its own group with a 128-row box; now the taps of one column offset and row parity share one halo box of
(BH + 2) BW BB rows (tc_plan_groups in csrc/tc_gemm.cu, mirrored by `tap_groups` below).  Without a GPU this prints the bytes
each layer's plan moves per batch.  With a GPU it also times the layers (aae_encoder_profile stage times, median over the
rounds, L2 flushed between batches) and divides the bytes by the time: the achieved L2 -> SMEM rate.

    python scripts/time_tap_reuse.py [--batch 256] [--precision tc|fp16] [--rounds 20]
"""
import argparse
import os
import statistics
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from oracle import aae_oracle as O  # noqa: E402

KCH, N_TILE, A_RING_BYTES = 64, 128, 128 * 1024


def tap_groups(di, dj, ch, BW, BH, BB, planes):
    """Mirror of tc_plan_groups: (list of tap-index lists in K order, rows per plane of the A box)."""
    taps = len(di)
    halo_rows = (BH + 2) * BW * BB
    halo = (taps > 1 and BW % 8 == 0 and (BB == 1 or (BB == 2 and BH * BW == 64))
            and 2 * planes * halo_rows * KCH * 2 <= A_RING_BYTES and BH + 2 <= 256 and all(-1 <= d <= 1 for d in di))
    if not halo:
        return [[t] for t in range(taps)], 128
    keys = []
    for t in range(taps):
        if (ch[t], dj[t]) not in keys:
            keys.append((ch[t], dj[t]))
    return [[t for t in range(taps) if (ch[t], dj[t]) == k] for k in keys], halo_rows


def encoder_conv_taps(cin):
    """5 x 5 stride-2 taps on the space-to-depth input: block offsets (di, dj) and parity-plane channel offsets."""
    di = [(t // 5 + 1) // 2 - 1 for t in range(25)]
    dj = [(t % 5 + 1) // 2 - 1 for t in range(25)]
    ch = [((((t // 5) + 1) & 1) * 2 + (((t % 5) + 1) & 1)) * cin for t in range(25)]
    return di, dj, ch


def encoder_plan(batch=256, planes=2, filters=O.NUM_FILTER, hw=128):
    """Per encoder tensor-core conv layer: tiles, groups, A box rows and L2 -> SMEM bytes per batch, before and after."""
    rows = []
    h, c = hw // 2, filters[0]
    for l in range(1, len(filters)):
        oh, cout = h // 2, filters[l]
        BW = oh
        BH = min(oh, 128 // BW)
        BB = 128 // (BW * BH)
        di, dj, ch = encoder_conv_taps(c)
        groups, a_rows = tap_groups(di, dj, ch, BW, BH, BB, planes)
        cpt = c // KCH
        m_tiles = -(-batch * oh * oh // 128)
        tiles = m_tiles * -(-cout // N_TILE)
        w_box = planes * N_TILE * KCH * 2
        before = tiles * 25 * cpt * (planes * 128 * KCH * 2 + w_box)
        after = tiles * (len(groups) * cpt * planes * a_rows * KCH * 2 + 25 * cpt * w_box)
        rows.append({"layer": "conv%d" % (l + 1), "BW": BW, "BH": BH, "BB": BB, "tiles": tiles, "groups": len(groups),
                     "a_rows": a_rows, "bytes_before": before, "bytes_after": after})
        h, c = oh, cout
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--precision", default="tc", choices=["tc", "fp16"])
    ap.add_argument("--rounds", type=int, default=20)
    args = ap.parse_args()
    planes = 2 if args.precision == "tc" else 1
    plan = encoder_plan(args.batch, planes)
    stage = None
    try:
        import torch
        gpu = torch.cuda.is_available()
    except ImportError:
        gpu = False
    if gpu:
        import ctypes as C
        from augmentedautoencoder_b200 import _lib
        from bench import make_model
        prec = _lib.PREC_TC_SPLIT if planes == 2 else _lib.PREC_TC_FP16
        enc, _ = make_model(prec, args.batch, 42, with_codebook=False)
        lib, h = _lib.lib(), enc.handle(torch.device("cuda", 0))
        x = torch.randint(0, 256, (args.batch, 128, 128, 3), dtype=torch.uint8, device="cuda")
        flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
        for _ in range(5):
            enc.encode_device(x)
        lib.aae_encoder_profile(h, 1, None, 0)
        buf, runs = (C.c_float * 16)(), []
        for _ in range(args.rounds):
            flush.zero_()
            enc.encode_device(x)
            torch.cuda.synchronize()
            n = lib.aae_encoder_profile(h, 1, buf, 16)
            runs.append([buf[j] for j in range(n)])
        lib.aae_encoder_profile(h, 0, None, 0)
        stage = [statistics.median(col) for col in zip(*runs)]      # conv1, conv2, conv3, conv4, dense
        print("device:", torch.cuda.get_device_name(0))
    print("batch %d, %s operands: L2 -> shared-memory bytes of the encoder GEMMs" % (args.batch, "split (hi, lo)" if planes == 2 else "fp16"))
    print("%-6s %4s %4s %4s %6s %7s %6s %10s %10s %7s %s" % ("layer", "BW", "BH", "BB", "tiles", "groups", "A rows", "before GB", "after GB",
                                                           "change", "   stage ms   TB/s" if stage else ""))
    tot_b = tot_a = 0
    for i, r in enumerate(plan):
        tot_b += r["bytes_before"]
        tot_a += r["bytes_after"]
        extra = ""
        if stage:
            ms = stage[i + 1]
            extra = "   %8.3f %6.2f" % (ms, r["bytes_after"] / (ms * 1e-3) / 1e12)
        print("%-6s %4d %4d %4d %6d %7d %6d %10.2f %10.2f %6.0f%%%s" % (r["layer"], r["BW"], r["BH"], r["BB"], r["tiles"], r["groups"], r["a_rows"],
                                                                   r["bytes_before"] / 1e9, r["bytes_after"] / 1e9,
                                                                   100.0 * (r["bytes_after"] / r["bytes_before"] - 1), extra))
    print("total  %58.2f %10.2f %6.0f%%" % (tot_b / 1e9, tot_a / 1e9, 100.0 * (tot_a / tot_b - 1)))
    if not stage:
        print("(no GPU: stage times and rates not measured)")


if __name__ == "__main__":
    main()
