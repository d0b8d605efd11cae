"""Tap-group plan of the tensor-core conv GEMMs (scripts/time_tap_reuse.py mirrors tc_plan_groups): group counts, halo box
sizes and the L2 -> shared-memory bytes of the encoder layers at 256 crops.  No GPU needed."""
from scripts.time_tap_reuse import encoder_conv_taps, encoder_plan, tap_groups


def test_encoder_layers_group_taps_by_column_and_row_parity():
    plan = encoder_plan(256, planes=2)
    assert [(r["layer"], r["groups"], r["a_rows"]) for r in plan] == [("conv2", 10, 192), ("conv3", 10, 160), ("conv4", 10, 160)]
    di, dj, ch = encoder_conv_taps(128)
    groups, _ = tap_groups(di, dj, ch, 32, 4, 1, 2)
    assert groups[0] == [0, 10, 20] and groups[1] == [1, 11, 21] and sorted(len(g) for g in groups) == [2] * 5 + [3] * 5
    assert sorted(t for g in groups for t in g) == list(range(25))
    for g in groups:                      # one box per group: same parity plane and column offset, rows -1, 0, +1 apart
        assert len({(ch[t], dj[t]) for t in g}) == 1 and sorted(di[t] for t in g) in ([-1, 0, 1], [0, 1])


def test_encoder_bytes_per_batch():
    gb = [(round(r["bytes_before"] / 1e9, 1), round(r["bytes_after"] / 1e9, 1)) for r in encoder_plan(256, planes=2)]
    assert gb == [(13.4, 10.7), (13.4, 10.1), (6.7, 5.0)]
    tot = [sum(r[k] for r in encoder_plan(256, planes=2)) / 1e9 for k in ("bytes_before", "bytes_after")]
    assert abs(tot[0] - 33.55) < 0.01 and abs(tot[1] - 25.84) < 0.01
    # single-pass fp16 operands: half of every box
    assert [r["bytes_after"] * 2 for r in encoder_plan(256, planes=1)] == [r["bytes_after"] for r in encoder_plan(256, planes=2)]


def test_decoder_and_dgrad_3x3_taps_group_by_column_offset():
    di = [t // 3 - 1 for t in range(9)]
    dj = [t % 3 - 1 for t in range(9)]
    for bw in (8, 16, 32, 64):
        bh = min(bw, 128 // bw)
        groups, rows = tap_groups(di, dj, [0] * 9, bw, bh, 128 // (bw * bh), 2)
        assert groups == [[0, 3, 6], [1, 4, 7], [2, 5, 8]] and rows == (bh + 2) * bw * (128 // (bw * bh))


def test_geometries_without_a_halo_box_keep_one_box_per_tap():
    di, dj, ch = encoder_conv_taps(64)
    assert tap_groups(di, dj, ch, 4, 4, 8, 2) == ([[t] for t in range(25)], 128)     # BW % 8 != 0, BB > 2
    assert tap_groups([0], [0], [0], 1, 1, 128, 2) == ([[0]], 128)                     # dense layer: one tap
