"""The operand-traffic model and the per-class grouping of tools/gemm_launch_table.py (no GPU)."""
import importlib.util
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parents[1]
spec = importlib.util.spec_from_file_location("gemm_launch_table", ROOT / "tools" / "gemm_launch_table.py")
glt = importlib.util.module_from_spec(spec)
spec.loader.exec_module(glt)


def test_streaming_operand_bytes():
    # 3x3 conv 64^2 320 -> 320 at batch 64: 2048 x 2 tiles of 128 x 160, 45 slabs of a 16 KB A and a 20 KB B tile
    got = glt.operand_bytes(64 * 64 * 64, 320, 2880, 1, 160, False, 132)
    assert got == 2048 * 2 * 45 * (16384 + 160 * 64 * 2)
    # a batched view: every batch entry streams its own tiles; a ragged edge counts as a whole tile
    assert glt.operand_bytes(200, 100, 64, 3, 128, False, 132) == 3 * 2 * 1 * 1 * (16384 + 128 * 128)


def test_b_stationary_operand_bytes():
    # K 320 projection: the A stream plus one whole 320 x 160 weight tile per CTA, (132 // 2) * 2 CTAs
    got = glt.operand_bytes(64 * 4096, 320, 320, 1, 160, True, 132)
    assert got == 2048 * 2 * 5 * 16384 + 132 * 5 * 160 * 64 * 2


def test_table_groups_and_averages_per_evaluation():
    row = dict(conv=1, M=16384, N=1280, K=11520, batch=1, splits=1, bn=160)
    rows = [dict(row, ms="2.0")] * 4 + [dict(conv=0, M=64, N=1280, K=320, batch=1, splits=1, bn=1160, ms="0.5")] * 2
    t = glt.table(rows, reps=2, num_sms=132)
    assert [c["conv"] for c in t] == [1, 0]          # sorted by time, heaviest first
    conv, bres = t
    assert conv["launches"] == 2 and conv["ms"] == pytest.approx(4.0)
    assert conv["tflop"] == pytest.approx(2 * 2 * 16384 * 1280 * 11520 / 1e12)
    assert conv["tflops"] == pytest.approx(conv["tflop"] / 4e-3)
    assert conv["l2_tbs"] == pytest.approx(conv["l2_gb"] / 1e3 / 4e-3)
    assert bres["bres"] and bres["bn"] == 160 and bres["launches"] == 1
