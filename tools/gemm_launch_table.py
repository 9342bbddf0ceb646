#!/usr/bin/env python
"""Per-layer-class table of the tensor-core kernel (k_tc_gemm) over one CFG UNet evaluation; one JSON line.

Random-init SD-1.5 UNet weights (as bench.py), latents (`--batch`, 4, 64, `--width` / 8) and N(0, 1) text embeddings.
After one warm-up evaluation, `--reps` eager evaluations run between rf_tc_profile_begin / rf_tc_profile_end with
RF_TC_PROFILE_DUMP pointed at a temporary file, so every GEMM / conv launch carries its CUDA-event time.  Launches with
the same (conv, M, N, K, batch, BN, splits, B-stationary) form one class.  Per class and evaluation:

  launches, ms, TFLOP/s     2MNK with the true extents over the summed event time
  l2_gb, l2_tbs             operand bytes the CTAs fetch from L2: tiles x slabs x (A tile + B tile), A tile = 128 x 64
                            fp16 = 16 KB, B tile = BN x 64 fp16; for B-stationary launches the A stream plus one whole
                            K x BN weight tile per CTA

The shared library is the one `riffusion._native` loads (RF_B200_LIB selects another build).  The line also holds the
card, its power limit and the median SM clock sampled during the profiled evaluations.  Nothing is written to the
repository.
"""
from __future__ import annotations

import argparse
import csv
import ctypes
import json
import math
import os
import sys
import tempfile
from collections import OrderedDict
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
BM, BK = 128, 64
A_TILE_BYTES = BM * BK * 2


def launch_class(row: dict) -> tuple:
    bn = int(row["bn"])
    return (int(row["conv"]), int(row["M"]), int(row["N"]), int(row["K"]), int(row["batch"]), bn % 1000,
            int(row["splits"]), bn >= 1000)


def operand_bytes(M: int, N: int, K: int, batch: int, bn: int, bres: bool, num_sms: int) -> int:
    """bytes of A and B tiles one launch streams from L2 into shared memory (see the module docstring); split-K units
    together cover the same slabs as whole tiles"""
    tiles_m, tiles_n, slabs = math.ceil(M / BM), math.ceil(N / bn), math.ceil(K / BK)
    b_tile = bn * BK * 2
    if bres:
        ctas = (num_sms // tiles_n) * tiles_n
        return batch * (tiles_m * tiles_n * slabs * A_TILE_BYTES + ctas * slabs * b_tile)
    return batch * tiles_m * tiles_n * slabs * (A_TILE_BYTES + b_tile)


def table(rows: list[dict], reps: int, num_sms: int) -> list[dict]:
    cls: "OrderedDict[tuple, dict]" = OrderedDict()
    for r in rows:
        key = launch_class(r)
        c = cls.setdefault(key, {"launches": 0, "ms": 0.0})
        c["launches"] += 1
        c["ms"] += float(r["ms"])
    out = []
    for (conv, M, N, K, batch, bn, splits, bres), c in cls.items():
        n = c["launches"] / reps
        ms = c["ms"] / reps
        flop = 2.0 * M * N * K * batch * n
        l2 = operand_bytes(M, N, K, batch, bn, bres, num_sms) * n
        out.append({"conv": conv, "M": M, "N": N, "K": K, "batch": batch, "bn": bn, "splits": splits, "bres": bres,
                    "launches": n, "ms": ms, "tflop": flop / 1e12,
                    "tflops": flop / (ms / 1e3) / 1e12 if ms > 0 else None, "l2_gb": l2 / 1e9,
                    "l2_tbs": l2 / (ms / 1e3) / 1e12 if ms > 0 else None})
    out.sort(key=lambda d: -d["ms"])
    return out


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--batch", type=int, default=64, help="UNet batch (2 x clips of one CFG evaluation)")
    ap.add_argument("--width", type=int, default=512, help="spectrogram width; latents are width / 8 wide")
    ap.add_argument("--reps", type=int, default=3, help="profiled evaluations (the table is per evaluation)")
    ap.add_argument("--label", default="", help="copied into the JSON line")
    args = ap.parse_args()
    for p in (str(ROOT), str(ROOT / "riffusion-hobby_b200")):
        if p not in sys.path:
            sys.path.insert(0, p)
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("gemm_launch_table.py: no CUDA device (there is no CPU path)")
    from bench import ClockSampler
    from riffusion import _native, sd15_spec
    from riffusion.unet_b200 import UNetB200
    from tools.bench_text_to_audio import gpu_info

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    lib = _native.lib()
    unet = UNetB200({k: v.to(dev) for k, v in sd15_spec.random_state_dict(sd15_spec.unet_spec(), 0).items()}, device="cuda")
    g = torch.Generator(device=dev).manual_seed(0)
    lat = torch.randn((args.batch, 4, 64, args.width // 8), generator=g, device=dev, dtype=torch.float16)
    ctx = torch.randn((args.batch, 77, 768), generator=g, device=dev, dtype=torch.float16)
    unet(lat, 500, encoder_hidden_states=ctx)
    torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as td:
        dump = os.path.join(td, "launches.csv")
        os.environ["RF_TC_PROFILE_DUMP"] = dump
        sampler = ClockSampler(0)
        sampler.start()
        lib.rf_tc_profile_begin()
        for _ in range(args.reps):
            unet(lat, 500, encoder_hidden_states=ctx)
        tc_ms, tc_fl, tc_n = ctypes.c_double(), ctypes.c_double(), ctypes.c_long()
        _native.check(lib.rf_tc_profile_end(ctypes.byref(tc_ms), ctypes.byref(tc_fl), ctypes.byref(tc_n)))
        clocks = sampler.stop()
        del os.environ["RF_TC_PROFILE_DUMP"]
        with open(dump) as f:
            rows = list(csv.DictReader(f))
    num_sms = torch.cuda.get_device_properties(dev).multi_processor_count
    classes = table(rows, args.reps, num_sms)
    total_ms = tc_ms.value / args.reps
    for c in classes:
        print(f"{'conv' if c['conv'] else 'gemm'} M={c['M']:>7} N={c['N']:>5} K={c['K']:>6} b={c['batch']:>4} "
              f"BN={c['bn']:>3} sp={c['splits']} bres={int(c['bres'])} n={c['launches']:>5.1f} "
              f"{c['ms']:8.3f} ms {c['tflops'] or 0:6.1f} TFLOP/s L2 {c['l2_gb']:7.2f} GB {c['l2_tbs'] or 0:5.2f} TB/s",
              file=sys.stderr)
    print(json.dumps({"label": args.label, "lib": str(_native._LIB_PATH), "batch": args.batch, "width": args.width,
                      "reps": args.reps, "launches_per_eval": tc_n.value / args.reps,
                      "tflop_per_eval": tc_fl.value / args.reps / 1e12, "ms_per_eval": total_ms,
                      "tflops": tc_fl.value / (tc_ms.value / 1e3) / 1e12, "gpu": gpu_info(), "clocks": clocks,
                      "classes": classes}))


if __name__ == "__main__":
    main()
