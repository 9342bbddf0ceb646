#!/usr/bin/env python
"""Throughput of audio to audio (`RiffusionPipeline.audio_to_audio`) on one H100; prints one JSON line.

Input: a seeded synthetic stereo track of `--seconds` s (a few decaying tones over noise), riffed over its whole length
with the app's defaults (mono 0-10 kHz, 5.0 s clips, 0.2 s overlap, denoising 0.55, 25 DPM-Solver++ steps, guidance
7.0).  Random-init SD-1.5 UNet and VAE weights and N(0, 1) text embeddings (the text encoder is not timed).  Every
shape is warmed up and its CUDA graph captured before a timed window.  The line holds:

  value       seconds of output audio per second, the whole call: slicing, device work, int16 / filters / stitch
  clips_per_s clips per second of the same runs
  serial      the reference's schedule on the same code: one clip after another at batch 1 (max_batch=1), and the
              batched / serial speed-up, both measured in this run
  unet        ms per CFG UNet evaluation (graph replay, batch 2 x clips)
  tc          k_tc_gemm TFLOP/s: sum of 2MNK over the GEMM / conv launches of one eager batched call over their CUDA-event
              time (rf_tc_profile_*, the accounting bench.py uses)
  gpu         card name, power limit and the median SM clock sampled during the timed window

With `--magic-mix` every clip is riffed with Magic Mix (`--kmin 0.3 --kmax 0.5 --mix-factor 0.5`, the app's values) in
place of img2img; the line then names the mode and carries its parameters instead of the denoising strength.

Nothing is written to the repository.
"""
from __future__ import annotations

import argparse
import contextlib
import ctypes
import json
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]


def output_seconds(n_clips: int, clip_duration_s: float, overlap_duration_s: float) -> float:
    """length of the stitched track: n clips, n - 1 crossfades"""
    return n_clips * clip_duration_s - (n_clips - 1) * overlap_duration_s


def magic_mix_evals(steps: int, kmax: float, scheduler: str) -> int:
    """CFG UNet evaluations of one Magic Mix call: len(timesteps) - t_max, t_max = steps - int(kmax * steps); PNDM's
    table has steps + 1 entries"""
    return steps + (scheduler == "PNDMScheduler") - (steps - int(kmax * steps))


def synthetic_track(seconds: float, seed: int = 0, rate: int = 44100):
    """a seeded stereo int16 track: decaying tones on a 0.5 s grid over low-level noise, slightly different per channel"""
    import numpy as np

    from riffusion.util.audio_util import AudioSegment

    rng = np.random.default_rng(seed)
    n = int(seconds * rate)
    t = np.arange(n) / rate
    out = np.zeros((n, 2))
    for onset in np.arange(0.0, seconds, 0.5):
        f = rng.choice([110.0, 220.0, 330.0, 440.0, 660.0, 880.0])
        m = t >= onset
        env = np.exp(-(t[m] - onset) * 4.0)
        for ch in range(2):
            out[m, ch] += env * np.sin(2 * np.pi * f * (1 + 0.002 * ch) * (t[m] - onset))
    out += 0.02 * rng.standard_normal(out.shape)
    out *= 0.8 * 32767 / np.abs(out).max()
    return AudioSegment(out.astype(np.int16), rate)


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--seconds", type=float, default=60.0, help="length of the synthetic track")
    ap.add_argument("--max-batch", type=int, default=32)
    ap.add_argument("--steps", type=int, default=25)
    ap.add_argument("--denoising", type=float, default=0.55)
    ap.add_argument("--scheduler", default="DPMSolverMultistepScheduler", choices=["DPMSolverMultistepScheduler", "PNDMScheduler"])
    ap.add_argument("--reps", type=int, default=2, help="timed repetitions of the batched call")
    ap.add_argument("--magic-mix", action="store_true", help="riff with Magic Mix instead of img2img")
    ap.add_argument("--kmin", type=float, default=0.3)
    ap.add_argument("--kmax", type=float, default=0.5)
    ap.add_argument("--mix-factor", type=float, default=0.5)
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("bench_audio_to_audio.py: no CUDA device (there is no CPU path)")
    for p in (str(ROOT), str(ROOT / "riffusion-hobby_b200"), str(ROOT / "tools")):
        if p not in sys.path:
            sys.path.insert(0, p)
    from bench import ClockSampler
    from bench_text_to_audio import _timed, gpu_info, tc_tflops
    from riffusion import _native
    from riffusion.riffusion_pipeline import RiffusionPipeline
    from riffusion.spectrogram_converter import SpectrogramConverter
    from riffusion.spectrogram_params import SpectrogramParams

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    lib = _native.lib()
    pipe = RiffusionPipeline.random_init(seed=0, device="cuda")
    params = SpectrogramParams(min_frequency=0, max_frequency=10000, stereo=False)
    conv = SpectrogramConverter(params, device="cuda")
    g = torch.Generator(device=dev).manual_seed(1000)
    text = torch.randn((1, 77, 768), generator=g, device=dev, dtype=torch.float16)
    uncond = torch.randn((1, 77, 768), generator=g, device=dev, dtype=torch.float16)
    track = synthetic_track(args.seconds)
    kw = dict(params=params, duration_s=args.seconds, denoising=args.denoising, num_inference_steps=args.steps,
              scheduler=args.scheduler, text_embeddings=text, uncond_embeddings=uncond, converter=conv)
    if args.magic_mix:
        kw.update(magic_mix=True, kmin=args.kmin, kmax=args.kmax, mix_factor=args.mix_factor)

    def run(max_batch: int):
        with contextlib.redirect_stdout(sys.stderr):         # the per-clip channel warnings; stdout is the JSON line
            out = pipe.audio_to_audio(track, "", max_batch=max_batch, **kw)
        torch.cuda.synchronize()
        return out

    def wall(max_batch: int, reps: int) -> float:
        t0 = time.perf_counter()
        for _ in range(reps):
            run(max_batch)
        return (time.perf_counter() - t0) / reps

    out = run(args.max_batch)               # warm-up: plans, graph capture for both batch shapes
    run(1)
    n = len(out["clip_start_times"])
    secs = output_seconds(n, 5.0, 0.2)
    assert abs(out["segment"].duration_seconds - secs) < 0.01, (out["segment"].duration_seconds, secs)
    n_evals = out["n_unet_evals"][0]
    if args.magic_mix:
        want = magic_mix_evals(args.steps, args.kmax, args.scheduler)
        assert n_evals == want, (n_evals, want)
    sampler = ClockSampler(0)
    sampler.start()
    s_batched = wall(args.max_batch, args.reps)
    clocks = sampler.stop()
    s_serial = wall(1, 1)

    b = min(n, args.max_batch)
    graphed = next(v for k, v in pipe._graphs.items() if k[0] == (b, 4, 64, 64))
    lat = torch.randn((b, 4, 64, 64), generator=g, device=dev, dtype=torch.float16)
    ms_unet = _timed(lambda: graphed(lat, 500), 10)

    pipe.use_cuda_graph = False             # one eager call with CUDA events around every GEMM / conv launch
    run(args.max_batch)
    lib.rf_tc_profile_begin()
    run(args.max_batch)
    tc_ms, tc_fl, tc_n = ctypes.c_double(), ctypes.c_double(), ctypes.c_long()
    lib.rf_tc_profile_end(ctypes.byref(tc_ms), ctypes.byref(tc_fl), ctypes.byref(tc_n))
    pipe.use_cuda_graph = True
    line = {
        "metric": "audio-to-audio output seconds per second", "value": secs / s_batched, "unit": "s/s",
        "clips_per_s": n / s_batched, "s_per_call": s_batched,
        "serial": {"max_batch": 1, "s_per_call": s_serial, "value": secs / s_serial, "speedup": s_serial / s_batched},
        "unet": {"ms_per_cfg_eval": ms_unet, "batch": 2 * b, "latents": [64, 64]},
        "tc": {"kernel": "k_tc_gemm", "tflops": tc_tflops(tc_fl.value, tc_ms.value), "kernel_ms_per_call": tc_ms.value,
               "flops_per_call": tc_fl.value, "launches_per_call": tc_n.value},
        "config": {"track_s": args.seconds, "clips": n, "output_s": secs, "max_batch": args.max_batch,
                   "steps": args.steps, "denoising": args.denoising, "scheduler": args.scheduler,
                   "n_unet_evals": n_evals, "guidance": 7.0, "weights": "random-init SD-1.5",
                   "text": "N(0,1) embeddings", "reps": args.reps},
        "gpu": gpu_info(), "clocks": clocks,
    }
    if args.magic_mix:
        line["metric"] = "audio-to-audio (Magic Mix) output seconds per second"
        line["config"]["magic_mix"] = {"kmin": args.kmin, "kmax": args.kmax, "mix_factor": args.mix_factor}
        del line["config"]["denoising"]
    print(json.dumps(line))


if __name__ == "__main__":
    main()
