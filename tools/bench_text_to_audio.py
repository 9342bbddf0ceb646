#!/usr/bin/env python
"""Throughput of text-to-audio (`RiffusionPipeline.text_to_audio`) on one H100; prints one JSON line.

Random-init SD-1.5 UNet and VAE weights and N(0, 1) text embeddings (the text encoder is not timed), `--clips` clips
per step in one CFG batch, `--steps` scheduler steps, mono 0-10 kHz params, a 512-row spectrogram of `--width` columns.
Every shape is warmed up and its CUDA graph captured before the timed window.  The line holds:

  value       clips/s with everything device-resident: denoising loop + VAE decode + image -> mel -> waveform
  e2e         clips/s of text_to_audio through host WAV bytes (peak-normalised int16 PCM copied back per clip)
  unet        ms per CFG UNet evaluation (graph replay, batch 2 x clips)
  tc          k_tc_gemm TFLOP/s: sum of 2MNK over the GEMM / conv launches of one eager step over their CUDA-event time
              (rf_tc_profile_*, the accounting bench.py uses)
  gpu         card name, power limit and the median SM clock sampled during the timed window

`--unet-only` measures only the ms per CFG UNet evaluation, from the package directory `--pkg` (so two builds of the
library can be compared in one process tree).  Nothing is written to the repository.
"""
from __future__ import annotations

import argparse
import ctypes
import json
import subprocess
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]


def n_unet_evals(scheduler: str, steps: int) -> int:
    """CFG evaluations of one txt2img call: one per timestep; PNDM's PLMS table has steps + 1 entries."""
    if scheduler in ("DPMSolverMultistepScheduler", "DDIMScheduler", "EulerAncestralDiscreteScheduler"):
        return steps
    if scheduler == "PNDMScheduler":
        return steps + 1
    raise ValueError(scheduler)


def tc_tflops(flops: float, ms: float) -> float:
    """achieved rate of the tensor-core kernel: FLOPs (2MNK) over its summed CUDA-event time"""
    return flops / (ms / 1e3) / 1e12


def audio_samples(width: int, hop: int = 441) -> int:
    """waveform length of a `width`-column spectrogram: hop * (frames - 1)"""
    return hop * (width - 1)


def gpu_info() -> dict:
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits",
                              "-i", "0"], capture_output=True, text=True, timeout=30).stdout.strip().split(",")
        return {"name": out[0].strip(), "power_limit_w": float(out[1]), "sm_max_mhz": float(out[2])}
    except Exception as exc:  # noqa: BLE001
        return {"error": repr(exc)}


def _timed(fn, reps: int) -> float:
    import torch

    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def unet_only(args) -> None:
    pkg = Path(args.pkg).resolve()
    sys.path.insert(0, str(pkg))
    import torch

    from riffusion import sd15_spec
    from riffusion.graphed import GraphedUNet
    from riffusion.unet_b200 import UNetB200

    dev = torch.device("cuda", 0)
    unet = UNetB200({k: v.to(dev) for k, v in sd15_spec.random_state_dict(sd15_spec.unet_spec(), 0).items()}, device="cuda")
    g = torch.Generator(device=dev).manual_seed(0)
    lat = torch.randn((args.clips, 4, 64, args.width // 8), generator=g, device=dev, dtype=torch.float16)
    ctx = torch.randn((2 * args.clips, 77, 768), generator=g, device=dev, dtype=torch.float16)
    graphed = GraphedUNet(unet, lat.shape, ctx)
    for _ in range(3):
        graphed(lat, 500)
    ms = _timed(lambda: graphed(lat, 500), args.reps)
    print(json.dumps({"pkg": str(pkg), "width": args.width, "clips": args.clips, "ms_per_cfg_eval": ms, "reps": args.reps,
                      "gpu": gpu_info()}))


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--width", type=int, default=512, choices=[512, 768])
    ap.add_argument("--clips", type=int, default=32, help="clips per step (one CFG batch of 2 x clips)")
    ap.add_argument("--steps", type=int, default=30, help="scheduler steps")
    ap.add_argument("--scheduler", default="DPMSolverMultistepScheduler",
                    choices=["DPMSolverMultistepScheduler", "PNDMScheduler", "DDIMScheduler",
                             "EulerAncestralDiscreteScheduler"])
    ap.add_argument("--reps", type=int, default=3, help="timed repetitions of the whole step")
    ap.add_argument("--unet-only", action="store_true")
    ap.add_argument("--pkg", default=str(ROOT / "riffusion-hobby_b200"))
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("bench_text_to_audio.py: no CUDA device (there is no CPU path)")
    if args.unet_only:
        return unet_only(args)
    for p in (str(ROOT), str(ROOT / "riffusion-hobby_b200")):
        if p not in sys.path:
            sys.path.insert(0, p)
    from bench import ClockSampler
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
    B = args.clips
    g = torch.Generator(device=dev).manual_seed(1000)
    text = torch.randn((B, 77, 768), generator=g, device=dev, dtype=torch.float16)
    uncond = torch.randn((1, 77, 768), generator=g, device=dev, dtype=torch.float16)
    kw = dict(num_clips=B, num_inference_steps=args.steps, guidance_scale=7.0, width=args.width,
              scheduler=args.scheduler, text_embeddings=text, uncond_embeddings=uncond, params=params, converter=conv)

    def step_device():
        return pipe.text_to_audio("", **kw)

    def step_e2e():
        w = step_device()["waveform"]
        pcm = torch.empty((B, w.shape[-1]), dtype=torch.int16, device=dev)
        scratch = torch.zeros(1, dtype=torch.float32, device=dev)
        stream = torch.cuda.current_stream(dev)
        for i in range(B):
            scratch.zero_()
            _native.check(lib.rf_wave_to_int16(w[i].data_ptr(), 1, w.shape[-1], 1, pcm[i].data_ptr(), scratch.data_ptr(),
                                               stream.cuda_stream))
        return [bytes(pcm[i].cpu().numpy().tobytes()) for i in range(B)]

    out = step_device()                     # warm-up: plans, graph capture for this shape
    step_device()
    n_evals = out["n_unet_evals"]
    assert n_evals == n_unet_evals(args.scheduler, args.steps)
    assert out["waveform"].shape == (B, 1, audio_samples(args.width))
    sampler = ClockSampler(0)
    sampler.start()
    ms_step = _timed(step_device, args.reps)
    clocks = sampler.stop()
    step_e2e()
    t0 = time.perf_counter()
    for _ in range(args.reps):
        step_e2e()
    ms_e2e = (time.perf_counter() - t0) * 1e3 / args.reps

    graphed = next(v for k, v in pipe._graphs.items() if k[0] == (B, 4, 64, args.width // 8))
    lat = out["latents_unscaled"]
    ms_unet = _timed(lambda: graphed(lat, 500), 10)

    pipe.use_cuda_graph = False             # one eager step with CUDA events around every GEMM / conv launch
    step_device()
    lib.rf_tc_profile_begin()
    step_device()
    tc_ms, tc_fl, tc_n = ctypes.c_double(), ctypes.c_double(), ctypes.c_long()
    lib.rf_tc_profile_end(ctypes.byref(tc_ms), ctypes.byref(tc_fl), ctypes.byref(tc_n))
    pipe.use_cuda_graph = True
    line = {
        "metric": "text-to-audio clips/sec", "value": B / (ms_step / 1e3), "unit": "clips/s", "ms_per_step": ms_step,
        "e2e": {"value": B / (ms_e2e / 1e3), "unit": "clips/s", "ms_per_step": ms_e2e,
                "api": "RiffusionPipeline.text_to_audio + rf_wave_to_int16, int16 PCM bytes on the host"},
        "unet": {"ms_per_cfg_eval": ms_unet, "batch": 2 * B, "latents": [64, args.width // 8]},
        "tc": {"kernel": "k_tc_gemm", "tflops": tc_tflops(tc_fl.value, tc_ms.value), "kernel_ms_per_step": tc_ms.value,
               "flops_per_step": tc_fl.value, "launches_per_step": tc_n.value},
        "config": {"width": args.width, "height": 512, "clips": B, "steps": args.steps, "scheduler": args.scheduler,
                   "n_unet_evals": n_evals, "guidance": 7.0, "weights": "random-init SD-1.5", "text": "N(0,1) embeddings",
                   "reps": args.reps},
        "gpu": gpu_info(), "clocks": clocks,
    }
    print(json.dumps(line))


if __name__ == "__main__":
    main()
