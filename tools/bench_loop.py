#!/usr/bin/env python
"""Cost of seamless loops (`text_to_audio(loop=True)`) against ordinary clips on one H100; prints one JSON line.

Random-init SD-1.5 UNet and VAE, N(0, 1) text embeddings, `--clips` clips per CFG batch, `--steps` DPM-Solver++
steps, mono 0-10 kHz, 512-row spectrograms at each `--widths` width.  Loop and non-loop calls alternate within every
repetition (same process, same clocks), after every shape has been warmed up and its CUDA graph captured.  Per width:

  clips_per_s      {loop, plain}: whole text_to_audio calls, device-resident (denoise + VAE decode + mel + waveform)
  ms_per_cfg_eval  {loop, plain}: one CFG UNet evaluation (graph replay); the difference is the cost of the bordered
                   copies in front of every 3x3 convolution
  gl_ms            {loop, plain}: Griffin-Lim of the batch (inverse mel + 32 iterations) on its own, CUDA events
  gpu / clocks     card name, power limit, max SM clock; median SM clock sampled during the timed windows

Nothing is written to the repository.
"""
from __future__ import annotations

import argparse
import json
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
for _p in (str(ROOT), str(ROOT / "tools"), str(ROOT / "riffusion-hobby_b200")):
    if _p not in sys.path:
        sys.path.insert(0, _p)


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--widths", type=int, nargs="+", default=[512, 768])
    ap.add_argument("--clips", type=int, default=32)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--reps", type=int, default=2, help="alternated loop / plain repetitions per width")
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("bench_loop.py: no CUDA device (there is no CPU path)")
    from bench import ClockSampler
    from bench_text_to_audio import _timed, gpu_info
    from riffusion.riffusion_pipeline import RiffusionPipeline
    from riffusion.spectrogram_converter import SpectrogramConverter
    from riffusion.spectrogram_params import SpectrogramParams

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    pipe = RiffusionPipeline.random_init(seed=0, device="cuda")
    params = SpectrogramParams(min_frequency=0, max_frequency=10000, stereo=False)
    conv = SpectrogramConverter(params, device="cuda")
    B = args.clips
    g = torch.Generator(device=dev).manual_seed(1000)
    text = torch.randn((B, 77, 768), generator=g, device=dev, dtype=torch.float16)
    uncond = torch.randn((1, 77, 768), generator=g, device=dev, dtype=torch.float16)
    out = {"metric": "seamless-loop text-to-audio", "widths": {}}
    sampler = ClockSampler(0)
    sampler.start()
    for width in args.widths:
        kw = dict(num_clips=B, num_inference_steps=args.steps, guidance_scale=7.0, width=width,
                  scheduler="DPMSolverMultistepScheduler", text_embeddings=text, uncond_embeddings=uncond, params=params,
                  converter=conv)
        res = {}
        for loop in (False, True):       # warm-up: plans, graph capture of both shapes
            r = pipe.text_to_audio("", loop=loop, **kw)
            want = params.hop_length * (width if loop else width - 1)
            assert r["waveform"].shape == (B, 1, want), r["waveform"].shape
            res[loop] = r
        ms = {False: [], True: []}
        for _ in range(args.reps):
            for loop in (False, True):
                ms[loop].append(_timed(lambda: pipe.text_to_audio("", loop=loop, **kw), 1))
        lat = res[False]["latents_unscaled"]
        shape = tuple(lat.shape)
        unet_ms = {}
        for loop in (False, True):
            key = (shape, (2 * B, 77, 768)) + (("wrap_w",) if loop else ())
            graphed = pipe._graphs[key]
            unet_ms[loop] = _timed(lambda: graphed(lat, 500), 10)
        mel = torch.rand((B, 1, 512, width), device=dev) * 3e6
        ang = torch.rand((B, 1, params.n_fft // 2 + 1, width), dtype=torch.complex64, device=dev)
        gl_ms = {}
        for loop in (False, True):
            conv.waveform_from_mel_amplitudes(mel, ang, periodic=loop)
            gl_ms[loop] = _timed(lambda: conv.waveform_from_mel_amplitudes(mel, ang, periodic=loop), 3)
        name = {False: "plain", True: "loop"}
        out["widths"][str(width)] = {
            "clips_per_s": {name[k]: B / (min(v) / 1e3) for k, v in ms.items()},
            "ms_per_call": {name[k]: v for k, v in ms.items()},
            "ms_per_cfg_eval": {name[k]: v for k, v in unet_ms.items()},
            "gl_ms": {name[k]: v for k, v in gl_ms.items()},
        }
    out["clocks"] = sampler.stop()
    out["config"] = {"clips": B, "steps": args.steps, "scheduler": "DPMSolverMultistepScheduler", "height": 512,
                     "weights": "random-init SD-1.5", "text": "N(0,1) embeddings", "reps": args.reps}
    out["gpu"] = gpu_info()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
