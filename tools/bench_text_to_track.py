#!/usr/bin/env python
"""Long tracks (`text_to_track`) on one H100; prints one JSON line.

Random-init SD-1.5 UNet and VAE, N(0, 1) text embeddings, `--steps` DPM-Solver++ steps, mono 0-10 kHz, 512-pixel windows
at stride 256 (50 % overlap), `--max-batch` 32.  A 60 s track is 6001 frames on a 6144-column canvas: 23 windows, one
CFG batch of 46.  Arms, alternated within every repetition after each shape has been warmed up and its CUDA graph
captured:

  track_1x{dur}s    one track of `--duration-s` seconds
  track_4x{dur}s    four tracks (one loop each at the default max batch)
  clips_12x512      text_to_audio of 12 independent 512-pixel clips in one CFG batch of 24, for reference

  audio_s_per_s     output audio seconds per wall second of the whole call (denoise + decode + mel + Griffin-Lim)
  ms_per_cfg_eval   one CFG UNet evaluation of the track's windows (graph replay), CUDA events
  decode_ms         VAE decode + uint8 of one track's canvas
  gl_ms             inverse mel + Griffin-Lim of one track's canvas
  gpu / clocks      card name, power limit, max SM clock; median SM clock sampled during the timed windows

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
    ap.add_argument("--duration-s", type=float, default=60.0)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--max-batch", type=int, default=32)
    ap.add_argument("--reps", type=int, default=2, help="alternated repetitions of every arm")
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("bench_text_to_track.py: no CUDA device (there is no CPU path)")
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
    g = torch.Generator(device=dev).manual_seed(1000)
    text = torch.randn((1, 77, 768), generator=g, device=dev, dtype=torch.float16)
    uncond = torch.randn((1, 77, 768), generator=g, device=dev, dtype=torch.float16)
    common = dict(num_inference_steps=args.steps, guidance_scale=7.0, scheduler="DPMSolverMultistepScheduler",
                  text_embeddings=text, uncond_embeddings=uncond, params=params, converter=conv)
    dur = args.duration_s
    arms = {
        f"track_1x{dur:g}s": (dur, lambda: pipe.text_to_track("", duration_s=dur, num_tracks=1,
                                                               max_batch=args.max_batch, **common)),
        f"track_4x{dur:g}s": (4 * dur, lambda: pipe.text_to_track("", duration_s=dur, num_tracks=4,
                                                                   max_batch=args.max_batch, **common)),
        "clips_12x512": (12 * params.hop_length * 511 / params.sample_rate,
                         lambda: pipe.text_to_audio("", num_clips=12, width=512, **common)),
    }
    first = {name: fn() for name, (_, fn) in arms.items()}       # warm-up: plans, graph capture of every shape
    track = first[f"track_1x{dur:g}s"]
    assert track["waveform"].shape == (1, 1, round(dur * params.sample_rate)), track["waveform"].shape
    sampler = ClockSampler(0)
    sampler.start()
    ms = {name: [] for name in arms}
    for _ in range(args.reps):
        for name, (_, fn) in arms.items():
            ms[name].append(_timed(fn, 1))
    n = len(track["windows"])
    lat = track["latents_unscaled"]
    win_lat = torch.randn((n, 4, lat.shape[2], 64), generator=g, device=dev, dtype=torch.float16)
    graphed = pipe._graphs[(tuple(win_lat.shape), (2 * n, 77, 768))]
    unet_ms = _timed(lambda: graphed(win_lat, 500), 10)
    decode_ms = _timed(lambda: pipe._decode_u8(track["latents"]), 3)
    mel = torch.rand((1, 1, 512, lat.shape[-1] * 8), device=dev) * 3e6
    ang = torch.rand((1, 1, params.n_fft // 2 + 1, lat.shape[-1] * 8), dtype=torch.complex64, device=dev)
    gl_ms = _timed(lambda: conv.waveform_from_mel_amplitudes(mel, ang), 3)
    out = {"metric": "text-to-track", "arms": {
        name: {"audio_s_per_s": audio_s / (min(ms[name]) / 1e3), "ms_per_call": ms[name]}
        for name, (audio_s, _) in arms.items()}}
    out.update(windows=n, canvas_px=lat.shape[-1] * 8, ms_per_cfg_eval=unet_ms, cfg_batch=2 * n, decode_ms=decode_ms,
               gl_ms=gl_ms, clocks=sampler.stop(), gpu=gpu_info(),
               config={"duration_s": dur, "steps": args.steps, "scheduler": "DPMSolverMultistepScheduler",
                       "window_width": 512, "stride": 256, "max_batch": args.max_batch,
                       "weights": "random-init SD-1.5", "text": "N(0,1) embeddings", "reps": args.reps})
    print(json.dumps(out))


if __name__ == "__main__":
    main()
