#!/usr/bin/env python
"""Throughput of the interpolation walk (`RiffusionPipeline.interpolation`) on one H100; prints one JSON line.

Input: a synthetic 512x512 seed spectrogram (a seeded 5.12 s track of decaying tones, as an image) and the page's
defaults: 12 alphas, 50 PNDM steps, guidance 7.0, seeds 42 / 43.  Random-init SD-1.5 UNet and VAE weights and a seeded
stub text encoder (token table + positions, 768 wide), so the prompts' weighted embeddings are real tensors without CLIP
weights.  Two workloads: both ends at denoising 0.75 ("same") and ends at 0.5 / 0.9 ("diff").

Each workload alternates, in the same run, the single-loop call with the composition a caller had before it:
`riffuse_batch` over the same requests (one loop per group of equal strength, guidance and steps) plus the same audio
tail.  Every shape is warmed up and its CUDA graph captured before the timed calls.  Per workload the line holds:

  value / grouped.value   seconds of output audio per second, whole call (text, draws, loops, decode, audio, stitch)
  rows / grouped          loops, CFG UNet evaluations, CFG batch, row evaluations and rows evaluated before their start
  image_diff              per-row |difference| of the two paths' uint8 images (mean and max LSB, fraction within 1)
  gpu                     card name, power limit and the median SM clock sampled during the timed window

Nothing is written to the repository.
"""
from __future__ import annotations

import argparse
import contextlib
import json
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
PROMPT_A, PROMPT_B = "church bells on sunday", "jazz with (piano:1.2)"


def walk_accounting(n: int, steps: int, denoising_a: float, denoising_b: float, max_batch: int,
                    alpha_power: float = 1.0, guidance: float = 7.0) -> dict:
    """UNet work of an n-alpha walk: in `interpolation` (rows joining one loop at their own start, max_batch rows per
    loop) and in `riffuse_batch` (one loop per (strength, guidance, steps) group, CFG batch 2 x group size)"""
    from riffusion.riffusion_pipeline import RiffusionPipeline
    from riffusion.scheduler_b200 import PNDMSchedulerB200

    s = PNDMSchedulerB200()
    s.set_timesteps(steps)
    n_t = len(s.timesteps)
    alphas = RiffusionPipeline.interpolation_alphas(n, alpha_power)
    starts, groups = [], {}
    for a in alphas:
        strength = (1 - a) * denoising_a + a * denoising_b
        g = guidance * (1.0 - a) + guidance * a
        t_start = RiffusionPipeline._img2img_steps(s, steps, strength)[1]
        starts.append(t_start)
        groups.setdefault((strength, g, steps), t_start)
    evals, rows_evals, idle = 0, 0, 0
    for lo in range(0, n, max_batch):
        chunk = starts[lo:lo + max_batch]
        e = n_t - min(chunk)
        evals += e
        rows_evals += e * len(chunk)
        idle += sum(t - min(chunk) for t in chunk)
    return {"rows": {"loops": -(-n // max_batch), "unet_evals": evals, "cfg_batch": 2 * min(n, max_batch),
                     "row_evals": rows_evals, "idle_row_evals": idle},
            "grouped": {"loops": len(groups), "unet_evals": sum(n_t - t for t in groups.values())}}


class StubTextEncoder:
    """seeded token table + positions: (B, 77) ids -> ((B, 77, 768) fp16,) on the device"""

    def __init__(self, device, dim: int = 768, rows: int = 4096):
        import torch

        g = torch.Generator().manual_seed(77)
        self.table = torch.randn(rows, dim, generator=g).to(device)
        self.pos = torch.randn(77, dim, generator=g).to(device)

    def __call__(self, ids):
        return ((self.table[ids.to(self.table.device) % self.table.shape[0]] + self.pos[None]).half(),)


def seed_image():
    """512x512 RGB spectrogram image of a seeded synthetic 5.12 s track (mono 0-10 kHz)"""
    from bench_audio_to_audio import synthetic_track
    from PIL import Image

    from riffusion.riffusion_pipeline import DEFAULT_PARAMS
    from riffusion.spectrogram_image_converter import SpectrogramImageConverter

    with contextlib.redirect_stdout(sys.stderr):
        img = SpectrogramImageConverter(DEFAULT_PARAMS, device="cuda").spectrogram_image_from_audio(
            synthetic_track(5.2).set_channels(1))
    return img.crop((0, 0, 512, 512)).convert("RGB") if img.size[0] >= 512 else img.resize((512, 512), Image.BICUBIC)


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--alphas", type=int, default=12)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--max-batch", type=int, default=32)
    ap.add_argument("--reps", type=int, default=2, help="timed (single loop, grouped) pairs per workload")
    args = ap.parse_args()
    import numpy as np
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("bench_interpolation.py: no CUDA device (there is no CPU path)")
    for p in (str(ROOT), str(ROOT / "riffusion-hobby_b200"), str(ROOT / "tools"), str(ROOT / "tests" / "golden")):
        if p not in sys.path:
            sys.path.insert(0, p)
    from bench import ClockSampler
    from bench_text_to_audio import gpu_info
    from prompt_stub import StubTokenizer

    from riffusion.datatypes import PromptInput
    from riffusion.riffusion_pipeline import DEFAULT_PARAMS, RiffusionPipeline
    from riffusion.util import audio_util

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    pipe = RiffusionPipeline.random_init(seed=0, device="cuda")
    pipe.tokenizer, pipe.text_encoder = StubTokenizer(), StubTextEncoder(dev)
    init = seed_image()
    converter = pipe._converter(DEFAULT_PARAMS, None)

    def single(a, b):
        out = pipe.interpolation(a, b, init, num_interpolation_steps=args.alphas, num_inference_steps=args.steps,
                                 max_batch=args.max_batch)
        torch.cuda.synchronize()
        return out

    def grouped(requests):
        """riffuse_batch + the same device and host audio tail as `interpolation`"""
        images = pipe.riffuse_batch(requests, init)
        u8 = torch.from_numpy(np.stack([np.asarray(im) for im in images])).to(dev)
        wave = pipe._u8_to_waveform(u8, converter, False, None)
        segs = [audio_util.apply_filters(audio_util.audio_from_waveform(samples=w, sample_rate=44100, normalize=True))
                for w in wave.cpu().numpy()]
        seg = audio_util.stitch_segments(segs, crossfade_s=0)
        torch.cuda.synchronize()
        return u8, seg

    line = {"metric": "interpolation output seconds per second", "unit": "s/s", "workloads": {}}
    sampler = ClockSampler(0)
    sampler.start()
    for name, (den_a, den_b) in (("same", (0.75, 0.75)), ("diff", (0.5, 0.9))):
        a = PromptInput(prompt=PROMPT_A, seed=42, denoising=den_a, guidance=7.0)
        b = PromptInput(prompt=PROMPT_B, seed=43, denoising=den_b, guidance=7.0)
        out = single(a, b)                                  # warm-up: graphs for every batch shape, plans, caches
        u8_g, seg_g = grouped(out["requests"])
        t_single, t_grouped = [], []
        for _ in range(args.reps):
            t0 = time.perf_counter()
            out = single(a, b)
            t_single.append(time.perf_counter() - t0)
            t0 = time.perf_counter()
            u8_g, seg_g = grouped(out["requests"])
            t_grouped.append(time.perf_counter() - t0)
        secs = out["segment"].duration_seconds
        d = np.abs(out["images"].cpu().numpy().astype(np.int16) - u8_g.cpu().numpy().astype(np.int16))
        acc = walk_accounting(args.alphas, args.steps, den_a, den_b, args.max_batch)
        if acc["rows"]["loops"] == 1:
            assert out["n_unet_evals"] == [acc["rows"]["unet_evals"]], out["n_unet_evals"]
        line["workloads"][name] = {
            "denoising": [den_a, den_b], "output_s": secs, "grouped_output_s": seg_g.duration_seconds,
            "value": secs / min(t_single), "s_per_call": t_single,
            "rows": acc["rows"],
            "grouped": {**acc["grouped"], "value": secs / min(t_grouped), "s_per_call": t_grouped},
            "speedup": min(t_grouped) / min(t_single),
            "image_diff": {"mean_lsb_per_row": d.reshape(len(d), -1).mean(axis=1).round(4).tolist(),
                           "max_lsb": int(d.max()), "within_1_lsb": float((d <= 1).mean())},
        }
    line["clocks"] = sampler.stop()
    line["value"] = line["workloads"]["diff"]["value"]
    line["config"] = {"alphas": args.alphas, "steps": args.steps, "max_batch": args.max_batch, "guidance": 7.0,
                      "weights": "random-init SD-1.5", "text": "seeded stub text encoder", "reps": args.reps,
                      "timing": "min over reps, wall clock, alternating single loop / grouped"}
    line["gpu"] = gpu_info()
    print(json.dumps(line))


if __name__ == "__main__":
    main()
