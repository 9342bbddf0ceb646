#!/usr/bin/env python
"""Throughput of the text-to-audio batch task (`RiffusionPipeline.text_to_audio_batch`) on one H100; prints one JSON
line.

Random-init SD-1.5 UNet and VAE weights and the seeded 768-wide stub text encoder of tools/bench_interpolation.py.  The
workload is the typical comparison of param sets: 3 sets (DPM-Solver++, 50 steps, width 512, guidance 5 / 7 / 9) x 4
entries x 1 seed = 12 clips.  Three schedules of the same clips, alternated in the same run, every shape warmed up and
its CUDA graph captured first, best of `--reps`:

  batch     `text_to_audio_batch`: the sets differ only in guidance, so one loop of 12 rows
  per_set   one loop per param set (3 loops of 4 rows): `txt2img` with per-row embeddings and draws, same audio tail
  app       the app's schedule, one clip at a time (`text_to_audio_batch` with max_batch=1)

Per schedule the line holds output audio seconds per second of call, clips/s, ms per CFG UNet evaluation (call time over
the schedule's evaluations, tails included), the accounting (loops, evaluations, row evaluations) and the wall times;
`gpu` is the card name, power limit and the median SM clock sampled during the timed window.  Nothing is written to the
repository.
"""
from __future__ import annotations

import argparse
import json
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
PROMPTS = [("church bells on sunday", None, 42), ("electronic beats", "drums", 100),
           ("classical violin concerto", None, 4), ("jazz with piano", "vocals", 7)]


def default_batch(guidances=(5.0, 7.0, 9.0), steps: int = 50, width: int = 512) -> dict:
    """the benchmark's batch JSON object: one DPM-Solver++ param set per guidance, the four PROMPTS entries"""
    params = [dict(name=f"g{g:g}", scheduler="DPMSolverMultistepScheduler", num_inference_steps=steps, guidance=g,
                   width=width) for g in guidances]
    entries = [dict(prompt=p, seed=s, **({} if n is None else {"negative_prompt": n})) for p, n, s in PROMPTS]
    return dict(params=params, entries=entries)


def schedule_accounting(batch: dict, num_seeds: int = 1, max_batch: int = 32) -> dict:
    """clips, loops, CFG UNet evaluations and row evaluations of each schedule: `batch` (plan_batch at max_batch),
    `per_set` (one loop per param set, every clip of the set as one row, chunked at max_batch) and `app` (max_batch 1)"""
    from riffusion.text_to_audio_batch import n_unet_evals, parse_batch, plan_batch

    param_sets, entries = parse_batch(batch)

    def summary(loops):
        return {"loops": len(loops), "unet_evals": sum(e for _, e in loops), "row_evals": sum(r * e for r, e in loops)}

    clips, loops = plan_batch(param_sets, entries, num_seeds, max_batch)
    per_set_rows = len(entries) * num_seeds
    per_set = [(min(max_batch, per_set_rows - lo), n_unet_evals(ps.scheduler, ps.num_inference_steps))
               for ps in param_sets for lo in range(0, per_set_rows, max_batch)]
    _, app = plan_batch(param_sets, entries, num_seeds, 1)
    return {"clips": len(clips),
            "batch": summary([(len(lp.rows), lp.n_unet_evals) for lp in loops]),
            "per_set": summary(per_set),
            "app": summary([(len(lp.rows), lp.n_unet_evals) for lp in app])}


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--width", type=int, default=512)
    ap.add_argument("--reps", type=int, default=2, help="timed rounds of the three schedules")
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("bench_text_to_audio_batch.py: no CUDA device (there is no CPU path)")
    for p in (str(ROOT), str(ROOT / "riffusion-hobby_b200"), str(ROOT / "tools"), str(ROOT / "tests" / "golden")):
        if p not in sys.path:
            sys.path.insert(0, p)
    from bench import ClockSampler
    from bench_interpolation import StubTextEncoder
    from bench_text_to_audio import gpu_info
    from prompt_stub import StubTokenizer

    from riffusion.riffusion_pipeline import DEFAULT_PARAMS, RiffusionPipeline
    from riffusion.text_to_audio_batch import parse_batch
    from riffusion.util import audio_util

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    pipe = RiffusionPipeline.random_init(seed=0, device="cuda")
    pipe.tokenizer, pipe.text_encoder = StubTokenizer(), StubTextEncoder(dev)
    converter = pipe._converter(DEFAULT_PARAMS, None)
    batch = default_batch(steps=args.steps, width=args.width)
    param_sets, entries = parse_batch(batch)
    acc = schedule_accounting(batch)

    def batched(max_batch):
        out = pipe.text_to_audio_batch(batch, max_batch=max_batch, converter=converter)
        torch.cuda.synchronize()
        return out

    def per_set():
        """one txt2img loop per param set, rows = the entries, plus text_to_audio_batch's device and host tail"""
        segs = []
        texts = torch.cat([pipe.embed_text(e.prompt) for e in entries])
        unconds = torch.cat([pipe.embed_text(e.negative_prompt or "") for e in entries])
        for ps in param_sets:
            draws = torch.cat([torch.randn((1, 4, 64, ps.width // 8), generator=torch.Generator("cuda").manual_seed(e.seed),
                                           device="cuda", dtype=torch.float16) for e in entries])
            out = pipe.txt2img("", num_inference_steps=ps.num_inference_steps, guidance_scale=ps.guidance,
                               width=ps.width, height=512, scheduler=ps.scheduler, output_type="latent",
                               text_embeddings=texts, uncond_embeddings=unconds, latents=draws, num_clips=len(entries))
            u8 = pipe._decode_u8(out["latents"])
            for w in pipe._u8_to_waveform(u8, converter, False, None).cpu().numpy():
                segs.append(audio_util.apply_filters(audio_util.audio_from_waveform(samples=w, sample_rate=44100,
                                                                                    normalize=True), compression=False))
        torch.cuda.synchronize()
        return segs

    schedules = {"batch": lambda: batched(32), "per_set": per_set, "app": lambda: batched(1)}
    for run in schedules.values():                   # warm-up: graphs for every batch shape, caches
        run()
    out = batched(32)
    assert [lp["n_unet_evals"] for lp in out["loops"]] == [args.steps], out["loops"]
    output_s = sum(c["segment"].duration_seconds for c in out["clips"])
    times = {name: [] for name in schedules}
    sampler = ClockSampler(0)
    sampler.start()
    for _ in range(args.reps):
        for name, run in schedules.items():
            t0 = time.perf_counter()
            run()
            times[name].append(time.perf_counter() - t0)
    clocks = sampler.stop()
    line = {"metric": "text-to-audio batch output seconds per second", "unit": "s/s", "schedules": {}}
    for name, ts in times.items():
        best = min(ts)
        line["schedules"][name] = {"value": output_s / best, "clips_per_s": acc["clips"] / best,
                                   "ms_per_unet_eval": 1e3 * best / acc[name]["unet_evals"], **acc[name],
                                   "s_per_call": ts}
    line["value"] = line["schedules"]["batch"]["value"]
    line["speedup_vs_per_set"] = min(times["per_set"]) / min(times["batch"])
    line["speedup_vs_app"] = min(times["app"]) / min(times["batch"])
    line["clocks"] = clocks
    line["config"] = {"clips": acc["clips"], "output_s": output_s, "steps": args.steps, "width": args.width,
                      "guidance": [ps.guidance for ps in param_sets], "scheduler": "DPMSolverMultistepScheduler",
                      "weights": "random-init SD-1.5", "text": "seeded stub text encoder", "reps": args.reps,
                      "timing": "min over reps, wall clock, alternating batch / per_set / app"}
    line["gpu"] = gpu_info()
    print(json.dumps(line))


if __name__ == "__main__":
    main()
