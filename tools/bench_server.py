#!/usr/bin/env python
"""The model server under concurrent load on one H100; prints one JSON line.

Setup as tools/bench_interpolation.py: random-init SD-1.5 UNet and VAE, the seeded stub text encoder, a synthetic
512x512 seed spectrogram and a mask image whose right half is white, written to a temporary seed-image directory.

K closed-loop clients (K in --clients, default 1 4 12 24) each walk alpha 0 -> 1 in steps of 0.25 as the web app does,
one request after the other, with their own prompt pair and seeds; 50 steps, denoising 0.75, guidance 7 by default.
A fraction --mask-share of the clients send the mask.  Two arms, alternated for each K in one run:

  serial    `run_inference` behind one lock: the reference server's schedule, one request at a time at CFG batch 2
  batched   `InferenceBatcher` (max_batch 16, max_wait_s 0.02): requests coalesce into `riffuse_requests` loops

Per arm and K the line holds requests/s, seconds of output audio per second, p50 / p95 request latency, the loops run
(CFG evaluations and CFG batch of each), the filler-row fraction and the share of wall time spent in the host tail
(int16, loudness filters, audio export, JPEG and base64, timed around those calls alike in both arms).  Also the card, its power limit and the
median SM clock sampled during the timed window.  Nothing is written to the repository.
"""
from __future__ import annotations

import argparse
import json
import sys
import tempfile
import threading
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
PROMPTS = [("church bells on sunday", "jazz with (piano:1.2)"), ("lo-fi beat", "orchestral strings"),
           ("techno kick", "acoustic guitar"), ("rain on a tin roof", "choir singing"),
           ("funk bassline", "ambient pads"), ("reggae", "heavy metal riff")]


def client_requests(client: int, steps: int = 50, denoising: float = 0.75, guidance: float = 7.0,
                    masked: bool = False) -> list:
    """The JSON payloads one client sends, in order: alpha 0, 0.25, .., 1 between its prompt pair"""
    a, b = PROMPTS[client % len(PROMPTS)]
    out = []
    for k in range(5):
        p = {"alpha": 0.25 * k, "num_inference_steps": steps, "seed_image_id": "seed",
             "start": {"prompt": a, "seed": 1000 + client, "denoising": denoising, "guidance": guidance},
             "end": {"prompt": b, "seed": 2000 + client, "denoising": denoising, "guidance": guidance}}
        if masked:
            p["mask_image_id"] = "mask"
        out.append(p)
    return out


def _starts(requests):
    from riffusion.riffusion_pipeline import RiffusionPipeline
    from riffusion.scheduler_b200 import PNDMSchedulerB200

    out = []
    for r in requests:
        s = PNDMSchedulerB200()
        s.set_timesteps(r.num_inference_steps)
        strength = (1 - r.alpha) * r.start.denoising + r.alpha * r.end.denoising
        out.append((len(s.timesteps), RiffusionPipeline._img2img_steps(s, r.num_inference_steps, strength)[1]))
    return out


def loop_accounting(requests, max_batch: int) -> dict:
    """The loops `riffuse_requests` runs for these InferenceInputs, all on one seed-image size with 77-token prompts:
    loops, requests, CFG evaluations, CFG batch per loop (2 x rows with guidance, rows without), rows, filler rows,
    row evaluations (rows x evaluations, filler included) and the filler share of the rows"""
    from riffusion.riffusion_pipeline import RiffusionPipeline

    guid = [r.start.guidance * (1.0 - r.alpha) + r.end.guidance * r.alpha for r in requests]
    keys = [(r.num_inference_steps, g > 1.0) for r, g in zip(requests, guid)]
    starts = _starts(requests)
    evals, batches, rows, fill, row_evals = 0, [], 0, 0, 0
    loops = RiffusionPipeline.request_loops(keys, max_batch)
    for idx, batch in loops:
        n_t = starts[idx[0]][0]
        e = n_t - min(starts[i][1] for i in idx)
        evals += e
        batches.append(2 * batch if guid[idx[0]] > 1.0 else batch)
        rows += batch
        fill += batch - len(idx)
        row_evals += e * batch
    return {"loops": len(loops), "requests": len(requests), "unet_evals": evals, "cfg_batch": batches, "rows": rows,
            "filler_rows": fill, "row_evals": row_evals, "filler_fraction": fill / rows if rows else 0.0}


def serial_accounting(requests) -> dict:
    """The loops `riffuse` runs for these requests one at a time: one loop each, at CFG batch 2 (1 without guidance)"""
    starts = _starts(requests)
    guid = [r.start.guidance * (1.0 - r.alpha) + r.end.guidance * r.alpha for r in requests]
    return {"loops": len(requests), "unet_evals": sum(n - t for n, t in starts),
            "cfg_batch": [2 if g > 1.0 else 1 for g in guid]}


def _pct(xs, q):
    import numpy as np

    return float(np.percentile(np.asarray(xs), q)) if xs else None


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--clients", type=int, nargs="+", default=[1, 4, 12, 24])
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--denoising", type=float, default=0.75)
    ap.add_argument("--guidance", type=float, default=7.0)
    ap.add_argument("--mask-share", type=float, default=0.5, help="fraction of the clients that send the mask")
    ap.add_argument("--max-batch", type=int, default=16)
    ap.add_argument("--max-wait-s", type=float, default=0.02)
    args = ap.parse_args()
    import numpy as np
    import torch
    from PIL import Image

    if not torch.cuda.is_available():
        raise SystemExit("bench_server.py: no CUDA device (there is no CPU path)")
    for p in (str(ROOT), str(ROOT / "riffusion-hobby_b200"), str(ROOT / "tools"), str(ROOT / "tests" / "golden")):
        if p not in sys.path:
            sys.path.insert(0, p)
    from bench import ClockSampler
    from bench_interpolation import StubTextEncoder, seed_image
    from bench_text_to_audio import gpu_info
    from prompt_stub import StubTokenizer

    from riffusion import server
    from riffusion.datatypes import InferenceInput
    from riffusion.riffusion_pipeline import RiffusionPipeline

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    pipe = RiffusionPipeline.random_init(seed=0, device="cuda")
    pipe.tokenizer, pipe.text_encoder = StubTokenizer(), StubTextEncoder(dev)
    tmp = tempfile.TemporaryDirectory()
    seed_dir = tmp.name
    seed_image().save(Path(seed_dir, "seed.png"))
    mask = np.zeros((512, 512), np.uint8)
    mask[:, 256:] = 255
    Image.fromarray(mask, mode="L").save(Path(seed_dir, "mask.png"))

    # loop accounting, recorded around the pipeline's batch call
    record = {"batches": [], "loops": [], "tail_s": 0.0}
    real_requests = pipe.riffuse_requests

    def riffuse_requests(inputs, *a, **kw):
        outs = real_requests(inputs, *a, **kw)
        record["batches"].append(loop_accounting(inputs, kw.get("max_batch", 16)))
        loops = {o["loop"]: (o["n_unet_evals"], o["filler_rows"]) for o in outs}
        record["loops"].extend(loops.values())
        return outs

    pipe.riffuse_requests = riffuse_requests

    # the host tail, timed directly and alike in both arms: int16 (`audio_from_waveform`, called with a host array),
    # loudness filters (`apply_filters`), MP3 / WAV export, JPEG and base64 (`server._response`).  Only the thread
    # that owns the pipeline runs them (the serial arm's lock holder, the batcher's worker), so one counter serves.
    from riffusion.util import audio_util

    def timed(fn):
        def run(*a, **kw):
            t0 = time.perf_counter()
            try:
                return fn(*a, **kw)
            finally:
                record["tail_s"] += time.perf_counter() - t0
        return run

    audio_util.audio_from_waveform = timed(audio_util.audio_from_waveform)
    audio_util.apply_filters = timed(audio_util.apply_filters)
    server._response = timed(server._response)

    def run_arm(kind: str, n_clients: int) -> dict:
        n_mask = int(round(args.mask_share * n_clients))
        payloads = [client_requests(c, args.steps, args.denoising, args.guidance, c < n_mask) for c in range(n_clients)]
        latencies, durations, errors = [], [], []
        lock = threading.Lock()
        batcher = (server.InferenceBatcher(pipe, seed_dir, max_batch=args.max_batch, max_wait_s=args.max_wait_s)
                   if kind == "batched" else None)

        def client(c):
            for p in payloads[c]:
                t0 = time.perf_counter()
                if batcher is None:
                    with lock:
                        resp = server.run_inference(p, pipe, seed_dir)
                else:
                    resp = batcher.submit(p).result()
                latencies.append(time.perf_counter() - t0)
                if isinstance(resp, tuple):
                    errors.append(resp)
                else:
                    durations.append(json.loads(resp)["duration_s"])

        record.update(batches=[], loops=[], tail_s=0.0)
        threads = [threading.Thread(target=client, args=(c,)) for c in range(n_clients)]
        t0 = time.perf_counter()
        for t in threads:
            t.start()
        for t in threads:
            t.join()
        wall = time.perf_counter() - t0
        if batcher is not None:
            batcher.close()
        if errors:
            raise SystemExit(f"bench_server.py: {kind} arm answered {errors[:3]}")
        n_req = len(latencies)
        all_reqs = [InferenceInput.from_dict(p) for ps in payloads for p in ps]
        out = {"requests": n_req, "wall_s": wall, "requests_per_s": n_req / wall, "audio_s_per_s": sum(durations) / wall,
               "p50_latency_s": _pct(latencies, 50), "p95_latency_s": _pct(latencies, 95),
               "host_tail_share": record["tail_s"] / wall}
        if kind == "batched":
            fill = sum(b["filler_rows"] for b in record["batches"])
            rows = sum(b["rows"] for b in record["batches"])
            out.update(batch_sizes=list(batcher.batch_sizes), loops=len(record["loops"]),
                       unet_evals_per_loop=_pct([e for e, _ in record["loops"]], 50),
                       cfg_batch_per_loop=[c for b in record["batches"] for c in b["cfg_batch"]],
                       unet_evals=sum(b["unet_evals"] for b in record["batches"]), filler_fraction=fill / rows)
            assert sum(e for e, _ in record["loops"]) == out["unet_evals"], (record["loops"], out["unet_evals"])
        else:
            acc = serial_accounting(all_reqs)
            out.update(loops=acc["loops"], unet_evals=acc["unet_evals"],
                       unet_evals_per_loop=_pct([acc["unet_evals"] / acc["loops"]], 50), cfg_batch_per_loop=[2],
                       filler_fraction=0.0)
        return out

    # warm-up: every CFG batch shape the batched arm can use (1, 2, 4, .., max_batch rows), plans and caches
    warm = [server.InferenceInput.from_dict(p) for p in client_requests(0, args.steps, args.denoising, args.guidance)]
    seed_pil = Image.open(Path(seed_dir, "seed.png")).convert("RGB")
    b = 1
    while True:
        reqs = (warm * args.max_batch)[:b]
        pipe.riffuse_requests(reqs, [seed_pil] * b, [None] * b, max_batch=args.max_batch)
        if b >= args.max_batch:
            break
        b = min(2 * b, args.max_batch)
    server.run_inference(client_requests(0, args.steps, args.denoising, args.guidance, True)[1], pipe, seed_dir)

    line = {"metric": "model server requests per second under K closed-loop clients", "unit": "req/s", "clients": {}}
    sampler = ClockSampler(0)
    sampler.start()
    for k in args.clients:
        serial = run_arm("serial", k)
        batched = run_arm("batched", k)
        line["clients"][str(k)] = {"serial": serial, "batched": batched,
                                   "speedup": batched["requests_per_s"] / serial["requests_per_s"]}
        print(json.dumps({"K": k, "serial_rps": serial["requests_per_s"], "batched_rps": batched["requests_per_s"]}),
              file=sys.stderr, flush=True)
    line["clocks"] = sampler.stop()
    line["value"] = line["clients"][str(args.clients[-1])]["batched"]["requests_per_s"]
    line["config"] = {"steps": args.steps, "denoising": args.denoising, "guidance": args.guidance,
                      "mask_share": args.mask_share, "max_batch": args.max_batch, "max_wait_s": args.max_wait_s,
                      "requests_per_client": 5, "weights": "random-init SD-1.5", "text": "seeded stub text encoder",
                      "timing": "wall clock per arm, arms alternated for each K"}
    line["gpu"] = gpu_info()
    tmp.cleanup()
    print(json.dumps(line))


if __name__ == "__main__":
    main()
